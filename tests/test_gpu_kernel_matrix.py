"""The kernel matrix (pytest -m gpu): every solver kernel instantiation of the library, reached through
the C ABI and compared BIT FOR BIT with the checker (the compiled reference where oracle/_ref was
built, else the oracle restatement that test_oracle.py pins to it).  Batch cases are compared with
the checker frame by frame.

Every case also counts its launches (`j2p_session_launches`) and compares them with what
tests/kernel_paths.py predicts for the frame and mode, so the Python restatement of the host's
kernel choice is held to the real dispatch.  tests/test_kernel_coverage.py (no GPU) checks that the
named cases below reach every kernel in the library.

Case groups: sampling layouts x channel counts x TGV weight, single sessions and batches; objective
logging; the J2P_GRAD_SCALAR=1 and J2P_PROJ_TILE22=0 switches (child processes: the switches are
read once per process); values outside the fast paths' proven ranges in subsampled planes; extreme
tables and coefficients; tall narrow frames whose last gradient band is short; and a seeded sweep of
widths around the gradient's 60 / 240-column strips and the projection tiles.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import os
import subprocess
import sys

import numpy as np
import pytest

from jpeg2png_b200 import abi, synth
from tests import helpers as H
from tests import kernel_paths as K

G = K.PlaneGeom


@dataclasses.dataclass(frozen=True)
class Case:
    name: str
    planes: tuple                 # PlaneGeom per channel
    weight: float
    pweight: tuple
    iters: int
    nframes: int = 1              # > 1: one batch session of that many frames
    log: bool = False             # objective logging
    switch: str = ''              # '' | 'grad_scalar' (J2P_GRAD_SCALAR=1) | 'no_tile22' (J2P_PROJ_TILE22=0)
    device_decode: bool = False   # upload without the caller's decode (k_decode on the device)
    plant: str = ''               # '' | 'tiny' | 'patches' | 'zero_coefs' (test_gpu_parity.test_guard_fallback_rows) | 'subnormal' | 'island'
    extreme: str = ''             # '' | 'ones' (all-ones tables) | 'u16' (tables up to 65535) | 'coefs' (+-32767/-32768)
    seed: int = 0
    tall: bool = False            # heights re-chosen on the device: last gradient band 1..7 rows (tall_on_device)
    sweep: bool = False           # geometry sweep (not counted for kernel coverage)

    def mode(self) -> K.Mode:
        return K.Mode(nframes=self.nframes, log=self.log, grad_scalar=self.switch == 'grad_scalar',
                      tile22=self.switch != 'no_tile22', device_decode=self.device_decode)

    def describe(self) -> str:
        W, Hh = K.frame_size(self.planes)
        pl = ', '.join(f'{p.cw}x{p.ch}@({p.sw},{p.sh})' for p in self.planes)
        return (f'{self.name}: frame {W}x{Hh}, planes [{pl}], weight {self.weight}, pweight {list(self.pweight)}, '
                f'{self.iters} iterations, frames {self.nframes}, log {self.log}, switch {self.switch or "-"}, '
                f'device decode {self.device_decode}, plant {self.plant or "-"}, extreme {self.extreme or "-"}, seed {self.seed}')


# ---- frame layouts -------------------------------------------------------------------------
# (w_samp, h_samp) are the per-plane factors of struct coef, not the JPEG component factors.
LAYOUTS = {
    'y':     (G(72, 40, 1, 1),),                                        # one full-resolution plane
    's21':   (G(40, 48, 2, 1),),                                        # -s, a 4:2:2 chroma plane
    's12':   (G(48, 24, 1, 2),),                                        # -s, a 4:4:0 chroma plane
    'yy':    (G(64, 40, 1, 1), G(64, 40, 1, 1)),
    'y21':   (G(64, 40, 1, 1), G(32, 40, 2, 1)),
    '444':   (G(72, 48, 1, 1),) * 3,
    '422':   (G(80, 40, 1, 1), G(40, 40, 2, 1), G(40, 40, 2, 1)),
    '440':   (G(48, 64, 1, 1), G(48, 32, 1, 2), G(48, 32, 1, 2)),
    '411':   (G(64, 32, 1, 1), G(32, 32, 2, 1), G(16, 32, 4, 1)),       # component factors Y 4x1, Cb 2x1, Cr 1x1
    '420':   (G(64, 40, 1, 1), G(32, 24, 2, 2), G(32, 24, 2, 2)),       # luma grid 8 rows short of the frame
    'odd34': (G(40, 24, 1, 1), G(24, 16, 2, 2), G(16, 8, 3, 4)),
    'odd32': (G(48, 16, 1, 1), G(16, 8, 3, 2), G(16, 16, 3, 1)),
}
# Component factors Y 4x1, Cb 2x1, Cr 1x2 at 36 x 40 pixels (what the reader makes of such a file):
# Cb is a (2,2) plane 48 pixels wide in a 64-pixel frame.  The only named case whose single-frame
# projection runs k_step_uncovered22<false>.
Y4_CB2_CR12 = (G(40, 24, 1, 2), G(24, 24, 2, 2), G(16, 40, 4, 1))
# 4:2:0 whose chroma grid covers only the top 32 of 48 frame rows (batch: k_step_uncovered22<true>)
SHORT22 = (G(64, 48, 1, 1), G(32, 16, 2, 2), G(32, 16, 2, 2))
# larger frames for the planted values (the plantings address rows up to 60 and columns up to 104)
ADV = {
    '420': (G(208, 144, 1, 1), G(104, 72, 2, 2), G(104, 72, 2, 2)),
    '422': (G(208, 72, 1, 1), G(104, 72, 2, 1), G(104, 72, 2, 1)),
    'odd': (G(200, 72, 1, 1), G(112, 48, 2, 2), G(72, 24, 3, 4)),
}


def _named_cases():
    cases = []
    seed = 100

    def add(name, planes, weight, iters=8, pweight=None, **kw):
        nonlocal seed
        seed += 1
        pw = tuple(pweight) if pweight is not None else (0.001,) * len(planes)
        cases.append(Case(name, tuple(planes), weight, pw, iters, seed=seed, **kw))

    # every gradient group (channels x full / 4:2:0 / generic) x TGV on/off, single and batched
    for lay in ('y', 's21', 's12', 'yy', 'y21', '444', '422', '440', '411', '420'):
        for w in (0.0, 0.3):
            pw = (0.001, 0.0, 0.01) if lay == '422' and w else None        # a plane without the DCT-distance term
            add(f'{lay}_w{w}', LAYOUTS[lay], w, pweight=pw)
            n = 3 if w else 2
            add(f'{lay}_w{w}_batch{n}', LAYOUTS[lay], w, pweight=pw, nframes=n, device_decode=not w)
    for lay in ('odd34', 'odd32'):
        add(lay, LAYOUTS[lay], 0.4)
    add('odd34_batch2', LAYOUTS['odd34'], 0.4, nframes=2)
    add('y4_cb2_cr12', Y4_CB2_CR12, 0.3)
    add('short22_batch2', SHORT22, 0.3, nframes=2)
    # objective logging: every k_gradient<NC, true, TGV>
    for lay in ('y', 'y21', '420'):
        for w in (0.0, 0.3):
            add(f'log_{lay}_w{w}', LAYOUTS[lay], w, iters=6, log=True)
    # J2P_GRAD_SCALAR=1: every k_gradient<NC, false, TGV>; a batch keeps the packed kernel
    for lay in ('y', 'y21', '422'):
        for w in (0.0, 0.3):
            add(f'scalar_{lay}_w{w}', LAYOUTS[lay], w, switch='grad_scalar')
    add('scalar_420_batch2', LAYOUTS['420'], 0.3, nframes=2, switch='grad_scalar')
    # J2P_PROJ_TILE22=0: k_project<2,2> in place of the tile kernel (and of k_step_uncovered22)
    add('notile22_420', LAYOUTS['420'], 0.3, switch='no_tile22')
    add('notile22_420_batch2', LAYOUTS['420'], 0.3, nframes=2, switch='no_tile22')
    add('notile22_y4_cb2_cr12', Y4_CB2_CR12, 0.3, switch='no_tile22')
    add('notile22_short22', SHORT22, 0.0, switch='no_tile22')
    # the IEEE fallbacks of the projection in subsampled planes: k_project_tile22, k_project<2,1>, k_project<0,0>
    for lay in ('420', '422', 'odd'):
        for plant in ('tiny', 'patches', 'zero_coefs', 'subnormal'):
            for iters in (1, 6):
                add(f'{plant}_{lay}_x{iters}', ADV[lay], 0.3, iters=iters, plant=plant)
        # Normal luma keeps the joint TV norm O(1), so the chroma sub-gradient on a subnormal-range
        # island is itself below 2^-60 while the plane's norm stays normal: the step's quotient
        # g / norm and the residual's quotient num / q^2 both land in the subnormal range, where the
        # shared-reciprocal division can round differently from IEEE division.  Cb with the
        # DCT-distance term (residual fallback), Cr without it.
        for iters in (1, 2):
            add(f'island_{lay}_x{iters}', ADV[lay], 0.3, iters=iters, plant='island', pweight=(0.001, 0.001, 0.0))
        for extreme in ('ones', 'u16', 'coefs'):
            add(f'{extreme}_{lay}', ADV[lay], 0.3, iters=5, extreme=extreme, device_decode=extreme == 'coefs')
    add('u16_coefs_420_batch2', ADV['420'], 0.3, iters=5, extreme='u16+coefs', nframes=2, device_decode=True)
    # tall narrow frames whose last gradient band is 1..7 rows at the documented residency
    # (2 CTAs per SM for the joint builds, 5 for the one-channel builds; 132 SMs)
    h420 = K.short_last_band_heights(112, (K.GRAD_CTAS_PER_SM[3],), 2100, 4400)[0]
    h444 = K.short_last_band_heights(232, (2, 3), 2100, 4400)[0]
    h1 = K.short_last_band_heights(232, (K.GRAD_CTAS_PER_SM[1],), 5300, 6000)[0]
    add('tall_420', (G(112, h420, 1, 1), G(56, h420 // 2, 2, 2), G(56, h420 // 2, 2, 2)), 0.3, iters=3, tall=True)
    add('tall_444', (G(232, h444, 1, 1),) * 3, 0.0, iters=2, tall=True)
    add('tall_y', (G(232, h1, 1, 1),), 0.3, iters=3, tall=True)
    add('tall_420_batch2', (G(112, h420, 1, 1), G(56, h420 // 2, 2, 2), G(56, h420 // 2, 2, 2)), 0.3, iters=2, nframes=2, tall=True)
    return cases


# widths with W mod 60 in {0, 4, 56}, W mod 240 in {0, 8, 232}, and just below / above 128, 256, 512
SWEEP_WIDTHS = (120, 64, 176, 240, 248, 232, 480, 488, 472, 120, 136, 248, 264, 504, 520)


def _sweep_cases(n=40):
    cases = []
    for i in range(n):
        seed = 9000 + i
        rng = np.random.default_rng(seed)
        W = SWEEP_WIDTHS[i % len(SWEEP_WIDTHS)]
        Hf = int(rng.choice([16, 24, 40, 64, 96, 136]))
        nc = int(rng.choice([1, 2, 3, 3]))
        planes = []
        for c in range(nc):
            if c == 0 and nc > 1:
                sw = sh = 1
            elif c == 2 and rng.random() < 0.6:
                planes.append(planes[1])              # Cr like Cb: planes of one geometry share a launch
                continue
            else:
                sw, sh = int(rng.integers(1, 5)), int(rng.integers(1, 5))
            cw = max(8, (W // sw) // 8 * 8)
            ch = max(8, (Hf // sh) // 8 * 8)
            if rng.random() < 0.3 and cw > 8:
                cw -= 8                               # stops short of the frame on the right
            if rng.random() < 0.3 and ch > 8:
                ch -= 8                               # ... or at the bottom
            planes.append(G(cw, ch, sw, sh))
        weight = float(rng.choice([0.0, 0.3]))
        pweight = tuple(float(x) for x in rng.choice([0.0, 0.001, 0.01], size=nc))
        iters = int(rng.integers(1, 26))
        nframes = 2 if i % 8 == 7 else 1
        cases.append(Case(f'sweep{i}', tuple(planes), weight, pweight, iters, nframes=nframes, seed=seed, sweep=True))
    return cases


NAMED = _named_cases()
SWEEP = _sweep_cases()
CASES = NAMED + SWEEP


# ---- running one case ------------------------------------------------------------------------
def _plant(case, fd, rng):
    """The plantings of test_gpu_parity.test_guard_fallback_rows, on the caller's decode."""
    if case.plant == 'tiny':                  # every FISTA value far below 2^-35, some exactly 0
        return [(p * np.float32(2.0 ** -60) * (rng.random(p.shape) < 0.8)).astype(np.float32) for p in fd]
    if case.plant == 'patches':               # denormal, tiny and huge islands in a normal image
        for p, v in zip(fd, (1e-42, 3e-13, 4e21)):
            # the rows and columns of the 200 x 72 original, scaled to the plane
            h, w = p.shape
            r = lambda y: y * h // 72
            c = lambda x: x * w // 200
            spots = [(slice(r(10), r(14)), slice(c(30), c(90))), (slice(r(40), r(40) + 1), slice(0, w)),
                     (slice(r(50), r(60)), slice(c(100), c(104)))]
            assert all(p[s].size for s in spots), f'a patch misses the {w}x{h} plane'
            p[spots[0]] = np.float32(v) * rng.standard_normal(p[spots[0]].shape).astype(np.float32)
            p[spots[1]] = np.float32(v)
            p[spots[2]] = 0.0
        return fd
    if case.plant == 'island':                # chroma: subnormal-range values on whole coefficient blocks
        for p in fd[1:]:
            isl = _island(p.shape)
            mag = np.exp2(rng.uniform(-140, -112, p[isl].shape))
            p[isl] = (np.where(rng.random(mag.shape) < 0.5, -mag, mag)).astype(np.float32)
            assert (p[isl] != 0).mean() > 0.9
        return fd
    if case.plant == 'zero_coefs':            # all-zero coefficients, unit tables: tiny values survive the projection
        return [(rng.standard_normal(p.shape) * 1e-14).astype(np.float32) for p in fd]
    if case.plant == 'subnormal':             # all-zero coefficients, tables of 3..255: residuals below 2^-60, quotients subnormal
        return [(rng.standard_normal(p.shape) * 10.0 ** rng.uniform(-44, -20, p.shape)).astype(np.float32) for p in fd]
    return fd


def _island(shape):
    """Interior coefficient blocks of a plane (two blocks from every edge): the island of 'island'."""
    h, w = shape
    return slice(16, max(24, h - 16)), slice(16, max(24, w - 16))


def build_frames(case):
    """(frames, caller decodes per frame) of a case; deterministic in case.seed."""
    frames, fdata = [], []
    for f in range(case.nframes):
        img = synth.random_coefs([(p.cw, p.ch) for p in case.planes], [(p.sw, p.sh) for p in case.planes],
                                 case.seed * 16 + f)
        rng = np.random.default_rng(case.seed * 16 + f + 1)
        for pl in img.planes:
            if case.plant == 'zero_coefs':
                pl.data[:] = 0
                pl.quant[:] = 1
            if case.plant == 'subnormal':
                pl.data[:] = 0
                pl.quant[:] = rng.integers(3, 256, size=64).astype(np.uint16)
            if case.plant == 'island' and pl is not img.planes[0]:
                # zero coefficients on the island, small tables: the clamp keeps the tiny block values
                # (|v| <= q/2), so residuals stay below 2^-60 and their quotients by q^2 are subnormal
                blocks = pl.data.reshape(pl.h // 8, pl.w // 8, 64)
                rows, cols = _island((pl.h, pl.w))
                blocks[rows.start // 8:rows.stop // 8, cols.start // 8:cols.stop // 8] = 0
                pl.quant[:] = rng.choice([3, 5, 6, 7], size=64).astype(np.uint16)
            if 'ones' in case.extreme:
                pl.quant[:] = 1
            if 'u16' in case.extreme:             # q*q is inexact in fp32 above 4096; RN(1/q^2) at its extreme
                pl.quant[:] = rng.integers(1, 65536, size=64).astype(np.uint16)
                pl.quant[rng.integers(0, 64, size=8)] = 65535
                pl.quant[0] = 65535
            if 'coefs' in case.extreme:
                n = pl.data.size
                pl.data[rng.integers(0, n, size=max(1, n // 16))] = 32767
                pl.data[rng.integers(0, n, size=max(1, n // 16))] = -32768
                pl.data[0] = -32768
        frames.append(img)
        fdata.append(_plant(case, H.decode_planes(img, range(len(case.planes))), rng))
    return frames, fdata


def _checker():
    return 'ref' if H.have_ref() else 'oracle'


def tall_on_device(case):
    """The tall case with its height chosen for THIS device: the SM count from torch and the
    residency of the single-frame gradient instantiation (what grad_geometry is given, batches
    included) from the library's register and shared-memory use, so the last band is 1..7 rows."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    kernel = K.gradient_kernel(case.planes, case.weight, K.Mode())
    res = K.library_resources(abi.PRODUCT_LIB)
    assert res and kernel in res, f'no resource usage for {kernel}: the CUDA toolkit is needed to size this case'
    per_sm = K.resident_ctas(*res[kernel])
    W = K.frame_size(case.planes)[0]
    heights = K.short_last_band_heights(W, (per_sm,), 2100, 12000, sms)
    assert heights, f'no height with a short last band for {sms} SMs x {per_sm} CTAs'
    Hf = heights[0]
    planes = tuple(G(p.cw, Hf // p.sh, p.sw, p.sh) for p in case.planes)
    band = K.last_band_rows(W, Hf, sms * per_sm)
    assert 1 <= band <= 7
    return dataclasses.replace(case, planes=planes, name=f'{case.name} ({sms} SMs x {per_sm} CTAs of {kernel}: last band {band} rows)')


def run_case(lib, case):
    if case.tall:
        case = tall_on_device(case)
    frames, fdata = build_frames(case)
    nc = len(case.planes)
    chans = list(range(nc))
    mode = case.mode()
    _, per_iter = K.iteration(case.planes, case.weight, mode)
    _, n_setup = K.setup(case.planes, mode)
    what = case.describe()
    desc = abi.frame_desc(frames[0], chans, case.weight, case.pweight, case.iters)
    assert (int(desc.plane_w[0]), int(desc.plane_h[0])) == (case.planes[0].cw, case.planes[0].ch)
    log = []
    with abi.Session(lib, desc, case.nframes, batch=case.nframes > 1) as s:
        if case.log:
            assert lib.j2p_session_set_logging(s.s, 1) == 0, lib.j2p_last_error()
        s.upload(frames, chans, None if case.device_decode else [[p.copy() for p in fd] for fd in fdata])
        after_upload = s.launches
        if case.log:
            for i in range(case.iters):
                s.iterate(i, 1)
                o = (C.c_double * 4)()
                assert lib.j2p_session_objective(s.s, o) == 0, lib.j2p_last_error()
                log.append(list(o))
        else:
            s.iterate(0, case.iters)
        total = s.launches
        got = s.download()
    # a single session is armed by its last upload, a batch by its first iteration
    decodes = nc * case.nframes if case.device_decode else 0
    assert after_upload == (decodes if case.nframes > 1 else n_setup), f'{after_upload} set-up launches; {what}'
    assert total == n_setup + case.iters * per_iter, \
        f'{total - n_setup} solver launches for {case.iters} iterations, kernel_paths says {per_iter} each; {what}'
    checker = _checker()
    if 'u16' in case.extreme and checker == 'ref':
        # The reference's SIMD build converts the tables with _mm_cvtpi16_ps, a SIGNED 16-bit
        # conversion, so entries above 32767 become negative there; its scalar build, the oracle
        # and this library read struct coef's uint16_t.  The scalar build is the checker here.
        checker = 'ref_c'
    for f, img in enumerate(frames):
        want = H.run_compute(checker, img, chans, case.weight, case.pweight, case.iters, [p.copy() for p in fdata[f]])
        H.assert_bit_identical(got[f], want, f'frame {f} vs {checker}; {what};')
    if case.log:
        planes_o, log_o = H.run_compute('oracle', frames[0], chans, case.weight, case.pweight, case.iters,
                                        [p.copy() for p in fdata[0]], want_log=True)
        np.testing.assert_allclose(np.array(log), log_o, rtol=1e-9, atol=1e-12, err_msg=what)


# ---- the tests -------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def lib():
    lib = abi.load_product()
    assert lib.j2p_device_count() > 0, 'no CUDA device visible: the product has no CPU fallback'
    return lib


@pytest.mark.gpu
@pytest.mark.parametrize('case', [c for c in NAMED if not c.switch], ids=lambda c: c.name)
def test_named_case_matches_checker(lib, case):
    run_case(lib, case)


@pytest.mark.gpu
@pytest.mark.parametrize('case', SWEEP, ids=lambda c: c.name)
def test_geometry_sweep_matches_checker(lib, case):
    run_case(lib, case)


_SWITCH_CHILD = r'''
import sys
sys.path.insert(0, sys.argv[1])
from jpeg2png_b200 import abi
from tests import test_gpu_kernel_matrix as M
lib = abi.load_product()
cases = [c for c in M.NAMED if c.switch == sys.argv[2]]
for c in cases:
    M.run_case(lib, c)
print('switch cases ok', len(cases))
'''

_SWITCH_ENV = {'grad_scalar': ('J2P_GRAD_SCALAR', '1'), 'no_tile22': ('J2P_PROJ_TILE22', '0')}


@pytest.mark.gpu
@pytest.mark.parametrize('switch', sorted(_SWITCH_ENV))
def test_switch_cases_match_checker(switch):
    """The A/B switches are read once per process: their cases run in a child process."""
    var, val = _SWITCH_ENV[switch]
    env = dict(os.environ, **{var: val})
    r = subprocess.run([sys.executable, '-c', _SWITCH_CHILD, H.ROOT, switch], capture_output=True, text=True,
                       env=env, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert 'switch cases ok' in r.stdout
