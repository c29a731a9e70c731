"""Row-strip sessions on ONE GPU (pytest -m gpu): several strips of a frame on device 0, driven in
lock step by this process (tests/strip_backend.LockStep), so the strip-mode arithmetic of every
solver kernel is checked on a one-GPU box.  tests/test_gpu_strips.py needs 2, 4 or 8 GPUs.

The sessions are never bound to a j2p_comm: StripSync::nranks stays 0, so the kernels never wait on
flags, and the host does what the NCCL fallback queues between the kernels (gather the sums in rank
order, fold them in j2p_session_project, copy the border rows to the neighbours).

Every case makes two checks:
  (a) step by step against N oracle strips (tests/strip_backend.OracleStrip).  Both projections are
      fed the ORACLE's gathered sums, which takes the association of the sums (DESIGN.md §3) out of
      the comparison: after every iteration the owned rows of every strip must match the oracle's
      bit for bit, and each strip's sums of g^2 must lie within the rigorous bound for one set of
      non-negative fp64 summands added in two different orders.
  (b) end to end: the product strips fold their own sums, and the concatenated result must match
      the checker's compute() (the compiled reference where it was built, else the oracle) bit for
      bit.
and compares each strip's launch count with tests/kernel_paths.py in strip mode.  The A/B switches
(J2P_PROJ_TMA=1, J2P_GRAD_SCALAR=1, J2P_PROJ_TILE22=0) are read once per process: their cases run in
child processes.  tests/test_kernel_coverage.py checks (no GPU) that the named cases reach every
kernel a strip session can launch.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import os
import subprocess
import sys

import numpy as np
import pytest

from jpeg2png_b200 import abi, strips
from tests import helpers as H
from tests import kernel_paths as K
from tests import test_gpu_kernel_matrix as M
from tests.strip_backend import LockStep, OracleStrip, cuts_to_strips, fold

G = K.PlaneGeom


@dataclasses.dataclass(frozen=True)
class StripCase:
    name: str
    purpose: str
    planes: tuple                 # PlaneGeom per channel (the whole frame)
    weight: float
    pweight: tuple
    iters: int
    n: int = 0                    # strips.plan_strips into n strips, or
    cuts: tuple = ()              # explicit MCU-aligned cut rows
    plant: str = ''               # a planting of test_gpu_kernel_matrix._plant
    switch: str = ''              # '' | 'tma' | 'grad_scalar' | 'no_tile22' (child processes)
    device_decode: bool = False   # upload without the caller's decode (k_decode on the device)
    tall: bool = False            # strip heights re-chosen on the device: last gradient band 1..7 rows
    oracle: str = 'every'         # 'every' iteration | 'ends': iterations 1, 2 and the last | 'none': (b) only
    reset: bool = False           # re-solve after j2p_session_reset over poisoned stale halo rows
    seed: int = 0

    def plan(self):
        Hf = K.frame_size(self.planes)[1]
        if self.cuts:
            return cuts_to_strips(Hf, self.cuts)
        return strips.plan_strips(Hf, 8 * max(p.sh for p in self.planes), self.n)

    def mode(self, strip) -> K.Mode:
        return K.Mode(strip=tuple(strip), grad_scalar=self.switch == 'grad_scalar', tile22=self.switch != 'no_tile22',
                      tma=self.switch == 'tma', device_decode=self.device_decode)

    def matrix_case(self) -> M.Case:
        return M.Case(self.name, self.planes, self.weight, self.pweight, self.iters, plant=self.plant, seed=self.seed)

    def describe(self) -> str:
        W, Hf = K.frame_size(self.planes)
        pl = ', '.join(f'{p.cw}x{p.ch}@({p.sw},{p.sh})' for p in self.planes)
        return (f'{self.name} ({self.purpose}): frame {W}x{Hf}, planes [{pl}], strips {self.plan()}, weight {self.weight}, '
                f'pweight {list(self.pweight)}, {self.iters} iterations, switch {self.switch or "-"}, plant {self.plant or "-"}, '
                f'device decode {self.device_decode}, seed {self.seed}')


# ---- frames --------------------------------------------------------------------------------------
C420 = (G(96, 128, 1, 1), G(48, 64, 2, 2), G(48, 64, 2, 2))              # eight 16-row MCU rows
ODD34 = (G(40, 72, 1, 1), G(24, 48, 2, 2), G(16, 24, 3, 4))              # 32-row MCUs, three of them
ODD32 = (G(48, 48, 1, 1), G(16, 24, 3, 2), G(16, 48, 3, 1))
# three 1x1 planes, the last 8 rows short: the whole frame and the last 8-row-aligned strip take the
# generic gradient (and project plane 2 on its own); interior strips take the `full` instantiation
# and project all three planes in one launch
DISPATCH = (G(64, 48, 1, 1), G(64, 48, 1, 1), G(64, 40, 1, 1))
# luma 1928 wide in a 1936-wide frame: stepped-only columns in every strip
UNCOVERED = (G(1928, 64, 1, 1), G(968, 32, 2, 2), G(968, 32, 2, 2))
# the 1080p shape: luma grid 8 rows short of the frame; with 16-row strips the last one has 8 luma rows
LUMA_SHORT = M.LAYOUTS['420']


def _tall_template(nc):
    return (G(112, 16, 1, 1), G(56, 8, 2, 2), G(56, 8, 2, 2)) if nc == 3 else (G(232, 16, 1, 1),)


def tall_geometry(template, weight, sms, per_sm):
    """Two strips whose owned rows each give a last gradient band of 1..7 rows at `per_sm` resident
    CTAs on `sms` SMs: (whole-frame planes, cuts)."""
    W = K.frame_size(template)[0]
    lo = 2100 if per_sm <= 2 else 5300
    hs = K.short_last_band_heights(W, (per_sm,), lo, lo + 8000, sms)
    assert len(hs) >= 2, f'no strip heights with a short last band for {sms} SMs x {per_sm} CTAs'
    h1, h2 = hs[0], hs[1]
    return tuple(G(p.cw, (h1 + h2) // p.sh, p.sw, p.sh) for p in template), (h1,)


def _named_cases():
    cases = []
    seed = 500

    def add(name, purpose, planes, weight=0.3, iters=8, pweight=None, **kw):
        nonlocal seed
        seed += 1
        pw = tuple(pweight) if pweight is not None else (0.001,) * len(planes)
        cases.append(StripCase(name, purpose, tuple(planes), weight, pw, iters, seed=seed, **kw))

    for n in (2, 3, 5, 8):
        add(f'c420_n{n}', f'4:2:0 in {n} even strips' + (' (one 16-row MCU each)' if n == 8 else ''), C420, n=n)
    add('c444_8row', '4:4:4 in 8-row strips, the smallest the ABI accepts', M.LAYOUTS['444'], cuts=(8, 16, 24, 32, 40))
    add('uneven_first', 'one MCU row, then the rest', C420, cuts=(16,))
    add('uneven_last', 'the rest, then one MCU row', C420, cuts=(112,))
    add('luma_short', 'luma 8 rows short: the last strip has 8 of its 16 rows in luma (GPM 2 gp-row guards)', LUMA_SHORT, cuts=(16, 32))
    add('dispatch', 'interior strips take the full gradient and one projection launch, the last strip the generic ones',
        DISPATCH, cuts=(16, 32))
    add('uncovered_cols', 'luma 1928 in a 1936 frame: k_step_uncovered in every strip', UNCOVERED, n=4)
    add('short22_last', 'chroma grid ends in the last strip: k_step_uncovered22 there only', M.SHORT22, cuts=(16,))
    # every packed gradient instantiation (channels x full / 4:2:0 / generic x TGV) and projection kernel
    for lay in ('y', 's21', 's12', 'yy', 'y21', '444', '422', '440', '411', '420'):
        for w in (0.0, 0.3):
            pw = (0.001, 0.0, 0.01) if lay == '422' and w else None      # a plane without the DCT-distance term
            add(f'{lay}_w{w}', f'layout {lay}, TGV weight {w}' + (', Cb pweight 0' if pw else ''), M.LAYOUTS[lay], w,
                pweight=pw, n=3, device_decode=lay == '420' and w == 0.0)
    add('odd34', '(3,4) chroma: 32-row MCUs', ODD34, 0.4, n=3)
    add('odd32', '(3,2) and (3,1) chroma', ODD32, 0.4, n=3)
    add('y4_cb2_cr12', 'a (2,2) plane narrower than the frame: k_step_uncovered22 in every strip', M.Y4_CB2_CR12, n=3)
    # the plantings of test_guard_fallback_rows, cut through the planted rows
    adv_cuts = {'420': (80, 112),    # luma patch row 80 and chroma rows 80-81 at a border; rows 111 | 112 113 across one
                '422': (40, 56),     # the one-row patch at row 40 is a border row; 50..59 straddle 56
                'odd': (32, 64)}
    for lay, cuts in adv_cuts.items():
        for plant in ('tiny', 'patches', 'zero_coefs', 'subnormal'):
            add(f'{plant}_{lay}', f'planting {plant}, cuts through the planted rows', M.ADV[lay], iters=6, plant=plant, cuts=cuts)
        add(f'island_{lay}', 'planting island: subnormal quotients in the chroma steps', M.ADV[lay], iters=2, plant='island',
            pweight=(0.001, 0.001, 0.0), cuts=cuts)
    # strips whose last gradient band is 1..7 rows (nominal geometry here; re-chosen on the device)
    for nm, nc, w, iters in (('tall_420', 3, 0.3, 3), ('tall_444', 3, 0.0, 2), ('tall_y', 1, 0.3, 3)):
        tmpl = _tall_template(nc) if nm != 'tall_444' else (G(232, 16, 1, 1),) * 3
        per_sm = K.GRAD_CTAS_PER_SM[nc]
        planes, cuts = tall_geometry(tmpl, w, K.H100_SMS, per_sm)
        add(nm, 'two strips, each with a last gradient band of 1..7 rows', planes, w, iters=iters, cuts=cuts, tall=True,
            oracle='ends')
    add('reset', 're-solve after j2p_session_reset over NaN-poisoned stale halo rows', C420, iters=5, n=3, reset=True)
    # child processes
    for nm, planes, n in (('444', M.LAYOUTS['444'], 3), ('luma_short', LUMA_SHORT, 3), ('dispatch', DISPATCH, 3),
                          ('uncovered_cols', UNCOVERED, 2)):
        add(f'tma_{nm}', 'J2P_PROJ_TMA=1: the TMA projection adds the strip offset itself', planes, n=n, switch='tma')
    for lay in ('y', 'y21', '420'):
        for w in (0.0, 0.3):
            add(f'scalar_{lay}_w{w}', 'J2P_GRAD_SCALAR=1: the scalar gradient in strips', M.LAYOUTS[lay], w, n=3,
                switch='grad_scalar')
    for nm, planes, cuts in (('420', M.LAYOUTS['420'], (32,)), ('y4_cb2_cr12', M.Y4_CB2_CR12, (16,)),
                             ('short22', M.SHORT22, (16,))):
        add(f'notile22_{nm}', 'J2P_PROJ_TILE22=0: k_project<2, 2> on the owned rows', planes, cuts=cuts, switch='no_tile22')
    return cases


NAMED = _named_cases()
BY_NAME = {c.name: c for c in NAMED}
# BASELINE config 4's frame in 8 strips: the strong-scaling workload of bench.py, (b) only
C8K = dict(w=7680, h=4320, q=10, ss='4:2:0', weight=0.3, pw=[0.001] * 3, iters=10)


# ---- running one case ------------------------------------------------------------------------
def tall_on_device(case):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    kernel = K.gradient_kernel(case.planes, case.weight, K.Mode())
    res = K.library_resources(abi.PRODUCT_LIB)
    assert res and kernel in res, f'no resource usage for {kernel}: the CUDA toolkit is needed to size this case'
    per_sm = K.resident_ctas(*res[kernel])
    tmpl = tuple(G(p.cw, 16 // p.sh, p.sw, p.sh) for p in case.planes)
    planes, cuts = tall_geometry(tmpl, case.weight, sms, per_sm)
    W = K.frame_size(planes)[0]
    bands = [K.last_band_rows(W, rows, sms * per_sm) for _, rows in cuts_to_strips(K.frame_size(planes)[1], cuts)]
    assert all(1 <= b <= 7 for b in bands), bands
    return dataclasses.replace(case, planes=planes, cuts=cuts,
                               name=f'{case.name} ({sms} SMs x {per_sm} CTAs of {kernel}: last bands {bands} rows)')


def _row_kind(case, plan, i, r, W):
    """Where local owned row r of strip i sits: next to a cut, in the last gradient band."""
    rows = plan[i][1]
    up, down = i > 0, i + 1 < len(plan)
    kinds = []
    if (up and r < 2) or (down and r >= rows - 2):
        kinds.append('border row (sent to a neighbour)')
    elif (up and r < 4) or (down and r >= rows - 4):
        kinds.append('halo-adjacent row (its stencil reads halo rows)')
    res = K.library_resources(abi.PRODUCT_LIB) or {}
    kernel = K.gradient_kernel(case.planes, case.weight, case.mode(plan[i]))
    if kernel in res:
        import torch
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        _, bands, band_rows = K.grad_geometry(W, rows, sms * K.resident_ctas(*res[kernel]))
        if r >= (bands - 1) * band_rows:
            kinds.append(f'in the last gradient band ({rows - (bands - 1) * band_rows} rows)')
    return ', '.join(kinds) or 'interior row'


def _gamma(k):
    u = 2.0 ** -53
    return k * u / (1 - k * u)


def _make_product(lib, case, img, fd, plan):
    fdata = None if case.device_decode else fd
    return [strips.ProductStrip(lib, img, case.weight, case.pweight, case.iters, row0, rows, 0, fdata=fdata)
            for row0, rows in plan]


def _check_launches(lib, case, plan, prod, iters, arms, what):
    for i, (strip, s) in enumerate(zip(plan, prod)):
        mode = case.mode(strip)
        _, n_setup = K.setup(case.planes, mode)
        _, per_iter = K.iteration(case.planes, case.weight, mode)
        n_init = len(case.planes)
        want = n_setup + (arms - 1) * n_init + iters * per_iter
        got = lib.j2p_session_launches(s.s)
        assert got == want, (f'strip {i} {strip}: {got} launches, kernel_paths says {want} '
                             f'({n_setup} set-up, {per_iter} per iteration, {arms} arms); {what}')


def run_a(lib, case, img, fd, plan):
    """Check (a).  Returns the oracle's gathered sums of every iteration."""
    import torch
    what = case.describe()
    prod = _make_product(lib, case, img, fd, plan)
    orc = [OracleStrip(img, case.weight, case.pweight, case.iters, row0, rows, fd) for row0, rows in plan]
    try:
        _check_launches(lib, case, plan, prod, 0, 1, what)
        pd = LockStep(prod, torch.cuda.synchronize, torch.device('cuda', 0))
        od = LockStep(orc)
        pd.start()
        od.start()
        W, N, nc = prod[0].width, len(plan), len(case.planes)
        history = []
        for it in range(1, case.iters + 1):
            gp = pd.gradient().cpu().numpy()
            go = od.gradient()
            history.append(go.numpy().copy())
            for i, (_, rows) in enumerate(plan):
                n = W * rows
                for c in range(nc):
                    sp, so = float(gp[3 * i + c]), float(go[3 * i + c])
                    bound = 2 * _gamma(n - 1) * so
                    assert abs(sp - so) <= bound, (f'iteration {it}, strip {i} {plan[i]}, plane {c}: sum of g^2 {sp!r}, '
                                                   f'oracle {so!r}, |diff| {abs(sp - so)!r} > bound {bound!r}; {what}')
            pd.project(go)
            od.project(go)
            if case.oracle == 'every' or it in (1, 2, case.iters):
                for i in range(N):
                    for c in range(nc):
                        a, b = H.bits(prod[i].download(c)), H.bits(orc[i].download(c))
                        diff = np.argwhere(a != b)
                        if diff.size:
                            r, x = (int(v) for v in diff[0])
                            raise AssertionError(
                                f'(a) first difference: iteration {it}, strip {i} {plan[i]}, plane {c}, local row {r} '
                                f'({_row_kind(case, plan, i, r, W)}), column {x}: {int(a[r, x]):#010x} vs oracle {int(b[r, x]):#010x}; '
                                f'{int((a != b).sum())} samples differ in that plane; {what}')
        _check_launches(lib, case, plan, prod, case.iters, 1, what)
        return history
    finally:
        for s in prod + orc:
            s.close()


def run_b(lib, case, img, fd, plan, history=None):
    """Check (b); `history`: the oracle's gathered sums from (a), to name a DESIGN §3 flip."""
    import torch
    what = case.describe()
    prod = _make_product(lib, case, img, fd, plan)
    try:
        pd = LockStep(prod, torch.cuda.synchronize, torch.device('cuda', 0))
        pd.start()
        own = []
        for _ in range(case.iters):
            g = pd.gradient()
            own.append(g.cpu().numpy())
            pd.project(g)
        got = pd.download()
        _check_launches(lib, case, plan, prod, case.iters, 1, what)
        if case.reset:
            # Stale halo rows must never be read: after an odd number of iterations the buffer that
            # becomes x_{-1} on re-arming is the current iterate; poison its halo rows (and, after the
            # reset, those of the new x_0) with NaN.  The fresh exchange and copy_halo_to_prev must
            # overwrite every one of them.
            assert case.iters % 2 == 1
            nan = float('nan')

            def poison():
                torch.cuda.synchronize()
                for s in prod:
                    for c in range(s.nc):
                        for side in (0, 1):
                            h = s.halo(c, side)
                            if h is not None:
                                h[1].fill_(nan)
                torch.cuda.synchronize()

            poison()
            for s in prod:
                assert lib.j2p_session_reset(s.s) == 0, lib.j2p_last_error().decode()
            poison()
            pd.start()
            for _ in range(case.iters):
                pd.project(pd.gradient())
            again = pd.download()
            H.assert_bit_identical(again, got, f'second solve after j2p_session_reset vs the first; {what}')
            _check_launches(lib, case, plan, prod, 2 * case.iters, 2, what)
    finally:
        for s in prod:
            s.close()
    checker = M._checker()
    want = H.run_compute(checker, img, list(range(len(case.planes))), case.weight, case.pweight, case.iters,
                         [p.copy() for p in fd])
    try:
        H.assert_bit_identical(got, want, f'(b) {len(plan)} strips folding their own sums vs {checker}; {what}')
    except AssertionError as e:
        if history is None:
            raise
        N, nc = len(plan), len(case.planes)
        flips = [(it + 1, c) for it in range(case.iters) for c in range(nc)
                 if fold(own[it], N, c) != fold(history[it], N, c)]
        if flips:
            it, c = flips[0]
            raise AssertionError(f'{e}\n(a) passed: this is the DESIGN.md §3 association flip: sqrtf((float)sum) of plane {c} '
                                 f'differs between the product\'s fold and the oracle\'s at iteration {it}') from None
        raise AssertionError(f'{e}\n(a) passed and no iteration\'s folded norm differs from the oracle\'s: not the §3 flip') from None


def run_case(lib, case):
    if case.tall:
        case = tall_on_device(case)
    frames, fdata = M.build_frames(case.matrix_case())
    img, fd = frames[0], fdata[0]
    plan = case.plan()
    history = run_a(lib, case, img, fd, plan) if case.oracle != 'none' else None
    run_b(lib, case, img, fd, plan, history)


# ---- the tests -------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def lib():
    lib = abi.load_product()
    assert lib.j2p_device_count() > 0, 'no CUDA device visible: the product has no CPU fallback'
    return lib


@pytest.mark.gpu
@pytest.mark.parametrize('case', [c for c in NAMED if not c.switch], ids=lambda c: c.name)
def test_strips_on_one_device(lib, case):
    run_case(lib, case)


@pytest.mark.gpu
def test_8k_frame_in_8_strips_on_one_device(lib):
    """7680x4320 4:2:0, 8 strips, 10 iterations, against the checker (check (b) only)."""
    from jpeg2png_b200 import synth
    base = synth.synth_coefs(-(-C8K['w'] // 64) * 16, -(-C8K['h'] // 64) * 16, C8K['q'], C8K['ss'], seed=1238)
    img = synth.tile_coefs(base, 4, 4, C8K['w'], C8K['h'])
    planes = tuple(G(p.w, p.h, p.w_samp, p.h_samp) for p in img.planes)
    case = StripCase('8k', 'BASELINE config 4 in 8 strips', planes, C8K['weight'], tuple(C8K['pw']), C8K['iters'], n=8,
                     device_decode=True, oracle='none')
    fd = H.decode_planes(img)
    run_b(lib, case, img, fd, case.plan())


_SWITCH_CHILD = r'''
import sys
sys.path.insert(0, sys.argv[1])
from jpeg2png_b200 import abi
from tests import test_gpu_strips_one_device as S
lib = abi.load_product()
cases = [c for c in S.NAMED if c.switch == sys.argv[2]]
for c in cases:
    S.run_case(lib, c)
print('switch cases ok', len(cases))
'''

_SWITCH_ENV = {'tma': ('J2P_PROJ_TMA', '1'), 'grad_scalar': ('J2P_GRAD_SCALAR', '1'), 'no_tile22': ('J2P_PROJ_TILE22', '0')}


@pytest.mark.gpu
@pytest.mark.parametrize('switch', sorted(_SWITCH_ENV))
def test_switch_strip_cases(switch):
    """The A/B switches are read once per process: their cases run in a child process."""
    var, val = _SWITCH_ENV[switch]
    env = dict(os.environ, **{var: val})
    r = subprocess.run([sys.executable, '-c', _SWITCH_CHILD, H.ROOT, switch], capture_output=True, text=True,
                       env=env, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert 'switch cases ok' in r.stdout


@pytest.mark.gpu
def test_strip_refusals(lib):
    """What a strip session refuses, once each."""
    def desc(planes):
        img = M.build_frames(M.Case('r', tuple(planes), 0.3, (0.001,) * len(planes), 1))[0][0]
        return img, abi.frame_desc(img, list(range(len(planes))), 0.3, [0.001] * len(planes), 1)

    def create(d, row0, rows):
        s = C.c_void_p()
        rc = lib.j2p_session_create_strip(C.byref(s), 0, C.byref(d), row0, rows)
        return rc, s

    _, d420 = desc(C420)
    rc, _ = create(d420, 8, 16)                               # 4:2:0 chroma blocks are 16 frame rows
    assert rc != 0 and b'not aligned' in lib.j2p_last_error()
    rc, _ = create(d420, 16, 24)
    assert rc != 0 and b'not aligned' in lib.j2p_last_error()
    _, d22 = desc(M.SHORT22)                                  # chroma covers frame rows 0..31 of 48
    rc, _ = create(d22, 32, 16)
    assert rc != 0 and b'starts below' in lib.j2p_last_error()

    img, _ = desc(C420)
    s = strips.ProductStrip(lib, img, 0.3, [0.001] * 3, 1, 16, 32, 0)
    try:
        p = s.s
        assert lib.j2p_session_iterate(p, 0, 1) != 0 and b'strip session' in lib.j2p_last_error()
        assert lib.j2p_session_set_logging(p, 1) != 0 and b'strip' in lib.j2p_last_error()
        buf = (C.c_ubyte * (16 * (96 * 3 + 1)))()
        assert lib.j2p_session_download_scanlines(p, 96, 16, 8, buf) != 0 and b'whole-frame' in lib.j2p_last_error()
        o = abi.ImageOut()
        assert lib.j2p_session_export(p, 0, 1, C.byref(o), C.cast(buf, C.c_void_p), None) != 0
        assert b'whole-frame' in lib.j2p_last_error()
        sums = (C.c_double * 6)()
        assert lib.j2p_session_project(p, C.cast(sums, C.c_void_p), 0) != 0 and b'bad argument' in lib.j2p_last_error()
        sp, rp, n = C.c_void_p(), C.c_void_p(), C.c_size_t()
        assert lib.j2p_session_halo(p, 0, 2, C.byref(sp), C.byref(rp), C.byref(n)) != 0
        assert b'bad channel or side' in lib.j2p_last_error()
        assert lib.j2p_session_halo(p, 3, 0, C.byref(sp), C.byref(rp), C.byref(n)) != 0
        assert b'bad channel or side' in lib.j2p_last_error()
        assert lib.j2p_session_halo(p, 2, 1, C.byref(sp), C.byref(rp), C.byref(n)) == 0 and n.value == 2 * 96
    finally:
        s.close()
