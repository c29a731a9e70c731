"""Solver parameters on the GPU (pytest -m gpu): every regime of tests/solver_param_cases.py (step norms
inside, on and above the 2^40 guard of the shared-reciprocal division, overflowed norms, partly and
wholly NaN results, negative, -0 and subnormal weights, separate planes in different regimes, and
runs of thousands of iterations) through every solver kernel family that can see it, compared with
the checker (the compiled reference where oracle/_ref was built, else the oracle): the same NaN
positions and the same bits on every other sample.

Families: the case's own synth frame (luma 72x56 in an 80x64 4:2:0 frame: k_project_tile,
k_project_tile22 and k_step_uncovered), and the kernel matrix's layouts with the case's weights:
4:4:4, 4:2:0 with a short luma grid, 4:2:2 and 4:4:0 chroma (k_project<2,1>, <1,2>), a chroma grid
short of the frame (k_step_uncovered22), one-plane sessions, batches and objective logging; the
J2P_GRAD_SCALAR=1, J2P_PROJ_TILE22=0 and J2P_PROJ_TMA=1 switches in child processes; two and three
row strips on one device, step by step against the oracle's strips; decode_jpeg and the command line.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from jpeg2png_b200 import abi, decode_jpeg, strips
from tests import helpers as H
from tests import kernel_paths as K
from tests import solver_param_cases as P
from tests import test_gpu_kernel_matrix as M
from tests.strip_backend import LockStep, OracleStrip, fold
from tests.test_codecs import CLI_DIR, codecs, make_jpeg, read_jpeg  # noqa: F401  (codecs is a fixture)

pytestmark = pytest.mark.gpu
G = K.PlaneGeom
same = P.assert_same_or_nan


@pytest.fixture(scope='module')
def lib():
    lib = abi.load_product()
    assert lib.j2p_device_count() > 0, 'no CUDA device visible: the product has no CPU fallback'
    return lib


def mode_of(mc) -> K.Mode:
    """kernel_paths' mode of a kernel-matrix case; `switch` may also be 'tma' (J2P_PROJ_TMA=1) here."""
    return K.Mode(nframes=mc.nframes, log=mc.log, grad_scalar=mc.switch == 'grad_scalar', tile22=mc.switch != 'no_tile22',
                  tma=mc.switch == 'tma', device_decode=mc.device_decode)


# ---- the case's own frame ---------------------------------------------------------------------
def run_own_frame(lib, case, nframes=1, switch=''):
    """Each solve of the case on its synth frame in one session (a batch of `nframes` copies when > 1),
    against the checker; also counts the launches against tests/kernel_paths.py (`switch`: the process's
    A/B switch, as in M.Case)."""
    img = case.image()
    checker = M._checker()
    want = P.run_checker(checker, case, img)
    got = []
    for s in case.solves:
        sub = P.planes_of(img, s.channels)
        n = len(s.channels)
        fd = H.decode_planes(sub, range(n))
        planes = tuple(G(p.w, p.h, p.w_samp, p.h_samp) for p in sub.planes)
        mode = mode_of(M.Case('', planes, s.weight, s.pweight, s.iters, nframes=nframes, switch=switch))
        n_setup = K.setup(planes, mode)[1] if nframes > 1 else 0      # a batch is armed by its first iteration
        desc = abi.frame_desc(sub, list(range(n)), s.weight, s.pweight, s.iters)
        with abi.Session(lib, desc, nframes, batch=nframes > 1) as ss:
            ss.upload([sub] * nframes, list(range(n)), [[p.copy() for p in fd] for _ in range(nframes)])
            before = ss.launches
            ss.iterate(0, s.iters)
            per_iter = K.iteration(planes, s.weight, mode)[1]
            assert ss.launches - before == n_setup + s.iters * per_iter, \
                f'{ss.launches - before - n_setup} launches for {s.iters} iterations, kernel_paths says {per_iter} each; {case.describe()}'
            out = ss.download()
        for f in range(1, nframes):
            same(out[f], out[0], f'batch frame {f} vs frame 0; {case.describe()}')
        got += out[0]
    same(got, want, f'{nframes} frame(s) vs {checker}; {case.describe()}')


@pytest.mark.parametrize('case', P.CASES, ids=lambda c: c.name)
def test_own_frame(lib, case):
    run_own_frame(lib, case)
    run_own_frame(lib, case, nframes=2)


# ---- the kernel matrix's layouts ----------------------------------------------------------------
JOINT_FAMILIES = {'444': M.LAYOUTS['444'], '420': M.LAYOUTS['420'], '422': M.LAYOUTS['422'], '440': M.LAYOUTS['440'],
                  'short22': M.SHORT22}
ONE_FAMILIES = {'y': M.LAYOUTS['y'], 's21': M.LAYOUTS['s21'], 's12': M.LAYOUTS['s12']}


def matrix_cases(case, switch=''):
    """The case's weights on the kernel matrix's layouts: one M.Case per (solve, layout, mode)."""
    out = []
    for k, s in enumerate(case.solves):
        fams = JOINT_FAMILIES if len(s.channels) == 3 else ONE_FAMILIES
        for lay, planes in fams.items():
            name = f'{case.name}[{k}]_{lay}'
            out.append(M.Case(name, planes, s.weight, s.pweight, s.iters, seed=700 + k, switch=switch))
            if switch:
                continue
            if lay in ('420', 'y', 'short22'):
                out.append(M.Case(name + '_batch3', planes, s.weight, s.pweight, s.iters, nframes=3, seed=710 + k))
            if lay in ('420', 'y'):
                out.append(M.Case(name + '_log', planes, s.weight, s.pweight, s.iters, log=True, seed=720 + k))
    return out


def run_matrix_case(lib, mc):
    """test_gpu_kernel_matrix.run_case for results that may hold NaN: the launch counts against
    kernel_paths, every frame against the checker with assert_same_or_nan, and the objective log
    against the oracle's (inf and NaN entries equal where they match)."""
    frames, fdata = M.build_frames(mc)
    chans = list(range(len(mc.planes)))
    mode = mode_of(mc)
    _, per_iter = K.iteration(mc.planes, mc.weight, mode)
    _, n_setup = K.setup(mc.planes, mode)
    what = mc.describe()
    desc = abi.frame_desc(frames[0], chans, mc.weight, mc.pweight, mc.iters)
    log = []
    with abi.Session(lib, desc, mc.nframes, batch=mc.nframes > 1) as s:
        if mc.log:
            assert lib.j2p_session_set_logging(s.s, 1) == 0, lib.j2p_last_error()
        s.upload(frames, chans, [[p.copy() for p in fd] for fd in fdata])
        after_upload = s.launches
        if mc.log:
            for i in range(mc.iters):
                s.iterate(i, 1)
                o = (C.c_double * 4)()
                assert lib.j2p_session_objective(s.s, o) == 0, lib.j2p_last_error()
                log.append(list(o))
        else:
            s.iterate(0, mc.iters)
        total = s.launches
        got = s.download()
    # a single session is armed by its last upload, a batch by its first iteration
    assert after_upload == (0 if mc.nframes > 1 else n_setup), f'{after_upload} set-up launches; {what}'
    assert total == n_setup + mc.iters * per_iter, \
        f'{total - n_setup} solver launches for {mc.iters} iterations, kernel_paths says {per_iter} each; {what}'
    checker = M._checker()
    for f, img in enumerate(frames):
        want = H.run_compute(checker, img, chans, mc.weight, mc.pweight, mc.iters, [p.copy() for p in fdata[f]])
        same(got[f], want, f'frame {f} vs {checker}; {what};')
    if mc.log:
        _, log_o = H.run_compute('oracle', frames[0], chans, mc.weight, mc.pweight, mc.iters,
                                 [p.copy() for p in fdata[0]], want_log=True)
        np.testing.assert_allclose(np.array(log), log_o, rtol=1e-9, atol=1e-12, err_msg=what)


@pytest.mark.parametrize('case', P.CASES, ids=lambda c: c.name)
def test_kernel_families(lib, case):
    for mc in matrix_cases(case):
        run_matrix_case(lib, mc)


_SWITCH_CHILD = r'''
import sys
sys.path.insert(0, sys.argv[1])
from jpeg2png_b200 import abi
from tests import solver_param_cases as P
from tests import test_gpu_solver_params as T
lib = abi.load_product()
n = 0
for case in P.CASES:
    T.run_own_frame(lib, case, switch=sys.argv[2])
    for mc in T.matrix_cases(case, sys.argv[2]):
        T.run_matrix_case(lib, mc)
        n += 1
print('switch cases ok', n)
'''

_SWITCH_ENV = {'grad_scalar': ('J2P_GRAD_SCALAR', '1'), 'no_tile22': ('J2P_PROJ_TILE22', '0'), 'tma': ('J2P_PROJ_TMA', '1')}


@pytest.mark.parametrize('switch', sorted(_SWITCH_ENV))
def test_switches(switch):
    """The switches are read once per process: every case runs in a child process."""
    var, val = _SWITCH_ENV[switch]
    env = dict(os.environ, **{var: val})
    r = subprocess.run([sys.executable, '-c', _SWITCH_CHILD, H.ROOT, switch], capture_output=True, text=True,
                       env=env, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert 'switch cases ok' in r.stdout


# ---- row strips on one device ---------------------------------------------------------------------
def _norms_equal(a, b):
    return (np.isnan(a) and np.isnan(b)) or a == b


@pytest.mark.parametrize('n', [2, 3])
@pytest.mark.parametrize('case', [c for c in P.CASES if not c.separate], ids=lambda c: c.name)
def test_strips_step_by_step(lib, case, n):
    """(a) Product and oracle strips fed the oracle's gathered sums: the planes after every iteration,
    NaN-aware, and the narrowed norm of the product's own sums against the oracle's, so a fold that
    narrows differently shows where it happens.  (b) The product strips folding their own sums against
    the checker."""
    img = case.image()
    s = case.solves[0]
    sub = P.planes_of(img, s.channels)
    nc = len(s.channels)
    fd = H.decode_planes(sub, range(nc))
    Hf = max(p.h * p.h_samp for p in sub.planes)
    plan = strips.plan_strips(Hf, 8 * max(p.h_samp for p in sub.planes), n)
    pw = list(s.pweight) + [0.0] * (3 - nc)
    what = f'{case.describe()}; strips {plan}'
    dev = torch.device('cuda', 0)
    prod = [strips.ProductStrip(lib, sub, s.weight, pw, s.iters, r0, rows, 0, fdata=fd) for r0, rows in plan]
    orc = [OracleStrip(sub, s.weight, pw, s.iters, r0, rows, fd) for r0, rows in plan]
    try:
        pd, od = LockStep(prod, torch.cuda.synchronize, dev), LockStep(orc)
        pd.start()
        od.start()
        for it in range(1, s.iters + 1):
            gp = pd.gradient().cpu().numpy()
            go = od.gradient()
            for c in range(nc):
                a, b = fold(gp, n, c), fold(go.numpy(), n, c)
                assert _norms_equal(a, b), f'iteration {it}, plane {c}: folded norm {a!r} vs oracle {b!r}; {what}'
            pd.project(go)
            od.project(go)
            same(pd.download(), od.download(), f'(a) iteration {it}; {what}')
    finally:
        for x in prod + orc:
            x.close()
    prod = [strips.ProductStrip(lib, sub, s.weight, pw, s.iters, r0, rows, 0, fdata=fd) for r0, rows in plan]
    try:
        pd = LockStep(prod, torch.cuda.synchronize, dev)
        pd.start()
        for _ in range(s.iters):
            pd.project(pd.gradient())
        got = pd.download()
    finally:
        for x in prod:
            x.close()
    checker = M._checker()
    same(got, H.run_compute(checker, img, list(s.channels), s.weight, s.pweight, s.iters), f'(b) vs {checker}; {what}')


# ---- long runs --------------------------------------------------------------------------------------
def _first_norm_difference(lib, img, s):
    """A long run that mismatches, re-run step by step as one strip on each side, each folding its own
    sums: the first (iteration, plane) whose narrowed norm differs, or None."""
    sub = P.planes_of(img, s.channels)
    nc = len(s.channels)
    fd = H.decode_planes(sub, range(nc))
    Hf = max(p.h * p.h_samp for p in sub.planes)
    pw = list(s.pweight) + [0.0] * (3 - nc)
    p = strips.ProductStrip(lib, sub, s.weight, pw, s.iters, 0, Hf, 0, fdata=fd)
    o = OracleStrip(sub, s.weight, pw, s.iters, 0, Hf, fd)
    try:
        pd, od = LockStep([p], torch.cuda.synchronize, torch.device('cuda', 0)), LockStep([o])
        pd.start()
        od.start()
        for it in range(1, s.iters + 1):
            gp, go = pd.gradient(), od.gradient()
            a, b = gp.cpu().numpy(), go.numpy()
            for c in range(nc):
                if not _norms_equal(fold(a, 1, c), fold(b, 1, c)):
                    return it, c, fold(a, 1, c), fold(b, 1, c)
            pd.project(gp)
            od.project(go)
    finally:
        p.close()
        o.close()
    return None


@pytest.mark.parametrize('case', P.LONG, ids=lambda c: c.name)
def test_long_runs(lib, case):
    img = case.image()
    checker = M._checker()
    for s in case.solves:
        sub = P.planes_of(img, s.channels)
        n = len(s.channels)
        desc = abi.frame_desc(sub, list(range(n)), s.weight, s.pweight, s.iters)
        with abi.Session(lib, desc, 1, batch=False) as ss:
            ss.upload([sub], list(range(n)), [H.decode_planes(sub, range(n))])
            ss.iterate(0, s.iters)
            got = ss.download()[0]
        want = H.run_compute(checker, img, list(s.channels), s.weight, s.pweight, s.iters)
        try:
            same(got, want, f'planes {list(s.channels)} x{s.iters} vs {checker}; {case.describe()}')
        except AssertionError as e:
            flip = _first_norm_difference(lib, img, s)
            if flip is None:
                raise AssertionError(f'{e}\nno iteration\'s narrowed norm differs from the oracle\'s: not the DESIGN §3 flip') from None
            raise AssertionError(f'{e}\nfirst narrowed-norm difference (iteration, plane, product, oracle): {flip}: '
                                 'the DESIGN §3 association flip') from None


# ---- decode_jpeg and the command line ---------------------------------------------------------------
def _checker_planes(img, joint, iters, weights, pweights):
    if joint:
        return H.run_compute('oracle', img, [0, 1, 2], weights[0], pweights, iters[0])
    return [H.run_compute('oracle', img, [c], weights[c], [pweights[c]], iters[c])[0] for c in range(3)]


def checker_samples(img, planes, bits):
    """The checker's C conversion (png.c:39-62 restated) of solved planes: (h, w, 3), uint8 or uint16;
    NaN samples become whatever that conversion makes of them on x86."""
    y = np.ascontiguousarray(planes[0] + np.float32(128.0), np.float32)
    cb, cr = (np.ascontiguousarray(p, np.float32) for p in planes[1:])
    out = np.zeros(img.width * img.height * 3 * bits // 8, np.uint8)
    H.load_oracle().oracle_ycc_to_rgb(img.width, img.height, bits, y.ctypes.data, y.shape[1], cb.ctypes.data, cb.shape[1],
                                      cr.ctypes.data, cr.shape[1], out.ctypes.data)
    if bits == 8:
        return out.reshape(img.height, img.width, 3)
    return out.view('>u2').astype(np.uint16).reshape(img.height, img.width, 3)


def checker_floats(img, planes):
    """The clamped float samples (png.c:44-46 before the scaling): (h, w, 3) float32, NaN passed through."""
    h, w = img.height, img.width
    y = (planes[0][:h, :w] + np.float32(128.0)).astype(np.float64)
    cb, cr = (p[:h, :w].astype(np.float64) for p in planes[1:])
    out = []
    with np.errstate(invalid='ignore', over='ignore'):
        for v in (y + 1.402 * cr, (y - 0.34414 * cb) - 0.71414 * cr, y + 1.772 * cb):
            x = v.astype(np.float32)
            x = np.where(x.astype(np.float64) > 255.0, np.float32(255.0), np.where(x.astype(np.float64) < 0.0, np.float32(0.0), x))
            out.append(x.astype(np.float32))
    return np.stack(out, axis=-1)


# name -> (joint flags, separate flags): decode_jpeg keywords; weights of -s are per plane
DECODE = {
    'above_guard_w': (dict(weight=1e12), dict(weight=(1e12, 0.3, 0.0))),
    'above_guard_p': (dict(pweight=(1e12, 0.001, 1e12)), dict(weight=(0.3, 0.0, 0.3), pweight=(1e12, 0.001, 1e12))),
    'norm_inf_w': (dict(weight=1e18), dict(weight=(1e18, 0.0, 1e18))),
    'norm_inf_p': (dict(pweight=(1e30, 0.001, 1e30)), dict(weight=(0.3, 0.3, 0.0), pweight=(1e30, 0.001, 1e30))),
    'negative': (dict(weight=-0.3, pweight=(0.001, -0.001, 0.001)), dict(weight=(-0.3, 0.0, -0.3), pweight=(0.001, -0.001, 0.001))),
    # separate: luma alone at 1e38 for one iteration leaves some of its samples NaN
    'partial_nan': (dict(weight=1e38), dict(weight=(1e38, 0.0, 0.0), iterations=(1, 6, 6))),
}


@pytest.fixture(scope='module')
def jpeg(codecs):  # noqa: F811
    """A Pillow-written 72x56 4:2:0 file and the reader's coefficients of it."""
    data = make_jpeg(72, 56, 30, '4:2:0', False, seed=5)
    img, err = read_jpeg(codecs, data)
    assert img is not None, err
    return data, img


def _flags(kw, sep):
    it = kw.get('iterations', 6)
    w = kw.get('weight', 0.3)
    pw = kw.get('pweight', 0.001)
    weights = list(w) if sep else [w, 0.0, 0.0]
    pweights = list(pw) if isinstance(pw, tuple) else [pw] * 3
    return list(it) if isinstance(it, tuple) else [it] * 3, weights, pweights


@pytest.mark.parametrize('sep', [False, True], ids=['joint', 'separate'])
@pytest.mark.parametrize('name', list(DECODE))
def test_decode_jpeg(jpeg, name, sep):
    data, img = jpeg
    kw = {'iterations': 6, **DECODE[name][1 if sep else 0]}
    iters, weights, pweights = _flags(kw, sep)
    planes = _checker_planes(img, not sep, iters, weights, pweights)
    what = f'{name} {"separate" if sep else "joint"}: {kw}'
    for dtype, bits in ((torch.uint8, 8), (torch.uint16, 16)):
        got = decode_jpeg(data, separate=sep, dtype=dtype, layout='HWC', **kw).cpu().numpy()
        want = checker_samples(img, planes, bits)
        assert (got == want).all(), f'{dtype}: {int((got != want).sum())} of {got.size} samples differ; {what}'
    got = decode_jpeg(data, separate=sep, dtype=torch.float32, layout='HWC', **kw).cpu().numpy()
    same([got], [checker_floats(img, planes)], f'float32; {what}')


CLI_ARGS = [['-w', '-0.3'], ['-w', '1e12'], ['-w', '1e40'], ['-w', 'nan'], ['-p', '1e30']]


@pytest.mark.parametrize('sep', [False, True], ids=['joint', 'separate'])
@pytest.mark.parametrize('args', CLI_ARGS, ids=lambda a: ' '.join(a))
def test_cli(jpeg, tmp_path, args, sep):
    from PIL import Image
    data, img = jpeg
    subprocess.run(['make', '-C', CLI_DIR, 'jpeg2png'], check=True, capture_output=True)
    src = tmp_path / 'in.jpg'
    src.write_bytes(data)
    r = subprocess.run([os.path.join(CLI_DIR, 'jpeg2png'), '-q', '-i', '6', *(['-s'] if sep else []), *args, str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = np.asarray(Image.open(tmp_path / 'in.png'))
    w = float(args[1]) if args[0] == '-w' else 0.3
    pw = float(args[1]) if args[0] == '-p' else 0.001
    planes = _checker_planes(img, not sep, [6] * 3, [w, 0.0, 0.0], [pw] * 3)
    want = checker_samples(img, planes, 8)
    assert (got == want).all(), f'{args}: {int((got != want).sum())} of {got.size} samples differ'
