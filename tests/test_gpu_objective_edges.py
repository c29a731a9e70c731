"""The recording kernels (libj2pobjective.so) at the solver's edges (pytest -m gpu): every case of
tests/objective_edge_cases.py recorded, compared with the unrecorded solve and with the checker.

Planes: the recorded planes equal the unrecorded batch's and the checker's (the compiled reference
where oracle/_ref was built, else the oracle): the same NaN positions and the same bits on every other
sample (solver_param_cases.assert_same_or_nan).  A recording session's planes are what
decode_jpeg(..., return_objective=True) returns, so a recording kernel that rounded one fallback
differently would change the user's pixels.

History against the oracle's log (`assert_history`), per frame and iteration:
  - NaN positions are equal; NaN signs and payloads are not compared (DESIGN §8);
  - infinities are equal, sign included;
  - prob_dist, tv and tv2 are each a sum of terms of one sign (a float product a·norm widened to
    double, or a square): each is compared at rtol 1e-9, where only the order of the fp64 sums differs;
  - the objective (tv + tv2 + prob_dist) / total_alpha can cancel (a negative weight makes tv2 <= 0
    while tv >= 0), so it is compared against 1e-9 times the sum of its terms' magnitudes over
    |total_alpha|, not against itself;
  - iteration 0's prob_dist is exactly 0, and tv2 is exactly 0 without TGV.
Batch independence: a frame's history and planes are bit-identical alone and anywhere in a batch
(objective.cu: every recording kernel runs with batch addressing).  Launch counts: the recording
dispatch restated in tests/objective_edge_cases.py, the row split and the per-frame generic launches included.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import jpeg2png_b200
from jpeg2png_b200 import abi, decode_jpeg
from tests import helpers as H
from tests import objective_edge_cases as E
from tests import solver_param_cases as P
from tests import test_gpu_kernel_matrix as M
from tests import test_gpu_limits as L
from tests.test_codecs import CLI_DIR, codecs  # noqa: F401  (codecs is a fixture)
from tests.test_gpu_solver_params import CLI_ARGS, DECODE, _flags, jpeg  # noqa: F401  (jpeg is a fixture)

pytestmark = pytest.mark.gpu
RTOL = 1e-9                                  # test_gpu_objective.py, test_gpu_parity.py::test_objective_log_matches_oracle
same = P.assert_same_or_nan


@pytest.fixture(scope='module')
def lib():
    lib = abi.load_product()
    assert lib.j2p_device_count() > 0, 'no CUDA device visible: the product has no CPU fallback'
    return lib


def _check(lib, rc):
    assert rc == 0, lib.j2p_last_error().decode()


def total_alpha(weight, pweight):
    """objective_terms' total_alpha (session.cu, compute.c:244-260), in float."""
    ta = np.float32(0.0)
    for p in pweight:
        if p != 0.0:
            ta = np.float32(ta + np.float32(p))
    nc = np.float32(len(pweight))
    ta = np.float32(ta + nc)
    if weight != 0.0:
        with np.errstate(over='ignore', invalid='ignore'):
            ta = np.float32(ta + np.float32(np.float32(weight) / np.sqrt(np.float32(2.0))) * nc)
    return float(ta)


def assert_history(got, want, weight, pweight, what):
    """One frame's recorded history (iterations, 4) against the oracle's log, by the contract above."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, f'{what}: history {got.shape} vs log {want.shape}'
    cols = ('objective', 'prob_dist', 'tv', 'tv2')
    gn, wn = np.isnan(got), np.isnan(want)
    if (gn != wn).any():
        i, c = np.argwhere(gn != wn)[0]
        raise AssertionError(f'{what}: NaN positions differ, first iteration {i} {cols[c]}: {got[i, c]!r} vs {want[i, c]!r}')
    gi, wi = np.isinf(got), np.isinf(want)
    if (gi != wi).any() or (got[gi] != want[wi]).any():
        i, c = np.argwhere((gi != wi) | (gi & wi & (got != want)))[0]
        raise AssertionError(f'{what}: infinities differ, first iteration {i} {cols[c]}: {got[i, c]!r} vs {want[i, c]!r}')
    fin = ~(gn | gi)
    for c in (1, 2, 3):
        m = fin[:, c]
        np.testing.assert_allclose(got[m, c], want[m, c], rtol=RTOL, atol=0, err_msg=f'{what}: {cols[c]}')
    m = fin[:, 0]
    ta = abs(total_alpha(weight, pweight))
    with np.errstate(invalid='ignore', over='ignore'):
        bound = RTOL * np.abs(want[:, 1:]).sum(axis=1) / ta + 4 * np.finfo(np.float64).eps * np.abs(want[:, 0])
        bad = m & ~(np.abs(got[:, 0] - want[:, 0]) <= bound)
    if bad.any():
        i = int(np.argwhere(bad)[0][0])
        raise AssertionError(f'{what}: objective at iteration {i}: {got[i, 0]!r} vs {want[i, 0]!r}, bound {bound[i]!r} '
                             f'(terms {want[i, 1:].tolist()}, total_alpha {ta!r})')
    if len(got):
        assert got[0, 1] == 0.0, f'{what}: iteration 0 prob_dist {got[0, 1]!r}'
    if weight == 0.0:
        assert (got[:, 3] == 0.0).all(), f'{what}: tv2 without TGV'


def _session(lib, frames, chans, mc, batch):
    return abi.Session(lib, abi.frame_desc(frames[0], chans, mc.weight, mc.pweight, mc.iters), len(frames), batch=batch)


def recorded(lib, frames, chans, mc, fdata=None, batch=None):
    """(planes per frame, history (frames, iterations, 4), solve launches) of a recording session."""
    batch = len(frames) > 1 if batch is None else batch
    with _session(lib, frames, chans, mc, batch) as s:
        _check(lib, lib.j2p_session_record_objective(s.s, 1))
        s.upload(frames, chans, None if fdata is None else [[p.copy() for p in fd] for fd in fdata])
        s.iterate(0, 0)                                   # arm
        before = s.launches
        s.iterate(0, mc.iters)
        launches = s.launches - before
        hist = np.zeros((len(frames), mc.iters, 4))
        _check(lib, lib.j2p_session_objective_history(s.s, 0, mc.iters, hist.ctypes.data_as(C.POINTER(C.c_double))))
        return s.download(), hist, launches


def unrecorded(lib, frames, chans, mc, fdata=None):
    with _session(lib, frames, chans, mc, len(frames) > 1) as s:
        s.upload(frames, chans, None if fdata is None else [[p.copy() for p in fd] for fd in fdata])
        s.iterate(0, 0)
        before = s.launches
        s.iterate(0, mc.iters)
        return s.download(), s.launches - before


def checker_of(mc):
    if not H.have_ref():
        return 'oracle'
    # tables above 32767: the reference's SIMD build reads them signed (DESIGN §8), its scalar build is the checker
    return 'ref_c' if 'u16' in mc.extreme else 'ref'


def check_frame(img, fd, got, hist, mc, what):
    """One frame's recorded planes and history against the checker and the oracle's log."""
    chans = list(range(len(mc.planes)))
    planes_o, log = H.run_compute('oracle', img, chans, mc.weight, mc.pweight, mc.iters, [p.copy() for p in fd], want_log=True)
    checker = checker_of(mc)
    want = planes_o if checker == 'oracle' else H.run_compute(checker, img, chans, mc.weight, mc.pweight, mc.iters, [p.copy() for p in fd])
    same(got, want, f'{what}: recorded vs {checker}')
    assert_history(hist, log, mc.weight, mc.pweight, what)


def run_case(lib, ec):
    mc = M.tall_on_device(ec.mc) if ec.mc.tall else ec.mc
    frames, fdata = M.build_frames(mc)
    chans = list(range(len(mc.planes)))
    what = f'{ec.name} [{ec.cls} {ec.reaches or ec.limit}]; {mc.describe()}'
    if ec.limit == 'split':
        L._need_device_gb(2)
    got, hist, launches = recorded(lib, frames, chans, mc, fdata)
    plain, plain_launches = unrecorded(lib, frames, chans, mc, fdata)
    per_iter = E.recording_iteration(mc.planes, mc.weight, mc.nframes)[1]
    assert launches == mc.iters * per_iter, f'{launches} recorded launches for {mc.iters} iterations, kernel_paths says {per_iter} each; {what}'
    assert launches == plain_launches, f'{launches} recorded launches, {plain_launches} unrecorded; {what}'
    for f, img in enumerate(frames):
        same(got[f], plain[f], f'{what}: frame {f} recorded vs unrecorded')
        check_frame(img, fdata[f], got[f], hist[f], mc, f'{what}: frame {f}')
    if mc.nframes > 1:                                    # each frame alone: the same bits
        for f in range(mc.nframes):
            one, h1, _ = recorded(lib, frames[f:f + 1], chans, mc, fdata[f:f + 1], batch=False)
            same(one[0], got[f], f'{what}: frame {f} alone vs in the batch')
            assert (h1[0].view(np.uint64) == hist[f].view(np.uint64)).all(), f'{what}: frame {f} history alone vs in the batch'


SMALL_CASES = [c for c in E.CASES if c.limit not in ('full',)]


@pytest.mark.parametrize('case', SMALL_CASES, ids=lambda c: c.name)
def test_recorded_case_matches_the_checker(lib, case):
    run_case(lib, case)


def test_history_does_not_depend_on_the_neighbours(lib):
    """Frames of one geometry in different fallback regimes (plantings, extreme coefficients): each
    frame's history and planes are the same bits alone, first, last and between the others."""
    mcs = [E.BY_NAME[n].mc for n in ('tiny_adv420', 'island_adv420', 'coefs_adv420', 'patches_adv420', 'zero_coefs_adv420')]
    frames, fdata = [], []
    for mc in mcs:
        fr, fd = M.build_frames(M.Case(mc.name, mc.planes, 0.3, (0.001,) * 3, 3, nframes=1, plant=mc.plant,
                                       extreme=mc.extreme, seed=mc.seed))
        frames.append(fr[0])
        fdata.append(fd[0])
    mc = M.Case('neighbours', mcs[0].planes, 0.3, (0.001, 0.001, 0.0), 3)
    chans = [0, 1, 2]
    alone = [recorded(lib, [frames[k]], chans, mc, [fdata[k]], batch=False) for k in range(len(frames))]
    for k, (planes, hist, _) in enumerate(alone):
        check_frame(frames[k], fdata[k], planes[0], hist[0], mc, f'{mcs[k].name} alone')
    for order in ([0, 1, 2, 3, 4], [4, 3, 2, 1, 0], [2, 0], [3, 1, 4]):
        got, hist, _ = recorded(lib, [frames[k] for k in order], chans, mc, [fdata[k] for k in order])
        for pos, k in enumerate(order):
            same(got[pos], alone[k][0][0], f'{mcs[k].name} at {pos} of {order}: planes')
            assert (hist[pos].view(np.uint64) == alone[k][1][0].view(np.uint64)).all(), f'{mcs[k].name} at {pos} of {order}: history'


@pytest.mark.parametrize('name', ['full_444', 'full_420', 'full_422'])
def test_full_batch(lib, name):
    """65535 frames at 2 iterations: every frame's history and planes equal its source recorded alone
    (frames 0, 1, 32767, 32768, 65533 and 65534 have sources of their own), the sources equal the
    checker and the oracle's log, and the recorded planes equal the unrecorded batch's."""
    ec = E.BY_NAME[name]
    mc = ec.mc
    planes = L.SMALL[name.split('_')[1]]
    chans = list(range(len(planes)))
    n = mc.nframes
    sources = [L._random_frame(planes, 9100 + k) for k in range(8 + len(E.FULL_DISTINCT))]
    src = np.arange(n) % 8
    src[list(E.FULL_DISTINCT)] = 8 + np.arange(len(E.FULL_DISTINCT))
    alone_planes, alone_hist = [], []
    for k, img in enumerate(sources):
        p1, h1, _ = recorded(lib, [img], chans, mc, batch=False)
        check_frame(img, H.decode_planes(img, chans), p1[0], h1[0], mc, f'{name} source {k}')
        alone_planes.append(np.stack(p1[0]))
        alone_hist.append(h1[0])
    L._need_device_gb(2)
    frames = [sources[s] for s in src]
    got, hist, launches = recorded(lib, frames, chans, mc)
    per_iter = ec.launches()
    assert launches == mc.iters * per_iter, f'{name}: {launches} launches, kernel_paths says {per_iter} per iteration'
    got = np.stack([np.stack(fr) for fr in got])
    L._first_difference(got, np.stack(alone_planes)[src], f'{name}: recorded batch of {n}')
    want_hist = np.stack(alone_hist)[src]
    diff = (hist.view(np.uint64) != want_hist.view(np.uint64)).reshape(n, -1).any(axis=1)
    assert not diff.any(), f'{name}: {int(diff.sum())} frames record another history than alone; first {int(np.argwhere(diff)[0][0])}'
    plain, plain_launches = unrecorded(lib, frames, chans, mc)
    assert plain_launches == launches
    L._first_difference(got, np.stack([np.stack(fr) for fr in plain]), f'{name}: recorded vs unrecorded batch of {n}')


# ---- decode_jpeg and the command line ---------------------------------------------------------------
_MIXED = P.BY_NAME['mixed_separate'].solves
DECODE_REC = dict(DECODE, mixed_separate=(None, dict(iterations=tuple(s.iters for s in _MIXED), weight=tuple(s.weight for s in _MIXED),
                                                     pweight=tuple(s.pweight[0] for s in _MIXED))))
DECODE_RUNS = [(name, sep) for name, flags in DECODE_REC.items() for sep in (False, True) if flags[sep] is not None]


@pytest.mark.parametrize('name,sep', DECODE_RUNS, ids=[f'{n}-{"separate" if s else "joint"}' for n, s in DECODE_RUNS])
def test_decode_jpeg_records_the_regimes(jpeg, name, sep):  # noqa: F811
    data, img = jpeg
    kw = {'iterations': 6, **DECODE_REC[name][1 if sep else 0]}
    iters, weights, pweights = _flags(kw, sep)
    what = f'{name} {"separate" if sep else "joint"}: {kw}'
    plain = decode_jpeg(data, separate=sep, dtype=torch.float32, **kw)
    image, log = decode_jpeg(data, separate=sep, dtype=torch.float32, return_objective=True, **kw)
    same([image.cpu().numpy()], [plain.cpu().numpy()], f'{what}: image recorded vs not')
    solves = [(3, [0, 1, 2], weights[0], pweights, iters[0])] if not sep else \
        [(c, [c], weights[c], [pweights[c]], iters[c]) for c in range(3)]
    assert sorted(log) == [k for k, *_ in solves], f'{what}: channels {sorted(log)}'
    for key, chans, w, pw, it in solves:
        _, want = H.run_compute('oracle', img, chans, w, pw, it, want_log=True)
        assert_history(log[key].numpy(), want, w, pw, f'{what}: channel {key}')


def _parse_csv(text):
    lines = text.strip().splitlines()
    assert lines[0] == 'filename,channel,iteration,objective,prob_dist,tv,tv2'
    return {tuple(f[:3]): [float(v) for v in f[3:]] for f in (line.split(',') for line in lines[1:])}


@pytest.mark.parametrize('sep', [False, True], ids=['joint', 'separate'])
@pytest.mark.parametrize('args', CLI_ARGS, ids=lambda a: ' '.join(a))
def test_csv_matches_the_command_line(jpeg, tmp_path, args, sep):  # noqa: F811
    data, _ = jpeg
    subprocess.run(['make', '-C', CLI_DIR, 'jpeg2png'], check=True, capture_output=True)
    src = tmp_path / 'in.jpg'
    src.write_bytes(data)
    cli = tmp_path / 'cli.csv'
    r = subprocess.run([os.path.join(CLI_DIR, 'jpeg2png'), '-q', '-f', '-i', '6', *(['-s'] if sep else []), *args, '-c', str(cli),
                        str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    kw = {'weight': float(args[1])} if args[0] == '-w' else {'pweight': float(args[1])}
    _, logs = decode_jpeg([str(src)], mode='UNCHANGED', separate=sep, iterations=6, return_objective=True, **kw)
    ours = tmp_path / 'ours.csv'
    jpeg2png_b200.write_objective_csv(ours, [str(src)], logs)
    want, got = _parse_csv(cli.read_text()), _parse_csv(ours.read_text())
    assert sorted(got) == sorted(want)
    for key in want:
        g, w = np.array(got[key]), np.array(want[key])
        assert (np.isnan(g) == np.isnan(w)).all(), (key, g, w)
        assert (np.isinf(g) == np.isinf(w)).all() and (g[np.isinf(g)] == w[np.isinf(w)]).all(), (key, g, w)
        m = np.isfinite(w)
        np.testing.assert_allclose(g[m], w[m], rtol=1e-6, atol=1.5e-6, err_msg=str(key))
