"""Solver parameters on the CPU (no GPU): the oracle equals both reference builds at every case of
tests/solver_param_cases.py, every case reaches the regime it is named for, and the command line
and decode_jpeg accept the -w / -p values the reference's sscanf("%f") accepts."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from jpeg2png_b200.decode import solver_flags
from tests import helpers as H
from tests import solver_param_cases as P
from tests.test_codecs import CLI_DIR

need_ref = pytest.mark.skipif(not H.have_ref(), reason='oracle/_ref (the compiled reference) was not built')


@need_ref
@pytest.mark.parametrize('case', P.CASES + P.LONG, ids=lambda c: c.name)
def test_oracle_equals_both_reference_builds(case):
    img = case.image()
    want = P.run_checker('oracle', case, img)
    for kind in ('ref', 'ref_c'):
        P.assert_same_or_nan(P.run_checker(kind, case, img), want, f'{kind} vs oracle; {case.describe()};')


@pytest.mark.parametrize('case', P.CASES, ids=lambda c: c.name)
def test_case_reaches_its_regime(case):
    img = case.image()
    runs = P.oracle_norms(case, img)
    norms = np.concatenate([n.reshape(-1) for n, _ in runs])
    planes = [p for _, pl in runs for p in pl]
    # the strip interface with one strip is the solver itself
    P.assert_same_or_nan(planes, P.run_checker('oracle', case, img), f'one-strip oracle vs oracle_compute; {case.describe()}')
    nan = sum(int(np.isnan(p).sum()) for p in planes)
    size = sum(p.size for p in planes)
    what = f'{case.describe()}: norms {norms.min()!r}..{norms.max()!r}, {nan} of {size} samples NaN'
    finite = norms[np.isfinite(norms)]
    if case.regime == 'inside':
        assert ((norms >= P.GUARD_LO) & (norms <= P.GUARD_HI)).all(), what
    elif case.regime == 'above':
        assert (finite > P.GUARD_HI).any(), what
    elif case.regime in ('straddle_lo', 'straddle_hi'):
        n1 = runs[0][0][0, 0]
        lo = case.regime == 'straddle_lo'
        assert float(n1) == P.STRADDLE_NORMS[0 if lo else 1], what
        assert (n1 <= P.GUARD_HI) if lo else (n1 > P.GUARD_HI), what
        # the other side is one float32 ulp of the weight away
        other = P.STRADDLE_HI if lo else P.STRADDLE_LO
        assert abs(int(np.float32(other).view(np.uint32)) - int(np.float32(case.solves[0].weight).view(np.uint32))) == 1
    elif case.regime == 'norm_inf':
        assert np.isinf(norms).any(), what
    elif case.regime == 'partial_nan':
        assert 0 < nan < size, what
    elif case.regime == 'all_nan':
        assert nan == size, what
    elif case.regime == 'mixed':
        assert (finite > P.GUARD_HI).any() and np.isinf(norms).any(), what
    else:
        # sign and magnitude of the weights: compare with the same case at +0 in place of the
        # negative, -0 or tiny weights; -0 switches a term off and a negative weight on, and
        # subnormal weights switch the terms on without changing a bit
        zeroed = P.ParamCase(case.name + '+0', case.regime, case.frame, tuple(
            P.Solve(s.channels, 0.0 if (s.weight < 0 or s.weight < 1e-30) else s.weight,
                    tuple(0.0 if (w < 0 or w < 1e-30) else w for w in s.pweight), s.iters) for s in case.solves))
        base = P.run_checker('oracle', zeroed, img)
        if case.regime in ('tgv_off', 'tiny'):
            H.assert_bit_identical(planes, base, what)
        else:
            assert nan == 0, what
            assert any((H.bits(a) != H.bits(b)).any() for a, b in zip(planes, base)), what
    if case.regime in ('straddle_lo', 'straddle_hi', 'inside', 'above'):
        assert nan == 0, what


def test_straddle_and_canonical_frames():
    """The frame the straddle weights were bisected on: 72x56 4:2:0, luma 72x56 in an 80x64 frame
    (stepped-only luma rows and columns: k_step_uncovered)."""
    img = P.BY_NAME['straddle_lo'].image()
    assert [(p.w, p.h, p.w_samp, p.h_samp) for p in img.planes] == [(72, 56, 1, 1), (40, 32, 2, 2), (40, 32, 2, 2)]
    img = P.BY_NAME['partial_nan'].image()
    assert [(p.w, p.h, p.w_samp) for p in img.planes][0] == (72, 56, 1)
    for c in P.LONG:
        assert c.image().width <= 128 and c.image().height <= 96


# ---- argument parsing -----------------------------------------------------------------------------
VALUES = ['-0.3', '-0', '0', '1e12', '1e40', '-1e40', 'nan', 'NaN', '-nan', 'inf', '-inf', 'Infinity', '1e-45', '1e-50',
          '3e38', '0x1p3', '+.5', '.', '', '-', 'e5', 'x', '1e', '0.3x', 'nan(1)']
_libc = C.CDLL(None)


def sscanf_floats(s, fmt=b'%f,%f,%f'):
    """(count, values) of the reference's sscanf(arg, "%f,%f,%f", ...) (jpeg2png.c:209, :224)."""
    v = (C.c_float * 3)()
    n = _libc.sscanf(s.encode(), fmt, C.byref(v, 0), C.byref(v, 4), C.byref(v, 8))
    return n, list(v)


@pytest.fixture(scope='module')
def exe():
    subprocess.run(['make', '-C', CLI_DIR, 'jpeg2png'], check=True, capture_output=True)
    return os.path.join(CLI_DIR, 'jpeg2png')


@pytest.mark.parametrize('flag', ['-w', '-p'])
@pytest.mark.parametrize('sep', [False, True], ids=['joint', 'separate'])
def test_cli_accepts_what_sscanf_accepts(exe, tmp_path, flag, sep):
    """A value the reference's sscanf reads gets past the flags (the run stops at the missing input
    file, before any device is touched); one it does not read is refused with the reference's message."""
    for v in VALUES:
        n, _ = sscanf_floats(v)
        args = (['-s'] if sep else []) + [flag, v, 'missing.jpg']
        r = subprocess.run([exe, *args], capture_output=True, text=True, cwd=str(tmp_path), timeout=60)
        last = r.stderr.strip().splitlines()[-1] if r.stderr.strip() else ''
        if n == 1:
            assert last == 'jpeg2png: could not open input file `missing.jpg`', (args, r.stderr)
        else:
            msg = 'invalid weight' if flag == '-w' else 'invalid probability weight'
            assert r.returncode == 1 and last == 'jpeg2png: ' + msg, (args, n, r.stderr)


def test_solver_flags_take_the_values_the_command_line_takes():
    """decode_jpeg's weight / pweight: every value sscanf reads reaches the solver as the same float."""
    for v in VALUES:
        n, vals = sscanf_floats(v)
        if n != 1:
            continue
        x = vals[0]
        for sep in (False, True):
            _, weights, pweights = solver_flags(6, x, x, sep)
            for got in (weights[0], *pweights):
                a, b = np.float32(got), np.float32(x)
                assert (math.isnan(a) and math.isnan(b)) or H.bits(np.array([a]))[0] == H.bits(np.array([b]))[0], (v, got, x)
            assert weights[1:] == (0.0, 0.0)
        _, weights, _ = solver_flags(6, [x, -x, x], 0.001, True)
        assert np.float32(weights[1]).tobytes() == np.float32(-x).tobytes() or math.isnan(x)
