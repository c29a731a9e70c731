"""Solver parameter regimes (test infrastructure): TGV weights, DCT-distance weights (pweights) and
iteration counts well outside the defaults, each named for the side of a kernel guard it puts a frame on.

Every projection kernel divides the sub-gradient by the step norm sqrtf((float)sum g^2) with the
shared-reciprocal sequence when the norm lies in [2^-40, 2^40] (qdiv_divisor_ok, numerics.cuh) and
with IEEE division otherwise.  Once sum g^2 exceeds FLT_MAX the norm is inf, RN(1/inf) = 0, and only
the IEEE fallback gives the reference's g / inf = +-0.  The weights and pweights below put the
canonical frame (CANON: 72x56 4:2:0, synth_coefs quality 30, seed 5) inside the guard, above it, on
either side of 2^40, at an overflowed norm, at partly and wholly NaN results, and at negative, -0 and
subnormal values, which the host's `weight != 0` / `pweight != 0` must treat as on, off and on.
tests/test_solver_params_host.py checks (no GPU) that every case still reaches its regime and that
the oracle equals both reference builds on it; tests/test_gpu_solver_params.py runs each regime
through every solver kernel family.

Results that hold NaN are compared with `assert_same_or_nan`: the same NaN positions and the same
bits on every other sample.  NaN payloads and signs are not compared: x86's default NaN is
0xffc00000 (and the reference also makes 0x7fc00000), the GPU's canonical NaN is 0x7fffffff.
"""
from __future__ import annotations

import dataclasses

import numpy as np

from jpeg2png_b200 import synth
from jpeg2png_b200.synth import CoefImage
from tests import helpers as H

GUARD_LO = np.float32(2.0 ** -40)
GUARD_HI = np.float32(2.0 ** 40)

# (width, height, quality, subsampling, seed) of synth.synth_coefs
CANON = (72, 56, 30, '4:2:0', 5)
CANON444 = (72, 56, 30, '4:4:4', 5)

# Bisected over float32 weights on CANON (joint, pweight 0.001, 6 iterations: the count changes the
# first sub-gradient): consecutive floats whose first iteration's luma norm is exactly 2^40, the
# guard's inclusive bound, at STRADDLE_LO and 2^40 + 131072, the next float the norm reaches, at
# STRADDLE_HI (one ulp of the weight moves the norm by about 36.8 * 2048).
STRADDLE_LO = 29849311232.0
STRADDLE_HI = 29849313280.0
STRADDLE_NORMS = (1099511627776.0, 1099511758848.0)


@dataclasses.dataclass(frozen=True)
class Solve:
    """One compute() call: planes `channels` of the frame solved together."""
    channels: tuple
    weight: float
    pweight: tuple                # one per channel
    iters: int


@dataclasses.dataclass(frozen=True)
class ParamCase:
    name: str
    regime: str                   # see REGIMES
    frame: tuple                  # synth_coefs arguments
    solves: tuple                 # one Solve (joint or one-plane) or three (separate mode, -s)

    @property
    def separate(self) -> bool:
        return len(self.solves) > 1

    def image(self) -> CoefImage:
        return synth.synth_coefs(*self.frame)

    def describe(self) -> str:
        s = '; '.join(f'planes {list(v.channels)} weight {v.weight!r} pweight {list(v.pweight)} x{v.iters}' for v in self.solves)
        return f'{self.name} ({self.regime}): synth_coefs{self.frame}: {s}'


# regime -> what tests/test_solver_params_host.py checks of the case on the oracle
REGIMES = {
    'inside': 'every (iteration, channel) step norm lies in [2^-40, 2^40]',
    'above': 'some step norm is finite and above 2^40',
    'straddle_lo': "the first iteration's luma norm is STRADDLE_NORMS[0] <= 2^40",
    'straddle_hi': "the first iteration's luma norm is STRADDLE_NORMS[1] > 2^40",
    'norm_inf': 'some step norm is inf',
    'partial_nan': 'some, not all, result samples are NaN',
    'all_nan': 'every result sample is NaN',
    'tgv_off': 'the result equals the one with weight +0 and pweight +0 where the case has -0',
    'tgv_on': 'the result differs from the one with the negative weights set to +0',
    'tiny': 'the terms are on (kernel_paths picks the TGV instantiations), but a2 and the DCT-distance scale round '
            'to 0 or contribute nothing: the result equals the one with the tiny weights set to +0',
    'mixed': 'separate planes in different regimes: one above the guard, one at an inf norm',
}


def _joint(name, regime, weight, pweight, iters=6, frame=CANON):
    return ParamCase(name, regime, frame, (Solve((0, 1, 2), weight, tuple(pweight), iters),))


def _one(name, regime, weight, pweight, iters, frame=CANON444):
    return ParamCase(name, regime, frame, (Solve((0,), weight, (pweight,), iters),))


PW = (0.001, 0.001, 0.001)
CASES = [
    _joint('inside_big', 'inside', 1e10, PW),
    _joint('above_guard_w', 'above', 1e12, PW),
    _joint('above_guard_p', 'above', 0.3, (1e12, 0.001, 1e12)),
    _joint('straddle_lo', 'straddle_lo', STRADDLE_LO, PW),
    _joint('straddle_hi', 'straddle_hi', STRADDLE_HI, PW),
    _joint('norm_inf_w', 'norm_inf', 1e18, PW),
    _joint('norm_inf_p', 'norm_inf', 0.3, (1e30, 0.001, 1e30)),
    # one channel, 4:4:4: 1856 of 4032 samples NaN after one iteration (all of them after two)
    _one('partial_nan', 'partial_nan', 1e38, 0.001, 1),
    _joint('all_nan_inf', 'all_nan', float('inf'), PW, 2),
    _joint('all_nan_nan', 'all_nan', float('nan'), PW, 2),
    # one channel: a2 = weight / sqrt(2) = 1.77e38, so 2 * a2 overflows (kernels_gradient_packed.cu
    # computes (-2 a2) (M / n)); the reference is already all NaN here, as it is at 2e38 where it
    # does not overflow, so the planes cannot show where that rewrite stops being exact
    _one('all_nan_2a2', 'all_nan', 2.5e38, 0.001, 2),
    _joint('negative', 'tgv_on', -0.3, (0.001, -0.001, 0.001)),
    _joint('neg_zero', 'tgv_off', -0.0, (0.001, -0.0, 0.001)),
    _joint('subnormal', 'tiny', 1e-45, (1e-45, 1e-40, 0.001)),
    ParamCase('mixed_separate', 'mixed', CANON, (Solve((0,), 1e12, (0.001,), 6), Solve((1,), -0.3, (1e30,), 4),
                                                 Solve((2,), 1e37, (-0.001,), 3))),
]
BY_NAME = {c.name: c for c in CASES}

# Long runs on small frames: every association of the solver runs thousands of times.
LONG = [
    _joint('long_420', 'long', 0.3, PW, 2000, frame=(128, 96, 30, '4:2:0', 7)),
    _joint('long_444', 'long', 0.3, PW, 1000, frame=(96, 64, 40, '4:4:4', 8)),
    ParamCase('long_separate', 'long', (120, 88, 30, '4:2:0', 9),
              (Solve((0,), 0.3, (0.001,), 2000), Solve((1,), 0.1, (0.001,), 1), Solve((2,), 0.0, (0.001,), 0))),
]
LONG_BY_NAME = {c.name: c for c in LONG}


def planes_of(img: CoefImage, channels) -> CoefImage:
    """The frame cut down to planes `channels` (what a one-plane session of -s holds)."""
    return CoefImage(width=img.width, height=img.height, planes=[img.planes[c] for c in channels])


def run_checker(kind, case: ParamCase, img=None):
    """Every plane of the case's result, in channel order, from one checker ('ref', 'ref_c', 'oracle')."""
    img = img or case.image()
    out = []
    for s in case.solves:
        out += H.run_compute(kind, img, list(s.channels), s.weight, s.pweight, s.iters)
    return out


def narrowed(sum_g2) -> np.float32:
    """sqrtf((float)sum) (compute.c:205); inf once the sum exceeds FLT_MAX."""
    with np.errstate(over='ignore'):
        return np.sqrt(np.float32(float(sum_g2)), dtype=np.float32)


def oracle_norms(case: ParamCase, img=None):
    """Per solve: the step norms [iteration, channel] and the result planes, from the oracle's strip
    interface with one strip covering the frame."""
    from tests.strip_backend import OracleStrip
    img = img or case.image()
    out = []
    for s in case.solves:
        sub = planes_of(img, s.channels)
        fd = H.decode_planes(sub, range(len(s.channels)))
        pw = list(s.pweight) + [0.0] * (3 - len(s.channels))
        st = OracleStrip(sub, s.weight, pw, s.iters, 0, max(p.h * p.h_samp for p in sub.planes), fd)
        try:
            norms = []
            for _ in range(s.iters):
                g = st.gradient().clone()
                norms.append([narrowed(g[c]) for c in range(st.nc)])
                st.project(g, 1)
            planes = [st.download(c) for c in range(st.nc)]
        finally:
            st.close()
        out.append((np.array(norms, np.float32).reshape(s.iters, len(s.channels)), planes))
    return out


def assert_same_or_nan(a, b, what=''):
    """Plane by plane: identical NaN masks and identical bits on every other sample.  Reports the first
    differing sample as helpers.assert_bit_identical does."""
    for k, (p, q) in enumerate(zip(a, b)):
        assert p.shape == q.shape, f'{what} plane {k}: shape {p.shape} vs {q.shape}'
        pn, qn = np.isnan(p), np.isnan(q)
        diff = (pn != qn) | (~pn & ~qn & (H.bits(p) != H.bits(q)))
        if diff.any():
            idx = tuple(np.argwhere(diff)[0])
            with np.errstate(invalid='ignore', over='ignore'):
                d = np.abs(p.astype(np.float64) - q.astype(np.float64))
            raise AssertionError(
                f'{what} plane {k}: {int(diff.sum())} of {diff.size} samples differ (NaN positions: '
                f'{int((pn != qn).sum())}); first at {idx}: {p[idx]!r} ({int(H.bits(p)[idx]):#010x}) vs '
                f'{q[idx]!r} ({int(H.bits(q)[idx]):#010x}); max abs diff where both are numbers {float(np.nanmax(np.where(pn | qn, 0.0, d)))}')
    assert len(a) == len(b), f'{what}: {len(a)} planes vs {len(b)}'
