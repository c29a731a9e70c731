"""The recording kernels (libj2pobjective.so) at the solver's edges: named cases of
tests/test_gpu_objective_edges.py.

Each case is a kernel-matrix case (tests/test_gpu_kernel_matrix.py `Case`: planes, weight, pweights,
iterations, frames of the batch, planting, extreme) plus the class it stands for and where its frames
come from.  The recording kernels a case reaches and its launches come from `recording_iteration`
below.  tests/test_objective_edges_host.py (no GPU) checks that
every kernel of the library is reached in each class, that every regime case still reaches its
regime on the oracle and that every limit case still crosses its limit.

Classes:
  regime    the weights of a tests/solver_param_cases.py case on a layout; `reaches` names what the
            oracle shows on the case's first frame: 'inside' (every step norm in [2^-40, 2^40]),
            'above' (a finite norm above 2^40), 'inf' (an overflowed norm), 'nan' (NaN samples) or
            'finite' (no NaN and no inf norm)
  fallback  the kernel matrix's plantings (IEEE fallbacks of the sub-gradient and the projection)
            and extreme tables and coefficients
  limit     frames whose last gradient band is 1..7 rows (`band`), frames more than 65535 block rows
            tall (`split`), 65535-frame batches (`full`) and a 2000-iteration run (`long`)
"""
from __future__ import annotations

import dataclasses
import re

from tests import kernel_paths as K
from tests import solver_param_cases as P
from tests import test_gpu_kernel_matrix as M
from tests import test_gpu_limits as L

G = K.PlaneGeom
MAX_GRID_ROWS = L.GRID_YZ                   # kMaxGridRows (kernels.cuh): the launchers split taller grids
NONFINITE = ('above', 'inf', 'nan')         # the regimes of the first coverage class


# The recording dispatch (session.cu record_gradient / record_project, objective/objective.cu) makes the
# solver's choice of kernels for the session and swaps each solve kernel for its recording variant,
# batch addressing always; the uncovered-pixel steps stay the solver's.  So the recording kernels are
# tests/kernel_paths.py's choice renamed, and the launches are the solver's, row split included.
_RECORDING = ((re.compile(r'^k_gradient_packed<(\d), (\w+), (\d), \w+>$'), r'k_gradient_packed_rec<\1, \2, \3>'),
              (re.compile(r'^k_project_tile<(\w+), \w+>$'), r'k_project_tile_rec<\1>'),
              (re.compile(r'^k_project_tile22<\w+>$'), 'k_project_tile22_rec'),
              (re.compile(r'^k_project<(\d), (\d)>$'), r'k_project_rec<\1, \2>'))


def recording_kernel(name: str) -> str:
    """The recording variant of one solver launch of a batch or single-frame session (uncovered steps: itself)."""
    for pattern, rec in _RECORDING:
        if pattern.match(name):
            return pattern.sub(rec, name)
    assert name.startswith('k_step_uncovered'), f'{name} has no recording variant'
    return name


def recording_iteration(planes, weight, nframes):
    """(names of the launches of one recording iteration, without the row split; launches with it).
    j2p_objective_project splits every projection grid at 65535 CTA rows, as the solver's launchers do
    (test_gpu_limits._tall_launches counts that for one frame)."""
    names, n = K.iteration(planes, weight, K.Mode(nframes=nframes))
    names = [recording_kernel(k) for k in names]
    _, Hf = K.frame_size(planes)
    rows = [p.ch // 8 if (p.sw, p.sh) in ((1, 1), (2, 2)) else -(-Hf // (8 * p.sh)) for p in planes]
    if max(rows) > MAX_GRID_ROWS:
        assert nframes == 1, 'a batch of frames taller than one grid'
        n = L._tall_launches([(p.cw, p.ch, p.sw, p.sh) for p in planes], weight)
    return names, n


@dataclasses.dataclass(frozen=True)
class EdgeCase:
    name: str
    cls: str                      # 'regime' | 'fallback' | 'limit'
    mc: M.Case                    # the frame, its planes and the solver settings
    reaches: str = ''             # regime cases: see the module docstring
    limit: str = ''               # limit cases: 'band' | 'split' | 'full' | 'long'
    regime: str = ''              # regime cases: the solver_param_cases case the weights come from

    def kernels(self):
        """The recording kernels one iteration of the case launches."""
        return sorted({k for k in recording_iteration(self.mc.planes, self.mc.weight, self.mc.nframes)[0] if '_rec' in k})

    def launches(self):
        """Solve launches per iteration: the recording kernels, the uncovered-pixel steps, the row split."""
        return recording_iteration(self.mc.planes, self.mc.weight, self.mc.nframes)[1]


# ---- layouts that between them reach all 20 recording kernels ------------------------------------------
LAYOUTS = {
    '444': M.LAYOUTS['444'],                      # k_gradient_packed_rec<3, *, 1>, k_project_tile_rec<false>
    '420': M.ADV['420'],                          # <3, *, 2>, k_project_tile22_rec
    'short_luma': M.LAYOUTS['420'],               # <3, *, 2>, k_project_tile_rec<true>
    '422': M.LAYOUTS['422'],                      # <3, *, 0>, k_project_rec<2, 1>
    '440': M.LAYOUTS['440'],                      # k_project_rec<1, 2>
    'odd': M.LAYOUTS['odd34'],                    # k_project_rec<0, 0>
    'y': M.LAYOUTS['y'],                          # <1, *, 1>
    's21': M.LAYOUTS['s21'],                      # <1, *, 0>, k_project_rec<2, 1>
    'two_444': M.LAYOUTS['yy'],                   # <2, *, 1>
    'two_420': M.LAYOUTS['420'][1:],              # <2, *, 0>, k_project_tile22_rec
}
# the ADV layouts of the plantings, and a 4:4:0 frame of their size (k_project_rec<1, 2>'s fallbacks)
ADV = dict(M.ADV, **{'440': (G(208, 144, 1, 1), G(208, 72, 1, 2), G(208, 72, 1, 2))})
REGIMES = [c for c in P.CASES if not c.separate]
# what the oracle shows of each regime's weights on the layouts (checked by the host test).  The
# straddle weights were bisected on solver_param_cases.CANON: on these frames both lie above the guard.
REACHES = {'inside_big': 'inside', 'above_guard_w': 'above', 'above_guard_p': 'above', 'straddle_lo': 'above',
           'straddle_hi': 'above', 'norm_inf_w': 'inf', 'norm_inf_p': 'inf', 'partial_nan': 'nan', 'all_nan_inf': 'nan',
           'all_nan_nan': 'nan', 'all_nan_2a2': 'nan', 'negative': 'finite', 'neg_zero': 'finite', 'subnormal': 'finite'}
# layouts where a regime shows something else: weight 1e10 goes above the guard on the larger or
# one-plane frames, and weight 1e38 overflows the joint norm (g / inf = 0: no NaN) wherever luma
# shares the norm with another plane
REACHES_ON = {**{('inside_big', lay): 'above' for lay in ('420', 'y', 's21')},
              **{('partial_nan', lay): 'inf' for lay in ('444', '420', 'short_luma', '422', '440', 'odd', 'two_420')}}


def _fit(values, n):
    """A regime's per-plane pweights for an n-plane layout: its first n, the last repeated."""
    v = list(values)
    return tuple((v + [v[-1]] * n)[:n])


def _cases():
    out = []
    seed = 3000

    def add(name, cls, planes, weight, pweight, iters, nframes=1, **kw):
        nonlocal seed
        seed += 1
        ekw = {k: kw.pop(k) for k in ('reaches', 'limit', 'regime') if k in kw}
        out.append(EdgeCase(name, cls, M.Case(name, tuple(planes), weight, tuple(pweight), iters, nframes=nframes, seed=seed, **kw), **ekw))

    # regimes on every recording kernel family, TGV on and off: the pweight regimes also at weight 0
    for rc in REGIMES:
        s = rc.solves[0]
        variants = [('', s.weight)] + ([('_w0', 0.0)] if rc.name in ('above_guard_p', 'norm_inf_p') else [])
        for lay, planes in LAYOUTS.items():
            for suffix, w in variants:
                add(f'{rc.name}{suffix}_{lay}', 'regime', planes, w, _fit(s.pweight, len(planes)), s.iters, nframes=2,
                    reaches=REACHES_ON.get((rc.name, lay), REACHES[rc.name]), regime=rc.name)
    # the fallbacks: plantings on the ADV layouts (the luma-side ones reach the sub-gradient's slow rows)
    for lay, planes in ADV.items():
        for plant in ('tiny', 'patches', 'zero_coefs', 'subnormal'):
            add(f'{plant}_adv{lay}', 'fallback', planes, 0.3, (0.001,) * 3, 4, nframes=2, plant=plant)
        add(f'island_adv{lay}', 'fallback', planes, 0.3, (0.001, 0.001, 0.0), 2, nframes=2, plant='island')
        for extreme in ('ones', 'u16', 'coefs'):
            add(f'{extreme}_adv{lay}', 'fallback', planes, 0.3, (0.001,) * 3, 5, extreme=extreme)
    add('u16_coefs_adv420_batch2', 'fallback', ADV['420'], 0.3, (0.001,) * 3, 5, nframes=2, extreme='u16+coefs')
    # slow sub-gradient rows of every other gradient family, TGV on and off
    for w in (0.0, 0.3):
        for lay in ('444', 'short_luma', '422', 'y', 's21', 'two_444', 'two_420', 'odd'):
            add(f'tiny_{lay}_w{w}', 'fallback', LAYOUTS[lay], w, (0.001,) * len(LAYOUTS[lay]), 3, nframes=2, plant='tiny')
    for lay in ('420', '422'):
        add(f'tiny_adv{lay}_w0.0', 'fallback', ADV[lay], 0.0, (0.001,) * 3, 3, nframes=2, plant='tiny')
    # bands: the matrix's tall narrow frames (heights chosen on the device: last band 1..7 rows) and the
    # same on the other gradient families and generic projections
    for mc in M.NAMED:
        if mc.tall:
            add(mc.name, 'limit', mc.planes, mc.weight, mc.pweight, mc.iters, nframes=mc.nframes, tall=True, limit='band')
    h = lambda W, nc: K.short_last_band_heights(W, (K.GRAD_CTAS_PER_SM[3 if nc == 3 else 1],), 2100, 6000)[0]
    for name, planes in (('y', (G(232, 0, 1, 1),)), ('420', (G(112, 0, 1, 1), G(56, 0, 2, 2), G(56, 0, 2, 2))),
                         ('yy', (G(232, 0, 1, 1),) * 2), ('s21', (G(112, 0, 2, 1),)), ('c22', (G(112, 0, 2, 2),) * 2),
                         ('420narrow', (G(216, 0, 1, 1), G(112, 0, 2, 2), G(112, 0, 2, 2))),   # luma 8 columns short
                         ('422', (G(224, 0, 1, 1), G(112, 0, 2, 1), G(112, 0, 2, 1))),
                         ('440', (G(112, 0, 1, 1), G(112, 0, 1, 2), G(112, 0, 1, 2))),
                         ('odd32', (G(48, 0, 1, 1), G(16, 0, 3, 2), G(16, 0, 3, 1)))):
        W = K.frame_size(planes)[0]
        Hf = h(W, len(planes))
        planes = tuple(G(p.cw, Hf // p.sh, p.sw, p.sh) for p in planes)
        for w in (0.0, 0.3):
            add(f'tall_{name}_w{w}', 'limit', planes, w, (0.001,) * len(planes), 2, tall=True, limit='band')
    # split launches: more than 65535 CTA rows in one projection grid
    for name in ('one_plane', '420', '422'):
        planes = tuple(G(*p) for p in L.TALL[name])
        add(f'split_{name}', 'limit', planes, 0.3, tuple(L.PW3[:len(planes)]), 3, limit='split')
    # full batches of 16 x 16 frames
    for name in ('444', '420', '422'):
        planes = tuple(G(*p) for p in L.SMALL[name])
        add(f'full_{name}', 'limit', planes, 0.3, tuple(L.PW3), 2, nframes=L.MAX_FRAMES, limit='full')
    # a long run
    lc = P.LONG_BY_NAME['long_420']
    img = lc.image()
    add('long_420', 'limit', tuple(G(p.w, p.h, p.w_samp, p.h_samp) for p in img.planes), lc.solves[0].weight,
        lc.solves[0].pweight, lc.solves[0].iters, limit='long')
    return out


CASES = _cases()
BY_NAME = {c.name: c for c in CASES}
assert len(BY_NAME) == len(CASES)

# (class, kernel) pairs no case of the class reaches, each with the reason
EXEMPT = {}

# frames of the full batches that get distinct content and are compared with the same frame recorded alone
FULL_DISTINCT = (0, 1, 32767, 32768, 65533, 65534)


def coverage_classes(case: EdgeCase):
    """The coverage classes a case counts for: 'nonfinite' (a regime case that goes above the guard, to
    an inf norm or to NaN), 'fallback' (a planting or an extreme), 'limit' (tall or full batch)."""
    if case.cls == 'regime':
        return ['nonfinite'] if case.reaches in NONFINITE else []
    if case.cls == 'fallback':
        return ['fallback']
    return ['limit'] if case.limit in ('band', 'split', 'full') else []
