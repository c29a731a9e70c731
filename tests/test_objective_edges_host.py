"""Without a GPU: the case table of tests/test_gpu_objective_edges.py (tests/objective_edge_cases.py)
stays honest.  Every kernel of libj2pobjective.so is reached in each coverage class (a non-finite or
above-guard regime, a fallback planting or extreme, a tall frame or a full batch) or exempt with a
reason; every regime case still reaches what it claims on the oracle; every limit case still crosses
its limit."""
import dataclasses

import numpy as np
import pytest

from jpeg2png_b200 import abi
from tests import kernel_paths as K
from tests import objective_cases as OC
from tests import objective_edge_cases as E
from tests import solver_param_cases as P
from tests import test_gpu_kernel_matrix as M
from tests import test_gpu_limits as L
from tests.test_objective_host import LIB, _kernels

CLASSES = ('nonfinite', 'fallback', 'limit')


def reached_by_class(cases):
    out = {c: {} for c in CLASSES}
    for case in cases:
        for cls in E.coverage_classes(case):
            for k in case.kernels():
                out[cls].setdefault(k, []).append(case.name)
    return out


def missing(lib_kernels, cases):
    """(class, kernel) pairs of the library no case of the class reaches and no exemption covers."""
    reached = reached_by_class(cases)
    return sorted((cls, k) for cls in CLASSES for k in lib_kernels if k not in reached[cls] and (cls, k) not in E.EXEMPT)


def test_every_recording_kernel_is_reached_in_every_class():
    lib = _kernels(LIB)
    assert len(lib) == 20
    assert missing(lib, E.CASES) == [], 'recording kernels a class of cases does not reach (class, kernel)'
    named = {k for c in E.CASES for k in c.kernels()}
    assert sorted(named - lib) == [], 'cases name kernels the library lacks'
    assert sorted(k for _, k in E.EXEMPT if k not in lib) == [], 'exemptions name kernels the library lacks'
    assert all(reason for reason in E.EXEMPT.values())


def test_removing_a_sole_case_names_its_kernel():
    """Deleting the only case of a class that reaches a kernel makes the coverage check name that kernel."""
    lib = _kernels(LIB)
    reached = reached_by_class(E.CASES)
    sole = [(cls, k, names[0]) for cls in CLASSES for k, names in reached[cls].items() if len(names) == 1]
    assert sole, 'no kernel rests on a single case: nothing to check'
    for cls, k, name in sole:
        assert (cls, k) in missing(lib, [c for c in E.CASES if c.name != name]), (cls, k, name)


def _norms_and_nan(ec):
    mc = ec.mc
    frames, _ = M.build_frames(dataclasses.replace(mc, nframes=1))
    img = frames[0]
    case = P.ParamCase(ec.name, ec.reaches, None, (P.Solve(tuple(range(len(mc.planes))), mc.weight, mc.pweight, mc.iters),))
    (norms, planes), = P.oracle_norms(case, img)
    return norms, planes


@pytest.mark.parametrize('case', [c for c in E.CASES if c.cls == 'regime'], ids=lambda c: c.name)
def test_regime_case_reaches_its_regime(case):
    norms, planes = _norms_and_nan(case)
    nan = sum(int(np.isnan(p).sum()) for p in planes)
    finite = norms[np.isfinite(norms)]
    what = f'{case.name}: norms {norms.min()!r}..{norms.max()!r}, {nan} NaN samples; {case.mc.describe()}'
    if case.reaches == 'inside':
        assert ((norms >= P.GUARD_LO) & (norms <= P.GUARD_HI)).all() and nan == 0, what
    elif case.reaches == 'above':
        assert (finite > P.GUARD_HI).any() and nan == 0, what
    elif case.reaches == 'inf':
        assert np.isinf(norms).any(), what
    elif case.reaches == 'nan':
        assert nan > 0, what
    else:
        assert case.reaches == 'finite', case.reaches
        assert nan == 0 and np.isfinite(norms).all(), what


def test_limit_cases_cross_their_limits():
    res = K.library_resources(abi.PRODUCT_LIB)
    if res is None:
        pytest.skip('cuobjdump or the built library is missing (run __graft_entry__.build())')
    for ec in E.CASES:
        mc = ec.mc
        W, Hf = K.frame_size(mc.planes)
        if ec.limit == 'band':
            # the height the H100 run picks (M.tall_on_device): a last band of 1..7 rows exists for this width
            per_sm = K.resident_ctas(*res[K.gradient_kernel(mc.planes, mc.weight, K.Mode())])
            assert K.short_last_band_heights(W, (per_sm,), 2100, 12000, K.H100_SMS), ec.name
            assert Hf >= 2100, ec.name
        elif ec.limit == 'split':
            rows = [p.ch // 8 if (p.sw, p.sh) in ((1, 1), (2, 2)) else -(-Hf // (8 * p.sh)) for p in mc.planes]
            assert max(rows) > E.MAX_GRID_ROWS, ec.name
            if ec.name == 'split_422':                      # the generic per-frame path with a non-zero row0
                assert min(r for r, p in zip(rows, mc.planes) if (p.sw, p.sh) == (2, 1)) > E.MAX_GRID_ROWS
            assert ec.launches() > K.iteration(mc.planes, mc.weight)[1], ec.name   # the frame needs the row split
        elif ec.limit == 'full':
            assert mc.nframes == L.MAX_FRAMES and mc.iters == 2, ec.name
        elif ec.limit == 'long':
            assert mc.iters == 2000, ec.name
    assert {ec.name for ec in E.CASES if ec.limit == 'full'} == {'full_444', 'full_420', 'full_422'}
    assert E.FULL_DISTINCT == (0, 1, 32767, 32768, L.MAX_FRAMES - 2, L.MAX_FRAMES - 1)
    n422 = E.recording_iteration(E.BY_NAME['full_422'].mc.planes, 0.3, L.MAX_FRAMES)[0]
    assert n422.count('k_project_rec<2, 1>') == 2 * L.MAX_FRAMES


def test_recording_dispatch_names_what_the_objective_cases_list():
    """The restated recording dispatch gives, on every case of tests/objective_cases.py, the kernels
    that table lists for it."""
    for name, (make, channels, weight, _, _, listed) in OC.CASES.items():
        img = make(0)
        planes = [K.PlaneGeom(img.planes[c].w, img.planes[c].h, img.planes[c].w_samp, img.planes[c].h_samp) for c in channels]
        got = {k for k in E.recording_iteration(planes, weight, 3)[0] if '_rec' in k}
        assert sorted(got) == sorted(listed), name


def test_the_table_has_what_it_is_named_for():
    names = set(E.BY_NAME)
    for rc in E.REGIMES:
        for lay in E.LAYOUTS:
            assert f'{rc.name}_{lay}' in names
    for lay in E.ADV:
        for plant in ('tiny', 'patches', 'zero_coefs', 'subnormal', 'island'):
            assert f'{plant}_adv{lay}' in names
    assert any(ec.mc.extreme == 'u16+coefs' and ec.mc.nframes == 2 for ec in E.CASES)
    assert {(ec.mc.weight != 0.0) for ec in E.CASES if ec.cls == 'regime' and ec.reaches in E.NONFINITE} == {True, False}
