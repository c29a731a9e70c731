"""Batch sessions without a GPU: the entry point refuses like every other one (no CPU fallback),
and the batched kernel instantiations are built on the same Hopper techniques as the single-frame
ones (cuobjdump over the in-tree library)."""
import ctypes as C

import pytest

from jpeg2png_b200 import abi
from tests.test_sass_techniques import sass_by_kernel


@pytest.fixture(scope='module')
def lib():
    return abi.load_product()


def _desc():
    d = abi.FrameDesc()
    d.nchannel = 1
    d.plane_w[0] = d.plane_h[0] = 8
    d.w_samp[0] = d.h_samp[0] = 1
    d.iterations = 1
    return d


def test_batch_without_gpu_is_an_error_not_a_fallback(lib):
    if lib.j2p_device_count() > 0:
        pytest.skip('a CUDA device is present')
    d = _desc()
    s = C.c_void_p()
    rc = lib.j2p_session_create_batch(C.byref(s), 0, C.byref(d), 4)
    assert rc == -3 and not s.value                      # J2P_ERR_NODEVICE
    assert b'no CPU fallback' in lib.j2p_last_error()


def test_empty_batch_is_refused(lib):
    d = _desc()
    s = C.c_void_p()
    assert lib.j2p_session_create_batch(C.byref(s), 0, C.byref(d), 0) == -1 and not s.value
    assert b'at least one frame' in lib.j2p_last_error()


def test_batched_kernels_keep_the_async_staging_and_the_launch_chain():
    sass = sass_by_kernel()
    # batched instantiations: the last template argument (BATCH) is true
    grads = {n: o for n, o in sass.items() if 'k_gradient_packed' in n and n.split('EEEv')[0].endswith('ELb1')}
    tiles = {n: o for n, o in sass.items() if ('k_project_tileILb' in n and 'ELb1EEEv' in n) or 'k_project_tile22ILb1' in n}
    steps = {n: o for n, o in sass.items() if 'k_step_uncoveredILb1' in n or 'k_step_uncovered22ILb1' in n}
    assert len(grads) == 14 and len(tiles) == 3 and len(steps) == 2, (sorted(grads), sorted(tiles), sorted(steps))
    for name, ops in grads.items():
        assert ops['LDGSTS'] >= 6, f'{name}: the cp.async row ring is gone'
        assert ops['ACQBULK'] >= 1 and ops['PREEXIT'] >= 1, f'{name}: griddepcontrol.wait / launch_dependents missing'
    for name, ops in tiles.items():
        assert ops['LDGSTS'] >= 6, f'{name}: cp.async staging is gone'
        assert ops['ACQBULK'] >= 1 and ops['PREEXIT'] >= 1, name
    for name, ops in {**grads, **tiles, **steps}.items():
        assert not any(op.startswith(('HMMA', 'IMMA', 'UTCMMA', 'UTCHMMA', 'WGMMA')) for op in ops), name
