"""Batch sessions on the GPU (pytest -m gpu): every frame of a batch must be bit-identical to the
same frame solved alone in a single-frame session, and to the checker (the compiled reference when
it travelled, else the oracle).  Every batch mixes frames of different quality (tables) and seeds."""
import ctypes as C

import numpy as np
import pytest

from jpeg2png_b200 import abi, synth
from tests import helpers as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def lib():
    lib = abi.load_product()
    assert lib.j2p_device_count() > 0, 'no CUDA device visible: the product has no CPU fallback'
    return lib


def _checker():
    return 'ref' if H.have_ref() else 'oracle'


def _single(lib, img, channels, weight, pw, iters, fdata=None):
    """The frame alone in an ordinary session (j2p_session_create)."""
    with abi.Session(lib, abi.frame_desc(img, channels, weight, pw, iters), batch=False) as s:
        s.upload([img], channels, None if fdata is None else [fdata])
        s.iterate(0, iters)
        return s.download()[0]


def _frames(case, n):
    """n frames of one geometry, each with its own seed and tables.  Returns (frames, channels, weight, pweight)."""
    qs = [10, 35, 75, 90, 50, 20]
    if case == '444':
        return [synth.synth_coefs(136, 72, qs[k % 6], '4:4:4', 100 + k) for k in range(n)], [0, 1, 2], 0.7, [0.001, 0.0, 0.01]
    if case == '420':
        return [synth.synth_coefs(256, 128, qs[k % 6], '4:2:0', 200 + k) for k in range(n)], [0, 1, 2], 0.3, [0.001] * 3
    if case == '1080p':      # luma grid 1080 rows, frame 1088: the luma plane is 8 rows short
        return [synth.random_coefs([(1920, 1080), (960, 544), (960, 544)], [(1, 1), (2, 2), (2, 2)], 300 + k)
                for k in range(n)], [0, 1, 2], 0.3, [0.001] * 3
    if case == '422':
        return [synth.random_coefs([(96, 48), (48, 48), (48, 48)], [(1, 1), (2, 1), (2, 1)], 400 + k)
                for k in range(n)], [0, 1, 2], 0.3, [0.001] * 3
    if case == 'odd':        # (3,4) sampling
        return [synth.random_coefs([(40, 24), (24, 16), (16, 8)], [(1, 1), (2, 2), (3, 4)], 500 + k)
                for k in range(n)], [0, 1, 2], 0.4, [0.001] * 3
    if case == 'sep_luma':
        return [synth.synth_coefs(120, 64, qs[k % 6], '4:2:0', 600 + k) for k in range(n)], [0], 0.3, [0.001]
    if case == 'sep_chroma':
        return [synth.synth_coefs(120, 64, qs[k % 6], '4:2:0', 700 + k) for k in range(n)], [1], 0.3, [0.001]
    if case == 'no_tgv':
        return [synth.synth_coefs(64, 64, qs[k % 6], '4:4:4', 800 + k) for k in range(n)], [0, 1, 2], 0.0, [0.001, 0.002, 0.0]
    raise ValueError(case)


@pytest.mark.parametrize('n', [1, 3, 16])
@pytest.mark.parametrize('case', ['444', '420', '1080p', '422', 'odd', 'sep_luma', 'sep_chroma', 'no_tgv'])
def test_batch_frames_match_single_sessions(lib, case, n):
    frames, ch, w, pw = _frames(case, n)
    iters = 5 if case == '1080p' else 12
    got = abi.solve_batch(frames, ch, w, pw, iters, lib=lib)          # device decode
    assert len(got) == n
    for f, img in enumerate(frames):
        H.assert_bit_identical(got[f], _single(lib, img, ch, w, pw, iters), f'{case} batch of {n}, frame {f}')


def test_config1_batch_of_8_matches_the_checker(lib):
    """BASELINE config 1's frame (256x256 Q10 4:2:0, 50 iterations), eight per batch."""
    frames = [synth.synth_coefs(256, 256, 10 + 5 * (k % 3), '4:2:0', 1234 + k) for k in range(8)]
    fd = [H.decode_planes(img) for img in frames]
    got = abi.solve_batch(frames, [0, 1, 2], 0.3, [0.001] * 3, 50, fdata=fd, lib=lib)
    for f, img in enumerate(frames):
        want = H.run_compute(_checker(), img, [0, 1, 2], 0.3, [0.001] * 3, 50, fd[f])
        H.assert_bit_identical(got[f], want, f'config 1 frame {f}')


def test_config5_two_1080p_frames_full_length(lib):
    """BASELINE config 5's frame (1920x1080 Q75 4:2:0) at its full 100 iterations, two per batch."""
    frames = [synth.synth_coefs(1920, 1080, q, '4:2:0', seed) for q, seed in ((75, 1240), (60, 1241))]
    fd = [H.decode_planes(img) for img in frames]
    got = abi.solve_batch(frames, [0, 1, 2], 0.3, [0.001] * 3, 100, fdata=fd, lib=lib)
    for f, img in enumerate(frames):
        want = H.run_compute(_checker(), img, [0, 1, 2], 0.3, [0.001] * 3, 100, fd[f])
        H.assert_bit_identical(got[f], want, f'config 5 frame {f}')


@pytest.mark.parametrize('case', ['tiny', 'patches'])
def test_guard_rows_in_one_frame_of_a_batch(lib, case):
    """One frame carries the planted values of test_gpu_parity.test_guard_fallback_rows (values
    outside the proven range of the fast division / roots); its neighbours are normal."""
    frames = [synth.synth_coefs(200, 72, q, '4:4:4', seed) for q, seed in ((40, 4321), (70, 11), (25, 12))]
    fd = [H.decode_planes(img) for img in frames]
    rng = np.random.default_rng(7)
    f = fd[0]
    if case == 'tiny':
        fd[0] = [(p * np.float32(2.0 ** -60) * (rng.random(p.shape) < 0.8)).astype(np.float32) for p in f]
    else:
        for p, v in zip(f, (1e-42, 3e-13, 4e21)):
            p[10:14, 30:90] = np.float32(v) * rng.standard_normal((4, 60)).astype(np.float32)
            p[40:41, :] = np.float32(v)
            p[50:60, 100:104] = 0.0
    order = [1, 0, 2]                                       # the planted frame in the middle
    frames, fd = [frames[k] for k in order], [fd[k] for k in order]
    for iters in (1, 6):
        got = abi.solve_batch(frames, [0, 1, 2], 0.3, [0.001] * 3, iters, fdata=[[p.copy() for p in x] for x in fd], lib=lib)
        for k, img in enumerate(frames):
            single = _single(lib, img, [0, 1, 2], 0.3, [0.001] * 3, iters, [p.copy() for p in fd[k]])
            H.assert_bit_identical(got[k], single, f'guard {case} x{iters} frame {k} vs single session')
            want = H.run_compute(_checker(), img, [0, 1, 2], 0.3, [0.001] * 3, iters, [p.copy() for p in fd[k]])
            H.assert_bit_identical(got[k], want, f'guard {case} x{iters} frame {k} vs checker')


def test_pieces_reupload_and_reset(lib):
    frames, ch, w, pw = _frames('420', 3)
    others = [synth.synth_coefs(256, 128, q, '4:2:0', seed) for q, seed in ((15, 900), (85, 901), (45, 902))]
    desc = abi.frame_desc(frames[0], ch, w, pw, 50)
    with abi.Session(lib, desc, 3) as s:
        s.upload(frames, ch)
        s.iterate(0, 50)
        whole = s.download()
        s.iterate(0, 30)
        s.iterate(30, 20)
        H.assert_bit_identical(sum(s.download(), []), sum(whole, []), 'iterate(0,30) + iterate(30,20) vs iterate(0,50)')
        assert lib.j2p_session_reset(s.s) == 0, lib.j2p_last_error()
        s.iterate(0, 50)
        H.assert_bit_identical(sum(s.download(), []), sum(whole, []), 'after reset')
        # new frames into the same batch: re-armed once by the next solve
        s.upload(others, ch)
        before = s.launches
        s.iterate(0, 50)
        resets = s.launches - before - 50 * _launches_per_iteration(lib, others, ch, w, pw, 1, batch=False)
        assert resets == 3 * len(ch), f'{resets} set-up launches for one re-arm of 3 frames'
        again = s.download()
    fresh = abi.solve_batch(others, ch, w, pw, 50, lib=lib)
    H.assert_bit_identical(sum(again, []), sum(fresh, []), 're-uploaded batch vs fresh batch')


def _launches_per_iteration(lib, frames, ch, w, pw, n, batch=True):
    with abi.Session(lib, abi.frame_desc(frames[0], ch, w, pw, 20), n, batch=batch) as s:
        s.upload(frames[:n], ch)
        s.iterate(0, 1)                                     # re-arms the batch
        before = s.launches
        s.iterate(1, 10)
        return (s.launches - before) / 10


@pytest.mark.parametrize('case', ['444', '1080p'])
def test_launches_per_iteration_do_not_grow_with_the_batch(lib, case):
    frames, ch, w, pw = _frames(case, 16)
    one = _launches_per_iteration(lib, frames, ch, w, pw, 1, batch=False)
    assert _launches_per_iteration(lib, frames, ch, w, pw, 1) == one
    assert _launches_per_iteration(lib, frames, ch, w, pw, 16) == one


@pytest.mark.parametrize('bits', [8, 16])
def test_frame_scanlines_match_single_sessions(lib, bits):
    frames, ch, w, pw = _frames('420', 3)
    iters = 10
    img0 = frames[0]
    vw, vh = img0.width, img0.height
    size = vh * (vw * 3 * bits // 8 + 1)
    with abi.Session(lib, abi.frame_desc(img0, ch, w, pw, iters), 3) as s:
        s.upload(frames, ch)
        s.iterate(0, iters)
        got = []
        for f in range(3):
            buf = np.empty(size, np.uint8)
            assert lib.j2p_session_download_frame_scanlines(s.s, f, vw, vh, bits, buf.ctypes.data) == 0, lib.j2p_last_error()
            got.append(buf)
        frame0 = np.empty(size, np.uint8)
        assert lib.j2p_session_download_scanlines(s.s, vw, vh, bits, frame0.ctypes.data) == 0
        assert (frame0 == got[0]).all(), 'download_scanlines is frame 0'
    for f, img in enumerate(frames):
        with abi.Session(lib, abi.frame_desc(img, ch, w, pw, iters), batch=False) as s1:
            s1.upload([img], ch)
            s1.iterate(0, iters)
            want = np.empty(size, np.uint8)
            assert lib.j2p_session_download_scanlines(s1.s, vw, vh, bits, want.ctypes.data) == 0
        assert (got[f] == want).all(), f'frame {f}: {int((got[f] != want).sum())} bytes differ'


def test_refused_calls(lib):
    frames, ch, w, pw = _frames('444', 2)
    desc = abi.frame_desc(frames[0], ch, w, pw, 10)
    s = C.c_void_p()
    assert lib.j2p_session_create_batch(C.byref(s), 0, C.byref(desc), 0) == -1 and not s.value
    assert b'at least one frame' in lib.j2p_last_error()

    def refused(rc, words):
        assert rc == -1, rc
        msg = lib.j2p_last_error()
        assert words in msg, msg

    with abi.Session(lib, desc, 2) as b:
        assert lib.j2p_session_frames(b.s) == 2
        b.upload(frames, ch)
        b.iterate(0, 2)
        p = frames[0].planes[0]
        data, quant = np.ascontiguousarray(p.data), np.ascontiguousarray(p.quant)
        out = np.empty((b.H, b.W), np.float32)
        refused(lib.j2p_session_upload(b.s, 6, data.ctypes.data, quant.ctypes.data, None), b'out of range')
        refused(lib.j2p_session_download(b.s, 6, out.ctypes.data), b'out of range')
        assert lib.j2p_session_plane_ptr(b.s, 6) is None and b'out of range' in lib.j2p_last_error()
        assert lib.j2p_session_plane_ptr(b.s, 5) is not None
        buf = np.empty(b.H * (b.W * 3 + 1), np.uint8)
        refused(lib.j2p_session_download_frame_scanlines(b.s, 2, b.W, b.H, 8, buf.ctypes.data), b'out of range')
        refused(lib.j2p_session_set_logging(b.s, 1), b'batch')
        refused(lib.j2p_session_gradient(b.s), b'batch')
        sums = (C.c_double * 3)()
        refused(lib.j2p_session_project(b.s, C.cast(sums, C.c_void_p), 1), b'batch')
        send, recv, count = C.c_void_p(), C.c_void_p(), C.c_size_t()
        refused(lib.j2p_session_halo(b.s, 0, 0, C.byref(send), C.byref(recv), C.byref(count)), b'batch')
        refused(lib.j2p_session_copy_halo_to_prev(b.s), b'batch')
        refused(lib.j2p_session_strip_info(b.s, None, None, None), b'batch')
        refused(lib.j2p_session_iterate_strip(b.s, None, 1), b'batch')
        assert lib.j2p_session_sums_ptr(b.s) is None and b'batch' in lib.j2p_last_error()
        # the batch is still usable after the refusals
        b.iterate(0, 2)
        b.sync()
