"""Groups of sessions of different frame sizes on the GPU (pytest -m gpu): j2p_session_iterate_group
runs every frame of every session in one launch per grouped kernel (libj2pmixed.so), and each frame
must be bit-identical to the same frame solved alone in a single-frame session."""
import ctypes as C
import io

import numpy as np
import pytest
import torch
from PIL import Image

from jpeg2png_b200 import abi, decode, decode_jpeg, synth
from tests import helpers as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def lib():
    lib = abi.load_product()
    assert lib.j2p_device_count() > 0, 'no CUDA device visible: the product has no CPU fallback'
    return lib


def _single(lib, img, channels, weight, pw, iters):
    with abi.Session(lib, abi.frame_desc(img, channels, weight, pw, iters), batch=False) as s:
        s.upload([img], channels)
        s.iterate(0, iters)
        launches = s.launches
        return s.download()[0], launches


def _sessions(lib, groups, channels, weight, pw, iters):
    """One session per list of frames of one geometry: a batch when it holds several, else an ordinary one."""
    out = []
    for frames in groups:
        s = abi.Session(lib, abi.frame_desc(frames[0], channels, weight, pw, iters), nframes=len(frames), batch=len(frames) > 1)
        s.upload(frames, channels)
        out.append(s)
    return out


def _group(lib, sessions, first, count):
    arr = (C.c_void_p * len(sessions))(*[s.s.value for s in sessions])
    return lib.j2p_session_iterate_group(arr, len(sessions), first, count)


def _run_group(lib, sessions, first, count):
    rc = _group(lib, sessions, first, count)
    assert rc == 0, lib.j2p_last_error().decode()


def _same(got, want, what):
    for c, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g.view(np.int32), w.view(np.int32)), f'{what}, plane {c}: {int((g.view(np.int32) != w.view(np.int32)).sum())} samples differ'


def _420(w, h, q, seed):
    return synth.synth_coefs(w, h, q, '4:2:0', seed)


def _short_luma(seed):
    """1080p-style: the luma grid is 8 rows short of the frame (frame 48 rows, luma 40), uncovered rows stepped only."""
    return synth.random_coefs([(64, 40), (32, 24), (32, 24)], [(1, 1), (2, 2), (2, 2)], seed)


# layout -> (groups of frames, channels, weight, pweights)
def _layout(name):
    qs = [10, 35, 75, 90, 50, 20]
    if name == '444':
        return ([[synth.synth_coefs(136, 72, 10, '4:4:4', 1), synth.synth_coefs(136, 72, 75, '4:4:4', 2), synth.synth_coefs(136, 72, 35, '4:4:4', 3)],
                 [synth.synth_coefs(64, 48, 50, '4:4:4', 4)], [synth.synth_coefs(8, 8, 90, '4:4:4', 5)],
                 [synth.synth_coefs(200, 40, 20, '4:4:4', 6)]], [0, 1, 2], 0.7, [0.001, 0.0, 0.01])
    if name == '420':
        return ([[_420(256, 128, qs[k], 10 + k) for k in range(3)], [_420(120, 64, 35, 20)], [_420(72, 56, 75, 21)],
                 [_420(16, 16, 90, 22)], [_420(40, 1000, 50, 23)]], [0, 1, 2], 0.3, [0.001] * 3)
    if name == '420_short_luma':
        return ([[_420(128, 64, 10, 30)], [_short_luma(31), _short_luma(32)], [_420(48, 32, 75, 33)]], [0, 1, 2], 0.3, [0.001] * 3)
    if name == 'gray':
        return ([[_420(96, 64, qs[k], 40 + k) for k in range(4)], [_420(8, 8, 50, 45)], [_420(64, 720, 20, 46)]], [0], 0.3, [0.001])
    if name == 'sep_chroma':
        return ([[_420(120, 64, qs[k], 50 + k) for k in range(2)], [_420(48, 48, 90, 55)], [_420(200, 16, 10, 56)]], [1], 0.3, [0.001])
    if name == 'weight0':
        return ([[_420(64, 64, 10, 60)], [_420(32, 48, 75, 61), _420(32, 48, 20, 62)]], [0, 1, 2], 0.0, [0.001] * 3)
    if name == 'pweight0':
        return ([[synth.synth_coefs(64, 40, 10, '4:4:4', 70)], [synth.synth_coefs(24, 16, 75, '4:4:4', 71)]], [0, 1, 2], 0.5, [0.0, 0.0, 0.0])
    raise ValueError(name)


LAYOUTS = ['444', '420', '420_short_luma', 'gray', 'sep_chroma', 'weight0', 'pweight0']


@pytest.mark.parametrize('name', LAYOUTS)
def test_group_frames_match_single_sessions(lib, name):
    groups, ch, w, pw = _layout(name)
    iters = 12
    ss = _sessions(lib, groups, ch, w, pw, iters)
    try:
        _run_group(lib, ss, 0, iters)
        for s, frames in zip(ss, groups):
            got = s.download()
            for f, img in enumerate(frames):
                want, launches = _single(lib, img, ch, w, pw, iters)
                _same(got[f], want, f'{name}: {img.planes[0].w}x{img.planes[0].h} frame {f}')
            if len(frames) == 1:       # the launch count advances as the session's own iterate would advance it
                assert s.launches == launches
    finally:
        for s in ss:
            s.close()


def test_a_few_frames_against_the_checker(lib):
    groups, ch, w, pw = _layout('420')
    ss = _sessions(lib, groups[1:3], ch, w, pw, 10)
    try:
        _run_group(lib, ss, 0, 10)
        for s, frames in zip(ss, groups[1:3]):
            img = frames[0]
            want = H.run_compute('oracle', img, ch, w, pw, 10, H.decode_planes(img))
            H.assert_bit_identical(s.download()[0], want, f'{img.planes[0].w}x{img.planes[0].h} against the oracle')
    finally:
        for s in ss:
            s.close()


def test_pieces_and_continuing_alone(lib):
    groups, ch, w, pw = _layout('420_short_luma')
    iters = 11
    whole = _sessions(lib, groups, ch, w, pw, iters)
    pieces = _sessions(lib, groups, ch, w, pw, iters)
    mixed = _sessions(lib, groups, ch, w, pw, iters)
    try:
        _run_group(lib, whole, 0, iters)
        _run_group(lib, pieces, 0, 3)
        _run_group(lib, pieces, 3, 0)
        _run_group(lib, pieces, 3, 5)
        _run_group(lib, pieces, 8, 3)
        _run_group(lib, mixed, 0, 6)            # then every session alone
        for s in mixed:
            s.iterate(6, iters - 6)
        for a, b, c in zip(whole, pieces, mixed):
            for f, (x, y, z) in enumerate(zip(a.download(), b.download(), c.download())):
                _same(y, x, f'pieces, frame {f}')
                _same(z, x, f'group then alone, frame {f}')
        _run_group(lib, whole, 0, iters)         # first == 0 re-arms: the same solve again
        for a, b in zip(whole, pieces):
            for f, (x, y) in enumerate(zip(a.download(), b.download())):
                _same(x, y, f're-armed, frame {f}')
    finally:
        for s in whole + pieces + mixed:
            s.close()


def test_sessions_on_their_own_streams_are_ordered(lib):
    """Sessions uploaded on their streams and downloaded after the group (downloads sync the session's own stream)."""
    groups, ch, w, pw = _layout('444')
    ss = _sessions(lib, groups, ch, w, pw, 6)
    try:
        _run_group(lib, ss, 0, 6)
        for s, frames in zip(ss[1:], groups[1:]):
            _same(s.download()[0], _single(lib, frames[0], ch, w, pw, 6)[0], 'second session')
    finally:
        for s in ss:
            s.close()


def _refused(lib, ss, first, count, words):
    rc = _group(lib, ss, first, count)
    assert rc == -1, rc
    msg = lib.j2p_last_error().decode()
    for w in words:
        assert w in msg, msg


def test_refusals(lib):
    a = _420(64, 32, 10, 80)
    base = _sessions(lib, [[a], [_420(32, 32, 20, 81)]], [0, 1, 2], 0.3, [0.001] * 3, 10)
    others = []
    try:
        assert lib.j2p_session_iterate_group(None, 0, 0, 1) == -1
        # 4:2:2 planes
        s422 = synth.random_coefs([(96, 48), (48, 48), (48, 48)], [(1, 1), (2, 1), (2, 1)], 82)
        others += _sessions(lib, [[s422]], [0, 1, 2], 0.3, [0.001] * 3, 10)
        _refused(lib, base + others[-1:], 0, 1, ['session 2', '2x1'])
        # other weight, pweight, iterations, plane count
        others += _sessions(lib, [[a]], [0, 1, 2], 0.4, [0.001] * 3, 10)
        _refused(lib, base + others[-1:], 0, 1, ['session 2', 'weight'])
        others += _sessions(lib, [[a]], [0, 1, 2], 0.3, [0.001, 0.0, 0.001], 10)
        _refused(lib, base + others[-1:], 0, 1, ['session 2', 'pweight'])
        others += _sessions(lib, [[a]], [0, 1, 2], 0.3, [0.001] * 3, 11)
        _refused(lib, base + others[-1:], 0, 1, ['session 2', 'iterations'])
        others += _sessions(lib, [[a]], [0], 0.3, [0.001], 10)
        _refused(lib, base + others[-1:], 0, 1, ['session 2', 'planes'])
        # logging
        lg = _sessions(lib, [[a]], [0, 1, 2], 0.3, [0.001] * 3, 10)[0]
        others.append(lg)
        assert lib.j2p_session_set_logging(lg.s, 1) == 0
        _refused(lib, [base[0], lg], 0, 1, ['session 1', 'logs'])
        # a strip session
        st = C.c_void_p()
        assert lib.j2p_session_create_strip(C.byref(st), 0, C.byref(abi.frame_desc(a, [0, 1, 2], 0.3, [0.001] * 3, 10)), 0, 16) == 0
        try:
            arr = (C.c_void_p * 2)(base[0].s.value, st.value)
            assert lib.j2p_session_iterate_group(arr, 2, 0, 1) == -1
            assert 'session 1' in lib.j2p_last_error().decode() and 'strip' in lib.j2p_last_error().decode()
        finally:
            lib.j2p_session_destroy(st)
        # 4:4:0 and odd sampling factors
        s440 = synth.random_coefs([(48, 96), (48, 48), (48, 48)], [(1, 1), (1, 2), (1, 2)], 85)
        others += _sessions(lib, [[s440]], [0, 1, 2], 0.3, [0.001] * 3, 10)
        _refused(lib, base + others[-1:], 0, 1, ['session 2', '1x2'])
        odd = synth.random_coefs([(40, 24), (24, 16), (16, 8)], [(1, 1), (2, 2), (3, 4)], 86)
        others += _sessions(lib, [[odd]], [0, 1, 2], 0.3, [0.001] * 3, 10)
        _refused(lib, base + others[-1:], 0, 1, ['session 2', '3x4'])
        # a refusal re-arms nobody: session 0 (at iteration 0 of a fresh solve) keeps its state
        # the same session twice
        _refused(lib, [base[0], base[1], base[0]], 0, 1, ['session 2', 'session 0 again'])
        # first is not every session's next iteration
        _run_group(lib, base, 0, 2)
        base[0].iterate(2, 1)
        _refused(lib, base, 3, 1, ['session 1', 'contiguous'])
        # more than 65535 frames
        big = abi.Session(lib, abi.frame_desc(synth.synth_coefs(8, 8, 50, '4:4:4', 83), [0, 1, 2], 0.3, [0.001] * 3, 10), nframes=65535)
        others.append(big)
        one = _sessions(lib, [[synth.synth_coefs(16, 8, 50, '4:4:4', 84)]], [0, 1, 2], 0.3, [0.001] * 3, 10)[0]
        others.append(one)
        _refused(lib, [big, one], 0, 1, ['session 1', '65535 frames'])
    finally:
        for s in base + others:
            s.close()


def test_refused_call_changes_nothing(lib):
    a, b = _420(64, 32, 10, 90), _420(32, 32, 20, 91)
    ss = _sessions(lib, [[a], [b]], [0, 1, 2], 0.3, [0.001] * 3, 8)
    try:
        _run_group(lib, ss, 0, 4)
        ss[1].iterate(4, 1)                                       # session 1 is one iteration ahead
        launches = [s.launches for s in ss]
        rc = _group(lib, [ss[0], ss[1]], 5, 1)                     # session 0 expects 4
        assert rc == -1 and 'session 0' in lib.j2p_last_error().decode()
        assert [s.launches for s in ss] == launches
        fresh = abi.Session(lib, abi.frame_desc(b, [0, 1, 2], 0.3, [0.001] * 3, 8), batch=False)   # nothing uploaded
        try:
            rc = _group(lib, [ss[0], fresh], 0, 1)              # first == 0 would re-arm session 0
            assert rc == -1 and 'session 1' in lib.j2p_last_error().decode()
        finally:
            fresh.close()
        assert [s.launches for s in ss] == launches
        ss[0].iterate(4, 4)                                       # session 0 continues where it was
        _same(ss[0].download()[0], _single(lib, a, [0, 1, 2], 0.3, [0.001] * 3, 8)[0], 'after a refused call')
    finally:
        for s in ss:
            s.close()


def _grouped_kernels(lib, ss, iters):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _run_group(lib, ss, 0, iters)
        for s in ss:
            s.sync()
    return sum(1 for e in prof.events() if 'grouped' in e.name)


def test_launches_per_iteration_do_not_grow_with_the_group(lib):
    """4:2:0 frames of whole MCUs: one gradient (GPM 2), one luma tile and one chroma tile launch per
    iteration, for 2 sessions or 9."""
    sizes = [(64, 32), (48, 48), (128, 16), (32, 96), (16, 16), (80, 64), (96, 32), (112, 48), (48, 144)]
    counts = []
    for n in (2, 9):
        ss = _sessions(lib, [[_420(w, h, 50, 100 + k)] for k, (w, h) in enumerate(sizes[:n])], [0, 1, 2], 0.3, [0.001] * 3, 5)
        try:
            counts.append(_grouped_kernels(lib, ss, 5))
        finally:
            for s in ss:
                s.close()
    assert counts == [3 * 5, 3 * 5], counts


# ---- decode_jpeg on mixed-size lists ---------------------------------------------------------------
def jpeg(w, h, seed, gray=False, subsampling='4:2:0', orientation=None, quality=40):
    im = Image.fromarray(synth.cartoon_image(w, h, seed).astype(np.uint8), 'RGB')
    if gray:
        im = im.convert('L')
    kw = {}
    if orientation is not None:
        e = Image.Exif()
        e[0x0112] = orientation
        kw['exif'] = e.tobytes()
    buf = io.BytesIO()
    im.save(buf, 'JPEG', quality=quality, subsampling=subsampling, **kw)
    return buf.getvalue()


class _GroupSpy:
    def __init__(self, monkeypatch):
        lib = abi.load_product()
        real = lib.j2p_session_iterate_group
        self.calls = []

        def spy(arr, n, first, count):
            self.calls.append(n)
            return real(arr, n, first, count)
        monkeypatch.setattr(lib, 'j2p_session_iterate_group', spy)


SIZES = [(64, 48), (80, 32), (48, 64), (96, 96), (32, 32), (120, 88), (16, 16), (200, 40)]


@pytest.mark.parametrize('dtype', [torch.uint8, torch.uint16, torch.float32])
@pytest.mark.parametrize('layout', ['CHW', 'HWC'])
def test_decode_mixed_sizes_equals_each_file_alone(monkeypatch, dtype, layout):
    files = [jpeg(w, h, k) for k, (w, h) in enumerate(SIZES)]
    alone = [decode_jpeg(f, iterations=6, dtype=dtype, layout=layout) for f in files]
    spy = _GroupSpy(monkeypatch)
    got = decode_jpeg(files, iterations=6, dtype=dtype, layout=layout)
    assert spy.calls == [len(SIZES)]                   # one pack, one group call
    for i, (t, a) in enumerate(zip(got, alone)):
        assert t.shape == a.shape and torch.equal(t, a), i


@pytest.mark.parametrize('mode', ['GRAY', 'UNCHANGED'])
def test_decode_gray_modes(monkeypatch, mode):
    files = [jpeg(w, h, k, gray=k % 2 == 0) for k, (w, h) in enumerate(SIZES)]
    alone = [decode_jpeg(f, iterations=6, mode=mode) for f in files]
    spy = _GroupSpy(monkeypatch)
    got = decode_jpeg(files, iterations=6, mode=mode)
    # GRAY: every colour file is a joint 3-plane chunk and every gray file a 1-plane chunk: two classes
    assert sorted(spy.calls) == [4, 4]
    for i, (t, a) in enumerate(zip(got, alone)):
        assert t.shape == a.shape and torch.equal(t, a), i


def test_decode_orientation_and_max_frames(monkeypatch):
    files = [jpeg(w, h, k, orientation=1 + k % 8) for k, (w, h) in enumerate(SIZES)]
    files += [jpeg(*SIZES[0], 50, orientation=6), jpeg(*SIZES[1], 51, orientation=3)]     # a second frame of two sizes
    alone = [decode_jpeg(f, iterations=6, apply_exif_orientation=True) for f in files]
    spy = _GroupSpy(monkeypatch)
    got = decode_jpeg(files, iterations=6, apply_exif_orientation=True)
    assert spy.calls == [len(SIZES)]                   # two frames of a size are one chunk (a batch of 2)
    for i, (t, a) in enumerate(zip(got, alone)):
        assert t.shape == a.shape and torch.equal(t, a), i
    spy.calls.clear()
    got = decode_jpeg(files, iterations=6, apply_exif_orientation=True, max_frames=1)
    # chunks in plan order: sizes 0 and 1 have two chunks each, so the packs are
    # [0] [0', 1] [1', 2 .. 7]: every pack holds one chunk per geometry
    assert spy.calls == [2, len(SIZES) - 1]
    for i, (t, a) in enumerate(zip(got, alone)):
        assert t.shape == a.shape and torch.equal(t, a), i


def test_switch_off_and_separate_and_large_frames_take_todays_path(monkeypatch):
    files = [jpeg(w, h, k) for k, (w, h) in enumerate(SIZES[:4])] + [jpeg(512, 512, 9)]
    spy = _GroupSpy(monkeypatch)
    on = decode_jpeg(files, iterations=6)
    assert spy.calls == [4]                            # the 512x512 file is over GROUP_MAX_PIXELS
    spy.calls.clear()
    monkeypatch.setattr(decode, '_group_chunks', False)
    off = decode_jpeg(files, iterations=6)
    assert spy.calls == []
    for t, a in zip(on, off):
        assert torch.equal(t, a)
    monkeypatch.setattr(decode, '_group_chunks', True)
    sep = decode_jpeg(files, iterations=6, separate=True)
    assert spy.calls == []
    for f, t in zip(files, sep):
        assert torch.equal(t, decode_jpeg(f, iterations=6, separate=True))
