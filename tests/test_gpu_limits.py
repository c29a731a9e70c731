"""The solver at the sizes its sessions accept: batches of up to 65535 frames, frames more than
65535 coefficient blocks tall, slabs and batches past 2^31 and 2^32 elements, exports past 2^32
bytes.  CUDA caps gridDim.y and gridDim.z at 65535, so these are the inputs whose launch grids
(one CTA row per block row, one z slice per frame and plane) or 64-bit offsets a kernel can get
wrong while every everyday size passes.

Every result is compared bit for bit: batch frames with their source solved alone in a single-frame
session, and each source (or the whole frame) with the checker (the compiled reference when it
travelled, else the oracle).  test_cases_cross_their_limits (no GPU) keeps each case above the
limit it is named after."""
import ctypes as C

import numpy as np
import pytest
import torch

from jpeg2png_b200 import abi, decode_jpeg, synth
from tests import helpers as H
from tests import kernel_paths as KP
from tests.test_codecs import make_jpeg

GRID_YZ = 65535                          # CUDA's gridDim.y / gridDim.z limit
MAX_FRAMES = 65535                       # j2p_session_create_batch, decode_jpeg's MAX_BATCH
PW3 = [0.001, 0.0, 0.01]


def slab_elems(W, H, nc):
    """Elements of one frame's slab (session.cu create_impl): x, xp, g, gp of every plane, 64-aligned planes."""
    return ((W * H + 63) & ~63) * 4 * nc


# ---- the cases: plane geometry (cw, ch, sw, sh), and what each one is meant to cross ------------
SMALL = {   # 16 x 16 frames for the full batches
    '444': [(16, 16, 1, 1)] * 3,
    '420': [(16, 16, 1, 1), (8, 8, 2, 2), (8, 8, 2, 2)],
    'yy': [(16, 16, 1, 1)] * 2,                         # two full-resolution planes: one tile launch of count 2
    '422': [(16, 16, 1, 1), (8, 16, 2, 1), (8, 16, 2, 1)],   # chroma on the per-frame generic path
}
# (layout, frames): 65535 frames of each layout, and for each grouping the first count whose
# frames x planes-per-launch pass gridDim.z's limit
BATCHES = [('444', 21846), ('444', MAX_FRAMES), ('420', 32768), ('420', MAX_FRAMES), ('yy', 32768), ('yy', MAX_FRAMES),
           ('422', MAX_FRAMES)]
GROUPED = {'444': 3, '420': 2, 'yy': 2}  # planes that share one projection launch (Y+Cb+Cr, Cb+Cr, Y+Y)
DECODE_BATCHES = [('4:4:4', 30000), ('4:2:0', 32800)]
TALL = {    # (planes, the block rows past the grid limit and which launch they belong to)
    'one_plane': [(16, 524296, 1, 1)],
    '444': [(16, 524296, 1, 1)] * 3,
    '420': [(16, 1048592, 1, 1), (8, 524296, 2, 2), (8, 524296, 2, 2)],
    '422': [(16, 524296, 1, 1), (8, 524296, 2, 1), (8, 524296, 2, 1)],
}
EXPORT_WH = (16, 65552)                  # taller than gridDim.y allows the epilogue's one-row CTAs
SLAB_444 = (13440, 13344)                # slab just past 2^31 elements
SLAB_444_MAX = (18912, 18912)            # the largest square 4:4:4 frame with a slab below 2^32
SLAB_444_REFUSED = (18920, 18920)
SLAB_ONE_PLANE = (23200, 23200)          # one plane, slab past 2^31
BIG_BATCH = (2048, 2048, 86)             # 86 frames of 4:4:4: 4.33e9 slab elements
BIG_BATCH_CHECKED = (0, 42, 85)          # first, the frames that straddle 2^31 and 2^32 elements, last


def _geoms(planes):
    return [KP.PlaneGeom(*p) for p in planes]


def test_cases_cross_their_limits():
    """CPU guard: each case's geometry really passes the limit it names (grid dimensions from the
    launchers' formulas, slab elements, export bytes), so that none can be shrunk into uselessness."""
    for layout, n in BATCHES:
        names, _ = KP.iteration(_geoms(SMALL[layout]), 0.3, KP.Mode(nframes=n))
        if layout == '422':
            assert names.count('k_project<2, 1>') == 2 * n and n == MAX_FRAMES   # a launch per frame and chroma plane
        else:
            group = GROUPED[layout]
            assert group * n > GRID_YZ, (layout, n)               # frames x planes per launch: the old gridDim.z
            assert group * (n - 1) <= GRID_YZ or n == MAX_FRAMES  # the first count that crosses it
    for subsampling, n in DECODE_BATCHES:
        assert GROUPED[{'4:4:4': '444', '4:2:0': '420'}[subsampling]] * n > GRID_YZ and n <= MAX_FRAMES
    assert SMALL['444'][0][:2] == SMALL['420'][0][:2] == (16, 16)
    for name, planes in TALL.items():
        g = _geoms(planes)
        W, Hh = KP.frame_size(g)
        assert W * Hh <= 2**31 - 1 and slab_elems(W, Hh, len(g)) <= 2**32 - 1
        tile_rows = [p.ch // 8 for p in g if (p.sw, p.sh) in ((1, 1), (2, 2))]
        generic_rows = [-(-Hh // (8 * p.sh)) for p in g if (p.sw, p.sh) not in ((1, 1), (2, 2))]
        assert max(tile_rows) > GRID_YZ, name
        if name == '420':
            assert g[1].ch // 8 > GRID_YZ                         # the 2x2 chroma launch too
        if name == '422':
            assert min(generic_rows) > GRID_YZ                    # k_project<2, 1>'s grid.y
        assert _tall_launches(planes, 0.3) > KP.iteration(g, 0.3)[1]   # the frame needs the row split
    assert EXPORT_WH[1] > GRID_YZ
    W, Hh = SLAB_444
    assert 2**31 < slab_elems(W, Hh, 3) < 2**31 + 2**26
    W, Hh = SLAB_444_MAX
    assert slab_elems(W, Hh, 3) <= 2**32 - 1 < slab_elems(*SLAB_444_REFUSED, 3)
    assert SLAB_444_REFUSED[0] - W == 8
    W, Hh = SLAB_ONE_PLANE
    assert slab_elems(W, Hh, 1) > 2**31 and W * Hh <= 2**31 - 1
    W, Hh, n = BIG_BATCH
    fs = slab_elems(W, Hh, 3)
    assert fs * n > 2**32
    assert 42 * fs < 2**31 < 43 * fs and 85 * fs < 2**32 < 86 * fs
    assert n * W * Hh * 3 * 4 > 2**32                             # the float32 export
    assert BIG_BATCH_CHECKED == (0, 42, n - 1)


# ---- GPU side ----------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def lib():
    lib = abi.load_product()
    assert lib.j2p_device_count() > 0, 'no CUDA device visible: the product has no CPU fallback'
    return lib


def _checker():
    return 'ref' if H.have_ref() else 'oracle'


def _need_device_gb(gb):
    """Fail (never skip) when the device does not have the memory a case was measured to need."""
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    assert free >= gb * 2**30, (f'this case needs {gb} GB of free device memory; {free / 2**30:.1f} of '
                                f'{total / 2**30:.1f} GB are free (the device is shared)')


def _random_frame(planes, seed):
    return synth.random_coefs([(p[0], p[1]) for p in planes], [(p[2], p[3]) for p in planes], seed)


def _large_frame(W, Hh, nc, seed):
    """A W x H frame of nc full-resolution planes: a random 512 x 512 frame's blocks tiled."""
    base = synth.random_coefs([(512, 512)] * nc, [(1, 1)] * nc, seed)
    return synth.tile_coefs(base, -(-W // 512), -(-Hh // 512), W, Hh)


def _single(lib, img, ch, w, pw, iters):
    with abi.Session(lib, abi.frame_desc(img, ch, w, pw, iters), batch=False) as s:
        s.upload([img], ch)
        s.iterate(0, iters)
        return s.download()[0]


def _first_difference(got, want, what):
    """got, want: arrays whose leading axis is the frame: fail naming the first frame that differs."""
    diff = H.bits(got) != H.bits(want)
    if diff.any():
        f = int(np.argwhere(diff.reshape(diff.shape[0], -1).any(axis=1))[0][0])
        raise AssertionError(f'{what}: frame {f} differs from its source solved alone '
                             f'({int(diff.sum())} samples differ over all frames)')


@pytest.mark.gpu
@pytest.mark.parametrize('layout,n', BATCHES, ids=[f'{a}-{n}' for a, n in BATCHES])
def test_full_batch_matches_single_sessions(lib, layout, n):
    planes = SMALL[layout]
    ch = list(range(len(planes)))
    w, pw, iters = 0.3, PW3[:len(planes)], 2
    sources = [_random_frame(planes, 9000 + k) for k in range(8)]
    singles = []
    for k, img in enumerate(sources):
        single = _single(lib, img, ch, w, pw, iters)
        H.assert_bit_identical(single, H.run_compute(_checker(), img, ch, w, pw, iters), f'{layout} source {k} vs checker')
        singles.append(np.stack(single))
    _need_device_gb(2)
    with abi.Session(lib, abi.frame_desc(sources[0], ch, w, pw, iters), n) as s:
        s.upload([sources[f % 8] for f in range(n)], ch)
        s.iterate(0, 1)                                     # re-arms the batch
        before = s.launches
        s.iterate(1, iters - 1)
        launches = (s.launches - before) / (iters - 1)
        got = np.stack([np.stack(fr) for fr in s.download()])
    assert launches == KP.iteration(_geoms(planes), w, KP.Mode(nframes=n))[1], f'{launches} launches per iteration'
    _first_difference(got, np.stack([singles[f % 8] for f in range(n)]), f'{layout} batch of {n}')


def _decode_alone(files):
    return [decode_jpeg(f, iterations=3) for f in files]


@pytest.mark.gpu
@pytest.mark.parametrize('subsampling,n', DECODE_BATCHES)
def test_decode_jpeg_one_batch_of_small_files(lib, subsampling, n):
    """decode_jpeg on tens of thousands of thumbnails of one geometry: one batch session (the
    tensors are views of one allocation), every tensor equal to its file decoded alone."""
    files = [make_jpeg(16, 16, q, subsampling, seed=s) for q, s in ((20, 1), (50, 2), (75, 3), (90, 4), (35, 5))]
    alone = _decode_alone(files)
    _need_device_gb(2)
    got = decode_jpeg([files[k % len(files)] for k in range(n)], iterations=3, max_frames=MAX_FRAMES)
    assert len(got) == n
    assert len({t.untyped_storage().data_ptr() for t in got}) == 1, 'the files did not land in one batch'
    want = torch.stack([alone[k % len(files)] for k in range(n)])
    same = (torch.stack(got) == want).flatten(1).all(dim=1)
    assert bool(same.all()), f'{int((~same).sum())} of {n} tensors differ from their file decoded alone; first {int((~same).nonzero()[0])}'


def _tall_launches(planes, w):
    """Launches per iteration of a single frame taller than the grid: kernel_paths.iteration's count
    for the frame, plus one launch per further 65535 CTA rows of each projection launch (the row
    split of launch_project_tile, launch_project_tile22 and launch_project; kMaxGridRows in
    kernels.cuh).  A projection launch has one CTA row per coefficient block row of its plane."""
    g = _geoms(planes)
    _, Hh = KP.frame_size(g)
    extra, c = 0, 0
    while c < len(g):
        p = g[c]
        tiled = (p.sw, p.sh) in ((1, 1), (2, 2))
        cta_rows = p.ch // 8 if tiled else -(-Hh // (8 * p.sh))
        extra += -(-cta_rows // GRID_YZ) - 1
        c += sum(1 for q in g[c:] if q == p) if tiled else 1        # planes of one geometry share a tiled launch
    return KP.iteration(g, w)[1] + extra


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(TALL))
def test_tall_frame_matches_the_checker(lib, name):
    planes = TALL[name]
    ch = list(range(len(planes)))
    w, pw, iters = 0.3, PW3[:len(planes)], 3
    img = _random_frame(planes, 77)
    fd = H.decode_planes(img, ch)
    want = H.run_compute(_checker(), img, ch, w, pw, iters, [p.copy() for p in fd])
    _need_device_gb(2)
    with abi.Session(lib, abi.frame_desc(img, ch, w, pw, iters), batch=False) as s:
        s.upload([img], ch, [fd])
        s.iterate(0, 1)
        before = s.launches
        s.iterate(1, iters - 1)
        launches = (s.launches - before) / (iters - 1)
        H.assert_bit_identical(s.download()[0], want, f'{name} session vs checker')
    assert launches == _tall_launches(planes, w), f'{launches} launches per iteration'
    H.assert_bit_identical(H.run_compute('product', img, ch, w, pw, iters, [p.copy() for p in fd]), want,
                           f'{name} compute() vs checker')


def _rgb_restatement(planes, w, h):
    """png.c:39-47 in numpy (test_gpu_decode.test_float_export_equals_numpy_restatement): (h, w, 3) float32."""
    y = (planes[0][:h, :w] + np.float32(128.0)).astype(np.float64)
    cb, cr = planes[1][:h, :w].astype(np.float64), planes[2][:h, :w].astype(np.float64)
    out = []
    for v in (y + 1.402 * cr, (y - 0.34414 * cb) - 0.71414 * cr, y + 1.772 * cb):
        x = v.astype(np.float32)
        out.append(np.where(x.astype(np.float64) > 255.0, np.float32(255.0), np.where(x.astype(np.float64) < 0.0, np.float32(0.0), x)))
    return np.stack(out, axis=-1).astype(np.float32)


def _samples(f, bits):
    return f if bits == 32 else (np.trunc(f).astype(np.uint8) if bits == 8 else np.trunc(f * np.float32(256.0)).astype(np.uint16))


@pytest.mark.gpu
def test_tall_exports_equal_numpy_restatement(lib):
    W, Hh = EXPORT_WH
    img = _random_frame([(W, Hh, 1, 1)] * 3, 31)
    for p in img.planes:                                    # samples beyond [0, 255] on both sides
        p.data[:] = np.clip(p.data.astype(np.int32) * 6, -1500, 1500).astype(np.int16)
    _need_device_gb(1)
    with abi.Session(lib, abi.frame_desc(img, [0, 1, 2], 0.3, PW3, 2), batch=False) as s:
        s.upload([img], [0, 1, 2])
        s.iterate(0, 2)
        planes = s.download()[0]
        rgb = _rgb_restatement(planes, W, Hh)
        gray = np.ascontiguousarray(_rgb_restatement([planes[0], np.zeros_like(planes[0]), np.zeros_like(planes[0])], W, Hh)[..., 0])
        assert rgb.min() == 0 and rgb.max() == 255, 'the case is meant to hit both clamps'
        for bits, dt in ((8, torch.uint8), (16, torch.uint16), (32, torch.float32)):
            want = _samples(rgb, bits)
            for layout in ('CHW', 'HWC'):
                out = torch.empty((3, Hh, W) if layout == 'CHW' else (Hh, W, 3), dtype=dt, device='cuda')
                o = abi.ImageOut(W, Hh, bits, abi.LAYOUT_CHW if layout == 'CHW' else abi.LAYOUT_HWC, out.numel() * out.element_size())
                assert lib.j2p_session_export(s.s, 0, 1, C.byref(o), C.c_void_p(out.data_ptr()), None) == 0, lib.j2p_last_error()
                torch.cuda.synchronize()
                got = out.cpu().numpy()
                got = np.ascontiguousarray(got.transpose(1, 2, 0) if layout == 'CHW' else got)
                assert (got.view(np.uint8) == want.view(np.uint8)).all(), f'export {bits} bit {layout}: rows {np.unique(np.argwhere(got != want)[:, 0])[:5]} differ'
            out = torch.empty((Hh, W), dtype=dt, device='cuda')
            o = abi.ImageOut(W, Hh, bits, abi.LAYOUT_CHW, out.numel() * out.element_size())
            assert lib.j2p_session_export_gray(s.s, 0, 1, C.byref(o), C.c_void_p(out.data_ptr()), None) == 0, lib.j2p_last_error()
            torch.cuda.synchronize()
            assert (out.cpu().numpy().view(np.uint8) == _samples(gray, bits).view(np.uint8)).all(), f'gray export {bits} bit'
        for bits in (8, 16):
            raw = np.empty(Hh * (W * 3 * bits // 8 + 1), np.uint8)
            assert lib.j2p_session_download_scanlines(s.s, W, Hh, bits, raw.ctypes.data) == 0, lib.j2p_last_error()
            raw = raw.reshape(Hh, -1)
            assert (raw[:, 0] == 0).all(), 'filter bytes'
            want = _samples(rgb, bits).reshape(Hh, -1)
            got = raw[:, 1:] if bits == 8 else raw[:, 1:].copy().view('>u2').astype(np.uint16)
            assert (got == want).all(), f'scanlines {bits} bit: rows {np.unique(np.argwhere(got != want)[:, 0])[:5]} differ'


def _slab_case(lib, W, Hh, nc, need_gb):
    ch = list(range(nc))
    w, pw, iters = 0.3, PW3[:nc], 2
    img = _large_frame(W, Hh, nc, 55)
    fd = H.decode_planes(img, ch)
    _need_device_gb(need_gb)
    with abi.Session(lib, abi.frame_desc(img, ch, w, pw, iters), batch=False) as s:
        s.upload([img], ch, [fd])
        s.iterate(0, iters)
        got = s.download()[0]
    want = H.run_compute(_checker(), img, ch, w, pw, iters, fd)
    H.assert_bit_identical(got, want, f'{W}x{Hh} x{nc} planes vs checker')


@pytest.mark.gpu
def test_slab_past_2_31_elements(lib):
    _slab_case(lib, *SLAB_444, 3, 13)


@pytest.mark.gpu
def test_largest_slab_and_the_next_size_refused(lib):
    d = abi.frame_desc(_random_frame([(8, 8, 1, 1)] * 3, 1), [0, 1, 2], 0.3, PW3, 2)
    for c in range(3):
        d.plane_w[c], d.plane_h[c] = SLAB_444_REFUSED
    s = C.c_void_p()
    assert lib.j2p_session_create(C.byref(s), 0, C.byref(d)) == -1 and not s.value   # J2P_ERR_ARG
    assert b'32-bit element offsets' in lib.j2p_last_error()
    _slab_case(lib, *SLAB_444_MAX, 3, 25)


@pytest.mark.gpu
def test_one_plane_slab_past_2_31_elements(lib):
    _slab_case(lib, *SLAB_ONE_PLANE, 1, 10)


@pytest.mark.gpu
def test_batch_past_2_32_elements(lib):
    W, Hh, n = BIG_BATCH
    ch, w, pw, iters = [0, 1, 2], 0.3, PW3, 2
    sources = [_random_frame([(W, Hh, 1, 1)] * 3, 4000 + k) for k in range(8)]
    singles, exports = [], []
    o = abi.ImageOut(W, Hh, 32, abi.LAYOUT_CHW, 3 * W * Hh * 4)
    for k, img in enumerate(sources):
        with abi.Session(lib, abi.frame_desc(img, ch, w, pw, iters), batch=False) as s:
            s.upload([img], ch)
            s.iterate(0, iters)
            single = s.download()[0]
            ex = torch.empty((3, Hh, W), dtype=torch.float32, device='cuda')
            assert lib.j2p_session_export(s.s, 0, 1, C.byref(o), C.c_void_p(ex.data_ptr()), None) == 0, lib.j2p_last_error()
            torch.cuda.synchronize()
        if k in {f % 8 for f in BIG_BATCH_CHECKED}:
            H.assert_bit_identical(single, H.run_compute(_checker(), img, ch, w, pw, iters), f'source {k} vs checker')
        singles.append(single)
        exports.append(ex)
    _need_device_gb(30)
    with abi.Session(lib, abi.frame_desc(sources[0], ch, w, pw, iters), n) as s:
        s.upload([sources[f % 8] for f in range(n)], ch)
        s.iterate(0, iters)
        for f in BIG_BATCH_CHECKED:
            got = []
            for c in range(3):
                a = np.empty((Hh, W), np.float32)
                assert lib.j2p_session_download(s.s, f * 3 + c, a.ctypes.data) == 0, lib.j2p_last_error()
                got.append(a)
            H.assert_bit_identical(got, singles[f % 8], f'frame {f} of {n} vs its source alone')
        out = torch.empty((n, 3, Hh, W), dtype=torch.float32, device='cuda')
        assert out.numel() * 4 > 2**32
        assert lib.j2p_session_export(s.s, 0, n, C.byref(o), C.c_void_p(out.data_ptr()), None) == 0, lib.j2p_last_error()
        torch.cuda.synchronize()
    for f in range(n):
        assert torch.equal(out[f].view(torch.int32), exports[f % 8].view(torch.int32)), f'float32 export of frame {f} differs'
