"""CPU tests of the PNG encoder through its serial host driver (j2p_png_encode_host, the same steps
as the kernels of libj2ppng.so): the container and its checksums, the filter heuristic, the round
trip, the size against zlib's run-length deflate, the block types and code-length limits, the
refusals, and the library's kernel inventory."""
import ctypes as C
import io
import os
import zlib

import numpy as np
import pytest

from jpeg2png_b200 import encode as E
from tests import codec_checks as CK
from tests import png_cases as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# kernel -> the GPU test that reaches it (every call of j2p_png_encode launches all four)
KERNELS = {
    'k_png_filter': 'tests/test_gpu_png.py::test_device_equals_host_driver (row filters)',
    'k_png_piece': 'tests/test_gpu_png.py::test_device_equals_host_driver (deflate and checksums of each piece)',
    'k_png_assemble': 'tests/test_gpu_png.py::test_device_equals_host_driver (file layout, joined checksums)',
    'k_png_copy': 'tests/test_gpu_png.py::test_device_equals_host_driver (pieces into the files)',
}

CASES = P.cases()


def _zlib_rle(stream):
    c = zlib.compressobj(1, zlib.DEFLATED, 15, 8, zlib.Z_RLE)
    return len(c.compress(stream) + c.flush())


def _check(png, x, layout):
    stream = P.check_png(png, x, layout)
    idat = P.chunks(png)[1][1]
    pieces = -(-len(stream) // P.PIECE)
    assert len(idat) <= 1.01 * (_zlib_rle(stream) + 6) + 128 * pieces, 'more than 1 % + 128 bytes per piece over zlib'
    return stream


@pytest.mark.parametrize('name', list(CASES))
def test_host_driver_case(name):
    x, layout = CASES[name]
    png = E.encode_host([x], layout)[0]
    _check(png, x, layout)
    a = P.hwc(x, layout)
    if a.size <= 30000:                             # the slow pure-Python unfilter
        stream = zlib.decompress(P.chunks(png)[1][1])
        h, w, _ = a.shape
        assert (P.unfilter(stream, h, w * 3 * a.itemsize, 3 * a.itemsize) == P.scanlines(a)).all()
    if a.dtype == np.uint8:
        from PIL import Image
        im = Image.open(io.BytesIO(png))
        assert im.mode == 'RGB' and (np.asarray(im) == a).all()


def test_many_images_in_one_call_equal_each_alone():
    names = ['1x1', 'stride_at_piece', 'noise_u16', 'chw', 'strided_hwc', 'constant_rem3']
    xs = [CASES[n] for n in names]
    alone = [E.encode_host([x], lay)[0] for x, lay in xs]
    hwc = [P.hwc(x, lay) for x, lay in xs]
    assert E.encode_host(hwc, 'HWC') == alone


def test_random_images():
    rc = P.random_cases()
    pngs = E.encode_host([x for x, _ in rc], 'HWC')
    for (x, lay), png in zip(rc, pngs):
        _check(png, x, lay)


def test_block_types():
    first = lambda name: P.first_block(P.chunks(E.encode_host([CASES[name][0]], CASES[name][1])[0])[1][1])
    assert first('noise_stored')[0] == 0                          # uniform noise: stored
    assert first('1x1')[0] == 1                                   # a few symbols: fixed codes
    t, lit, dist = first('smooth_200x300')
    assert t == 2 and dist == [1]                                 # dynamic, matches: one distance code
    t, lit, dist = first('fibonacci')
    assert t == 2 and max(lit) == 15                              # the 15-bit limit acted
    # no matches at all: still one distance code of one bit
    rng = np.random.default_rng(3)
    x = rng.choice(np.arange(0, 40, 2, dtype=np.uint8), size=(1, 3000, 3))
    x[0, :, :] = np.where(np.arange(9000).reshape(3000, 3) % 2, x[0], x[0] + 1)
    png = E.encode_host([x])[0]
    t, lit, dist = P.first_block(P.chunks(png)[1][1])
    stream = P.check_png(png, x, 'HWC')
    assert t == 2 and dist == [1] and not any(lit[257:])          # no length codes in the block


def test_constant_runs_hit_the_258_cap():
    for r in range(5):
        x, lay = CASES[f'constant_rem{r}']
        stream = P.check_png(E.encode_host([x], lay)[0], x, lay)
        assert set(stream) == {0} and (len(stream) - 1) % 258 == r


def test_sizes_on_deblocked_frames_against_the_host_writer(tmp_path):
    """The oracle solver's output on a few 256x256 frames: encode_png's file sizes against
    j2p_write_png_scanlines (reported, not bounded)."""
    from jpeg2png_b200 import synth
    from tests import helpers as H
    codecs = C.CDLL(os.path.join(ROOT, 'jpeg2png_b200', 'cli', 'libj2pcodecs.so'))
    libc = C.CDLL(None)
    libc.fopen.restype = C.c_void_p
    libc.fopen.argtypes = [C.c_char_p, C.c_char_p]
    libc.fclose.argtypes = [C.c_void_p]
    codecs.j2p_write_png_scanlines.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_void_p]
    ours = theirs = 0
    for seed in range(3):
        img = synth.synth_coefs(256, 256, 10, '4:2:0', seed=40 + seed)
        planes = H.run_compute('oracle', img, [0, 1, 2], 0.3, [0.001] * 3, 10)
        planes[0] = planes[0] + np.float32(128.0)
        ora = H.load_oracle()
        rgb = np.zeros(256 * 256 * 3, np.uint8)
        p = [np.ascontiguousarray(q, np.float32) for q in planes]
        ora.oracle_ycc_to_rgb(256, 256, 8, p[0].ctypes.data, p[0].shape[1], p[1].ctypes.data, p[1].shape[1],
                              p[2].ctypes.data, p[2].shape[1], rgb.ctypes.data)
        x = rgb.reshape(256, 256, 3)
        png = E.encode_host([x])[0]
        _check(png, x, 'HWC')
        ours += len(png)
        raw = np.zeros((256, 256 * 3 + 1), np.uint8)
        raw[:, 1:] = x.reshape(256, -1)
        path = str(tmp_path / f'{seed}.png').encode()
        f = libc.fopen(path, b'wb')
        assert codecs.j2p_write_png_scanlines(f, 256, 256, 8, raw.ctypes.data) == 0
        libc.fclose(f)
        theirs += os.path.getsize(path)
    print(f'3 deblocked 256x256 frames: encode_png {ours} bytes, host writer {theirs} bytes ({ours / theirs:.3f})')


def _descs(**kw):
    d = E.Image()
    d.data, d.width, d.height, d.sample_bytes, d.row_stride, d.col_stride, d.chan_stride = 1 << 20, 4, 4, 1, 12, 3, 1
    for k, v in kw.items():
        setattr(d, k, v)
    return (E.Image * 1)(d)


@pytest.mark.parametrize('bad,match', [
    (dict(data=None), 'null data'), (dict(width=0), 'width and height'), (dict(height=0), 'width and height'),
    (dict(width=1 << 31), 'width and height'), (dict(height=1 << 31), 'width and height'),
    (dict(sample_bytes=3), 'unknown sample size'), (dict(sample_bytes=4), 'unknown sample size')])
def test_abi_refusals(bad, match):
    lib = E.load_png()
    n = C.c_size_t()
    assert lib.j2p_png_plan(_descs(**bad), 1, C.byref(n), None) == -1
    assert match in lib.j2p_png_last_error().decode()
    offs = (C.c_uint64 * 2)()
    assert lib.j2p_png_encode(_descs(**bad), 1, 1 << 20, 1 << 30, None, offs, None, 0, None) == -1
    assert match in lib.j2p_png_last_error().decode()


@pytest.mark.parametrize('w,h,sb,ok', [(27000, 27000, 1, False), (26800, 26800, 1, False), (26700, 26700, 1, True),
                                       (19000, 19000, 2, False), (18900, 18900, 2, True), (2147483647, 2, 1, False),
                                       (1, 2147483647, 2, False)])
def test_plan_refuses_an_image_too_large_for_one_idat_chunk(w, h, sb, ok):
    """PNG caps a chunk at 2^31 - 1 bytes and the file has one IDAT: an image whose worst-case
    IDAT (every block stored) could exceed that is refused before any memory is sized."""
    lib = E.load_png()
    n = C.c_size_t()
    d = _descs(width=w, height=h, sample_bytes=sb, row_stride=3 * w, col_stride=3)
    rc = lib.j2p_png_plan(d, 1, C.byref(n), None)
    if ok:
        assert rc == 0
        # the worst case of the accepted image: header, every piece at its bound, trailer
        filtered = h * (1 + 3 * w * sb)
        assert filtered < 2 ** 31 and n.value > 2 * filtered
    else:
        assert rc == -1 and 'too large for one IDAT chunk' in lib.j2p_png_last_error().decode()
        offs = (C.c_uint64 * 2)()
        assert lib.j2p_png_encode(d, 1, 1 << 20, 1 << 40, None, offs, None, 0, None) == -1
        assert lib.j2p_png_encode_host(d, 1, 1 << 20, 1 << 40, offs) == -1
        assert 'too large for one IDAT chunk' in lib.j2p_png_last_error().decode()


def test_encode_host_refuses_an_image_too_large_with_value_error():
    big = np.lib.stride_tricks.as_strided(np.zeros(1, np.uint8), shape=(27000, 27000, 3), strides=(0, 0, 0))
    with pytest.raises(ValueError, match='too large for one IDAT chunk'):
        E.encode_host([big])


def test_abi_refuses_null_pointers_and_non_device_memory():
    lib = E.load_png()
    n = C.c_size_t()
    assert lib.j2p_png_plan(None, 1, C.byref(n), None) == -1
    assert lib.j2p_png_plan(_descs(), 0, C.byref(n), None) == -1
    x = np.zeros((4, 4, 3), np.uint8)
    d = _descs(data=x.ctypes.data)
    assert lib.j2p_png_plan(d, 1, C.byref(n), None) == 0
    work = np.zeros(n.value, np.uint8)
    offs = (C.c_uint64 * 2)()
    assert lib.j2p_png_encode(d, 1, None, n.value, None, offs, None, 0, None) == -1
    assert 'null' in lib.j2p_png_last_error().decode()
    assert lib.j2p_png_encode(d, 1, work.ctypes.data, n.value, None, None, None, 0, None) == -1
    assert lib.j2p_png_encode(d, 1, work.ctypes.data, n.value, None, offs, None, 0, None) == -1
    assert 'device memory' in lib.j2p_png_last_error().decode() or 'CUDA' in lib.j2p_png_last_error().decode() \
        or 'driver' in lib.j2p_png_last_error().decode()
    assert lib.j2p_png_encode_host(d, 1, work.ctypes.data, n.value - 1, offs) == -1
    assert 'smaller' in lib.j2p_png_last_error().decode()


def test_encode_png_argument_errors():
    import torch
    from jpeg2png_b200 import encode_png
    with pytest.raises(ValueError, match='layout'):
        encode_png(torch.zeros(3, 4, 4, dtype=torch.uint8), layout='NCHW')
    with pytest.raises(ValueError, match='uint8 or torch.uint16'):
        encode_png(torch.zeros(3, 4, 4, dtype=torch.float32))
    with pytest.raises(ValueError, match='CHW'):
        encode_png(torch.zeros(4, 4, 3, dtype=torch.uint8))
    with pytest.raises(ValueError, match='HWC'):
        encode_png(torch.zeros(3, 4, 4, dtype=torch.uint8), layout='HWC')
    with pytest.raises(ValueError, match='3-dimensional'):
        encode_png([torch.zeros(4, 4, dtype=torch.uint8)])
    with pytest.raises(ValueError, match='CUDA tensors'):
        encode_png([torch.zeros(3, 4, 4, dtype=torch.uint8)])
    with pytest.raises(ValueError, match='torch tensors'):
        encode_png(np.zeros((3, 4, 4), np.uint8))


def test_encode_png_without_a_device_raises_runtime_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip('a CUDA device is present')
    from jpeg2png_b200 import encode_png
    with pytest.raises(RuntimeError, match='needs a CUDA device'):
        encode_png([])


def test_kernel_inventory_is_covered_and_does_not_spill():
    CK.check_kernel_inventory('png/libj2ppng.so', KERNELS)
