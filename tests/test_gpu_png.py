"""encode_png and libj2ppng.so on the GPU: the device writes the host driver's bytes on every CPU
case (one mixed call and one call per image), an 8K 16-bit image, JPEG files through
decode_jpeg + encode_png against the checker pipeline, a producer on a side stream, a forced
split, the refusals and launch counts."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

from jpeg2png_b200 import decode_jpeg, encode_png
from jpeg2png_b200 import encode as E
from tests import codec_checks as CK
from tests import png_cases as P
from tests.test_codecs import codecs, read_jpeg  # noqa: F401  (codecs is a fixture)
from tests.test_gpu_cli import expected_rgb
from tests.test_gpu_decode import FILES, PW, _case, expected_rgb16

pytestmark = pytest.mark.gpu

CASES = P.cases()


def _cuda(x):
    """A CUDA tensor with x's values (contiguous)."""
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def test_device_equals_host_driver():
    items = list(CASES.values()) + P.random_cases()
    want = [E.encode_host([x], lay)[0] for x, lay in items]
    hwc = [P.hwc(x, lay) for x, lay in items]
    got_one_call = encode_png([_cuda(x) for x in hwc], layout='HWC')
    for k, (g, w) in enumerate(zip(got_one_call, want)):
        assert g == w, f'image {k} of the mixed call'
    for k, (x, lay) in enumerate(items):
        assert encode_png(_cuda(x), layout=lay) == want[k], f'image {k} alone'


def test_strided_device_views_equal_host_driver():
    big = P.cases()['smooth_200x300'][0]
    g = _cuda(big)
    views = [(big[5:180:2, 7:290:3], g[5:180:2, 7:290:3], 'HWC'), (big.transpose(2, 0, 1), g.permute(2, 0, 1), 'CHW'),
             (big[::-1].copy()[10:20], g.flip(0)[10:20], 'HWC')]
    u16 = P.cases()['smooth_u16'][0]
    gu = _cuda(u16)
    views.append((u16.transpose(2, 1, 0)[:, ::2], gu.permute(2, 1, 0)[:, ::2], 'CHW'))
    for host, dev, lay in views:
        assert encode_png(dev, layout=lay) == E.encode_host([host], lay)[0]


def test_8k_uint16_equals_host_driver_and_round_trips():
    h, w = 4320, 7680
    x = P._smooth(h, w, np.uint16, seed=77)
    got = encode_png(_cuda(x), layout='HWC')
    assert got == E.encode_host([x], 'HWC')[0]
    ch = P.chunks(got)
    stream = zlib.decompress(ch[1][1])
    raw = P.scanlines(x)
    rb = w * 6 + 1
    assert len(stream) == h * rb
    for y0 in range(0, h, 256):                        # the numpy restatement in bands of rows
        y1 = min(h, y0 + 256)
        lo = max(0, y0 - 1)
        _, want = P.filter_rows(raw[lo:y1], 6)
        assert stream[y0 * rb:y1 * rb] == want[(y0 - lo) * rb:]


def _png_pixels(png):
    ch = P.chunks(png)
    w, h, depth = int.from_bytes(ch[0][1][:4], 'big'), int.from_bytes(ch[0][1][4:8], 'big'), ch[0][1][8]
    sb = depth // 8
    raw = P.unfilter(zlib.decompress(ch[1][1]), h, w * 3 * sb, 3 * sb)
    if sb == 2:
        return raw.view('>u2').astype(np.uint16).reshape(h, w, 3)
    return raw.reshape(h, w, 3)


@pytest.mark.parametrize('sep', [False, True], ids=['joint', 'separate'])
@pytest.mark.parametrize('name', list(FILES))
def test_jpeg_files_through_decode_and_encode(codecs, name, sep):  # noqa: F811
    data, kw, iters, weights = _case(name, sep)
    img, err = read_jpeg(codecs, data)
    assert img is not None, err
    for dtype, want in ((torch.uint8, expected_rgb(img, not sep, iters, weights, PW)),
                        (torch.uint16, expected_rgb16(img, not sep, iters, weights, PW))):
        for layout in ('CHW', 'HWC'):
            t = decode_jpeg(data, dtype=dtype, layout=layout, **kw)
            px = _png_pixels(encode_png(t, layout=layout))
            tt = t.cpu().numpy()
            assert (px == (tt.transpose(1, 2, 0) if layout == 'CHW' else tt)).all()
            assert (px == want).all(), f'{dtype} {layout}: the PNG pixels differ from the command line pipeline'


def test_producer_on_a_side_stream_needs_no_sync():
    x = P._smooth(700, 900, seed=21)
    want = E.encode_host([x], 'HWC')[0]
    src = _cuda(x)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        t = torch.zeros_like(src)
        for _ in range(20):                            # keep the stream busy before the last write
            t.add_(1)
        t.copy_(src)
        got = encode_png(t, layout='HWC')
    assert got == want


def test_forced_split_gives_the_same_bytes(monkeypatch):
    ts = [_cuda(P._smooth(120 + 40 * k, 200, np.uint16 if k % 2 else np.uint8, seed=k)) for k in range(6)]
    CK.check_forced_split(monkeypatch, E.CODEC, ts, lambda: encode_png(ts, layout='HWC'))


def test_refusals():
    with pytest.raises(ValueError, match='CUDA tensors'):
        encode_png(torch.zeros(3, 8, 8, dtype=torch.uint8))
    lib = E.load_png()
    host = np.zeros((8, 8, 3), np.uint8)
    dev = torch.zeros(8, 8, 3, dtype=torch.uint8, device='cuda')

    def desc(ptr):
        d = (E.Image * 1)()
        d[0].data, d[0].width, d[0].height, d[0].sample_bytes = ptr, 8, 8, 1
        d[0].row_stride, d[0].col_stride, d[0].chan_stride = 24, 3, 1
        return d
    n, o = C.c_size_t(), C.c_size_t()
    assert lib.j2p_png_plan(desc(dev.data_ptr()), 1, C.byref(n), C.byref(o)) == 0
    work = torch.empty(n.value, dtype=torch.uint8, device='cuda')
    offs = (C.c_uint64 * 2)()
    assert lib.j2p_png_encode(desc(host.ctypes.data), 1, work.data_ptr(), n.value, None, offs, None, 0, None) == -1
    assert 'not device memory' in lib.j2p_png_last_error().decode()
    hwork = np.zeros(n.value, np.uint8)
    assert lib.j2p_png_encode(desc(dev.data_ptr()), 1, hwork.ctypes.data, n.value, None, offs, None, 0, None) == -1
    assert 'not device memory' in lib.j2p_png_last_error().decode()
    assert lib.j2p_png_encode(desc(dev.data_ptr()), 1, work.data_ptr(), n.value - 1, None, offs, None, 0, None) == -1
    # a good call, with the files copied to a host buffer by the library
    st = E.Stats()
    assert lib.j2p_png_encode(desc(dev.data_ptr()), 1, work.data_ptr(), n.value, None, offs, None, 0, C.byref(st)) == 0
    assert st.launches == 4 and st.pieces == 1
    buf = np.zeros(offs[1], np.uint8)
    assert lib.j2p_png_encode(desc(dev.data_ptr()), 1, work.data_ptr(), n.value, None, offs, buf.ctypes.data, buf.size - 1, None) == -1
    assert lib.j2p_png_encode(desc(dev.data_ptr()), 1, work.data_ptr(), n.value, None, offs, buf.ctypes.data, buf.size, None) == 0
    assert buf.tobytes() == E.encode_host([host], 'HWC')[0]


def test_launch_count_does_not_depend_on_the_images():
    """The kernels that run on the device, counted by the profiler: each of the four once per call,
    for one tiny image and for a mixed list alike, and as many as the call reports."""
    for _, st in CK.check_launch_count('png', ('k_png_filter', 'k_png_piece', 'k_png_assemble', 'k_png_copy')):
        assert st['launches'] == 4
