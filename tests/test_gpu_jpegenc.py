"""encode_jpeg and libj2pjpegenc.so on the GPU: the device writes the host driver's bytes on the
whole CPU corpus (one mixed call per quality and sampling, and one call per image), on strided
CUDA views, on decode_jpeg's tensors (where Pillow's bytes are also checked), on an 8K image and
on 64 1080p images in one call; a producer on a side stream, a forced split, launch counts and
the refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

from jpeg2png_b200 import decode_jpeg, encode_jpeg
from jpeg2png_b200 import jpeg_encode as J
from tests import codec_checks as CK
from tests import jpegenc_cases as JC
from tests.test_gpu_decode import FILES, _case

pytestmark = pytest.mark.gpu

CORPUS = JC.corpus()


def _cuda(x):
    """A CUDA tensor with x's values (contiguous)."""
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
@pytest.mark.parametrize('quality', JC.QUALITIES)
def test_device_equals_host_driver(quality, subsampling):
    names = list(CORPUS)
    want = [J.encode_host([CORPUS[n][1]], quality, subsampling, CORPUS[n][0])[0] for n in names]
    got = encode_jpeg([_cuda(CORPUS[n][2]) for n in names], quality=quality, subsampling=subsampling, layout='HWC')
    for n, g, w in zip(names, got, want):
        assert g == w, f'{n} in the mixed call'
    if quality in (1, 75, 100):
        for n, w in zip(names, want):
            lay, a, _ = CORPUS[n]
            assert encode_jpeg(_cuda(a), quality=quality, subsampling=subsampling, layout=lay) == w, f'{n} alone'


def test_strided_device_views_equal_host_driver():
    big = JC.content('cartoon', 200, 300, 7)
    g = _cuda(big)
    views = [(big[5:180:2, 7:290:3], g[5:180:2, 7:290:3], 'HWC'), (big.transpose(2, 0, 1), g.permute(2, 0, 1), 'CHW'),
             (big[::-1], g.flip(0), 'HWC'), (big[:, ::-1], g.flip(1), 'HWC'), (big[..., ::-1], g.flip(2), 'HWC'),
             (big.transpose(2, 1, 0)[:, ::2], g.permute(2, 1, 0)[:, ::2], 'CHW')]
    for s in JC.SAMPLINGS:
        for host, dev, lay in views:
            assert encode_jpeg(dev, quality=85, subsampling=s, layout=lay) == J.encode_host([host], 85, s, lay)[0]


@pytest.mark.parametrize('name', list(FILES))
def test_decoded_tensors_give_pillows_bytes(name):
    data, kw, _, _ = _case(name, False)
    for layout in ('CHW', 'HWC'):
        t = decode_jpeg(data, dtype=torch.uint8, layout=layout, **kw)
        x = t.cpu().numpy()
        hwc = x.transpose(1, 2, 0) if layout == 'CHW' else x
        for q, s in ((95, '4:4:4'), (90, '4:2:0'), (75, '4:2:2')):
            assert encode_jpeg(t, quality=q, subsampling=s, layout=layout) == JC.pillow(hwc, q, s), \
                f'{layout} q{q} {s} ({JC.turbo_version()})'


def test_8k_image_equals_host_driver():
    x = JC.content('cartoon', 4320, 7680, 77)
    for q, s in ((90, '4:2:0'), (100, '4:4:4')):
        assert encode_jpeg(_cuda(x), quality=q, subsampling=s, layout='HWC') == J.encode_host([x], q, s)[0]


def test_64_1080p_in_one_call_equal_host_driver():
    rng = np.random.default_rng(5)
    base = JC.content('cartoon', 1080, 1920, 3)
    xs = [np.clip(base.astype(np.int16) + rng.integers(-6, 7, base.shape), 0, 255).astype(np.uint8) for _ in range(64)]
    got = encode_jpeg([_cuda(x) for x in xs], quality=90, subsampling='4:2:0', layout='HWC')
    for k in range(0, 64, 9):                           # the serial driver on a sample of them
        assert got[k] == J.encode_host([xs[k]], 90, '4:2:0')[0], f'image {k}'
    assert got[63] == J.encode_host([xs[63]], 90, '4:2:0')[0]


def test_producer_on_a_side_stream_needs_no_sync():
    x = JC.content('cartoon', 700, 900, 21)
    want = J.encode_host([x], 80, '4:2:0')[0]
    src = _cuda(x)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        t = torch.zeros_like(src)
        a = torch.full((4096, 4096), 1e-3, device='cuda')
        b = torch.empty_like(a)
        for _ in range(30):                            # ~4 TFLOP: tens of milliseconds before the last write
            torch.mm(a, a, out=b)
            a, b = b, a
        t.copy_(src)
        got = encode_jpeg(t, quality=80, layout='HWC')
    assert got == want


def test_forced_split_gives_the_same_bytes(monkeypatch):
    names = [n for n in CORPUS if n.startswith(('97x61', '200x300', '31x33'))]
    ts = [_cuda(CORPUS[n][2]) for n in names]
    CK.check_forced_split(monkeypatch, J.codec(J.params(70, '4:2:0')), ts, lambda: encode_jpeg(ts, quality=70, layout='HWC'))


def test_refusals():
    with pytest.raises(ValueError, match='CUDA tensors'):
        encode_jpeg(torch.zeros(3, 8, 8, dtype=torch.uint8))
    lib = J.load_jpegenc()
    p = J.Params(75, 2)
    host = np.zeros((8, 8, 3), np.uint8)
    dev = torch.zeros(8, 8, 3, dtype=torch.uint8, device='cuda')

    def desc(ptr):
        d = (J.Image * 1)()
        d[0].data, d[0].width, d[0].height = ptr, 8, 8
        d[0].row_stride, d[0].col_stride, d[0].chan_stride = 24, 3, 1
        return d
    n, o = C.c_size_t(), C.c_size_t()
    assert lib.j2p_jpegenc_plan(desc(dev.data_ptr()), 1, C.byref(p), C.byref(n), C.byref(o)) == 0
    work = torch.empty(n.value, dtype=torch.uint8, device='cuda')
    offs = (C.c_uint64 * 2)()
    assert lib.j2p_jpegenc_encode(desc(host.ctypes.data), 1, C.byref(p), work.data_ptr(), n.value, None, offs, None, 0, None) == -1
    assert 'not device memory' in lib.j2p_jpegenc_last_error().decode()
    hwork = np.zeros(n.value, np.uint8)
    assert lib.j2p_jpegenc_encode(desc(dev.data_ptr()), 1, C.byref(p), hwork.ctypes.data, n.value, None, offs, None, 0, None) == -1
    assert 'not device memory' in lib.j2p_jpegenc_last_error().decode()
    assert lib.j2p_jpegenc_encode(desc(dev.data_ptr()), 1, C.byref(p), work.data_ptr(), n.value - 1, None, offs, None, 0, None) == -1
    # a good call, with the files copied to a host buffer by the library
    st = J.Stats()
    assert lib.j2p_jpegenc_encode(desc(dev.data_ptr()), 1, C.byref(p), work.data_ptr(), n.value, None, offs, None, 0, C.byref(st)) == 0
    assert st.launches == 7 and st.blocks == 6
    buf = np.zeros(offs[1], np.uint8)
    assert lib.j2p_jpegenc_encode(desc(dev.data_ptr()), 1, C.byref(p), work.data_ptr(), n.value, None, offs, buf.ctypes.data,
                                  buf.size - 1, None) == -1
    assert lib.j2p_jpegenc_encode(desc(dev.data_ptr()), 1, C.byref(p), work.data_ptr(), n.value, None, offs, buf.ctypes.data,
                                  buf.size, None) == 0
    assert buf.tobytes() == J.encode_host([host])[0]


def test_launch_count_does_not_depend_on_the_images():
    """The kernels that run on the device, counted by the profiler: each of the seven once per
    call, for one tiny image and for a mixed list alike, and as many as the call reports."""
    names = ('k_je_blocks', 'k_je_sizes', 'k_je_scan', 'k_je_emit', 'k_je_ffcount', 'k_je_offsets', 'k_je_stuff')
    for shapes, st in CK.check_launch_count('jpeg', names):
        assert st['blocks'] == sum(-(-h // 16) * -(-w // 16) * 6 for h, w in shapes)      # 4:2:0 MCUs, six blocks each
