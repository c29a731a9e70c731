"""encode_jpeg(..., progressive=True) and libj2pjpegprog.so on the GPU: the device writes the host
driver's bytes on the whole CPU corpus (one mixed call per quality and sampling, and images alone),
on strided and flipped CUDA views, on the crafted run cases and partial-MCU sizes, on an 8K image, a
flat 8K image (the longest run segments) and 64 1080p images in one call; decode_jpeg's tensors give
Pillow's progressive bytes; decode_jpeg reads a progressive file to the default file's tensors on
either front end; a producer on a side stream, a forced split and launch counts."""
import numpy as np
import pytest
import torch

from jpeg2png_b200 import decode_jpeg, encode_jpeg
from jpeg2png_b200 import jpeg_encode as J
from tests import codec_checks as CK
from tests import jpegenc_cases as JC
from tests import jpegprog_cases as PC
from tests.test_gpu_decode import FILES, _case
from tests.test_jpegprog_host import _reader_takes

pytestmark = pytest.mark.gpu

CORPUS = JC.corpus()


def _cuda(x):
    """A CUDA tensor with x's values (contiguous)."""
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _host(xs, q, s, layout='HWC'):
    return J.encode_host(xs, q, s, layout, progressive=True)


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
@pytest.mark.parametrize('quality', JC.QUALITIES)
def test_device_equals_host_driver(quality, subsampling):
    names = list(CORPUS)
    want = [_host([CORPUS[n][1]], quality, subsampling, CORPUS[n][0])[0] for n in names]
    got = encode_jpeg([_cuda(CORPUS[n][2]) for n in names], quality=quality, subsampling=subsampling, layout='HWC', progressive=True)
    for n, g, w in zip(names, got, want):
        assert g == w, f'{n} in the mixed call'
    if quality in (1, 75, 100):
        for n, w in zip(names, want):
            lay, a, _ = CORPUS[n]
            assert encode_jpeg(_cuda(a), quality=quality, subsampling=subsampling, layout=lay, progressive=True) == w, f'{n} alone'


def test_strided_and_flipped_device_views_equal_host_driver():
    big = JC.content('cartoon', 200, 300, 7)
    g = _cuda(big)
    views = [(big[5:180:2, 7:290:3], g[5:180:2, 7:290:3], 'HWC'), (big.transpose(2, 0, 1), g.permute(2, 0, 1), 'CHW'),
             (big[::-1], g.flip(0), 'HWC'), (big[:, ::-1], g.flip(1), 'HWC'), (big[..., ::-1], g.flip(2), 'HWC'),
             (big.transpose(2, 1, 0)[:, ::2], g.permute(2, 1, 0)[:, ::2], 'CHW')]
    for s in JC.SAMPLINGS:
        for host, dev, lay in views:
            assert encode_jpeg(dev, quality=85, subsampling=s, layout=lay, progressive=True) == _host([host], 85, s, lay)[0]


def test_crafted_run_cases_and_partial_mcu_sizes_equal_host_driver():
    for name, (x, q, s, _) in PC.crafted().items():
        assert encode_jpeg(_cuda(x), quality=q, subsampling=s, layout='HWC', progressive=True) == _host([x], q, s)[0], name
    for h, w, s in PC.partial_mcu():
        xs = [JC.content(kind, h, w, h * w) for kind in ('cartoon', 'noise')]
        assert encode_jpeg([_cuda(x) for x in xs], quality=95, subsampling=s, layout='HWC', progressive=True) == _host(xs, 95, s)


@pytest.mark.parametrize('name', list(FILES))
def test_decoded_tensors_give_pillows_progressive_bytes(name):
    data, kw, _, _ = _case(name, False)
    for layout in ('CHW', 'HWC'):
        t = decode_jpeg(data, dtype=torch.uint8, layout=layout, **kw)
        x = t.cpu().numpy()
        hwc = x.transpose(1, 2, 0) if layout == 'CHW' else x
        for q, s in ((95, '4:4:4'), (90, '4:2:0'), (75, '4:2:2')):
            assert encode_jpeg(t, quality=q, subsampling=s, layout=layout, progressive=True) == PC.pillow_progressive(hwc, q, s), \
                f'{layout} q{q} {s} ({JC.turbo_version()})'


def test_8k_image_equals_host_driver():
    x = JC.content('cartoon', 4320, 7680, 77)
    for q, s in ((90, '4:2:0'), (100, '4:4:4')):
        assert encode_jpeg(_cuda(x), quality=q, subsampling=s, layout='HWC', progressive=True) == _host([x], q, s)[0]


def test_flat_8k_equals_host_driver():
    """Every AC block of a flat image adds to one EOB run: each AC scan is one run segment of up to
    518,400 blocks, walked by one thread."""
    x = np.full((4320, 7680, 3), 77, np.uint8)
    for q, s in ((90, '4:2:0'), (95, '4:4:4')):
        got = encode_jpeg(_cuda(x), quality=q, subsampling=s, layout='HWC', progressive=True)
        assert got == _host([x], q, s)[0]


def test_64_1080p_in_one_call_equal_host_driver():
    rng = np.random.default_rng(5)
    base = JC.content('cartoon', 1080, 1920, 3)
    xs = [np.clip(base.astype(np.int16) + rng.integers(-6, 7, base.shape), 0, 255).astype(np.uint8) for _ in range(64)]
    got = encode_jpeg([_cuda(x) for x in xs], quality=90, subsampling='4:2:0', layout='HWC', progressive=True)
    for k in range(0, 64, 9):                           # the serial driver on a sample of them
        assert got[k] == _host([xs[k]], 90, '4:2:0')[0], f'image {k}'
    assert got[63] == _host([xs[63]], 90, '4:2:0')[0]


@pytest.mark.parametrize('dtype', [torch.uint8, torch.uint16, torch.float32])
def test_decode_of_progressive_file_equals_decode_of_default_file(dtype):
    xs = [JC.content('cartoon', 120, 160, 3), JC.content('noise', 64, 48, 4), JC.content('cartoon', 96, 62, 5)]
    assert all(_reader_takes(*x.shape[:2], '4:2:0') for x in xs)
    ts = [_cuda(x) for x in xs]
    prog = encode_jpeg(ts, quality=80, subsampling='4:2:0', layout='HWC', progressive=True)
    base = encode_jpeg(ts, quality=80, subsampling='4:2:0', layout='HWC')
    assert all(p != b for p, b in zip(prog, base))
    for on_device in (False, True):
        got = decode_jpeg(prog, iterations=10, dtype=dtype, progressive_on_device=on_device)
        want = decode_jpeg(base, iterations=10, dtype=dtype)
        assert len(got) == len(want) == 3
        for g, w in zip(got, want):
            assert torch.equal(g, w), on_device
        assert torch.equal(decode_jpeg(prog[0], iterations=10, dtype=dtype, progressive_on_device=on_device),
                           decode_jpeg(base[0], iterations=10, dtype=dtype))


def test_producer_on_a_side_stream_needs_no_sync():
    x = JC.content('cartoon', 700, 900, 21)
    want = _host([x], 80, '4:2:0')[0]
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
        got = encode_jpeg(t, quality=80, layout='HWC', progressive=True)
    assert got == want


def test_forced_split_gives_the_same_bytes(monkeypatch):
    names = [n for n in CORPUS if n.startswith(('97x61', '200x300', '31x33'))]
    ts = [_cuda(CORPUS[n][2]) for n in names]
    CK.check_forced_split(monkeypatch, J.codec(J.params(70, '4:2:0'), progressive=True), ts,
                          lambda: encode_jpeg(ts, quality=70, layout='HWC', progressive=True))


def test_launch_count_does_not_depend_on_the_images():
    """The kernels that run on the device, counted by the profiler: each of the ten once per call,
    for one tiny image and for a mixed list alike, and as many as the call reports."""
    names = ('k_jp_blocks', 'k_jp_runs', 'k_jp_hist', 'k_jp_tables', 'k_jp_sizes', 'k_jp_scan', 'k_jp_emit', 'k_jp_ffcount',
             'k_jp_offsets', 'k_jp_stuff')
    for shapes, st in PC.check_launch_count(names):
        assert st['launches'] == 10
        assert st['blocks'] == sum(-(-h // 16) * -(-w // 16) * 6 for h, w in shapes)      # 4:2:0 MCUs, six blocks each
