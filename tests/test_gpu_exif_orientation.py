"""decode_jpeg(..., apply_exif_orientation=True) and j2p_session_export_oriented on the GPU: every
orientation equals the numpy flip / transpose of the unrotated decode of the same file, and for uint8
what Pillow's ImageOps.exif_transpose makes of it, across dtypes, layouts, joint / separate / gray
exports, the three front ends and sizes that cut the 32 x 32 tiles unevenly; a chunk of mixed
orientations is one export launch; chunks with nothing to rotate take the plain export; the ABI
entry refuses what it should and is ordered with the session streams."""
import ctypes as C
import io

import numpy as np
import pytest
import torch
from PIL import Image, ImageOps

from jpeg2png_b200 import abi, decode, decode_jpeg, synth
from tests.test_gpu_decode import PW, _big_coefficient_session

pytestmark = pytest.mark.gpu

ITERS = 4
DTYPES = (torch.uint8, torch.uint16, torch.float32)


def jpeg(w, h, k, gray=False, progressive=False, seed=1, subsampling='4:4:4'):
    """A Pillow JPEG of a cartoon image carrying EXIF Orientation k (None: no EXIF at all); 4:4:4 by
    default, as the reader refuses 4:2:0 planes of some odd sizes as the reference does."""
    im = Image.fromarray(synth.cartoon_image(w, h, seed).astype(np.uint8), 'RGB')
    if gray:
        im = im.convert('L')
    kw = {}
    if k is not None:
        e = Image.Exif()
        e[0x0112] = k
        kw['exif'] = e.tobytes()
    buf = io.BytesIO()
    im.save(buf, 'JPEG', quality=70, progressive=progressive, subsampling=subsampling, **kw)
    return buf.getvalue()


def oriented_numpy(a, k):
    """a: (h, w, c); the orientation k applied as exif_transpose applies it."""
    return {1: lambda x: x, 2: lambda x: x[:, ::-1], 3: lambda x: x[::-1, ::-1], 4: lambda x: x[::-1],
            5: lambda x: x.transpose(1, 0, 2), 6: lambda x: np.rot90(x, -1), 7: lambda x: x.transpose(1, 0, 2)[::-1, ::-1],
            8: lambda x: np.rot90(x, 1)}[k](a)


def oriented_pillow(a, k):
    """a: (h, w, c) uint8; Pillow's ImageOps.exif_transpose of it with Orientation k."""
    im = Image.fromarray(a[:, :, 0] if a.shape[2] == 1 else a)
    im.getexif()[0x0112] = k
    out = np.asarray(ImageOps.exif_transpose(im))
    return out[:, :, None] if out.ndim == 2 else out


def hwc(t, layout):
    a = t.cpu().numpy()
    return a.transpose(1, 2, 0) if layout == 'CHW' else a


VARIANTS = {
    'joint': (False, {}),
    'separate': (False, dict(separate=True)),
    'gray_of_colour': (False, dict(mode='GRAY')),
    'unchanged_gray': (True, dict(mode='UNCHANGED')),
}
FRONT_ENDS = ('device', 'host', 'progressive')
SIZES = [(97, 61), (1, 40), (40, 1), (33, 65)]


def _check_all_orientations(files, kw, monkeypatch, front, w, h):
    """files[k - 1] carries orientation k; all have the same pixels."""
    if front == 'host':
        monkeypatch.setattr(decode, '_host_front_end', True)
    if front == 'progressive':
        kw = dict(kw, progressive_on_device=True)
    for dtype in DTYPES:
        for layout in ('CHW', 'HWC'):
            plain = decode_jpeg(files[0], iterations=ITERS, dtype=dtype, layout=layout, **kw)
            base = hwc(plain, layout)
            got = decode_jpeg(files, iterations=ITERS, dtype=dtype, layout=layout, apply_exif_orientation=True, **kw)
            for k, t in enumerate(got, 1):
                assert t.is_contiguous() and t.dtype == dtype
                a = hwc(t, layout)
                want = oriented_numpy(base, k)
                assert a.shape == want.shape, (k, a.shape, want.shape)
                assert (np.ascontiguousarray(a).view(np.uint8) == np.ascontiguousarray(want).view(np.uint8)).all(), (dtype, layout, k)
                if dtype == torch.uint8:
                    assert (a == oriented_pillow(base, k)).all(), (layout, k)
                if k >= 5:
                    assert a.shape[:2] == (w, h)


@pytest.mark.parametrize('front', FRONT_ENDS)
@pytest.mark.parametrize('variant', list(VARIANTS))
@pytest.mark.parametrize('size', SIZES, ids=[f'{w}x{h}' for w, h in SIZES])
def test_every_orientation_equals_numpy_and_pillow(monkeypatch, size, variant, front):
    w, h = size
    gray, kw = VARIANTS[variant]
    files = [jpeg(w, h, k, gray=gray, progressive=front == 'progressive', seed=w + h) for k in range(1, 9)]
    _check_all_orientations(files, kw, monkeypatch, front, w, h)


def test_1080p_frame(monkeypatch):
    files = [jpeg(1920, 1080, k, seed=3, subsampling='4:2:0') for k in range(1, 9)]
    plain = decode_jpeg(files[0], iterations=ITERS)
    got = decode_jpeg(files, iterations=ITERS, apply_exif_orientation=True)
    base = hwc(plain, 'CHW')
    for k, t in enumerate(got, 1):
        assert tuple(t.shape) == ((3, 1920, 1080) if k >= 5 else (3, 1080, 1920))
        assert (hwc(t, 'CHW') == oriented_numpy(base, k)).all(), k
        assert (hwc(t, 'CHW') == oriented_pillow(base, k)).all(), k


class _Spy:
    """Counts the export calls decode_jpeg makes and the launches each oriented export adds."""

    def __init__(self, monkeypatch):
        self.lib = abi.load_product()
        self.calls = {name: 0 for name in ('j2p_session_export', 'j2p_session_export_gray', 'j2p_session_export_separate',
                                           'j2p_session_export_oriented')}
        self.launches = []
        for name in self.calls:
            monkeypatch.setattr(self.lib, name, self._wrap(name, getattr(self.lib, name)))

    def _wrap(self, name, fn):
        def call(*args):
            self.calls[name] += 1
            if name != 'j2p_session_export_oriented':
                return fn(*args)
            s = args[0][0]
            before = self.lib.j2p_session_launches(s)
            rc = fn(*args)
            self.launches.append(self.lib.j2p_session_launches(s) - before)
            return rc
        return call


@pytest.mark.parametrize('layout', ['CHW', 'HWC'])
def test_mixed_chunk_is_one_launch_and_equals_each_file_alone(monkeypatch, layout):
    files = [jpeg(120, 88, 1 + i % 8, seed=i, subsampling='4:2:0') for i in range(24)]
    alone = [decode_jpeg(f, iterations=ITERS, layout=layout, apply_exif_orientation=True) for f in files]
    spy = _Spy(monkeypatch)
    got = decode_jpeg(files, iterations=ITERS, layout=layout, apply_exif_orientation=True)
    assert spy.calls['j2p_session_export_oriented'] == 1 and spy.launches == [1]
    assert sum(spy.calls.values()) == 1
    storage = got[0].untyped_storage().data_ptr()
    for i, (t, a) in enumerate(zip(got, alone)):
        assert t.shape == a.shape and torch.equal(t, a), i
        assert t.untyped_storage().data_ptr() == storage and t.is_contiguous()
    split = decode_jpeg(files, iterations=ITERS, layout=layout, apply_exif_orientation=True, max_frames=5)
    for i, (t, a) in enumerate(zip(split, alone)):
        assert t.shape == a.shape and torch.equal(t, a), i


def test_default_ignores_the_tag():
    tagged, untagged = jpeg(120, 88, 6, seed=9, subsampling='4:2:0'), jpeg(120, 88, None, seed=9, subsampling='4:2:0')
    want = decode_jpeg(untagged, iterations=ITERS)
    for got in (decode_jpeg(tagged, iterations=ITERS), decode_jpeg(tagged, iterations=ITERS, apply_exif_orientation=False)):
        assert got.shape == (3, 88, 120) and torch.equal(got, want)


@pytest.mark.parametrize('variant', list(VARIANTS))
def test_chunk_without_rotation_takes_the_plain_export(monkeypatch, variant):
    gray, kw = VARIANTS[variant]
    files = [jpeg(64, 48, k, gray=gray, seed=s, subsampling='4:2:0') for s, k in ((1, 1), (2, None), (3, 1))]
    want = decode_jpeg(files, iterations=ITERS, **kw)
    spy = _Spy(monkeypatch)
    got = decode_jpeg(files, iterations=ITERS, apply_exif_orientation=True, **kw)
    assert spy.calls['j2p_session_export_oriented'] == 0 and sum(spy.calls.values()) == 1
    for t, a in zip(got, want):
        assert t.shape == a.shape and torch.equal(t, a)
        assert t._base is not None and t._base.dim() == 4


def _oriented(lib, sessions, nframes, orient, w, h, dtype, layout, channels=3, stream=None):
    n = len(orient)
    out = torch.empty((n, channels * h * w), dtype=dtype, device='cuda')
    o = abi.ImageOut(w, h, {torch.uint8: 8, torch.uint16: 16, torch.float32: 32}[dtype],
                     abi.LAYOUT_CHW if layout == 'CHW' else abi.LAYOUT_HWC, out[0].numel() * out.element_size())
    ot = torch.tensor(orient, dtype=torch.uint8, device='cuda')
    ss = (C.c_void_p * len(sessions))(*sessions)
    rc = lib.j2p_session_export_oriented(ss, len(sessions), channels, 0, nframes, C.c_void_p(ot.data_ptr()), C.byref(o),
                                         C.c_void_p(out.data_ptr()), stream)
    assert rc == 0, lib.j2p_last_error()
    torch.cuda.synchronize()
    return out


def test_out_of_range_values_and_null_write_orientation_1():
    lib = abi.load_product()
    img, s = _big_coefficient_session(lib)
    with s:
        w, h = img.width, img.height
        for dtype in DTYPES:
            for layout in ('CHW', 'HWC'):
                plain = torch.empty((3 * h * w,), dtype=dtype, device='cuda')
                o = abi.ImageOut(w, h, {torch.uint8: 8, torch.uint16: 16, torch.float32: 32}[dtype],
                                 abi.LAYOUT_CHW if layout == 'CHW' else abi.LAYOUT_HWC, plain.numel() * plain.element_size())
                assert lib.j2p_session_export(s.s, 0, 1, C.byref(o), C.c_void_p(plain.data_ptr()), None) == 0
                ss = (C.c_void_p * 1)(s.s)
                null = torch.empty_like(plain)
                assert lib.j2p_session_export_oriented(ss, 1, 3, 0, 1, None, C.byref(o), C.c_void_p(null.data_ptr()), None) == 0
                torch.cuda.synchronize()
                assert torch.equal(null, plain)
                for v in (0, 9, 255):
                    assert torch.equal(_oriented(lib, [s.s], 1, [v], w, h, dtype, layout)[0], plain), (v, dtype, layout)


def test_session_stream_waits_for_an_oriented_export_on_another_stream():
    lib = abi.load_product()
    img1 = synth.synth_coefs(256, 128, 30, '4:2:0', seed=1)
    img2 = synth.synth_coefs(256, 128, 30, '4:2:0', seed=2)
    desc = abi.frame_desc(img1, [0, 1, 2], 0.3, PW, 20)

    def solved(img):
        with abi.Session(lib, desc, 1, 0, batch=False) as s:
            s.upload([img], [0, 1, 2])
            s.iterate(0, 20)
            out = _oriented(lib, [s.s], 1, [6], 256, 128, torch.uint8, 'HWC')
            s.sync()
            return out

    want1, want2 = solved(img1), solved(img2)
    assert not torch.equal(want1, want2)
    side = torch.cuda.Stream()
    with abi.Session(lib, desc, 1, 0, batch=False) as s:
        s.upload([img1], [0, 1, 2])
        s.iterate(0, 20)
        ot = torch.tensor([6], dtype=torch.uint8, device='cuda')
        torch.cuda.synchronize()
        got = torch.empty((1, 3 * 256 * 128), dtype=torch.uint8, device='cuda')
        o = abi.ImageOut(256, 128, 8, abi.LAYOUT_HWC, 3 * 256 * 128)
        with torch.cuda.stream(side):
            torch.cuda._sleep(100_000_000)                  # holds the export back
            assert lib.j2p_session_export_oriented((C.c_void_p * 1)(s.s), 1, 3, 0, 1, C.c_void_p(ot.data_ptr()), C.byref(o),
                                                   C.c_void_p(got.data_ptr()), C.c_void_p(side.cuda_stream)) == 0
        s.upload([img2], [0, 1, 2])                          # re-arms the session: overwrites the iterates
        s.iterate(0, 20)
        s.sync()
        torch.cuda.synchronize()
        assert torch.equal(got, want1), 'the session overwrote its planes before the export read them'


def test_export_oriented_refusals():
    lib = abi.load_product()
    img = synth.synth_coefs(64, 64, 30, '4:4:4', seed=3)
    joint = abi.frame_desc(img, [0, 1, 2], 0.3, PW, 2)
    one = abi.frame_desc(img, [0], 0.3, PW, 2)
    dst = torch.empty(64 * 64 * 3 * 4 * 2, dtype=torch.uint8, device='cuda')
    p = C.c_void_p(dst.data_ptr())
    orient = torch.tensor([6, 3], dtype=torch.uint8, device='cuda')
    op = C.c_void_p(orient.data_ptr())
    host = (C.c_ubyte * 2)(6, 3)

    def out(w=64, h=64, sample=8, layout=abi.LAYOUT_CHW, frame_bytes=None, c=3):
        fb = w * h * c * max(sample // 8, 1) if frame_bytes is None else frame_bytes
        return C.byref(abi.ImageOut(w, h, sample, layout, fb))

    def refused(rc):
        return rc == -1 and len(lib.j2p_last_error()) > 0

    def ss(*x):
        return (C.c_void_p * len(x))(*x)

    ex = lib.j2p_session_export_oriented
    with abi.Session(lib, joint, 1, 0, batch=False) as s, abi.Session(lib, joint, 2, 0) as b, \
            abi.Session(lib, one, 1, 0, batch=False) as y, abi.Session(lib, one, 1, 0, batch=False) as cb, \
            abi.Session(lib, one, 2, 0) as cr2:
        for x in (s, b):
            x.upload([img] * x.nframes, [0, 1, 2])
            x.iterate(0, 2)
        for x in (y, cb, cr2):
            x.upload([img] * x.nframes, [0])
            x.iterate(0, 2)
        assert ex(ss(s.s), 1, 3, 0, 1, op, out(), p, None) == 0, lib.j2p_last_error()       # the valid calls
        assert ex(ss(b.s), 1, 3, 0, 2, op, out(), p, None) == 0, lib.j2p_last_error()
        assert ex(ss(s.s), 1, 1, 0, 1, op, out(c=1), p, None) == 0, lib.j2p_last_error()
        assert ex(ss(y.s), 1, 1, 0, 1, None, out(c=1), p, None) == 0, lib.j2p_last_error()
        assert ex(ss(y.s, cb.s, y.s), 3, 3, 0, 1, op, out(), p, None) == 0, lib.j2p_last_error()
        assert refused(ex(None, 1, 3, 0, 1, op, out(), p, None))                            # null sessions
        assert refused(ex(ss(None), 1, 3, 0, 1, op, out(), p, None))                        # null session
        assert refused(ex(ss(y.s, None, y.s), 3, 3, 0, 1, op, out(), p, None))
        for n, c in ((0, 3), (2, 3), (3, 1), (1, 2), (1, 0), (4, 3)):                         # none of the three shapes
            assert refused(ex(ss(y.s, cb.s, y.s, cb.s), n, c, 0, 1, op, out(), p, None)), (n, c)
        assert refused(ex(ss(y.s), 1, 3, 0, 1, op, out(), p, None))                         # joint export of nchannel 1
        assert refused(ex(ss(y.s, s.s, cb.s), 3, 3, 0, 1, op, out(), p, None))              # separate with nchannel 3
        assert refused(ex(ss(y.s, cb.s, cr2.s), 3, 3, 0, 1, op, out(), p, None))            # different frame counts
        assert refused(ex(ss(s.s), 1, 3, 0, 1, op, out(), None, None))                      # null dst
        assert refused(ex(ss(s.s), 1, 3, 0, 1, op, None, p, None))                          # null description
        assert refused(ex(ss(s.s), 1, 3, 0, 0, op, out(), p, None))                         # nframes == 0
        assert refused(ex(ss(s.s), 1, 3, 1, 1, op, out(), p, None))                         # frame out of range
        assert refused(ex(ss(b.s), 1, 3, 1, 2, op, out(), p, None))
        assert refused(ex(ss(s.s), 1, 3, 0, 1, op, out(w=0), p, None))
        assert refused(ex(ss(s.s), 1, 3, 0, 1, op, out(h=65), p, None))                     # larger than the frame
        assert refused(ex(ss(s.s), 1, 3, 0, 1, op, out(sample=12), p, None))                # unknown sample
        assert refused(ex(ss(s.s), 1, 3, 0, 1, op, out(layout=2), p, None))                 # unknown layout
        assert refused(ex(ss(s.s), 1, 3, 0, 1, op, out(frame_bytes=64 * 64 * 3 - 1), p, None))
        assert refused(ex(ss(s.s), 1, 3, 0, 1, C.cast(host, C.c_void_p), out(), p, None))   # orientation in host memory
        d = C.c_void_p()
        assert lib.j2p_session_create_strip(C.byref(d), 0, C.byref(joint), 0, 32) == 0, lib.j2p_last_error()
        try:
            assert refused(ex(ss(d), 1, 3, 0, 1, op, out(), p, None))                       # a strip session
            assert refused(ex(ss(d), 1, 1, 0, 1, op, out(c=1), p, None))
        finally:
            lib.j2p_session_destroy(d)
        torch.cuda.synchronize()
