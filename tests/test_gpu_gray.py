"""Grayscale decode and encode on the GPU: decode_jpeg(mode='UNCHANGED') on one-component files is
bit-identical to the checker pipeline (reader coefficients -> oracle compute(1) -> +128 -> the
reference colour conversion with zero chroma, channel R) at 8, 16 and 32 bits in both layouts, with
both front ends and the progressive device decoder; mode='GRAY' on colour files gives the checker's
joint or separate luma; mixed lists, max_frames splits and a 64-file batch equal per-file results;
every refusal of j2p_session_export_gray; encode_png on gray tensors equals its host driver and
round-trips decode_jpeg's pixels."""
import ctypes as C
import io

import numpy as np
import pytest
import torch
from PIL import Image

from jpeg2png_b200 import abi, decode_jpeg, encode_png, synth
from jpeg2png_b200 import decode as D
from jpeg2png_b200 import encode as E
from tests import helpers as H
from tests import png_cases as P
from tests.test_gpu_decode import FILES, PW, _case
from tests.test_gray_host import CORPUS, GRAY_PNG, gray_jpeg, synth_colour

pytestmark = pytest.mark.gpu

ITERS, WEIGHT = 12, 0.3
SAMPLE = {torch.uint8: 8, torch.uint16: 16, torch.float32: 32}


def coef_image(data, flags=D.READ_GRAY):
    p = D.parse_jpeg(data, flags)
    return synth.CoefImage(width=p.w, height=p.h, planes=[synth.Plane(w=x.w, h=x.h, w_samp=x.w_samp, h_samp=x.h_samp,
                                                                      data=x.data, quant=x.quant) for x in p.planes])


def checker_gray(img, luma, dtype):
    """(h, w) samples of the solved luma plane `luma` through the reference conversion with zero
    chroma, channel R: 8-bit, 16-bit (as integers) or the float sample (numpy restatement)."""
    h, w = img.height, img.width
    y = np.ascontiguousarray(luma + np.float32(128.0), np.float32)
    if dtype == torch.float32:
        x = y[:h, :w].astype(np.float64).astype(np.float32)
        return np.where(x.astype(np.float64) > 255.0, np.float32(255.0), np.where(x.astype(np.float64) < 0.0, np.float32(0.0), x))
    bits = SAMPLE[dtype]
    zero = np.zeros_like(y)
    out = np.zeros(w * h * 3 * bits // 8, np.uint8)
    H.load_oracle().oracle_ycc_to_rgb(w, h, bits, y.ctypes.data, y.shape[1], zero.ctypes.data, zero.shape[1],
                                      zero.ctypes.data, zero.shape[1], out.ctypes.data)
    rgb = out.reshape(h, w, 3) if bits == 8 else out.view('>u2').astype(np.uint16).reshape(h, w, 3)
    assert (rgb[..., 0] == rgb[..., 1]).all() and (rgb[..., 0] == rgb[..., 2]).all()
    return rgb[..., 0]


def gray_luma(img, iterations=ITERS, weight=WEIGHT):
    return H.run_compute('oracle', img, [0], weight, [PW[0]], iterations)[0]


def plane_of(t, layout):
    a = t.cpu().numpy()
    assert a.ndim == 3
    return a[0] if layout == 'CHW' else a[..., 0]


def same(a, b):
    if a.dtype == np.float32:
        return (a.view(np.uint32) == b.view(np.uint32)).all()
    return (a == b).all()


@pytest.mark.parametrize('name', list(CORPUS))
def test_unchanged_gray_equals_checker_pipeline(name):
    data = CORPUS[name]
    img = coef_image(data)
    luma = gray_luma(img)
    for dtype in SAMPLE:
        want = checker_gray(img, luma, dtype)
        for layout in ('CHW', 'HWC'):
            got = decode_jpeg(data, mode='UNCHANGED', iterations=ITERS, weight=WEIGHT, dtype=dtype, layout=layout,
                              progressive_on_device=True)
            assert got.dtype == dtype and got.device.type == 'cuda'
            assert tuple(got.shape) == ((1, img.height, img.width) if layout == 'CHW' else (img.height, img.width, 1))
            g = plane_of(got, layout)
            assert same(g, want), f'{dtype} {layout}: {int((g != want).sum())} of {g.size} samples differ'
    # mode='GRAY' is the same for a gray file, and separate=True solves it with the first flags
    for kw in (dict(mode='GRAY'), dict(mode='UNCHANGED', separate=True, iterations=(ITERS, 3, 2), weight=(WEIGHT, 0.1, 0.0))):
        kw.setdefault('iterations', ITERS)
        kw.setdefault('weight', WEIGHT)
        got = plane_of(decode_jpeg(data, dtype=torch.float32, **kw), 'CHW')
        assert same(got, checker_gray(img, luma, torch.float32)), kw


def test_rgb_mode_still_refuses_gray_files():
    for name in ('baseline_64x48', 'progressive_97x61'):
        with pytest.raises(ValueError, match='only 3 component jpegs are supported'):
            decode_jpeg(CORPUS[name])
        with pytest.raises(ValueError, match='only 3 component jpegs are supported'):
            decode_jpeg(CORPUS[name], mode='RGB', progressive_on_device=True)


def test_front_ends_agree():
    files = list(CORPUS.values())
    results = []
    for host in (False, True):
        for prog in (False, True):
            old = D._host_front_end
            D._host_front_end = host
            try:
                results.append(decode_jpeg(files, mode='UNCHANGED', iterations=ITERS, dtype=torch.float32,
                                           progressive_on_device=prog))
            finally:
                D._host_front_end = old
    for k, r in enumerate(results[1:], 1):
        for i, (a, b) in enumerate(zip(results[0], r)):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f'front end {k}, file {i}'


@pytest.mark.parametrize('sep', [False, True], ids=['joint', 'separate'])
@pytest.mark.parametrize('name', list(FILES))
def test_gray_mode_on_colour_files_is_the_checker_luma(name, sep):
    data, kw, iters, weights = _case(name, sep)
    img = coef_image(data, 0)
    if sep:
        luma = H.run_compute('oracle', img, [0], weights[0], [PW[0]], iters[0])[0]
    else:
        luma = H.run_compute('oracle', img, [0, 1, 2], weights[0], PW, iters[0])[0]
    for dtype in (torch.uint8, torch.float32):
        want = checker_gray(img, luma, dtype)
        for layout in ('CHW', 'HWC'):
            got = decode_jpeg(data, mode='GRAY', dtype=dtype, layout=layout, progressive_on_device=True, **kw)
            assert tuple(got.shape) == ((1, img.height, img.width) if layout == 'CHW' else (img.height, img.width, 1))
            assert same(plane_of(got, layout), want), f'{dtype} {layout}'
    # UNCHANGED is RGB for a colour file
    assert torch.equal(decode_jpeg(data, mode='UNCHANGED', **kw), decode_jpeg(data, **kw))


def _mixed():
    g = [gray_jpeg(64, 48, seed=s) for s in (1, 2, 3)]
    g2 = [gray_jpeg(97, 61, seed=s, progressive=True) for s in (4, 5)]
    c = [synth_colour(64, 48, '4:2:0'), synth_colour(64, 48, '4:4:4', progressive=True)]
    return [g[0], c[0], g2[0], g[1], c[1], g2[1], g[2]]


@pytest.mark.parametrize('mode', ['UNCHANGED', 'GRAY'])
@pytest.mark.parametrize('sep', [False, True], ids=['joint', 'separate'])
def test_mixed_list_equals_each_file_alone(mode, sep):
    inputs = _mixed()
    kw = dict(iterations=(8, 6, 4), weight=(0.3, 0.1, 0.0), separate=True) if sep else dict(iterations=8)
    got = decode_jpeg(inputs, mode=mode, progressive_on_device=True, **kw)
    for i, (data, t) in enumerate(zip(inputs, got)):
        alone = decode_jpeg(data, mode=mode, **kw)
        assert t.shape == alone.shape and torch.equal(t, alone), f'input {i}'
    assert got[0].shape[0] == 1 and got[1].shape[0] == (1 if mode == 'GRAY' else 3)
    assert got[0].untyped_storage().data_ptr() == got[3].untyped_storage().data_ptr() == got[6].untyped_storage().data_ptr()
    split = decode_jpeg(inputs, mode=mode, max_frames=2, **kw)
    for i, (a, b) in enumerate(zip(got, split)):
        assert torch.equal(a, b), f'input {i} with max_frames=2'
    assert split[0].untyped_storage().data_ptr() == split[3].untyped_storage().data_ptr() != split[6].untyped_storage().data_ptr()


def test_64_file_gray_batch_equals_each_file():
    files = [gray_jpeg(120, 80, quality=40 + s % 50, seed=100 + s) for s in range(64)]
    got = decode_jpeg(files, mode='UNCHANGED', iterations=10, dtype=torch.float32, layout='HWC')
    assert len({t.untyped_storage().data_ptr() for t in got}) == 1
    for i in range(0, 64, 9):
        alone = decode_jpeg(files[i], mode='UNCHANGED', iterations=10, dtype=torch.float32, layout='HWC')
        assert torch.equal(got[i].view(torch.int32), alone.view(torch.int32)), i
    img = coef_image(files[63])
    assert same(got[63].cpu().numpy()[..., 0], checker_gray(img, gray_luma(img, 10), torch.float32))


def _gray_export(lib, s, w, h, dtype, layout, frame0=0, n=1):
    out = torch.empty((n, 1, h, w) if layout == 'CHW' else (n, h, w, 1), dtype=dtype, device='cuda')
    o = abi.ImageOut(w, h, SAMPLE[dtype], abi.LAYOUT_CHW if layout == 'CHW' else abi.LAYOUT_HWC, out[0].numel() * out.element_size())
    rc = lib.j2p_session_export_gray(s, frame0, n, C.byref(o), C.c_void_p(out.data_ptr()), None)
    assert rc == 0, lib.j2p_last_error()
    return out


def test_export_gray_of_a_joint_session_is_the_luma_with_zero_chroma():
    lib = abi.load_product()
    img = synth.synth_coefs(203, 117, 8, '4:2:0', seed=11)
    for pl in img.planes:
        pl.data[:] = np.clip(pl.data.astype(np.int32) * 3, -1000, 1000).astype(np.int16)
    desc = abi.frame_desc(img, [0, 1, 2], 0.3, PW, 6)
    with abi.Session(lib, desc, 2, 0) as s:
        s.upload([img, img], [0, 1, 2])
        s.iterate(0, 6)
        planes = s.download()
        got = {(dt, lay): _gray_export(lib, s.s, 203, 117, dt, lay, 0, 2) for dt in SAMPLE for lay in ('CHW', 'HWC')}
        torch.cuda.synchronize()
    want = checker_gray(img, planes[0][0], torch.float32)
    assert want.min() == 0 and want.max() == 255, 'the case is meant to hit both clamps'
    for (dt, lay), t in got.items():
        assert t.flatten().view(torch.uint8).numel() == 2 * 203 * 117 * SAMPLE[dt] // 8
        for f in range(2):
            a = plane_of(t[f], lay)
            if dt == torch.float32:
                assert same(a, want)
            else:
                assert same(a, checker_gray(img, planes[f][0], dt))
        assert torch.equal(got[dt, 'CHW'].flatten(), got[dt, 'HWC'].flatten()), 'CHW and HWC are the same bytes'


def test_export_gray_refusals():
    lib = abi.load_product()
    img = synth.synth_coefs(64, 64, 30, '4:4:4', seed=3)
    joint = abi.frame_desc(img, [0, 1, 2], 0.3, PW, 2)
    one = abi.frame_desc(img, [0], 0.3, PW, 2)
    two = abi.frame_desc(img, [0, 1], 0.3, PW, 2)
    dst = torch.empty(64 * 64 * 4 * 2, dtype=torch.uint8, device='cuda')
    p = C.c_void_p(dst.data_ptr())

    def out(w=64, h=64, sample=8, layout=abi.LAYOUT_CHW, frame_bytes=None):
        fb = w * h * max(sample // 8, 1) if frame_bytes is None else frame_bytes
        return C.byref(abi.ImageOut(w, h, sample, layout, fb))

    def refused(rc):
        return rc == -1 and len(lib.j2p_last_error()) > 0

    ex = lib.j2p_session_export_gray
    with abi.Session(lib, joint, 1, 0, batch=False) as s, abi.Session(lib, one, 2, 0) as y, \
            abi.Session(lib, two, 1, 0, batch=False) as t:
        s.upload([img], [0, 1, 2])
        y.upload([img, img], [0])
        for x in (s, y):
            x.iterate(0, 2)
        assert ex(s.s, 0, 1, out(), p, None) == 0, lib.j2p_last_error()      # the valid calls
        assert ex(y.s, 0, 2, out(), p, None) == 0, lib.j2p_last_error()
        assert ex(y.s, 1, 1, out(sample=32, layout=abi.LAYOUT_HWC), p, None) == 0, lib.j2p_last_error()
        assert refused(ex(None, 0, 1, out(), p, None))                        # null session
        assert refused(ex(s.s, 0, 1, out(), None, None))                      # null dst
        assert refused(ex(s.s, 0, 1, None, p, None))                          # null description
        assert refused(ex(s.s, 0, 0, out(), p, None))                         # nframes == 0
        assert refused(ex(s.s, 1, 1, out(), p, None))                         # frame out of range
        assert refused(ex(y.s, 1, 2, out(), p, None))
        assert refused(ex(s.s, 0, 1, out(w=0), p, None))
        assert refused(ex(s.s, 0, 1, out(h=0), p, None))
        assert refused(ex(s.s, 0, 1, out(w=65), p, None))                     # larger than the frame
        assert refused(ex(s.s, 0, 1, out(h=65), p, None))
        assert refused(ex(s.s, 0, 1, out(sample=12), p, None))                # unknown sample
        assert refused(ex(s.s, 0, 1, out(layout=2), p, None))                 # unknown layout
        assert refused(ex(s.s, 0, 1, out(frame_bytes=64 * 64 - 1), p, None))  # smaller than one image
        assert refused(ex(y.s, 0, 1, out(sample=16, frame_bytes=64 * 64), p, None))
        assert refused(ex(t.s, 0, 1, out(), p, None))                         # two planes (refused before any read)
        d = C.c_void_p()
        assert lib.j2p_session_create_strip(C.byref(d), 0, C.byref(joint), 0, 32) == 0, lib.j2p_last_error()
        try:
            assert refused(ex(d, 0, 1, out(), p, None))                       # a strip session
        finally:
            lib.j2p_session_destroy(d)
        torch.cuda.synchronize()


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def test_encode_png_gray_equals_host_driver():
    items = list(GRAY_PNG.values())
    want = [E.encode_host([x], lay)[0] for x, lay in items]
    got = encode_png([_cuda(P.hwc(x, lay)) for x, lay in items], layout='HWC')
    assert got == want
    for k, (x, lay) in enumerate(items):
        assert encode_png(_cuda(x), layout=lay) == want[k], k
    # views of device tensors, uint8 and uint16, mixed with RGB images in one call
    big = P._smooth(90, 130, seed=10)
    g = _cuda(big)
    u16 = P._smooth(70, 90, np.uint16, 12)
    gu = _cuda(u16)
    views = [(big[5:80:2, 7:120:3, 1:2], g[5:80:2, 7:120:3, 1:2], 'HWC'),
             (big.transpose(2, 0, 1)[2:3], g.permute(2, 0, 1)[2:3], 'CHW'),
             (u16[::3, ::2, :1], gu[::3, ::2, :1], 'HWC'),
             (u16.transpose(2, 1, 0)[:1, ::2], gu.permute(2, 1, 0)[:1, ::2], 'CHW')]
    for host, dev, lay in views:
        assert encode_png(dev, layout=lay) == E.encode_host([host], lay)[0]
    mixed = [g, g[..., :1], gu, gu[..., 2:3]]
    assert encode_png(mixed, layout='HWC') == E.encode_host([big, big[..., :1], u16, u16[..., 2:3]], 'HWC')


def test_decode_then_encode_png_round_trips_gray_pixels():
    files = [CORPUS['baseline_97x61_q20'], CORPUS['progressive_160x120_q95'], CORPUS['sof_2x2_97x61']]
    for dtype, mode in ((torch.uint8, 'L'), (torch.uint16, None)):
        ts = decode_jpeg(files, mode='UNCHANGED', iterations=ITERS, dtype=dtype)
        pngs = encode_png(ts)
        for t, png in zip(ts, pngs):
            im = Image.open(io.BytesIO(png))
            if mode:
                assert im.mode == mode
            assert (np.asarray(im).astype(np.int64) == t[0].cpu().numpy().astype(np.int64)).all()
    # and a colour file in mode 'GRAY'
    data = synth_colour(96, 64, '4:2:0')
    t = decode_jpeg(data, mode='GRAY', layout='HWC')
    im = Image.open(io.BytesIO(encode_png(t, layout='HWC')))
    assert im.mode == 'L' and (np.asarray(im) == t[..., 0].cpu().numpy()).all()
