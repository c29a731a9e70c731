"""CPU tests of one-component (grayscale) JPEGs and gray PNGs: the reader with J2P_READ_GRAY against
both layout passes and each entropy library's serial host driver, Pillow's own decode of the same
files, the refusals with and without the flag, decode_jpeg's mode argument and its batching of gray
keys, and gray files from the PNG encoder's host driver reopened in Pillow."""
import ctypes as C
import io
import zlib

import numpy as np
import pytest
from PIL import Image

from jpeg2png_b200 import decode as D
from jpeg2png_b200 import encode as E
from jpeg2png_b200 import pngcheck, synth
from tests import helpers as H
from tests import png_cases as P

GRAY = D.READ_GRAY


def gray_jpeg(w, h, quality=75, seed=1, **kw):
    """A Pillow 'L' JPEG of the synthetic cartoon's luma."""
    rgb = synth.cartoon_image(w, h, seed).astype(np.uint8)
    buf = io.BytesIO()
    Image.fromarray(rgb, 'RGB').convert('L').save(buf, 'JPEG', quality=quality, **kw)
    return buf.getvalue()


def with_sof_sampling(data, hv):
    """data with its one component's sampling byte in the SOF set to hv (0x22: 2x2)."""
    b = bytearray(data)
    i = 2
    while True:
        assert b[i] == 0xFF
        m, n = b[i + 1], int.from_bytes(b[i + 2:i + 4], 'big')
        if m in (0xC0, 0xC1, 0xC2):
            assert b[i + 9] == 1, 'not a one-component file'
            b[i + 11] = hv
            return bytes(b)
        i += 2 + n


def corpus():
    files = {
        'baseline_64x48': gray_jpeg(64, 48),
        'baseline_97x61_q20': gray_jpeg(97, 61, 20, seed=2),
        'baseline_1x1': gray_jpeg(1, 1, seed=3),
        'optimize_97x61': gray_jpeg(97, 61, 90, seed=4, optimize=True),
        'progressive_97x61': gray_jpeg(97, 61, 50, seed=5, progressive=True),
        'progressive_1x1': gray_jpeg(1, 1, seed=6, progressive=True),
        'progressive_160x120_q95': gray_jpeg(160, 120, 95, seed=7, progressive=True),
        'restart_rows1_97x61': gray_jpeg(97, 61, 75, seed=8, restart_marker_rows=1),
        'restart_rows1_progressive': gray_jpeg(80, 40, 75, seed=9, progressive=True, restart_marker_rows=1),
    }
    files['sof_2x2_97x61'] = with_sof_sampling(gray_jpeg(97, 61, seed=10), 0x22)
    files['sof_2x2_progressive'] = with_sof_sampling(gray_jpeg(97, 61, seed=11, progressive=True), 0x22)
    return files


CORPUS = corpus()


def host_planes(kind, layouts, subseq_bits=1024):
    """Decode layouts (all gray or all colour, any mix) with a host driver: per file, one int16
    array per plane.  Three out pointers per file, 0 for the planes a gray file does not have."""
    arrs, outs = [], []
    for lay in layouts:
        planes = [np.full(p.w * p.h, 0x5a5a, np.int16) for p in lay.planes]
        arrs.append(planes)
        outs += [a.ctypes.data for a in planes] + [0] * (3 - len(planes))
    make, lib, stats, name = ((D.entropy_plan, D.load_entropy(), D.EntropyStats(), 'entropy') if kind == 'seq' else
                              (D.progressive_plan, D.load_progressive(), D.ProgressiveStats(), 'progressive'))
    plan, addr, _, work_bytes = make(layouts, outs, subseq_bits)     # plan owns the buffer at addr
    work = np.zeros(work_bytes + 16, np.uint8)
    status = np.zeros(len(layouts), np.uint32)
    rc = getattr(lib, f'j2p_{name}_decode_host')(addr, (work.ctypes.data + 15) & ~15, status.ctypes.data, C.byref(stats))
    assert rc == 0, getattr(lib, f'j2p_{name}_last_error')()
    assert (status == 0).all()
    del plan
    return arrs


@pytest.mark.parametrize('name', list(CORPUS))
def test_reader_layout_and_host_drivers_agree(name):
    data = CORPUS[name]
    p = D.parse_jpeg(data, GRAY)
    assert len(p.planes) == 1
    pl = p.planes[0]
    assert (pl.w_samp, pl.h_samp) == (1, 1)
    assert (pl.w, pl.h) == (-(-p.w // 8) * 8, -(-p.h // 8) * 8)
    progressive = 'progressive' in name
    lay = D.FileLayout(data, GRAY)
    assert lay.device_decodable == (not progressive)
    if progressive:
        lay = D.ProgFileLayout(data, GRAY)
        assert lay.progressive_decodable
        assert lay.lay.ncomp == 1 and lay.lay.nscan == 6, 'libjpeg progression for one component'
    else:
        assert lay.lay.ncomp == 1 and lay.lay.nscan == 1 and lay.lay.scan[0].ncomp == 1
    assert (lay.w, lay.h) == (p.w, p.h)
    assert len(lay.planes) == 1
    assert (lay.planes[0].w, lay.planes[0].h, lay.planes[0].w_samp, lay.planes[0].h_samp) == (pl.w, pl.h, 1, 1)
    assert (lay.planes[0].quant == pl.quant).all()
    for bits in (32, 1024):
        got = host_planes('prog' if progressive else 'seq', [lay], bits)
        assert (got[0][0] == pl.data).all()


def test_sof_sampling_does_not_change_coefficients():
    for prog in (False, True):
        data = gray_jpeg(97, 61, seed=12, progressive=prog)
        a = D.parse_jpeg(data, GRAY)
        b = D.parse_jpeg(with_sof_sampling(data, 0x22), GRAY)
        assert (a.w, a.h) == (b.w, b.h)
        assert (a.planes[0].data == b.planes[0].data).all()


def test_host_drivers_take_gray_and_colour_files_in_one_call():
    seq = [CORPUS['baseline_64x48'], CORPUS['restart_rows1_97x61'], CORPUS['sof_2x2_97x61']]
    colour = [synth_colour(64, 48, '4:2:0'), synth_colour(40, 24, '4:4:4')]
    files = [seq[0], colour[0], seq[1], colour[1], seq[2]]
    lays = [D.FileLayout(d, GRAY) for d in files]
    got = host_planes('seq', lays)
    for d, planes in zip(files, got):
        want = D.parse_jpeg(d, GRAY).planes
        assert len(planes) == len(want)
        for a, b in zip(planes, want):
            assert (a == b.data).all()
    prog = [CORPUS['progressive_97x61'], synth_colour(64, 48, '4:2:0', progressive=True), CORPUS['progressive_1x1']]
    lays = [D.ProgFileLayout(d, GRAY) for d in prog]
    for d, planes in zip(prog, host_planes('prog', lays)):
        for a, b in zip(planes, D.parse_jpeg(d, GRAY).planes):
            assert (a == b.data).all()


def synth_colour(w, h, ss, progressive=False):
    rgb = synth.cartoon_image(w, h, 3).astype(np.uint8)
    buf = io.BytesIO()
    Image.fromarray(rgb, 'RGB').save(buf, 'JPEG', quality=60, subsampling=ss, progressive=progressive)
    return buf.getvalue()


@pytest.mark.parametrize('name', list(CORPUS))
def test_conventional_decode_within_one_of_pillow(name):
    data = CORPUS[name]
    p = D.parse_jpeg(data, GRAY)
    img = synth.CoefImage(width=p.w, height=p.h, planes=[synth.Plane(w=x.w, h=x.h, w_samp=x.w_samp, h_samp=x.h_samp,
                                                                     data=x.data, quant=x.quant) for x in p.planes])
    ours = H.decode_planes(img, [0])[0][:p.h, :p.w]
    im = Image.open(io.BytesIO(data))
    assert im.mode == 'L'
    theirs = np.asarray(im).astype(np.float64)
    assert np.abs(np.clip(np.rint(ours + 128.0), 0, 255) - theirs).max() <= 1.0


def test_refusals_with_and_without_the_flag():
    gray = CORPUS['baseline_64x48']
    for fn in (D.parse_jpeg, D.FileLayout):
        with pytest.raises(ValueError, match='^only 3 component jpegs are supported$'):
            fn(gray)
    with pytest.raises(ValueError, match='^only 3 component jpegs are supported$'):
        D.parse_jpeg(CORPUS['progressive_97x61'])
    with pytest.raises(ValueError, match='^only 3 component jpegs are supported$'):
        D.ProgFileLayout(CORPUS['progressive_97x61'])
    buf = io.BytesIO()
    Image.fromarray(np.arange(16 * 8 * 4, dtype=np.uint8).reshape(16, 8, 4), 'CMYK').save(buf, 'JPEG')
    cmyk = buf.getvalue()
    for fn in (D.parse_jpeg, D.FileLayout):
        with pytest.raises(ValueError, match='^only 3 component jpegs are supported$'):
            fn(cmyk)
        with pytest.raises(ValueError, match='^only 1 and 3 component jpegs are supported$'):
            fn(cmyk, GRAY)
    # a colour file reads the same with the flag
    colour = synth_colour(64, 48, '4:2:0')
    a, b = D.parse_jpeg(colour), D.parse_jpeg(colour, GRAY)
    assert len(b.planes) == 3 and all((x.data == y.data).all() for x, y in zip(a.planes, b.planes))


def test_decode_jpeg_mode_validation():
    data = CORPUS['baseline_64x48']
    for bad in ('rgb', 'L', 'gray', None, 3):
        with pytest.raises(ValueError, match="mode must be 'RGB', 'UNCHANGED' or 'GRAY'"):
            D.decode_jpeg(data, mode=bad)


def test_footprint_counts_planes_solved_and_channels_written():
    gray = D.parse_jpeg(gray_jpeg(96, 64, seed=4), GRAY).key()
    colour = D.parse_jpeg(synth_colour(96, 64, '4:2:0'), GRAY).key()
    assert len(gray[2]) == 1 and len(colour[2]) == 3
    w, h = 96, 64
    for sep in (False, True):
        for sb in (1, 2, 4):
            one = D.frame_footprint(gray, sep, sb, 'UNCHANGED')
            assert one == D.frame_footprint(gray, not sep, sb, 'GRAY'), 'a gray file is solved alike in both modes'
            assert D.frame_footprint(colour, True, sb, 'RGB') - D.frame_footprint(colour, True, sb, 'GRAY') > \
                D.frame_footprint(colour, False, sb, 'RGB') - D.frame_footprint(colour, False, sb, 'GRAY')
            assert D.frame_footprint(colour, sep, sb, 'RGB') - D.frame_footprint(colour, sep, sb, 'GRAY') >= 2 * w * h * sb
    # the luma session alone: the gray file's plane is the colour file's luma (same geometry)
    assert gray[2][0] == colour[2][0]
    assert D.frame_footprint(gray, True, 1, 'UNCHANGED') == D.frame_footprint(colour, True, 1, 'GRAY')
    assert D.frame_footprint(colour, True, 1, 'UNCHANGED') == D.frame_footprint(colour, True, 1)
    assert D.solved_planes(gray, False, 'UNCHANGED') == (1, 1)
    assert D.solved_planes(colour, False, 'GRAY') == (3, 1)
    assert D.solved_planes(colour, True, 'GRAY') == (1, 1)
    assert D.solved_planes(colour, True, 'UNCHANGED') == (3, 3)


def test_gray_and_colour_keys_group_apart():
    g1, g2 = D.parse_jpeg(gray_jpeg(64, 48, seed=1), GRAY), D.parse_jpeg(gray_jpeg(64, 48, seed=2), GRAY)
    c1, c2 = D.parse_jpeg(synth_colour(64, 48, '4:4:4'), GRAY), D.parse_jpeg(synth_colour(64, 48, '4:4:4'), GRAY)
    keys = [g1.key(), c1.key(), g2.key(), c2.key(), g1.key()]
    assert keys[0] == keys[2] != keys[1] == keys[3]
    assert D.plan(keys, lambda k: 2) == [(keys[0], [0, 2]), (keys[0], [4]), (keys[1], [1, 3])]


def _gray_cases():
    big = P._smooth(90, 130, seed=10)[..., :1]
    return {
        '1x1': (P._noise(1, 1)[..., :1], 'HWC'),
        'smooth_hwc': (np.ascontiguousarray(P._smooth(60, 70, seed=2)[..., 1:2]), 'HWC'),
        'noise_u16': (np.ascontiguousarray(P._noise(40, 90, np.uint16, 5)[..., :1]), 'HWC'),
        'chw_u16': (np.ascontiguousarray(P._smooth(33, 45, np.uint16, 9)[..., :1].transpose(2, 0, 1)), 'CHW'),
        'strided_hwc': (big[5:80:2, 7:120:3], 'HWC'),
        'channel_of_rgb_chw': (P._smooth(50, 61, seed=3).transpose(2, 0, 1)[2:3], 'CHW'),
        'three_pieces_plus_1': (np.ascontiguousarray(P._smooth(1, 196609)[..., :1]), 'HWC'),
        'constant_big': (np.full((400, 700, 1), 200, np.uint8), 'HWC'),
    }


GRAY_PNG = _gray_cases()


@pytest.mark.parametrize('name', list(GRAY_PNG))
def test_gray_png_host_driver(name):
    x, layout = GRAY_PNG[name]
    png = E.encode_host([x], layout)[0]
    a = P.hwc(x, layout)
    h, w, _ = a.shape
    sb = a.itemsize
    ch = P.chunks(png)
    assert [t for t, _ in ch] == [b'IHDR', b'IDAT', b'IEND']
    assert ch[0][1] == int.to_bytes(w, 4, 'big') + int.to_bytes(h, 4, 'big') + bytes([8 * sb, 0, 0, 0, 0])
    stream = zlib.decompress(ch[1][1])
    assert stream == pngcheck.filter_rows(pngcheck.scanlines(a), sb)[1]
    assert pngcheck.holds_pixels(png, a)
    if a.size <= 30000:
        assert (P.unfilter(stream, h, w * sb, sb) == pngcheck.scanlines(a)).all()
    im = Image.open(io.BytesIO(png))
    if sb == 1:
        assert im.mode == 'L'
    else:
        assert im.mode in ('I;16', 'I;16B', 'I')
    assert (np.asarray(im).astype(np.int64) == a[..., 0].astype(np.int64)).all()


def test_gray_and_rgb_mix_in_one_call():
    xs = [GRAY_PNG['smooth_hwc'], P.cases()['chw'], GRAY_PNG['chw_u16'], P.cases()['noise_u16'], GRAY_PNG['1x1']]
    alone = [E.encode_host([x], lay)[0] for x, lay in xs]
    assert E.encode_host([P.hwc(x, lay) for x, lay in xs], 'HWC') == alone
    assert [P.chunks(p)[0][1][9] for p in alone] == [0, 2, 0, 2, 0]


def test_holds_pixels_default_bpp_is_unchanged():
    x = P._smooth(20, 30, seed=1)
    png = E.encode_host([x], 'HWC')[0]
    assert pngcheck.holds_pixels(png, x) and pngcheck.holds_pixels(png, x, 3)
    assert not pngcheck.holds_pixels(png, x, 1)


def test_channel_counts_each_encoder_accepts():
    from jpeg2png_b200 import batch_encode as B
    from jpeg2png_b200 import jpeg_encode as J
    assert E.CODEC.channels == (3, 1)
    assert J.CODEC.channels == J.CODEC_OPT.channels == J.CODEC_PROG.channels == (3,)
    g = np.zeros((8, 8, 1), np.uint8)
    with pytest.raises(ValueError, match=r"^layout 'HWC' wants shape \(h, w, 3\); got \(8, 8, 1\)$"):
        J.encode_host([g], layout='HWC')
    with pytest.raises(ValueError, match=r"^layout 'CHW' wants shape \(3, h, w\) or \(1, h, w\); got \(2, 8, 8\)$"):
        E.encode_host([np.zeros((2, 8, 8), np.uint8)], 'CHW')
    assert B.axes((1, 5, 7), 'CHW', (3, 1)) == (5, 7, 1, 2, 0)


def test_png_abi_refuses_other_channel_counts():
    lib = E.load_png()
    for ch, ok in ((0, True), (1, True), (3, True), (2, False), (4, False)):
        d = (E.Image * 1)()
        d[0].data, d[0].width, d[0].height, d[0].sample_bytes = 1 << 20, 4, 4, 1
        d[0].row_stride, d[0].col_stride, d[0].chan_stride, d[0].channels = 12, 3, 1, ch
        n, o = C.c_size_t(), C.c_size_t()
        rc = lib.j2p_png_plan(d, 1, C.byref(n), C.byref(o))
        assert (rc == 0) == ok, ch
        if not ok:
            assert b'channels' in lib.j2p_png_last_error()
