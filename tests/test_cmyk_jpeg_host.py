"""CPU tests of CMYK JPEG encoding (encode_jpeg(..., cmyk=True) on four-channel tensors) through the
three encoders' serial host drivers: Pillow's 'CMYK' bytes on the CMYK corpus at every quality,
sampling and mode, with restart intervals and with given tables; the header of each kind of file;
the one-block interval bounds; the project's reader and layout pass on the files; keep_settings on
CMYK and YCCK files; the refusals; and one library call per kind for a mixed list."""
import ctypes as C
import io

import numpy as np
import pytest
import torch

from jpeg2png_b200 import batch_encode as B
from jpeg2png_b200 import decode as D
from jpeg2png_b200 import jpeg_encode as J
from tests import cmyk_jpeg_cases as K
from tests import cmyk_synth as S
from tests import gray_jpeg_cases as G
from tests import jpegenc_cases as JC
from tests.test_jpeg_restart_host import intervals

CORPUS = K.corpus()
SMALL = {k: v for k, v in CORPUS.items() if v.shape[0] * v.shape[1] <= JC.SMALL}
X = K.cmyk('cartoon', 61, 97, 5)


def _check(got, want, what):
    if got != want:
        k = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
        pytest.fail(f'{what}: {len(got)} bytes against Pillow\'s {len(want)}, first difference at byte {k} ({JC.turbo_version()})')


def host(xs, q=75, s='4:2:0', **kw):
    return J.encode_host(xs, q, s, 'HWC', **kw, cmyk=True)


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
@pytest.mark.parametrize('mode', list(K.MODES))
def test_host_drivers_equal_pillow_cmyk(mode, subsampling):
    for name, x in CORPUS.items():
        for q in (K.QUALITIES if x.size <= 4 * JC.SMALL else [75]):
            _check(host([x], q, subsampling, **K.MODES[mode])[0], K.pillow_cmyk(x, q, subsampling, **K.MODES[mode]), f'{name} q{q} {subsampling}')


@pytest.mark.parametrize('mode', list(K.MODES))
def test_host_drivers_equal_pillow_cmyk_with_restarts(mode):
    for name, x in SMALL.items():
        h, w = x.shape[:2]
        for q, s in ((1, '4:2:0'), (90, '4:4:4'), (75, '4:2:2')):
            for kw in K.restart_settings(h, w, s):
                _check(host([x], q, s, **K.MODES[mode], **kw)[0], K.pillow_cmyk(x, q, s, **K.MODES[mode], **kw), f'{name} q{q} {s} {kw}')


QTABLES = {
    'one': [list(range(1, 65))],
    'two': [list(range(1, 65)), [3] * 64],
    'three': [[2] * 64, list(range(64, 0, -1)), [5] * 64],
    'four': [[2] * 64, [4] * 64, list(range(10, 74)), [17] * 64],
    'four_wide': [[2] * 64, [300] * 64, [4] * 64, [1000 + k for k in range(64)]],
}


@pytest.mark.parametrize('mode', list(K.MODES))
def test_given_tables_equal_pillow(mode):
    for name, qt in QTABLES.items():
        for s in JC.SAMPLINGS:
            for q in (None, 60):
                want = K.pillow_cmyk(X, q, s, qtables=qt, **K.MODES[mode])
                _check(host([X], q, s, qtables=qt, **K.MODES[mode])[0], want, f'{name} {s} q{q}')
    # per image: each its own tables (or the quality tables) and its own subsampling, in one call
    xs = [X, K.cmyk('noise', 17, 13, 2), K.cmyk('cartoon', 31, 33, 3)]
    qts = [QTABLES['four'], None, QTABLES['two']]
    subs = ['4:2:0', '4:4:4', '4:2:2']
    got = J.encode_host(xs, None, subs, 'HWC', qtables=qts, **K.MODES[mode], cmyk=True)
    for g, x, qt, s in zip(got, xs, qts, subs):
        _check(g, K.pillow_cmyk(x, None, s, **({'qtables': qt} if qt else {}), **K.MODES[mode]), f'per image {s}')


def test_one_call_of_mixed_sizes_equals_calls_of_one():
    xs = list(SMALL.values())
    for mode in K.MODES.values():
        for kw in ({}, {'restart_marker_rows': 1}):
            assert host(xs, **mode, **kw) == [host([x], **mode, **kw)[0] for x in xs]


def test_layouts_and_strided_views_equal_contiguous():
    want = host([X], 80)[0]
    assert J.encode_host([np.ascontiguousarray(X.transpose(2, 0, 1))], 80, layout='CHW', cmyk=True)[0] == want
    big = np.zeros((130, 200, 6), np.uint8)
    big[3:125:2, 5:199:2, 1:5] = X
    assert J.encode_host([big[3:125:2, 5:199:2, 1:5]], 80, cmyk=True)[0] == want
    rev = np.ascontiguousarray(X[..., ::-1])
    assert J.encode_host([rev[..., ::-1]], 80, cmyk=True)[0] == want


def _sof(segs):
    (sof,) = [(m, p) for m, _, p in segs if m in (0xC0, 0xC1, 0xC2)]
    return sof


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
@pytest.mark.parametrize('mode', list(K.MODES))
def test_header_structure(mode, subsampling):
    h, w = X.shape[:2]
    hs, vs = K.FACTORS[subsampling]
    for kw in ({}, {'restart_marker_rows': 1}):
        f = host([X], 75, subsampling, **K.MODES[mode], **kw)[0]
        segs = G.segments(f)
        kinds = [m for m, _, _ in segs]
        assert f[2:18] == K.APP14 and 0xE0 not in kinds, 'APP14 Adobe, transform 0, and no JFIF APP0'
        dqt = [p for m, _, p in segs if m == 0xDB]
        assert len(dqt) == 1 and len(dqt[0]) == 65 and dqt[0][0] == 0, 'one DQT: table 0'
        sof = _sof(segs)
        assert sof[0] == (0xC2 if mode == 'progressive' else 0xC0)
        assert sof[1] == bytes([8, h >> 8, h & 255, w >> 8, w & 255, 4, 67, hs << 4 | vs, 0, 77, 0x11, 0, 89, 0x11, 0, 75, 0x11, 0])
        dht = [p[0] for m, _, p in segs if m == 0xC4]
        sos = [p for m, _, p in segs if m == 0xDA]
        if mode == 'progressive':
            assert len(sos) == 18 and len(K.SCRIPT) == 18
            assert [(p[-3], p[-2], p[-1] >> 4, p[-1] & 15) for p in sos] == K.SCRIPT
            assert [bytes(p[1:1 + 2 * p[0]:2]) for p in sos] == K.SCRIPT_COMPS
            assert all(set(p[2:1 + 2 * p[0]:2]) == {0} for p in sos), 'every component codes with table 0'
            assert dht == [0x00] + [0x10] * 16, 'seventeen tables, the DC refine has none'
        else:
            assert dht == [0x00, 0x10]
            assert sos == [bytes([4, 67, 0, 77, 0, 89, 0, 75, 0, 0, 63, 0])]
        if mode != 'progressive' and kw:
            (dri,) = [p for m, _, p in segs if m == 0xDD]
            assert dri == bytes([0, -(-w // (8 * hs))])
        if mode == 'baseline' and not kw and subsampling == '4:4:4':
            first_sos = next(i for m, i, _ in segs if m == 0xDA)
            assert first_sos + 2 + 14 == K.HEADER, 'the header is 341 bytes before the entropy-coded data'


def test_table_numbers_of_given_tables():
    """n given tables: component c uses min(c, n - 1), one DQT per table, the fourth written and
    used by K; a 16-bit table makes SOF1."""
    for n, want in ((1, [0, 0, 0, 0]), (2, [0, 1, 1, 1]), (3, [0, 1, 2, 2]), (4, [0, 1, 2, 3])):
        qt = [[k + 2] * 64 for k in range(n)]
        segs = G.segments(host([X], None, '4:4:4', qtables=qt)[0])
        assert [p[0] for m, _, p in segs if m == 0xDB] == list(range(n))
        assert list(_sof(segs)[1][8::3]) == want
    segs = G.segments(host([X], None, '4:4:4', qtables=QTABLES['four_wide'])[0])
    assert [p[0] for m, _, p in segs if m == 0xDB] == [0x00, 0x11, 0x02, 0x13] and _sof(segs)[0] == 0xC1


def test_dri_count_of_progressive_53x37_420():
    """A progressive AC scan counts its own component's blocks per row: C 7, M Y K 4, the DC scans
    4 MCUs, so the 18 scans of a 53 x 37 '4:2:0' file with restart_marker_rows=1 carry 9 DRIs."""
    x = K.cmyk('noise', 37, 53, 8)
    f = host([x], 75, '4:2:0', progressive=True, restart_marker_rows=1)[0]
    _check(f, K.pillow_cmyk(x, 75, '4:2:0', progressive=True, restart_marker_rows=1), '53x37')
    dri = [p for m, _, p in G.segments(f) if m == 0xDD]
    assert len(dri) == 9 and [p[1] for p in dri] == [4, 7, 4, 7, 4, 7, 4, 7, 4]


def test_samples_are_inverted():
    """The file codes 255 - t: at q100 (every table entry 1) a flat plane's DC is 8 (255 - t - 128), in
    the full-resolution C and the half-resolution M, Y and K alike, and every AC is 0.  (That the
    half-resolution planes average the inverted samples, with libjpeg's bias, is pinned by the
    corpus's byte equality with Pillow.)"""
    x = np.empty((24, 40, 4), np.uint8)
    x[:] = [0, 255, 100, 37]
    p = D.parse_jpeg4(host([x], 100, '4:2:0')[0])
    assert p.colour == D.CMYK
    for c, t in enumerate((0, 255, 100, 37)):
        b = p.planes[c].data.reshape(-1, 64)
        assert (b[:, 0] == 8 * (255 - t - 128)).all() and (b[:, 1:] == 0).all(), c


def test_one_block_intervals_of_noise_fit_the_bound():
    """Noise at q100 with restart_marker_blocks = 1: every interval of every scan fits its block's
    bound (7 pad bits included): baseline 1658 and optimize 1665 bits per block of the MCU, the
    progressive scans the gray script's per-scan bounds."""
    x = K.cmyk('noise', 48, 40, 4)
    bounds = {'baseline': [1658], 'optimize': [1665], 'progressive': K.PROG_BITS}
    for mode, bits in bounds.items():
        f = host([x], 100, '4:4:4', **K.MODES[mode], restart_marker_blocks=1)[0]
        _check(f, K.pillow_cmyk(x, 100, '4:4:4', **K.MODES[mode], restart_marker_blocks=1), mode)
        scans = intervals(f)
        assert len(scans) == len(bits)
        for k, segs in enumerate(scans):
            assert len(segs) == 5 * 6
            per = 4 if len(bits) == 1 or k in (0, 13) else 1      # blocks per MCU of the scan
            assert max(segs) <= (per * bits[k] + 7) // 8, (mode, k)


@pytest.mark.parametrize('mode', list(K.MODES))
def test_files_read_back(mode):
    """Every file at '4:4:4', and the subsampled ones of even sizes: the reader checks a plane's
    block grid against ceil(floor(W / 2) / 8), as the program it follows does, and so refuses an odd
    side's half-resolution planes, in colour files too."""
    for name, x in SMALL.items():
        even = x.shape[0] % 2 == 0 and x.shape[1] % 2 == 0
        for s in (JC.SAMPLINGS if even else ['4:4:4']):
            for kw in ({}, {'restart_marker_rows': 1}):
                f = host([x], 90, s, **K.MODES[mode], **kw)[0]
                p = D.parse_jpeg4(f)
                assert p.colour == D.CMYK and len(p.planes) == 4 and (p.w, p.h) == (x.shape[1], x.shape[0])
                if mode != 'progressive':
                    lay = D.FileLayout4(f)
                    assert lay.device_decodable and lay.colour == D.CMYK and lay.lay.ncomp == 4
                    assert all((a.quant == b.quant).all() for a, b in zip(lay.planes, p.planes))


def test_same_coefficients_in_every_mode():
    x = K.cmyk('cartoon', 62, 96, 3)
    planes = [D.parse_jpeg4(host([x], 85, '4:2:0', **kw)[0]).planes for kw in K.MODES.values()]
    for c in range(4):
        assert (planes[0][c].data == planes[1][c].data).all() and (planes[0][c].data == planes[2][c].data).all()


def _pillow_keep(data):
    from PIL import Image
    im = Image.open(io.BytesIO(data))
    buf = io.BytesIO()
    im.save(buf, 'JPEG', quality='keep')
    return np.asarray(im), buf.getvalue()


def test_keep_settings_of_cmyk_files_is_pillows_keep():
    files = [S.pillow_cmyk(97, 61, 75, 1), S.pillow_cmyk(40, 32, 20, 2, subsampling='4:2:0'),
             K.pillow_cmyk(K.cmyk('cartoon', 32, 34, 1), None, '4:2:2', qtables=QTABLES['four'])]
    for data in files:
        ks = J.keep_settings(data)
        assert ks['subsampling'] == '4:4:4'
        pixels, want = _pillow_keep(data)
        from PIL import Image
        assert ks['qtables'] == {k: list(v) for k, v in Image.open(io.BytesIO(data)).quantization.items()}
        for mode in K.MODES.values():
            from PIL import Image
            im = Image.open(io.BytesIO(data))
            buf = io.BytesIO()
            im.save(buf, 'JPEG', quality='keep', **mode)
            _check(J.encode_host([pixels], cmyk=True, **mode, **ks)[0], buf.getvalue(), f'keep {mode}')
        _check(J.encode_host([pixels], cmyk=True, **ks)[0], want, 'keep')
    lists = J.keep_settings(files)
    assert lists['subsampling'] == ['4:4:4'] * 3 and len(lists['qtables']) == 3


def test_keep_settings_of_ycck_files():
    """Four-component files of any sampling are '4:4:4', with their own tables."""
    for s in ([(1, 1)] * 4, [(2, 2), (1, 1), (1, 1), (2, 2)], [(2, 1), (1, 1), (1, 1), (1, 1)]):
        data, _ = S.ycck_file(48, 32, s, 3)
        ks = J.keep_settings(data)
        assert ks['subsampling'] == '4:4:4'
        assert ks['qtables'] and all(len(t) == 64 for t in ks['qtables'].values())
        lib = D.load_codecs()
        k = D.Keep()
        err = C.create_string_buffer(256)
        assert lib.j2p_jpeg_keep_settings(data, len(data), C.byref(k), err, 256) == 0, err.value
        assert k.ncomp == 4


def _abi_plan(lib, name, comps, cmyk):
    x = np.zeros((8, 8, 4), np.uint8)
    d = (J.Image * 1)()
    d[0].data, d[0].width, d[0].height = x.ctypes.data, 8, 8
    d[0].row_stride, d[0].col_stride, d[0].chan_stride = 32, 4, 1
    p = J.Params(75, 2, 0, 0, comps)
    p.cmyk = cmyk
    n, o = C.c_size_t(), C.c_size_t()
    return getattr(lib, f'j2p_{name}_plan')(d, 1, C.byref(p), C.byref(n), C.byref(o)), getattr(lib, f'j2p_{name}_last_error')()


def test_abi_refusals():
    for lib, name in ((J.load_jpegenc(), 'jpegenc'), (J.load_jpegopt(), 'jpegopt'), (J.load_jpegprog(), 'jpegprog')):
        assert _abi_plan(lib, name, 0, 1)[0] == 0
        for comps, cmyk in ((0, 2), (0, -1), (0, 4)):
            rc, err = _abi_plan(lib, name, comps, cmyk)
            assert rc == -1 and b'cmyk' in err, (name, cmyk)
        for comps in (1, 3):
            rc, err = _abi_plan(lib, name, comps, 1)
            assert rc == -1 and b'cmyk' in err, (name, comps)
        rc, err = _abi_plan(lib, name, 4, 0)
        assert rc == -1 and b'components' in err


def test_python_refusals():
    for bad in (1, 0, None, 'yes'):
        with pytest.raises(ValueError, match='cmyk must be True or False'):
            J.encode_host([X], cmyk=bad)
        with pytest.raises(ValueError, match='cmyk must be True or False'):
            J.encode_jpeg(torch.zeros(4, 8, 8, dtype=torch.uint8), cmyk=bad)
    with pytest.raises(ValueError, match='gray=True and cmyk=True'):
        J.encode_host([X], gray=True, cmyk=True)
    with pytest.raises(ValueError, match='does not combine with gray'):
        J.params(75, '4:2:0', components=1, cmyk=True)
    for bad in (2, 4, 0, True):
        with pytest.raises(ValueError, match='components must be 3 or 1'):
            J.params(75, '4:2:0', components=bad, cmyk=True)
    with pytest.raises(ValueError, match=r"^layout 'HWC' wants shape \(h, w, 4\); got \(8, 8, 3\)$"):
        J.encode_host([np.zeros((8, 8, 3), np.uint8)], cmyk=True)
    with pytest.raises(ValueError, match=r"^layout 'HWC' wants shape \(h, w, 3\) or \(h, w, 1\) or \(h, w, 4\); got \(8, 8, 2\)$"):
        J.encode_jpeg(torch.zeros(8, 8, 2, dtype=torch.uint8), layout='HWC', cmyk=True)
    with pytest.raises(ValueError, match=r"^layout 'CHW' wants shape \(3, h, w\) or \(1, h, w\) or \(4, h, w\); got \(5, 8, 8\)$"):
        J.encode_jpeg(torch.zeros(5, 8, 8, dtype=torch.uint8), cmyk=True)
    with pytest.raises(ValueError, match=r"^layout 'HWC' wants shape \(h, w, 3\) or \(h, w, 1\); got \(8, 8, 4\)$"):
        J.encode_jpeg(torch.zeros(8, 8, 4, dtype=torch.uint8), layout='HWC')
    with pytest.raises(ValueError, match='encodes CUDA tensors'):
        J.encode_jpeg(torch.zeros(4, 8, 8, dtype=torch.uint8), cmyk=True)
    p = J.params(75, '4:2:0', cmyk=True)
    assert (p.components, p.cmyk) == (0, 1)
    assert J.codec(p).channels == (4,)
    assert J.codec(J.params(75, '4:2:0')).channels == (3,) and J.params(75, '4:2:0').cmyk == 0


class _OnCuda(torch.Tensor):
    """A host tensor that says it is on a CUDA device, so that the driver's routing runs without one."""

    @property
    def device(self):
        return torch.device('cuda', 0)


def test_mixed_list_makes_one_call_per_kind(monkeypatch):
    calls = []

    def fake(codec, descs, device):
        calls.append((codec.channels, [(d.width, d.height) for d in descs]))
        return [f'{codec.channels[0]}:{d.width}x{d.height}'.encode() for d in descs]
    monkeypatch.setattr(B, 'encode_device', fake)
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: True)
    monkeypatch.setattr(torch.cuda, 'device_count', lambda: 1)
    shapes = [(4, 5, 7), (1, 6, 8), (3, 9, 10), (4, 11, 12), (1, 13, 14), (3, 15, 16)]
    ts = [torch.zeros(s, dtype=torch.uint8).as_subclass(_OnCuda) for s in shapes]
    for mode in K.MODES.values():
        calls.clear()
        got = J.encode_jpeg(ts, quality=60, **mode, cmyk=True)
        assert got == [f'{c}:{w}x{h}'.encode() for c, h, w in shapes]
        assert calls == [((4,), [(7, 5), (12, 11)]), ((1,), [(8, 6), (14, 13)]), ((3,), [(10, 9), (16, 15)])], 'in order of first appearance'
        calls.clear()
        assert J.encode_jpeg(ts[0], **mode, cmyk=True) == b'4:7x5' and len(calls) == 1
