"""CPU tests of gray JPEG encoding (encode_jpeg on one-channel tensors) through the three encoders'
serial host drivers: Pillow's 'L' bytes on the gray corpus at every quality, sampling and mode and
with restart intervals, the header of each kind of file, the project's reader and layout passes
on the files, the work-area bound, the refusals, and one library call per kind for a mixed list."""
import ctypes as C

import numpy as np
import pytest
import torch

from jpeg2png_b200 import batch_encode as B
from jpeg2png_b200 import decode as D
from jpeg2png_b200 import jpeg_encode as J
from tests import gray_jpeg_cases as G
from tests import jpegenc_cases as JC

CORPUS = G.corpus()
SMALL = {k: v for k, v in CORPUS.items() if v.shape[0] * v.shape[1] <= JC.SMALL}


def _check(got, want, what):
    if got != want:
        k = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
        pytest.fail(f'{what}: {len(got)} bytes against Pillow\'s {len(want)}, first difference at byte {k} ({JC.turbo_version()})')


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
@pytest.mark.parametrize('mode', list(G.MODES))
def test_host_drivers_equal_pillow_l(mode, subsampling):
    for name, x in CORPUS.items():
        qualities = G.QUALITIES if x.size <= JC.SMALL else [75]
        for q in qualities:
            want = G.pillow_l(x, q, subsampling, **G.MODES[mode])
            _check(J.encode_host([x], q, subsampling, 'HWC', **G.MODES[mode], gray=True)[0], want, f'{name} q{q} {subsampling}')


@pytest.mark.parametrize('mode', list(G.MODES))
def test_host_drivers_equal_pillow_l_with_restarts(mode):
    for name, x in SMALL.items():
        h, w = x.shape[:2]
        for q, s in ((1, '4:2:0'), (90, '4:4:4')):
            for kw in G.restart_settings(h, w):
                want = G.pillow_l(x, q, s, **G.MODES[mode], **kw)
                _check(J.encode_host([x], q, s, 'HWC', **G.MODES[mode], **kw, gray=True)[0], want, f'{name} q{q} {s} {kw}')


def test_one_call_of_mixed_sizes_equals_calls_of_one():
    xs = list(SMALL.values())
    for mode in G.MODES:
        alone = [J.encode_host([x], 75, '4:2:0', **G.MODES[mode], gray=True)[0] for x in xs]
        assert J.encode_host(xs, 75, '4:2:0', **G.MODES[mode], gray=True) == alone
        assert J.encode_host(xs, 75, '4:2:0', **G.MODES[mode], restart_marker_rows=1, gray=True) == \
            [J.encode_host([x], 75, '4:2:0', **G.MODES[mode], restart_marker_rows=1, gray=True)[0] for x in xs]


def test_layouts_and_strided_views_equal_contiguous():
    x = G.gray('cartoon', 61, 97, 5)
    want = J.encode_host([x], 80, gray=True)[0]
    assert J.encode_host([np.ascontiguousarray(x.transpose(2, 0, 1))], 80, layout='CHW', gray=True)[0] == want
    rgb = np.zeros((61, 97, 3), np.uint8)
    rgb[..., 2] = x[..., 0]
    assert J.encode_host([rgb[..., 2:3]], 80, gray=True)[0] == want
    big = np.zeros((130, 200, 1), np.uint8)
    big[3:125:2, 5:199:2] = x
    assert J.encode_host([big[3:125:2, 5:199:2]], 80, gray=True)[0] == want


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
@pytest.mark.parametrize('mode', list(G.MODES))
def test_header_structure(mode, subsampling):
    x = SMALL['97x61_cartoon'] if '97x61_cartoon' in SMALL else next(iter(SMALL.values()))
    h, w = x.shape[:2]
    for kw in ({}, {'restart_marker_rows': 1}):
        f = J.encode_host([x], 75, subsampling, **G.MODES[mode], **kw, gray=True)[0]
        segs = G.segments(f)
        kinds = [m for m, _, _ in segs]
        dqt = [p for m, _, p in segs if m == 0xDB]
        assert len(dqt) == 1 and len(dqt[0]) == 65 and dqt[0][0] == 0, 'one DQT: table 0'
        (sof,) = [(m, p) for m, _, p in segs if m in (0xC0, 0xC2)]
        assert sof[0] == (0xC2 if mode == 'progressive' else 0xC0)
        assert sof[1] == bytes([8, h >> 8, h & 255, w >> 8, w & 255, 1, 1, G.SOF_SAMPLING[subsampling], 0])
        dht = [p[0] for m, _, p in segs if m == 0xC4]
        sos = [p for m, _, p in segs if m == 0xDA]
        if mode == 'progressive':
            assert len(sos) == 6
            assert [(p[3], p[4], p[5] >> 4, p[5] & 15) for p in sos] == G.GRAY_SCRIPT
            assert all(p[:3] == bytes([1, 1, 0]) for p in sos)
            assert dht == [0x00, 0x10, 0x10, 0x10, 0x10], 'five tables, the DC refine has none'
        else:
            assert dht == [0x00, 0x10] and sos == [bytes([1, 1, 0, 0, 63, 0])]
        assert kinds.count(0xDD) == (1 if kw else 0), 'one DRI per file'
        if kw:
            (dri,) = [(i, p) for m, i, p in segs if m == 0xDD]
            assert dri[1] == bytes([0, -(-w // 8)]) and dri[0] < next(i for m, i, _ in segs if m == 0xDA)
        if mode == 'baseline' and not kw:
            assert f[89:91] == b'\xff\xc0'
            first_sos = next(i for m, i, _ in segs if m == 0xDA)
            assert first_sos + 10 == 328, 'the header is 328 bytes before the entropy-coded data'


def test_dri_of_97_wide_rows_1_is_13_once():
    x = G.gray('noise', 40, 97, 9)
    for mode in G.MODES:
        f = J.encode_host([x], 75, **G.MODES[mode], restart_marker_rows=1, gray=True)[0]
        _check(f, G.pillow_l(x, 75, **G.MODES[mode], restart_marker_rows=1), mode)
        assert [p for m, _, p in G.segments(f) if m == 0xDD] == [bytes([0, 13])]


@pytest.mark.parametrize('mode', list(G.MODES))
def test_files_read_back(mode):
    for name, x in SMALL.items():
        for kw in ({}, {'restart_marker_rows': 1}):
            f = J.encode_host([x], 90, **G.MODES[mode], **kw, gray=True)[0]
            p = D.parse_jpeg(f, D.READ_GRAY)
            assert len(p.planes) == 1 and (p.w, p.h) == (x.shape[1], x.shape[0])
            if mode == 'progressive':
                lay = D.ProgFileLayout(f, D.READ_GRAY)
                assert lay.progressive_decodable and lay.lay.ncomp == 1 and lay.lay.nscan == 6
            else:
                lay = D.FileLayout(f, D.READ_GRAY)
                assert lay.device_decodable and lay.lay.ncomp == 1
            assert (lay.planes[0].quant == p.planes[0].quant).all()


def test_same_coefficients_in_every_mode():
    x = G.gray('cartoon', 61, 97, 3)
    planes = [D.parse_jpeg(J.encode_host([x], 85, **kw, gray=True)[0], D.READ_GRAY).planes[0].data for kw in G.MODES.values()]
    assert (planes[0] == planes[1]).all() and (planes[0] == planes[2]).all()


def test_one_block_intervals_of_noise_fit_the_bound():
    """Noise at q100 with restart_marker_blocks = 1: every interval of every scan fits its block's
    bound (7 pad bits included)."""
    from tests.test_jpeg_restart_host import intervals
    x = G.gray('noise', 48, 40, 4)
    bounds = {'baseline': [1658], 'optimize': [1665], 'progressive': [27, 160, 1538, 1101, 1, 1101]}
    for mode, bits in bounds.items():
        f = J.encode_host([x], 100, **G.MODES[mode], restart_marker_blocks=1, gray=True)[0]
        _check(f, G.pillow_l(x, 100, **G.MODES[mode], restart_marker_blocks=1), mode)
        scans = intervals(f)
        assert len(scans) == len(bits)
        for k, segs in enumerate(scans):
            assert len(segs) == 5 * 6
            assert max(segs) <= (bits[k] + 7) // 8, (mode, k)


def test_abi_refuses_other_component_counts():
    libs = [(J.load_jpegenc(), 'jpegenc'), (J.load_jpegopt(), 'jpegopt'), (J.load_jpegprog(), 'jpegprog')]
    x = np.zeros((8, 8, 3), np.uint8)
    for comps, ok in ((0, True), (1, True), (3, True), (2, False), (4, False), (-1, False)):
        d = (J.Image * 1)()
        d[0].data, d[0].width, d[0].height = x.ctypes.data, 8, 8
        d[0].row_stride, d[0].col_stride, d[0].chan_stride = 24, 3, 1
        p = J.Params(75, 2, 0, 0, comps)
        for lib, name in libs:
            n, o = C.c_size_t(), C.c_size_t()
            rc = getattr(lib, f'j2p_{name}_plan')(d, 1, C.byref(p), C.byref(n), C.byref(o))
            assert (rc == 0) == ok, (name, comps)
            if not ok:
                assert b'components' in getattr(lib, f'j2p_{name}_last_error')()


def test_components_zero_is_colour():
    x = JC.content('cartoon', 31, 33, 1)
    want = J.encode_host([x], 75)[0]
    for name, lib in (('jpegenc', J.load_jpegenc()), ('jpegprog', J.load_jpegprog())):
        codec = J.codec(J.Params(75, 2), progressive=name == 'jpegprog')
        got = B.encode_host(codec, [x], 'HWC')[0]
        assert got == (want if name == 'jpegenc' else J.encode_host([x], 75, progressive=True)[0])


def test_python_refusals():
    with pytest.raises(ValueError, match=r"^layout 'HWC' wants shape \(h, w, 1\); got \(8, 8, 3\)$"):
        J.encode_host([np.zeros((8, 8, 3), np.uint8)], gray=True)
    with pytest.raises(ValueError, match=r"^layout 'HWC' wants shape \(h, w, 3\); got \(8, 8, 1\)$"):
        J.encode_host([np.zeros((8, 8, 1), np.uint8)])
    with pytest.raises(ValueError, match='gray must be True or False'):
        J.encode_host([np.zeros((8, 8, 1), np.uint8)], gray=1)
    for bad in (2, 4, 0, True):
        with pytest.raises(ValueError, match='components must be 3 or 1'):
            J.params(75, '4:2:0', components=bad)
    with pytest.raises(ValueError, match=r"^layout 'CHW' wants shape \(3, h, w\) or \(1, h, w\); got \(2, 8, 8\)$"):
        J.encode_jpeg(torch.zeros(2, 8, 8, dtype=torch.uint8))
    with pytest.raises(ValueError, match=r"^layout 'HWC' wants shape \(h, w, 3\) or \(h, w, 1\); got \(8, 8, 4\)$"):
        J.encode_jpeg(torch.zeros(8, 8, 4, dtype=torch.uint8), layout='HWC')
    with pytest.raises(ValueError, match='encodes CUDA tensors'):
        J.encode_jpeg(torch.zeros(1, 8, 8, dtype=torch.uint8))
    assert J.codec(J.params(75, '4:2:0', components=1)).channels == (1,)
    assert J.codec(J.params(75, '4:2:0')).channels == J.CODEC.channels == (3,)


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
    shapes = [(1, 5, 7), (3, 6, 8), (3, 9, 10), (1, 11, 12), (1, 13, 14)]
    ts = [torch.zeros(s, dtype=torch.uint8).as_subclass(_OnCuda) for s in shapes]
    for mode in G.MODES.values():
        calls.clear()
        got = J.encode_jpeg(ts, quality=60, **mode)
        assert got == [f'{c}:{w}x{h}'.encode() for c, h, w in shapes]
        assert calls == [((1,), [(7, 5), (12, 11), (14, 13)]), ((3,), [(8, 6), (10, 9)])], 'in order of first appearance'
        calls.clear()
        assert J.encode_jpeg(ts[0], **mode) == b'1:7x5' and len(calls) == 1
    # encode_png keeps one call for a mixed list
    from jpeg2png_b200 import encode as E
    calls.clear()
    E.encode_png(ts)
    assert [c for c, _ in calls] == [(3, 1)] and len(calls[0][1]) == len(shapes)
