"""CPU tests of restart markers in the three JPEG encoders (encode_jpeg(..., restart_marker_blocks=,
restart_marker_rows=)) through their serial host drivers: Pillow's bytes on the corpus for every
interval rule, the named cases (a luma AC grid wider than the MCU grid, the 65535-MCU cap, a DRI
that changes between progressive scans), the defaults, the refusals, the project's reader and
layout passes on the files, and the work-area bound of one-MCU intervals."""
import ctypes as C
import io

import numpy as np
import pytest

from jpeg2png_b200 import decode as D
from jpeg2png_b200 import jpeg_encode as J
from tests import entropy_cases as EC
from tests import jpegenc_cases as JC

MODES = {'baseline': {}, 'optimize': {'optimize': True}, 'progressive': {'progressive': True}}
QUALITIES = [1, 50, 90, 100]
SIZES = [(h, w) for h, w in JC.SIZES]
KINDS = ['cartoon', 'noise', 'flat128']
FACTORS = {'4:4:4': (1, 1), '4:2:2': (2, 1), '4:2:0': (2, 2)}


def pillow(x, q, s, **kw):
    """Pillow's file for the (h, w, 3) uint8 pixels with the save options kw.  Its output buffer
    must hold the whole file when the Huffman tables are optimized; its size changes no byte."""
    from PIL import Image, ImageFile
    old = ImageFile.MAXBLOCK
    ImageFile.MAXBLOCK = max(old, 4 * x.shape[0] * x.shape[1] * 3 + 65536)
    try:
        buf = io.BytesIO()
        Image.fromarray(np.ascontiguousarray(x), 'RGB').save(buf, 'JPEG', quality=q, subsampling=s, **kw)
        return buf.getvalue()
    finally:
        ImageFile.MAXBLOCK = old


def mcu_grid(h, w, s):
    hs, vs = FACTORS[s]
    return -(-w // (8 * hs)), -(-h // (8 * vs))


def settings(h, w, s):
    """The restart keywords of the corpus for an image: blocks around the MCU count, rows around the
    MCU rows, and both."""
    mx, my = mcu_grid(h, w, s)
    m = mx * my
    out = [dict(restart_marker_blocks=b) for b in sorted({1, 2, 3, 7, m - 1, m, m + 1, 65535}) if b > 0]
    out += [dict(restart_marker_rows=r) for r in sorted({1, 2, 5, my, my + 1})]
    out.append(dict(restart_marker_blocks=3, restart_marker_rows=2))
    return out


def corpus():
    """name -> (h, w, 3) pixels: every corpus size in cartoon, noise and flat content (cartoon and
    noise only above JC.SMALL pixels)."""
    out = {}
    for k, (h, w) in enumerate(SIZES):
        for kind in KINDS:
            if h * w > JC.SMALL and kind == 'flat128':
                continue
            out[f'{h}x{w}_{kind}'] = JC.content(kind, h, w, 300 + k)
    return out


CORPUS = corpus()


def markers(data):
    """[(marker, offset)] of a JPEG file's markers, entropy-coded data skipped (0xFF00 is a stuffed
    byte; RSTm and the others that follow data are listed)."""
    out, i = [], 2
    while i < len(data) - 1:
        if data[i] != 0xFF:
            i += 1
            continue
        m = data[i + 1]
        if m == 0 or m == 0xFF:
            i += 1 if m == 0xFF else 2
            continue
        out.append((m, i))
        if 0xD0 <= m <= 0xD7 or m == 0xD9:
            i += 2
            continue
        i += 2 + (data[i + 2] << 8 | data[i + 3])
    return out


def dris_per_scan(data):
    """[DRI interval written just before each SOS, or None]."""
    out, pending = [], None
    for m, i in markers(data):
        if m == 0xDD:
            pending = data[i + 4] << 8 | data[i + 5]
        elif m == 0xDA:
            out.append(pending)
            pending = None
    return out


def _check(got, want, what):
    if got != want:
        k = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
        pytest.fail(f'{what}: {len(got)} bytes against Pillow\'s {len(want)}, first difference at byte {k} ({JC.turbo_version()})')


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
@pytest.mark.parametrize('mode', list(MODES))
def test_host_drivers_equal_pillow_with_restarts(mode, subsampling):
    for name, x in CORPUS.items():
        h, w = x.shape[:2]
        for q in QUALITIES:
            for kw in settings(h, w, subsampling):
                want = pillow(x, q, subsampling, **MODES[mode], **kw)
                _check(J.encode_host([x], q, subsampling, 'HWC', **MODES[mode], **kw)[0], want, f'{name} q{q} {subsampling} {kw}')


def test_interval_per_scan_follows_each_scans_mcus_per_row():
    """4:2:0, W = 53: mcux 4, the luma grid 7 blocks wide, the chroma grids 4.  With rows = 1 the DC
    scans and the chroma AC scans get DRI 4 and the luma AC scans DRI 7, and a DRI is written only
    where the interval changes; with blocks, one DRI before scan 0; with both, rows wins."""
    for h, w in ((40, 53), (33, 17)):
        x = JC.content('cartoon', h, w, w)
        for q in (50, 95):
            for kw in (dict(restart_marker_rows=1), dict(restart_marker_blocks=5), dict(restart_marker_blocks=5, restart_marker_rows=1)):
                got = J.encode_host([x], q, '4:2:0', 'HWC', progressive=True, **kw)[0]
                _check(got, pillow(x, q, '4:2:0', progressive=True, **kw), f'{h}x{w} q{q} {kw}')
                base = J.encode_host([x], q, '4:2:0', 'HWC', **kw)[0]
                _check(base, pillow(x, q, '4:2:0', **kw), f'{h}x{w} q{q} {kw} baseline')
    x = JC.content('cartoon', 40, 53, 53)
    rows = dris_per_scan(J.encode_host([x], 90, '4:2:0', 'HWC', progressive=True, restart_marker_rows=1)[0])
    # scans: DC, Y 1..5, Cr, Cb, Y 6..63, Y refine, DC refine, Cr, Cb, Y
    assert rows == [4, 7, 4, None, 7, None, 4, None, None, 7]
    assert dris_per_scan(J.encode_host([x], 90, '4:2:0', 'HWC', progressive=True, restart_marker_blocks=5)[0]) == [5] + [None] * 9
    both = J.encode_host([x], 90, '4:2:0', 'HWC', progressive=True, restart_marker_blocks=5, restart_marker_rows=1)[0]
    assert dris_per_scan(both) == rows
    assert dris_per_scan(J.encode_host([x], 90, '4:2:0', 'HWC', restart_marker_rows=2)[0]) == [8]
    x17 = JC.content('cartoon', 33, 17, 17)             # W = 17: luma grid 3, MCU grid 2 x 2, chroma 2
    assert dris_per_scan(J.encode_host([x17], 90, '4:2:0', 'HWC', progressive=True, restart_marker_rows=1)[0]) == \
        [2, 3, 2, None, 3, None, 2, None, None, 3]


@pytest.mark.parametrize('mode', list(MODES))
def test_rows_are_capped_at_65535_mcus(mode):
    """4:4:4, 65500 pixels wide (libjpeg's widest): 8188 MCUs per row, so 9 rows would be 73692
    MCUs; 72 rows high, the interval is 65535 and its marker falls inside a row."""
    x = JC.content('noise', 72, 65500, 9)
    x[:, ::3] = 128
    got = J.encode_host([x], 75, '4:4:4', 'HWC', **MODES[mode], restart_marker_rows=9)[0]
    _check(got, pillow(x, 75, '4:4:4', **MODES[mode], restart_marker_rows=9), mode)
    assert set(d for d in dris_per_scan(got) if d is not None) == {65535}
    assert sum(1 for m, _ in markers(got) if 0xD0 <= m <= 0xD7) == (1 if mode != 'progressive' else 10)


@pytest.mark.parametrize('mode', list(MODES))
def test_zero_is_no_restarts(mode):
    for name in ('97x61_cartoon', '200x300_noise', '1x1_flat128'):
        x = CORPUS[name]
        for s in JC.SAMPLINGS:
            want = J.encode_host([x], 80, s, 'HWC', **MODES[mode])[0]
            assert J.encode_host([x], 80, s, 'HWC', **MODES[mode], restart_marker_blocks=0, restart_marker_rows=0)[0] == want
            assert 0xDD not in [m for m, _ in markers(want)]


def test_a_mixed_call_equals_each_image_alone():
    names = [n for n in CORPUS if not n.startswith('1023x')]
    xs = [CORPUS[n] for n in names]
    for mode in MODES:
        for kw in (dict(restart_marker_rows=1), dict(restart_marker_blocks=2)):
            alone = [J.encode_host([x], 70, '4:2:0', 'HWC', **MODES[mode], **kw)[0] for x in xs]
            assert J.encode_host(xs, 70, '4:2:0', 'HWC', **MODES[mode], **kw) == alone, (mode, kw)


@pytest.mark.parametrize('bad', [-1, 65536, 70000, True, False, 1.0, None, '1'])
@pytest.mark.parametrize('key', ['restart_marker_blocks', 'restart_marker_rows'])
def test_restart_keywords_are_checked(key, bad):
    import torch
    from jpeg2png_b200 import encode_jpeg
    x = np.zeros((8, 8, 3), np.uint8)
    for mode in MODES:
        with pytest.raises(ValueError, match=key):
            J.encode_host([x], **MODES[mode], **{key: bad})
        with pytest.raises(ValueError, match=key):
            encode_jpeg(torch.zeros(3, 8, 8, dtype=torch.uint8), **MODES[mode], **{key: bad})


def _descs():
    d = J.Image()
    d.data, d.width, d.height, d.row_stride, d.col_stride, d.chan_stride = 1 << 20, 4, 4, 12, 3, 1
    return (J.Image * 1)(d)


@pytest.mark.parametrize('lib,name', [(J.load_jpegenc, 'jpegenc'), (J.load_jpegopt, 'jpegopt'), (J.load_jpegprog, 'jpegprog')])
@pytest.mark.parametrize('par,match', [((75, 2, -1, 0), 'restart_marker_blocks'), ((75, 2, 65536, 0), 'restart_marker_blocks'),
                                       ((75, 2, 0, -1), 'restart_marker_rows'), ((75, 2, 0, 65536), 'restart_marker_rows')])
def test_abi_refuses_restart_values(lib, name, par, match):
    lb = lib()
    p = J.Params(*par)
    n = C.c_size_t()
    assert getattr(lb, f'j2p_{name}_plan')(_descs(), 1, C.byref(p), C.byref(n), None) == -1
    assert match in getattr(lb, f'j2p_{name}_last_error')().decode()
    offs = (C.c_uint64 * 2)()
    assert getattr(lb, f'j2p_{name}_encode_host')(_descs(), 1, C.byref(p), 1 << 20, 1 << 30, offs) == -1
    assert match in getattr(lb, f'j2p_{name}_last_error')().decode()
    assert J.Params(75, 2).restart_marker_blocks == 0 and J.Params(75, 2).restart_marker_rows == 0


def _reader_takes(h, w, s):
    hs, vs = FACTORS[s]
    return -(-w // (8 * hs)) == (w // hs + 7) // 8 and -(-h // (8 * vs)) == (h // vs + 7) // 8


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
def test_the_reader_takes_restart_files(subsampling):
    """j2p_read_jpeg_mem reads each restart file to the coefficients of the file without restarts;
    the sequential layout pass routes baseline and optimized ones to the device decoder and the
    progressive pass takes progressive ones; each scan has one segment per interval."""
    taken = 0
    for name, x in CORPUS.items():
        h, w = x.shape[:2]
        if name.startswith('1023x') or not _reader_takes(h, w, subsampling):
            continue
        mx, my = mcu_grid(h, w, subsampling)
        for mode in MODES:
            want, err = EC.reader(J.encode_host([x], 75, subsampling, 'HWC', **MODES[mode])[0])
            assert want is not None, err
            for kw in (dict(restart_marker_rows=1), dict(restart_marker_blocks=3)):
                f = J.encode_host([x], 75, subsampling, 'HWC', **MODES[mode], **kw)[0]
                got, err = EC.reader(f)
                assert got is not None, f'{name} {mode} {kw}: {err}'
                for c in range(3):
                    assert (got[c] == want[c]).all(), f'{name} {mode} {kw} component {c}'
                if mode == 'progressive':
                    lay = D.ProgFileLayout(f)
                    assert lay.progressive_decodable
                    scans = [lay.lay.scan[k].s for k in range(lay.lay.nscan)]
                else:
                    lay = D.FileLayout(f)
                    assert lay.device_decodable
                    scans = [lay.lay.scan[k] for k in range(lay.lay.nscan)]
                for sc in scans:
                    units = sc.mcux * sc.mcuy
                    ri = sc.restart_interval
                    assert ri == (kw['restart_marker_blocks'] if 'restart_marker_blocks' in kw else min(65535, sc.mcux))
                    assert sc.nseg == -(-units // ri), (name, mode, kw)
                taken += 1
    assert taken >= 30


# worst-case bits of a block in each scan (jpegenc.h, jpegopt.h, jpegprog_core.h)
BASE_BITS, OPT_BITS = 1658, 1665
PROG_BITS = [16 + 11, 5 * 26 + 30, 63 * 26 + 30, 63 * 26 + 30, 58 * 26 + 30, 63 * 17 + 30, 1, 63 * 17 + 30, 63 * 17 + 30, 63 * 17 + 30]


def intervals(data):
    """Per scan, the unstuffed byte counts of its intervals (between SOS, RSTm and the next marker)."""
    out, cur, start = [], None, None
    for m, i in markers(data):
        if cur is not None and start is not None:
            seg = data[start:i]
            cur.append(len(seg) - seg.count(b'\xff\x00'))
            start = None
        if m == 0xDA:
            cur = []
            out.append(cur)
            start = i + 2 + (data[i + 2] << 8 | data[i + 3])
        elif 0xD0 <= m <= 0xD7:
            start = i + 2
    return out


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
def test_one_mcu_intervals_of_noise_fit_the_bound(subsampling):
    """Noise at q100 with restart_marker_blocks = 1: every interval's bytes (its 7 pad bits at most
    included) fit its blocks' bound, for each encoder and scan."""
    x = JC.content('noise', 48, 40, 4)
    hs, vs = FACTORS[subsampling]
    bpm = hs * vs + 2
    for mode, bits in (('baseline', BASE_BITS), ('optimize', OPT_BITS)):
        f = J.encode_host([x], 100, subsampling, 'HWC', **MODES[mode], restart_marker_blocks=1)[0]
        _check(f, pillow(x, 100, subsampling, **MODES[mode], restart_marker_blocks=1), mode)
        (segs,) = intervals(f)
        assert len(segs) == np.prod(mcu_grid(48, 40, subsampling))
        assert max(segs) <= (bpm * bits + 7) // 8
    f = J.encode_host([x], 100, subsampling, 'HWC', progressive=True, restart_marker_blocks=1)[0]
    _check(f, pillow(x, 100, subsampling, progressive=True, restart_marker_blocks=1), 'progressive')
    for k, segs in enumerate(intervals(f)):
        per = bpm if k in (0, 6) else 1
        assert max(segs) <= (per * PROG_BITS[k] + 7) // 8, k
