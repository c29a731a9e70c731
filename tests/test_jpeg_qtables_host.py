"""CPU tests of given quantisation tables through the serial host drivers (the same steps as the
kernels of libj2pjpegenc.so, libj2pjpegopt.so and libj2pjpegprog.so): Pillow's bytes for every form
and count of tables, with and without quality, in every mode, sampling and kind; the frame and DQT
markers; the IJG tables given as qtables against the quality file; per-image tables and samplings
in one call; keep_settings against Pillow's quality='keep'; the quantiser over every entry; and the
refusals of the Python keywords and of the C ABI."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from jpeg2png_b200 import jpeg_encode as J
from jpeg2png_b200 import keep_settings
from tests import jpeg_qtables_cases as Q
from tests import jpegenc_cases as JC

HERE = os.path.dirname(os.path.abspath(__file__))
QUALITIES = [None, 20, 49, 50, 75, 100]


def _first_diff(got, want):
    return next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))


def _check(got, want, what):
    if got != want:
        pytest.fail(f'{what}: {len(got)} bytes against Pillow\'s {len(want)}, first difference at byte {_first_diff(got, want)} '
                    f'({JC.turbo_version()})')


@pytest.mark.parametrize('mode', list(Q.MODES))
def test_colour_equals_pillow(mode):
    kw = Q.MODES[mode]
    for h, w in Q.SIZES:
        x = Q.rgb(h, w, h * w)
        for n in (1, 2, 3, 4):
            for edge in (False, True):
                ts = Q.tables(n, seed=n * 100 + h + edge, edge=edge)
                for form, v in Q.forms(ts).items():
                    for q in QUALITIES:
                        s = JC.SAMPLINGS[(n + len(form) + (q or 0)) % 3]
                        got = J.encode_host([x], q, s, qtables=v, **kw)[0]
                        _check(got, Q.pillow(x, quality=q, subsampling=s, qtables=v, **kw), f'{h}x{w} {n} {form} edge={edge} q={q} {s}')


@pytest.mark.parametrize('mode', list(Q.MODES))
def test_gray_equals_pillow(mode):
    kw = Q.MODES[mode]
    for h, w in Q.SIZES:
        x = Q.rgb(h, w, h + w)[..., 1:2]
        for n in (1, 2, 3):
            ts = Q.tables(n, seed=n + h, edge=n == 2)
            for q in (None, 30, 90):
                for s in JC.SAMPLINGS:
                    got = J.encode_host([x], q, s, qtables=ts, gray=True, **kw)[0]
                    _check(got, Q.pillow(x, quality=q, subsampling=s, qtables=ts, **kw), f'gray {h}x{w} {n} q={q} {s}')


def test_every_quality_clamps_as_pillow():
    """Every quality scales given tables as Pillow does, the clamp to 255 included (a table of 300s
    at q=50), in all three samplings."""
    x = Q.rgb(31, 33, 7)
    for q in range(1, 101):
        v = [[300] * 64, Q.tables(1, q, 256)[0]]
        s = JC.SAMPLINGS[q % 3]
        _check(J.encode_host([x], q, s, qtables=v)[0], Q.pillow(x, quality=q, subsampling=s, qtables=v), f'q={q}')


def test_frame_and_dqt_markers():
    """One DQT per used table in component order, 16-bit exactly when an entry exceeds 255; SOF1
    with a 16-bit table in baseline and optimized files, SOF0 without, SOF2 in progressive ones."""
    x = Q.rgb(17, 13, 3)
    lo, hi = [[50] * 64, [60] * 64, [70] * 64, [80] * 64], [[50] * 63 + [256], [60] * 64, [8191] * 64, [1] * 64]
    for gray in (False, True):
        img = x[..., :1] if gray else x
        for n in (1, 2, 3, 4):
            for ts in (lo[:n], hi[:n]):
                used = 1 if gray else min(n, 3)
                wide = [max(t) > 255 for t in ts[:used]]
                for kw, sof in (({}, 0xC1 if any(wide) else 0xC0), ({'optimize': True}, 0xC1 if any(wide) else 0xC0),
                                ({'progressive': True}, 0xC2)):
                    f = J.encode_host([img], None, '4:4:4', qtables=ts, gray=gray, **kw)[0]
                    ms = Q.markers(f)
                    dqts = [s for m, s in ms if m == 0xDB]
                    assert [(d[0] >> 4, d[0] & 15, len(d)) for d in dqts] == [(int(w), k, 129 if w else 65) for k, w in enumerate(wide)]
                    frame = next(s for m, s in ms if m in (0xC0, 0xC1, 0xC2))
                    assert next(m for m, s in ms if m in (0xC0, 0xC1, 0xC2)) == sof
                    tq = [frame[6 + 3 * c + 2] for c in range(frame[5])]
                    assert tq == ([0] if gray else [0, min(1, n - 1), {1: 0, 2: 1}.get(n, 2)])
                    assert f == Q.pillow(img, subsampling='4:4:4', qtables=ts, **kw)


@pytest.mark.parametrize('gray', [False, True])
def test_ijg_tables_give_the_quality_file(gray):
    """qtables= the IJG tables of q is the quality=q file, for every q."""
    x = Q.rgb(33, 31, 11)
    img = x[..., :1] if gray else x
    for q in range(1, 101):
        assert J.encode_host([img], None, qtables=Q.ijg(q), gray=gray) == J.encode_host([img], q, gray=gray), q


def test_per_image_sets_in_one_call():
    """A call whose images each have their own set (and one the quality tables) writes each image's
    own Pillow file; so does a per-image subsampling list, in any mode."""
    xs = [Q.rgb(h, w, k) for k, (h, w) in enumerate(Q.SIZES * 2)]
    sets = [None if k == 3 else Q.tables(1 + k % 4, 500 + k, 400 if k % 2 else 200) for k in range(len(xs))]
    subs = [JC.SAMPLINGS[k % 3] for k in range(len(xs))]
    for kw in Q.MODES.values():
        got = J.encode_host(xs, None, subs, qtables=sets, **kw)
        for k, (x, t, s) in enumerate(zip(xs, sets, subs)):
            _check(got[k], Q.pillow(x, subsampling=s, qtables=t, **kw), f'image {k} {kw}')
        got = J.encode_host(xs, 60, subs, qtables=sets, **kw)
        for k, (x, t, s) in enumerate(zip(xs, sets, subs)):
            _check(got[k], Q.pillow(x, quality=60, subsampling=s, qtables=t, **kw), f'image {k} q60 {kw}')
    gray = [x[..., :1] for x in xs]
    got = J.encode_host(gray, None, subs, qtables=sets, gray=True)
    for k, (x, t, s) in enumerate(zip(gray, sets, subs)):
        _check(got[k], Q.pillow(x, subsampling=s, qtables=t), f'gray image {k}')


def test_distinct_sets_are_stored_once():
    x = Q.rgb(17, 13, 1)
    ts = Q.tables(2, 9)
    one = J.codec(J.params(75, '4:2:0'), sets=[ts])
    many = J.codec(J.params(75, '4:2:0'), sets=[ts] * 5)
    assert one.params[0]._obj.nqtables == many.params[0]._obj.nqtables == 1
    two = J.codec(J.params(75, '4:2:0'), sets=[ts, None, [list(t) for t in ts], None])
    assert two.params[0]._obj.nqtables == 2
    assert J.encode_host([x] * 4, None, qtables=[ts, None, ts, None]) == [J.encode_host([x], None, qtables=ts)[0], J.encode_host([x])[0]] * 2


def test_keep_settings_equal_pillow_keep():
    """encode_host with keep_settings on Pillow's decode of each source is Pillow's quality='keep'
    file of it: one input at a time, and the whole corpus as one per-image list (one call per kind)."""
    srcs = Q.keep_sources()
    want = {n: Q.pillow_keep(b) for n, b in srcs.items()}
    for n, b in srcs.items():
        ks = keep_settings(b)
        x = Q.pillow_pixels(b)
        _check(J.encode_host([x], None, ks['subsampling'], qtables=ks['qtables'], gray=x.shape[2] == 1)[0], want[n], n)
    for gray in (False, True):
        names = [n for n in srcs if n.startswith('gray') == gray]
        ks = keep_settings([srcs[n] for n in names])
        got = J.encode_host([Q.pillow_pixels(srcs[n]) for n in names], None, gray=gray, **ks)
        for n, g in zip(names, got):
            _check(g, want[n], f'{n} in a list')


def test_keep_settings_values(tmp_path):
    srcs = Q.keep_sources()
    ks = keep_settings(srcs['three_tables_420'])
    assert sorted(ks['qtables']) == [0, 1, 2] and ks['subsampling'] == '4:2:0'
    assert keep_settings(srcs['sampling_440'])['subsampling'] == '4:2:0'                # get_sampling's -1: libjpeg's 2 x 2
    assert keep_settings(srcs['gray_q80_62x96']) == {'qtables': {0: Q.ijg(80)[0]}, 'subsampling': '4:4:4'}
    assert max(max(t) for t in keep_settings(srcs['sixteen_bit_62x96'])['qtables'].values()) > 255
    p = tmp_path / 'a.jpg'
    p.write_bytes(srcs['ijg_q30_4:2:2_62x96'])
    assert keep_settings(str(p)) == keep_settings(p) == {'qtables': dict(enumerate(Q.ijg(30))), 'subsampling': '4:2:2'}
    assert keep_settings([p, srcs['one_table_30x46']])['subsampling'] == ['4:2:2', '4:2:0']


@pytest.mark.parametrize('data,match', [(b'not a jpeg', 'no SOI marker'), (b'\xff\xd8\xff\xda\x00\x02', 'scan before frame header'),
                                        (b'\xff\xd8\xff\xc0\x00\x0b\x0c\x00\x08\x00\x08\x01\x01\x11\x00', '12-bit samples')])
def test_keep_settings_refuses_what_the_reader_refuses(data, match):
    with pytest.raises(ValueError, match=match):
        keep_settings(data)
    with pytest.raises(ValueError, match='input 1'):
        keep_settings([Q.keep_sources()['one_table_30x46'], data])


def test_quantiser_over_every_entry(tmp_path):
    """j2p_je_quant with the plan's reciprocals is x / (8q) rounded half away from zero for every q
    in 1..8191 and every |x| < 2^15 (tests/qtables_quant_check.cu)."""
    exe = tmp_path / 'qtables_quant_check'
    subprocess.run(['/usr/local/cuda/bin/nvcc', '-O2', '-std=c++17', '--extended-lambda', '-gencode', 'arch=compute_90a,code=sm_90a',
                    '-o', str(exe), os.path.join(HERE, 'qtables_quant_check.cu')], check=True, capture_output=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert ' 0 mismatches' in r.stdout


GOOD = [[16] * 64]


@pytest.mark.parametrize('kw,match', [
    (dict(qtables=[[8192] * 64]), 'above 8191'), (dict(qtables=[[3000] * 64], quality=None), None),
    (dict(qtables=[[65535] * 64], quality=None), 'above 8191'), (dict(qtables=[[65536] * 64]), '0..65535'),
    (dict(qtables=[[-1] * 64]), '0..65535'), (dict(qtables=[[1.0] * 64]), '0..65535'), (dict(qtables=[[True] * 64]), '0..65535'),
    (dict(qtables=[[1] * 63]), '64 integers'), (dict(qtables=[[1] * 65]), '64 integers'), (dict(qtables=[]), '1..4 tables'),
    (dict(qtables={}), '1..4 tables'), (dict(qtables=GOOD * 5), '1..4 tables'), (dict(qtables='web_high'), 'text or as a preset'),
    (dict(qtables='1 2 3'), 'text or as a preset'), (dict(qtables=[GOOD, GOOD]), 'per-image qtables list has 2 elements for 1'),
    (dict(qtables=[None]), None), (dict(qtables=['medium']), 'text or as a preset'), (dict(qtables=7), 'list, tuple or dict'),
    (dict(quality=0), 'quality'), (dict(quality=101), 'quality'), (dict(quality=75.0), 'quality'), (dict(quality=True), 'quality'),
    (dict(quality='keep'), 'quality'), (dict(subsampling='4:1:1'), 'subsampling'), (dict(subsampling=['4:2:0', '4:4:4']), 'per-image'),
    (dict(subsampling=[None]), 'subsampling')])
def test_python_refusals(kw, match):
    x = Q.rgb(9, 8, 1)
    if match is None:
        assert J.encode_host([x], **kw)
        return
    with pytest.raises(ValueError, match=match):
        J.encode_host([x], **kw)


@pytest.mark.parametrize('lib', ['jpegenc', 'jpegopt', 'jpegprog'])
@pytest.mark.parametrize('case,match', [
    ('nqtables0', 'nqtables 0'), ('ntables0', 'set 1: ntables must be 1 .. 4 (got 0)'), ('ntables5', 'set 1: ntables must be 1 .. 4 (got 5)'),
    ('entry0', 'set 1: table 2 entry 5 is 0'), ('entry8192', 'set 1: table 0 entry 63 is 8192'), ('index', 'image 0: set 2 of qtables, which has 2'),
    ('null_ignores_index', None)])
def test_abi_refusals(lib, case, match):
    L = {'jpegenc': J.load_jpegenc, 'jpegopt': J.load_jpegopt, 'jpegprog': J.load_jpegprog}[lib]()
    d = (J.Image * 1)()
    d[0].data, d[0].width, d[0].height, d[0].row_stride, d[0].col_stride, d[0].chan_stride = 1 << 20, 4, 4, 12, 3, 1
    p = J.Params(75, 2)
    arr = (J.Qtables * 2)()
    for q in arr:
        q.ntables = 3
        for t in q.table:
            t[:] = [10] * 64
    p.qtables, p.nqtables = arr, 2
    if case == 'nqtables0':
        p.nqtables = 0
    elif case == 'ntables0':
        arr[1].ntables = 0
    elif case == 'ntables5':
        arr[1].ntables = 5
    elif case == 'entry0':
        arr[1].table[2][5] = 0
    elif case == 'entry8192':
        arr[1].table[0][63] = 8192
    elif case == 'index':
        d[0].qtables = 2
    else:
        p = J.Params(75, 2)
        d[0].qtables = 7
    n = C.c_size_t()
    rc = getattr(L, f'j2p_{lib}_plan')(d, 1, C.byref(p), C.byref(n), None)
    if match is None:
        assert rc == 0
        return
    assert rc == -1
    assert match in getattr(L, f'j2p_{lib}_last_error')().decode()
    offs = (C.c_uint64 * 2)()
    assert getattr(L, f'j2p_{lib}_encode_host')(d, 1, C.byref(p), 1 << 20, 1 << 30, offs) == -1
    assert match in getattr(L, f'j2p_{lib}_last_error')().decode()
