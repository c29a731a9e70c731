"""CMYK JPEG encoding on the GPU: encode_jpeg(..., cmyk=True) on four-channel tensors equals the
serial host drivers (and so Pillow's 'CMYK' files, tests/test_cmyk_jpeg_host.py) on the CMYK corpus
in every mode, with restart markers and given tables, for strided views, and for decode_jpeg's CMYK
tensors re-saved with keep_settings; mixed gray, RGB and CMYK lists make one call per kind; a CMYK
call launches each kernel once; large inputs and a forced split."""
import io

import numpy as np
import pytest
import torch

from jpeg2png_b200 import batch_encode as B
from jpeg2png_b200 import decode_jpeg, encode_jpeg, keep_settings
from jpeg2png_b200 import jpeg_encode as J
from tests import cmyk_jpeg_cases as K
from tests import codec_checks
from tests import cmyk_synth as S
from tests import gray_jpeg_cases as G
from tests import jpegenc_cases as JC

pytestmark = pytest.mark.gpu

CORPUS = K.corpus()
MODES = dict(K.MODES, restart_rows1={'restart_marker_rows': 1}, restart_blocks7_optimize={'optimize': True, 'restart_marker_blocks': 7},
             restart_rows2_progressive={'progressive': True, 'restart_marker_rows': 2},
             qtables_four_progressive={'progressive': True, 'qtables': [[2] * 64, [4] * 64, list(range(10, 74)), [300] * 64]})


def host(xs, q=75, s='4:2:0', **kw):
    return J.encode_host([np.ascontiguousarray(x) for x in xs], q, s, 'HWC', **kw, cmyk=True)


def cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@pytest.mark.parametrize('mode', list(MODES))
def test_device_equals_host_driver(mode):
    xs = list(CORPUS.values())
    ts = [cuda(x) for x in xs]
    kw = MODES[mode]
    for q in K.QUALITIES:
        for s in JC.SAMPLINGS:
            got = encode_jpeg(ts, quality=q, subsampling=s, layout='HWC', cmyk=True, **kw)
            assert got == host(xs, q, s, **kw), (q, s)
    for x, t in zip(xs[:12], ts[:12]):
        assert encode_jpeg(t, quality=90, subsampling='4:4:4', layout='HWC', cmyk=True, **kw) == K.pillow_cmyk(x, 90, '4:4:4', **kw)


def test_strided_views_equal_host_driver():
    x = K.cmyk('cartoon', 61, 97, 3)
    g = cuda(x)
    big = torch.zeros(130, 200, 6, dtype=torch.uint8, device='cuda')
    big[3:125:2, 5:199:2, 1:5] = g
    views = {
        'hwc': (g, 'HWC', x),
        'chw': (g.permute(2, 0, 1).contiguous(), 'CHW', x),
        'permuted_chw_view': (g.permute(2, 0, 1), 'CHW', x),
        'stepped': (big[3:125:2, 5:199:2, 1:5], 'HWC', x),
        'flipped': (torch.flip(g, [0, 1]), 'HWC', x[::-1, ::-1]),
        'transposed': (g.transpose(0, 1), 'HWC', x.transpose(1, 0, 2)),
        'window': (g[3:60:2, 5:90:3], 'HWC', x[3:60:2, 5:90:3]),
    }
    for name, (t, layout, want) in views.items():
        for kw in K.MODES.values():
            assert encode_jpeg(t, quality=80, layout=layout, cmyk=True, **kw) == host([want], 80, **kw)[0], name


def test_decoded_cmyk_resaved_with_keep_settings_is_pillows_save():
    """decode_jpeg(mode='UNCHANGED') on Pillow CMYK files, then encode_jpeg(cmyk=True,
    **keep_settings(files)): Pillow's save of the same pixels with the file's tables, 1 x 1; the
    files decode again."""
    from PIL import Image, ImageFile
    files = [S.pillow_cmyk(97, 61, 75, 1), S.pillow_cmyk(64, 48, 30, 2, subsampling='4:2:0'), S.pillow_cmyk(40, 24, 90, 3, subsampling='4:2:2')]
    for layout in ('CHW', 'HWC'):
        ts = decode_jpeg(files, iterations=8, mode='UNCHANGED', layout=layout)
        assert all(t.shape[0 if layout == 'CHW' else 2] == 4 for t in ts)
        for kw in K.MODES.values():
            got = encode_jpeg(ts, layout=layout, cmyk=True, **kw, **keep_settings(files))
            for t, f, src in zip(ts, got, files):
                a = t.cpu().numpy()
                a = a.transpose(1, 2, 0) if layout == 'CHW' else a
                buf = io.BytesIO()
                old = ImageFile.MAXBLOCK
                ImageFile.MAXBLOCK = max(old, 4 * a.size + 65536)
                try:
                    Image.fromarray(np.ascontiguousarray(a), 'CMYK').save(buf, 'JPEG', subsampling='4:4:4',
                                                                          qtables=Image.open(io.BytesIO(src)).quantization, **kw)
                finally:
                    ImageFile.MAXBLOCK = old
                assert f == buf.getvalue(), kw
            back = decode_jpeg(got, iterations=4, mode='UNCHANGED', layout=layout)
            assert [tuple(b.shape) for b in back] == [tuple(t.shape) for t in ts]


def test_mixed_lists_equal_per_kind_results(monkeypatch):
    cm = [cuda(x) for x in list(CORPUS.values())[:5]]
    grays = [cuda(G.gray('cartoon', h, w, 4)) for h, w in ((17, 13), (40, 33))]
    rgbs = [torch.from_numpy(JC.content('cartoon', h, w, 9)).cuda() for h, w in ((31, 33), (97, 61))]
    mixed = [cm[0], grays[0], rgbs[0], cm[1], cm[2], grays[1], rgbs[1], cm[3], cm[4]]
    for kw in MODES.values():
        if 'qtables' in kw:
            continue
        alone = {4: encode_jpeg(cm, layout='HWC', cmyk=True, **kw), 1: encode_jpeg(grays, layout='HWC', **kw),
                 3: encode_jpeg(rgbs, layout='HWC', **kw)}
        calls = []
        call = B.Codec.call

        def counting(self, fn, descs, *a, **k):
            if fn == 'encode':
                calls.append((self.channels, len(descs)))
            return call(self, fn, descs, *a, **k)
        monkeypatch.setattr(B.Codec, 'call', counting)
        got = encode_jpeg(mixed, layout='HWC', cmyk=True, **kw)
        monkeypatch.setattr(B.Codec, 'call', call)
        its = {c: iter(v) for c, v in alone.items()}
        assert got == [next(its[t.shape[2]]) for t in mixed]
        assert calls == [((4,), 5), ((1,), 2), ((3,), 2)]


@pytest.mark.parametrize('mode', list(K.MODES))
def test_launch_counts(mode):
    import json
    import subprocess
    import sys
    r = subprocess.run([sys.executable, '-c', f'from tests import cmyk_jpeg_cases; cmyk_jpeg_cases.launch_counts({mode!r})'],
                       cwd=codec_checks.ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    want = {'baseline': 7, 'optimize': 9, 'progressive': 10}[mode]
    for shapes, ran, st in json.loads(r.stdout.splitlines()[-1]):
        assert ran == {k: 1 for k in G.NAMES[mode]}, (ran, shapes)
        assert st['launches'] == want
        assert st['blocks'] == sum(K.blocks(h, w, '4:2:0') for h, w in shapes)


def test_8k_equals_host_driver():
    x = K.cmyk('cartoon', 4320, 7680, 21)
    t = cuda(x)
    for kw in (*K.MODES.values(), {'restart_marker_rows': 3, 'progressive': True}):
        assert encode_jpeg(t, quality=85, layout='HWC', cmyk=True, **kw) == host([x], 85, **kw)[0], kw


def test_flat_8k_progressive_equals_host_driver():
    x = np.full((4320, 7680, 4), 97, np.uint8)
    x[2000:2008, 3000:3008] = 200                   # one busy block in a sea of EOB runs
    t = cuda(x)
    for kw in ({}, {'restart_marker_blocks': 40000}):
        assert encode_jpeg(t, layout='HWC', progressive=True, cmyk=True, **kw) == host([x], progressive=True, **kw)[0]


def test_64_full_hd_in_one_call_sampled():
    xs = [K.cmyk('cartoon', 1080, 1920, 100 + i) for i in range(4)]
    ts = [cuda(xs[i % 4]) for i in range(64)]
    calls = []
    call = B.Codec.call
    try:
        def counting(self, fn, descs, *a, **k):
            if fn == 'encode':
                calls.append(len(descs))
            return call(self, fn, descs, *a, **k)
        B.Codec.call = counting
        for kw in K.MODES.values():
            calls.clear()
            got = encode_jpeg(ts, layout='HWC', subsampling='4:4:4', cmyk=True, **kw)
            assert calls == [64]
            for i in (0, 21, 63):
                assert got[i] == host([xs[i % 4]], 75, '4:4:4', **kw)[0], (kw, i)
    finally:
        B.Codec.call = call


def test_forced_split(monkeypatch):
    xs = list(CORPUS.values())[:8]
    ts = [cuda(x) for x in xs]
    for kw in K.MODES.values():
        p = J.params(75, '4:2:0', cmyk=True)
        codec_checks.check_forced_split(monkeypatch, J.codec(p, kw.get('optimize', False), kw.get('progressive', False)), ts,
                                        lambda: encode_jpeg(ts, layout='HWC', cmyk=True, **kw))
        monkeypatch.undo()
