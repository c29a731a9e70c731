"""Gray JPEG encoding on the GPU: encode_jpeg on one-channel tensors equals the serial host drivers
(and so Pillow's 'L' files, tests/test_gray_jpeg_host.py) on the gray corpus in every mode, with
restart markers, for strided views and for decode_jpeg's gray tensors; mixed gray and RGB lists make
one call per kind; a gray call launches each kernel once; large inputs, a forced split and the ABI's
refusal of other component counts."""
import ctypes as C

import numpy as np
import pytest
import torch

from jpeg2png_b200 import batch_encode as B
from jpeg2png_b200 import decode_jpeg, encode_jpeg, synth
from jpeg2png_b200 import jpeg_encode as J
from tests import codec_checks
from tests import gray_jpeg_cases as G
from tests import jpegenc_cases as JC
from tests.test_gray_host import CORPUS as GRAY_FILES
from tests.test_gray_host import synth_colour

pytestmark = pytest.mark.gpu

CORPUS = G.corpus()
MODES = dict(G.MODES, restart_rows1={'restart_marker_rows': 1}, restart_blocks7_optimize={'optimize': True, 'restart_marker_blocks': 7},
             restart_rows2_progressive={'progressive': True, 'restart_marker_rows': 2})


def host(xs, q=75, s='4:2:0', **kw):
    return J.encode_host([np.ascontiguousarray(x) for x in xs], q, s, 'HWC', **kw, gray=True)


def cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@pytest.mark.parametrize('mode', list(MODES))
def test_device_equals_host_driver(mode):
    xs = list(CORPUS.values())
    ts = [cuda(x) for x in xs]
    kw = MODES[mode]
    for q in G.QUALITIES:
        for s in JC.SAMPLINGS:
            got = encode_jpeg(ts, quality=q, subsampling=s, layout='HWC', **kw)
            assert got == host(xs, q, s, **kw), (q, s)
    for q in (1, 75, 100):
        for x, t in zip(xs, ts):
            assert encode_jpeg(t, quality=q, layout='HWC', **kw) == host([x], q, **kw)[0], q


def test_strided_views_equal_host_driver():
    rgb = JC.content('cartoon', 61, 97, 3)
    g = torch.from_numpy(rgb).cuda()
    chw = g.permute(2, 0, 1).contiguous()
    views = {
        'channel_of_hwc': (g[..., 1:2], 'HWC', rgb[..., 1:2]),
        'channel_of_chw': (chw[0:1], 'CHW', rgb[..., 0:1]),
        'permuted_chw_view': (g.permute(2, 0, 1)[2:3], 'CHW', rgb[..., 2:3]),
        'flipped': (torch.flip(g[..., 1:2], [0, 1]), 'HWC', rgb[::-1, ::-1, 1:2]),
        'transposed': (g[..., 0:1].transpose(0, 1), 'HWC', rgb[..., 0:1].transpose(1, 0, 2)),
        'stepped': (g[3:60:2, 5:90:3, 1:2], 'HWC', rgb[3:60:2, 5:90:3, 1:2]),
    }
    for name, (t, layout, want) in views.items():
        for kw in G.MODES.values():
            assert encode_jpeg(t, quality=80, layout=layout, **kw) == host([want], 80, **kw)[0], name


def _decode_inputs():
    files = list(GRAY_FILES.values()) + [synth_colour(64, 48, '4:2:0'), synth_colour(40, 24, '4:4:4')]
    return files


@pytest.mark.parametrize('mode', ['GRAY', 'UNCHANGED'])
def test_decoded_tensors_give_pillow_bytes(mode):
    files = _decode_inputs()
    for layout in ('CHW', 'HWC'):
        ts = decode_jpeg(files, iterations=8, mode=mode, layout=layout)
        gray = [t for t in ts if t.shape[0 if layout == 'CHW' else 2] == 1]
        assert len(gray) == (len(files) if mode == 'GRAY' else len(GRAY_FILES))
        for kw in G.MODES.values():
            got = encode_jpeg(gray, quality=90, layout=layout, **kw)
            for t, f in zip(gray, got):
                a = t.cpu().numpy()
                a = a[0] if layout == 'CHW' else a[..., 0]
                assert f == G.pillow_l(a, 90, **kw)
            for host_front in (False, True):
                from jpeg2png_b200 import decode as D
                old = D._host_front_end
                D._host_front_end = host_front
                try:
                    back = decode_jpeg(got, iterations=4, mode='UNCHANGED', progressive_on_device=True)
                finally:
                    D._host_front_end = old
                assert [tuple(b.shape) for b in back] == [(1,) + tuple(t.shape[1:] if layout == 'CHW' else t.shape[:2]) for t in gray]


def test_end_to_end_gray_file_to_pillow_bytes():
    data = GRAY_FILES['baseline_97x61_q20']
    t = decode_jpeg(data, mode='UNCHANGED')
    assert tuple(t.shape) == (1, 61, 97)
    assert encode_jpeg(t, quality=90) == G.pillow_l(t.cpu().numpy()[0], 90)


def test_mixed_lists_equal_per_kind_results(monkeypatch):
    grays = [cuda(x) for x in list(CORPUS.values())[:6]]
    rgbs = [torch.from_numpy(JC.content('cartoon', h, w, 9)).cuda() for h, w in ((31, 33), (17, 13), (97, 61))]
    mixed = [grays[0], rgbs[0], grays[1], grays[2], rgbs[1], grays[3], rgbs[2], grays[4], grays[5]]
    for kw in MODES.values():
        g_alone = encode_jpeg(grays, layout='HWC', **kw)
        c_alone = encode_jpeg(rgbs, layout='HWC', **kw)
        calls = []
        call = B.Codec.call

        def counting(self, fn, descs, *a, **k):
            if fn == 'encode':
                calls.append((self.channels, len(descs)))
            return call(self, fn, descs, *a, **k)
        monkeypatch.setattr(B.Codec, 'call', counting)
        got = encode_jpeg(mixed, layout='HWC', **kw)
        monkeypatch.setattr(B.Codec, 'call', call)
        gi, ci = iter(g_alone), iter(c_alone)
        assert got == [next(gi) if t.shape[2] == 1 else next(ci) for t in mixed]
        assert sorted(calls) == [((1,), 6), ((3,), 3)]


@pytest.mark.parametrize('mode', list(G.MODES))
def test_launch_counts(mode):
    import json
    import subprocess
    import sys
    r = subprocess.run([sys.executable, '-c', f'from tests import gray_jpeg_cases; gray_jpeg_cases.launch_counts({mode!r})'],
                       cwd=codec_checks.ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    want = {'baseline': 7, 'optimize': 9, 'progressive': 10}[mode]
    for shapes, ran, st in json.loads(r.stdout.splitlines()[-1]):
        assert ran == {k: 1 for k in G.NAMES[mode]}, (ran, shapes)
        assert st['launches'] == want
        assert st['blocks'] == sum(-(-h // 8) * -(-w // 8) for h, w in shapes)


def test_8k_equals_host_driver():
    x = G.gray('cartoon', 4320, 7680, 21)
    t = cuda(x)
    for kw in (*G.MODES.values(), {'restart_marker_rows': 3, 'progressive': True}):
        assert encode_jpeg(t, quality=85, layout='HWC', **kw) == host([x], 85, **kw)[0], kw


def test_flat_8k_progressive_equals_host_driver():
    x = np.full((4320, 7680, 1), 97, np.uint8)
    x[2000:2008, 3000:3008] = 200                   # one busy block in a sea of EOB runs
    t = cuda(x)
    for kw in ({}, {'restart_marker_blocks': 40000}):
        assert encode_jpeg(t, layout='HWC', progressive=True, **kw) == host([x], progressive=True, **kw)[0]


def test_64_full_hd_in_one_call_sampled():
    xs = [synth.cartoon_image(1920, 1080, 100 + i).astype(np.uint8)[..., 1:2] for i in range(4)]
    ts = [cuda(xs[i % 4]) for i in range(64)]
    calls = []
    call = B.Codec.call
    try:
        def counting(self, fn, descs, *a, **k):
            if fn == 'encode':
                calls.append(len(descs))
            return call(self, fn, descs, *a, **k)
        B.Codec.call = counting
        for kw in G.MODES.values():
            calls.clear()
            got = encode_jpeg(ts, layout='HWC', **kw)
            assert calls == [64]
            for i in (0, 21, 63):
                assert got[i] == host([xs[i % 4]], **kw)[0], (kw, i)
    finally:
        B.Codec.call = call


def test_forced_split(monkeypatch):
    xs = list(CORPUS.values())[:8]
    ts = [cuda(x) for x in xs]
    for kw in G.MODES.values():
        p = J.params(75, '4:2:0', components=1)
        codec_checks.check_forced_split(monkeypatch, J.codec(p, kw.get('optimize', False), kw.get('progressive', False)), ts,
                                        lambda: encode_jpeg(ts, layout='HWC', **kw))
        monkeypatch.undo()


def test_abi_refuses_two_components():
    t = torch.zeros(8, 8, 3, dtype=torch.uint8, device='cuda')
    d = (J.Image * 1)()
    d[0].data, d[0].width, d[0].height = t.data_ptr(), 8, 8
    d[0].row_stride, d[0].col_stride, d[0].chan_stride = 24, 3, 1
    work = torch.empty(1 << 20, dtype=torch.uint8, device='cuda')
    offs = (C.c_uint64 * 2)()
    for name, lib in (('jpegenc', J.load_jpegenc()), ('jpegopt', J.load_jpegopt()), ('jpegprog', J.load_jpegprog())):
        p = J.Params(75, 2, 0, 0, 2)
        rc = getattr(lib, f'j2p_{name}_encode')(d, 1, C.byref(p), work.data_ptr(), work.numel(), torch.cuda.current_stream().cuda_stream,
                                                offs, None, 0, None)
        assert rc == -1 and b'components' in getattr(lib, f'j2p_{name}_last_error')()
