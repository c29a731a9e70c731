"""Given quantisation tables on the GPU: encode_jpeg(..., qtables=) equals the serial host drivers
(and so Pillow, tests/test_jpeg_qtables_host.py) on the CPU corpus in every mode; 64 1080p images
with 64 distinct sets in one call, with the launches of a call without tables; decode_jpeg ->
encode_jpeg(**keep_settings) against Pillow's quality='keep' on a mixed list; a forced split; and a
producer on a side stream."""
import ctypes as C

import numpy as np
import pytest
import torch

from jpeg2png_b200 import batch_encode as B
from jpeg2png_b200 import decode_jpeg, encode_jpeg, keep_settings
from jpeg2png_b200 import jpeg_encode as J
from tests import jpeg_qtables_cases as Q
from tests import jpegenc_cases as JC

pytestmark = pytest.mark.gpu

LAUNCHES = {'default': 7, 'optimize': 9, 'progressive': 10}


def cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@pytest.mark.parametrize('mode', list(Q.MODES))
def test_device_equals_host_driver(mode):
    kw = Q.MODES[mode]
    xs = [Q.rgb(h, w, h * w) for h, w in Q.SIZES]
    ts = [cuda(x) for x in xs]
    for n in (1, 2, 3, 4):
        for edge in (False, True):
            tabs = Q.tables(n, seed=n * 100 + edge, edge=edge)
            for form, v in Q.forms(tabs).items():
                for q in (None, 20, 75, 100):
                    s = JC.SAMPLINGS[(n + len(form) + (q or 0)) % 3]
                    got = encode_jpeg(ts, quality=q, subsampling=s, layout='HWC', qtables=v, **kw)
                    assert got == J.encode_host(xs, q, s, qtables=v, **kw), (n, edge, form, q, s)
                    g = encode_jpeg([t[..., 1:2] for t in ts], quality=q, subsampling=s, layout='HWC', qtables=v, **kw)
                    assert g == J.encode_host([x[..., 1:2] for x in xs], q, s, qtables=v, gray=True, **kw), ('gray', n, edge, form, q, s)
    sets = [Q.tables(1 + k % 4, 700 + k, 500) for k in range(len(xs))]
    sets[2] = None
    subs = [JC.SAMPLINGS[k % 3] for k in range(len(xs))]
    mixed = ts + [t[..., :1] for t in ts]
    got = encode_jpeg(mixed, subsampling=subs * 2, layout='HWC', qtables=sets * 2, **kw)
    assert got[:len(xs)] == J.encode_host(xs, None, subs, qtables=sets, **kw)
    assert got[len(xs):] == J.encode_host([x[..., :1] for x in xs], None, subs, qtables=sets, gray=True, **kw)


def _stats_call(codec, ts):
    d = B.placed(codec, B.descs(codec, ts, 'CHW'))
    n, base = codec.plan(d)
    work = torch.empty(n, dtype=torch.uint8, device='cuda')
    offs = (C.c_uint64 * (len(ts) + 1))()
    st = J.Stats()
    codec.call('encode', d, work.data_ptr(), n, torch.cuda.current_stream().cuda_stream, offs, None, 0, C.byref(st))
    host = work[base:base + offs[len(ts)]].cpu().numpy()
    return [host[offs[i]:offs[i + 1]].tobytes() for i in range(len(ts))], st


@pytest.mark.parametrize('mode', list(LAUNCHES))
def test_64_1080p_images_with_64_sets(mode):
    """64 distinct sets in one call: the host driver's bytes, and as many launches as a call with
    the quality tables (7, 9 or 10)."""
    xs = [np.ascontiguousarray(JC.content('cartoon', 1080, 1920, k).transpose(2, 0, 1)) for k in range(64)]
    ts = [cuda(x) for x in xs]
    sets = [Q.tables(1 + k % 4, 900 + k, 60 + 4 * k, edge=k % 8 == 0) for k in range(64)]
    opt, prog = mode == 'optimize', mode == 'progressive'
    files, st = _stats_call(J.codec(J.params(75, '4:2:0'), opt, prog, [J.scaled_tables(t, None) for t in sets]), ts)
    assert st.launches == LAUNCHES[mode] and st.blocks == 64 * 120 * 68 * 6
    _, st0 = _stats_call(J.codec(J.params(90, '4:2:0'), opt, prog), ts)
    assert st0.launches == LAUNCHES[mode]
    assert files == encode_jpeg(ts, qtables=sets, optimize=opt, progressive=prog)
    for k in (0, 1, 2, 3, 8, 37, 63):               # the host driver is serial: a sample of the images
        assert files[k] == J.encode_host([xs[k]], None, layout='CHW', qtables=sets[k], optimize=opt, progressive=prog)[0], k


def test_keep_workflow_equals_pillow_keep():
    """decode_jpeg -> encode_jpeg(**keep_settings) on colour and gray files, three samplings, one
    and three tables: each file is Pillow's quality='keep' re-save of the decoded tensor's pixels."""
    srcs = Q.keep_sources()
    names = [n for n in srcs if not n.startswith('progressive')]
    files = [srcs[n] for n in names]
    tensors = decode_jpeg(files, mode='UNCHANGED', layout='HWC')
    got = encode_jpeg(tensors, layout='HWC', **keep_settings(files))
    for n, t, g in zip(names, tensors, got):
        assert g == Q.pillow_keep(srcs[n], t.cpu().numpy()), n
    chw = decode_jpeg(files, mode='UNCHANGED')
    assert encode_jpeg(chw, **keep_settings(files)) == got


def test_forced_split_gives_the_same_bytes(monkeypatch):
    xs = [Q.rgb(97, 61, k) for k in range(6)] + [Q.rgb(200, 300, 9)]
    ts = [cuda(x) for x in xs]
    sets = [Q.tables(1 + k % 3, 40 + k, 400) for k in range(len(xs))]
    whole = encode_jpeg(ts, layout='HWC', qtables=sets, optimize=True)
    codec = J.codec(J.params(75, '4:2:0'), True, sets=[J.scaled_tables(t, None) for t in sets])
    one = codec.plan(B.descs(codec, ts[:1], 'HWC'))[0]
    calls = []
    call = B.Codec.call

    def counting(self, fn, descs, *a, **kw):
        if fn == 'encode':
            calls.append(len(descs))
        return call(self, fn, descs, *a, **kw)
    monkeypatch.setattr(torch.cuda, 'mem_get_info', lambda *a: (8 * one, 80 << 30))
    monkeypatch.setattr(B.Codec, 'call', counting)
    assert encode_jpeg(ts, layout='HWC', qtables=sets, optimize=True) == whole
    assert len(calls) > 1 and sum(calls) == len(ts)
    assert whole == J.encode_host(xs, None, qtables=sets, optimize=True)


def test_producer_on_a_side_stream_needs_no_sync():
    xs = [Q.rgb(200, 300, k) for k in range(4)]
    sets = [Q.tables(2, k, 300) for k in range(4)]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        src = [cuda(x) for x in xs]
        torch.cuda._sleep(20_000_000)
        ts = [(x.float() * 1.0).to(torch.uint8) for x in src]
        got = encode_jpeg(ts, layout='HWC', qtables=sets, progressive=True)
    assert got == J.encode_host(xs, None, qtables=sets, progressive=True)
