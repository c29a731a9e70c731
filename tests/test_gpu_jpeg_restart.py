"""encode_jpeg with restart markers on the GPU: for the three encoders the device writes the host
driver's bytes on the restart corpus (HWC, CHW and strided views), in one mixed call and in a forced
split; a flat 8K progressive image with one interval per MCU row; each kernel runs once per call
with one interval per MCU row or per MCU; and decode_jpeg reads a restart file to the tensors of
the file without restarts, through the device Huffman front ends."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from jpeg2png_b200 import batch_encode as B
from jpeg2png_b200 import decode_jpeg, encode_jpeg
from jpeg2png_b200 import jpeg_encode as J
from tests import jpegenc_cases as JC
from tests.test_jpeg_restart_host import CORPUS, MODES, settings

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VIEWS = ['HWC', 'CHW', 'strided']


def _host(xs, q, s, layout='HWC', **kw):
    return J.encode_host(xs, q, s, layout, **kw)


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _device_view(x, how, seed):
    """x (h, w, 3) as (layout, CUDA tensor): contiguous HWC, contiguous CHW, or a strided view (a
    step-sliced window of a larger tensor)."""
    if how != 'strided':
        lay, a = JC.view(x, how, seed)
        return lay, _cuda(a)
    h, w, _ = x.shape
    big = torch.randint(0, 256, (2 * h + 3, 3 * w + 2, 3), dtype=torch.uint8, device='cuda', generator=torch.Generator('cuda').manual_seed(seed))
    big[1:1 + 2 * h:2, 2:2 + 3 * w:3] = _cuda(x)
    return 'HWC', big[1:1 + 2 * h:2, 2:2 + 3 * w:3]


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
@pytest.mark.parametrize('mode', list(MODES))
def test_device_equals_host_driver_with_restarts(mode, subsampling):
    names = [n for n in CORPUS if not n.startswith('1023x')]
    for k, n in enumerate(names):
        x = CORPUS[n]
        h, w = x.shape[:2]
        lay, t = _device_view(x, VIEWS[k % 3], k)
        for q in (1, 90):
            for kw in settings(h, w, subsampling):
                want = _host([x], q, subsampling, **MODES[mode], **kw)[0]
                got = encode_jpeg(t, quality=q, subsampling=subsampling, layout=lay, **MODES[mode], **kw)
                assert got == want, f'{n} {VIEWS[k % 3]} q{q} {kw}'


@pytest.mark.parametrize('mode', list(MODES))
def test_a_mixed_call_equals_host_driver(mode):
    xs = list(CORPUS.values())
    ts = [_cuda(x) for x in xs]
    for q, s in ((75, '4:2:0'), (100, '4:4:4'), (50, '4:2:2')):
        for kw in (dict(restart_marker_rows=1), dict(restart_marker_blocks=1), dict(restart_marker_blocks=7, restart_marker_rows=2)):
            got = encode_jpeg(ts, quality=q, subsampling=s, layout='HWC', **MODES[mode], **kw)
            assert got == _host(xs, q, s, **MODES[mode], **kw), (q, s, kw)


def _check_forced_split(monkeypatch, codec, ts, encode):
    """encode() on the HWC tensors ts, with the free memory faked so that the work areas do not fit
    in one call: more than one encode call, every image in exactly one, the bytes of one call."""
    whole = encode()
    one = codec.plan(B.descs(codec, ts[:1], 'HWC'))[0]
    calls = []
    call = B.Codec.call

    def counting(self, fn, descs, *a, **kw):
        if fn == 'encode':
            calls.append(len(descs))
        return call(self, fn, descs, *a, **kw)
    monkeypatch.setattr(torch.cuda, 'mem_get_info', lambda *a: (8 * one, 80 << 30))
    monkeypatch.setattr(B.Codec, 'call', counting)
    assert encode() == whole
    assert len(calls) > 1 and sum(calls) == len(ts)


@pytest.mark.parametrize('mode', list(MODES))
def test_forced_split_gives_the_same_bytes(monkeypatch, mode):
    names = [n for n in CORPUS if n.startswith(('97x61', '200x300', '31x33'))]
    ts = [_cuda(CORPUS[n]) for n in names]
    kw = dict(restart_marker_rows=1)
    codec = J.codec(J.params(70, '4:2:0', **kw), **MODES[mode])
    _check_forced_split(monkeypatch, codec, ts, lambda: encode_jpeg(ts, quality=70, layout='HWC', **MODES[mode], **kw))


def test_flat_8k_progressive_one_interval_per_row_equals_host_driver():
    """Without restarts each AC scan of a flat image is one run segment of up to 518,400 blocks;
    with one interval per MCU row the longest is one block row of a component."""
    x = np.full((4320, 7680, 3), 77, np.uint8)
    for q, s in ((90, '4:2:0'), (95, '4:4:4')):
        got = encode_jpeg(_cuda(x), quality=q, subsampling=s, layout='HWC', progressive=True, restart_marker_rows=1)
        assert got == _host([x], q, s, progressive=True, restart_marker_rows=1)[0]


# The child of the launch count: codec_checks.launch_counts's 'jpeg' calls, with the package's
# codec() choosing the mode's library and setting the restart keyword under test to 1.
_CHILD = ('import sys\n'
          'from jpeg2png_b200 import jpeg_encode as J\n'
          'codec = J.codec\n'
          'def restart_codec(p, *a, **kw):\n'
          '    setattr(p, sys.argv[2], 1)\n'
          '    return codec(p, optimize=sys.argv[1] == "optimize", progressive=sys.argv[1] == "progressive")\n'
          'J.codec = restart_codec\n'
          'from tests import codec_checks\n'
          'codec_checks.launch_counts("jpeg", tuple(sys.argv[3:]))\n')

KERNELS = {'baseline': ('k_je_blocks', 'k_je_sizes', 'k_je_scan', 'k_je_emit', 'k_je_ffcount', 'k_je_offsets', 'k_je_stuff'),
           'optimize': ('k_jo_blocks', 'k_jo_hist', 'k_jo_tables', 'k_jo_sizes', 'k_jo_scan', 'k_jo_emit', 'k_jo_ffcount', 'k_jo_offsets',
                        'k_jo_stuff'),
           'progressive': ('k_jp_blocks', 'k_jp_runs', 'k_jp_hist', 'k_jp_tables', 'k_jp_sizes', 'k_jp_scan', 'k_jp_emit', 'k_jp_ffcount',
                           'k_jp_offsets', 'k_jp_stuff')}


@pytest.mark.parametrize('key', ['restart_marker_rows', 'restart_marker_blocks'])
@pytest.mark.parametrize('mode', list(MODES))
def test_each_kernel_runs_once_per_call(mode, key):
    names = KERNELS[mode]
    r = subprocess.run([sys.executable, '-c', _CHILD, mode, key, *names], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    for shapes, ran, st in json.loads(r.stdout.splitlines()[-1]):
        assert ran == {k: 1 for k in names}, (ran, shapes)
        assert st['launches'] == len(names)


@pytest.mark.parametrize('progressive', [False, True])
def test_decode_of_restart_file_equals_decode_of_file_without(progressive):
    """Restart markers change no coefficient: decode_jpeg reads a file with one interval per MCU row
    to the tensors of the file without restarts (the device Huffman front end for baseline files,
    progressive_on_device=True for progressive ones)."""
    xs = [JC.content('cartoon', 120, 160, 3), JC.content('noise', 64, 48, 4), JC.content('cartoon', 96, 62, 5)]
    ts = [_cuda(x) for x in xs]
    kw = dict(progressive_on_device=True) if progressive else {}
    for optimize in (False, True):
        with_rst = encode_jpeg(ts, quality=80, layout='HWC', optimize=optimize, progressive=progressive, restart_marker_rows=1)
        without = encode_jpeg(ts, quality=80, layout='HWC', optimize=optimize, progressive=progressive)
        assert all(a != b for a, b in zip(with_rst, without))
        got = decode_jpeg(with_rst, iterations=10, dtype=torch.float32, **kw)
        want = decode_jpeg(without, iterations=10, dtype=torch.float32, **kw)
        for g, w in zip(got, want):
            assert torch.equal(g, w), optimize
