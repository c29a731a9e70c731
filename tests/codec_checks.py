"""Checks the codec libraries' tests share: the kernel inventory of a library (one cuobjdump parser),
and, for the two encoders through their shared driver (jpeg2png_b200/batch_encode.py), the forced
split of a list into several calls and the launch count of a call."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def kernels(lib):
    """{kernel name: (registers, stack bytes, local bytes)} of a library, from cuobjdump -res-usage."""
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump) or not os.path.exists(lib):
        pytest.skip('CUDA toolkit or the built library is missing')
    out = subprocess.run([cuobjdump, '-res-usage', lib], check=True, capture_output=True, text=True).stdout
    found = re.findall(r'Function (\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)', out)
    assert found, 'no kernels found in the library?'

    def name(m):                    # _Z<length><name><parameters>
        n = re.match(r'_Z(\d+)', m)
        return m[n.end():n.end() + int(n.group(1))] if n else m
    return {name(m): (int(r), int(s), int(l)) for m, r, s, l in found}


def check_kernel_inventory(lib, expected):
    """Every kernel of jpeg2png_b200/<lib> is a key of expected (kernel -> the GPU test that reaches
    it) and the reverse, and none uses stack or local memory."""
    ks = kernels(os.path.join(ROOT, 'jpeg2png_b200', lib))
    assert sorted(ks) == sorted(expected), f'kernels without a GPU test in KERNELS, or stale entries: {sorted(ks)}'
    for k, (reg, stack, local) in ks.items():
        assert stack == 0 and local == 0, f'{k} uses {stack} bytes of stack and {local} of local memory'


def check_forced_split(monkeypatch, codec, ts, encode):
    """encode() on the HWC tensors ts, with the free memory faked so that the work areas do not fit
    in one call: more than one encode call, every image in exactly one, the bytes of one call."""
    import torch
    from jpeg2png_b200 import batch_encode as B
    whole = encode()
    one = codec.plan(B.descs(codec, ts[:1], 'HWC'))[0]
    calls = []
    call = B.Codec.call

    def counting(self, fn, descs, *a, **kw):           # the images of each encode call
        if fn == 'encode':
            calls.append(len(descs))
        return call(self, fn, descs, *a, **kw)
    monkeypatch.setattr(torch.cuda, 'mem_get_info', lambda *a: (8 * one, 80 << 30))
    monkeypatch.setattr(B.Codec, 'call', counting)
    assert encode() == whole
    assert len(calls) > 1 and sum(calls) == len(ts)


def check_launch_count(encoder, names):
    """The kernels that run on the device, counted by the profiler: each of names once per call of
    encoder ('png' or 'jpeg'), for one tiny image and for a mixed list alike, and as many as the call
    reports.  Returns each call's (shapes, stats fields).

    The calls run in a child process: in a process that has already run many kernels and profiler
    sessions, a session can miss the first device records of a call."""
    r = subprocess.run([sys.executable, '-c', f'from tests import codec_checks; codec_checks.launch_counts({encoder!r}, {names!r})'],
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    out = []
    for shapes, ran, st in json.loads(r.stdout.splitlines()[-1]):
        assert ran == {k: 1 for k in names}, (ran, shapes)
        assert st['launches'] == sum(ran.values())
        out.append((shapes, st))
    return out


def launch_counts(encoder, names):
    """check_launch_count's child: prints, as JSON, each call's shapes, the profiler's count of each
    kernel of names, and the call's stats fields."""
    import torch
    from jpeg2png_b200 import batch_encode as B
    from jpeg2png_b200 import encode as E
    from jpeg2png_b200 import jpeg_encode as J
    codec, stats = (E.CODEC, E.Stats) if encoder == 'png' else (J.codec(J.Params(75, 2)), J.Stats)
    out = []
    for shapes in ([(1, 1)], [(300, 200)] * 5 + [(1, 1), (2000, 3000)]):
        ts = [torch.zeros(h, w, 3, dtype=torch.uint8, device='cuda') for h, w in shapes]
        d = B.descs(codec, ts, 'HWC')
        n, _ = codec.plan(d)
        work = torch.empty(n, dtype=torch.uint8, device='cuda')
        offs = (C.c_uint64 * (len(ts) + 1))()
        st = stats()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            codec.call('encode', d, work.data_ptr(), n, torch.cuda.current_stream().cuda_stream, offs, None, 0, C.byref(st))
            torch.cuda.synchronize()
        ran = {k: 0 for k in names}
        for ev in prof.key_averages():
            k = next((k for k in names if k in ev.key), None)
            if k:
                ran[k] += ev.count
        out.append((shapes, ran, {f: getattr(st, f) for f, _ in stats._fields_}))
    print(json.dumps(out))
