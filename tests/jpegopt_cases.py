"""What the optimizing JPEG encoder's CPU and GPU tests share: Pillow's `optimize=True` file, a
Python restatement of libjpeg's table builder (T.81 Annex K.2 with its tie rule, the K.3 limit),
and the launch count of a device call."""
import io
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# The child of check_launch_count: codec_checks.launch_counts's 'jpeg' calls, with the package's
# codec() choosing libj2pjpegopt.so for them.
_CHILD = ('import functools, sys\n'
          'from jpeg2png_b200 import jpeg_encode as J\n'
          'J.codec = functools.partial(J.codec, optimize=True)\n'
          'from tests import codec_checks\n'
          'codec_checks.launch_counts("jpeg", tuple(sys.argv[1:]))\n')


def check_launch_count(names):
    """The kernels that run on the device for a call of libj2pjpegopt.so, counted by the profiler:
    each of names once per call, for one tiny image and for a mixed list alike, and as many as the
    call reports.  Returns each call's (shapes, stats fields).  As codec_checks.check_launch_count,
    the calls run in a child process, where no earlier profiler session can hide a call's first
    device records."""
    r = subprocess.run([sys.executable, '-c', _CHILD, *names], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    out = []
    for shapes, ran, st in json.loads(r.stdout.splitlines()[-1]):
        assert ran == {k: 1 for k in names}, (ran, shapes)
        assert st['launches'] == sum(ran.values())
        out.append((shapes, st))
    return out


def pillow_optimized(x, quality, subsampling):
    """Pillow's `optimize=True` file for the (h, w, 3) uint8 pixels.  libjpeg cannot suspend in the
    second pass of an optimized file, so Pillow's output buffer must hold the whole file; its
    default does not for noisy images at high quality.  The buffer size changes no byte."""
    from PIL import Image, ImageFile
    old = ImageFile.MAXBLOCK
    ImageFile.MAXBLOCK = max(old, 4 * x.shape[0] * x.shape[1] * 3 + 65536)
    try:
        buf = io.BytesIO()
        Image.fromarray(np.ascontiguousarray(x), 'RGB').save(buf, 'JPEG', quality=quality, subsampling=subsampling, optimize=True)
        return buf.getvalue()
    finally:
        ImageFile.MAXBLOCK = old


def _fib(n):
    a, b, out = 1, 1, []
    for _ in range(n):
        out.append(a)
        a, b = b, a + b
    return out


def crafted():
    """name -> 256 counts: the table builder's hard cases (K.3, ties, counts past 2^32, one or two
    symbols)."""
    rng = np.random.default_rng(11)
    out = {}
    for m in (20, 24, 30, 36, 40):                      # Fibonacci: K.2 lengths past 16 from 36 symbols
        c = [0] * 256
        for k, f in enumerate(_fib(m)):
            c[(k * 37 + 5) % 256] = f
        out[f'fibonacci{m}'] = c
    out['one symbol'] = [0] * 255 + [9]
    out['one symbol at 0'] = [1] + [0] * 255
    out['two symbols'] = [0] * 17 + [3] + [0] * 100 + [3] + [0] * 137
    out['256 equal'] = [5] * 256
    out['ties at several levels'] = [(k % 3 + 1) * (1 + (k % 7 == 0)) for k in range(256)]
    out['powers of two'] = [1 << (k % 20) for k in range(256)]
    out['above 2^32'] = [int(v) for v in rng.integers(1 << 32, 1 << 40, 256)]
    out['above 2^32 and small'] = [int(v) if k % 5 else 1 for k, v in enumerate(rng.integers(1 << 32, 1 << 36, 256))]
    for s in range(4):
        c = rng.integers(0, 50, 256) * (rng.random(256) < 0.4)
        c[s] += 1
        out[f'sparse random {s}'] = [int(v) for v in c]
    return out


# the crafted cases whose K.2 lengths pass 16, so that the K.3 limit does the work
LONG = ('fibonacci36', 'fibonacci40', 'powers of two', 'above 2^32 and small')


def restated_table(counts):
    """(bits[16], vals, longest K.2 length) of the table for 256 symbol counts.

    K.2: a pseudo-symbol 256 of count 1 joins; while two nonzero counts remain, V1 is the
    highest-numbered symbol among those of least count, V2 the same without V1; they merge and both
    chains lengthen.  K.3: two codes at a length i > 16 move up while the longest shorter length j
    with codes gives one; then the longest length loses one code (the pseudo-symbol).  The symbols
    are sorted by K.2 length, then by value.  Every nonzero count takes part (no 10^9 cap)."""
    freq = [int(c) for c in counts] + [1]
    others, size = [-1] * 257, [0] * 257

    def least(skip):
        best = -1
        for i in range(257):
            if freq[i] and i != skip and (best < 0 or freq[i] <= freq[best]):
                best = i
        return best
    while True:
        c1 = least(-1)
        c2 = least(c1)
        if c2 < 0:
            break
        freq[c1] += freq[c2]
        freq[c2] = 0
        for c in (c1, c2):
            size[c] += 1
            while others[c] >= 0:
                c = others[c]
                size[c] += 1
        c = c1
        while others[c] >= 0:
            c = others[c]
        others[c] = c2
    longest = max(size)
    bits = [0] * (max(longest, 16) + 1)
    for s in size:
        if s:
            bits[s] += 1
    for i in range(longest, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1
    vals = [v for length in range(1, longest + 1) for v in range(256) if size[v] == length]
    return bits[1:17], vals, longest
