"""What the progressive JPEG encoder's CPU and GPU tests share: Pillow's `progressive=True` file, a
Python restatement of the AC scans' run rules (T.81 Annex G as libjpeg's progressive Huffman encoder
applies them) that counts how often each rule fires, the inputs crafted to make each fire, and the
launch count of a device call."""
import collections
import functools
import io
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# libjpeg's jpeg_simple_progression for YCbCr: (component or 'all', Ss, Se, Ah, Al)
SCRIPT = [('all', 0, 0, 0, 1), (0, 1, 5, 0, 2), (2, 1, 63, 0, 1), (1, 1, 63, 0, 1), (0, 6, 63, 0, 2), (0, 1, 63, 2, 1),
          ('all', 0, 0, 1, 0), (2, 1, 63, 1, 0), (1, 1, 63, 1, 0), (0, 1, 63, 1, 0)]

# natural index of each zig-zag position
NATURAL = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28, 35,
           42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63]

# The child of check_launch_count: codec_checks.launch_counts's 'jpeg' calls, with the package's
# codec() choosing libj2pjpegprog.so for them.
_CHILD = ('import functools, sys\n'
          'from jpeg2png_b200 import jpeg_encode as J\n'
          'J.codec = functools.partial(J.codec, progressive=True)\n'
          'from tests import codec_checks\n'
          'codec_checks.launch_counts("jpeg", tuple(sys.argv[1:]))\n')


def check_launch_count(names):
    """The kernels that run on the device for a call of libj2pjpegprog.so, counted by the profiler
    in a child process (as jpegopt_cases.check_launch_count): each of names once per call, for one
    tiny image and for a mixed list alike, and as many as the call reports."""
    r = subprocess.run([sys.executable, '-c', _CHILD, *names], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    out = []
    for shapes, ran, st in json.loads(r.stdout.splitlines()[-1]):
        assert ran == {k: 1 for k in names}, (ran, shapes)
        assert st['launches'] == sum(ran.values())
        out.append((shapes, st))
    return out


def pillow_progressive(x, quality, subsampling, **kw):
    """Pillow's `progressive=True` file for the (h, w, 3) uint8 pixels (kw: more save options).  As
    for an optimized file, Pillow's output buffer must hold the whole file; its size changes no
    byte."""
    from PIL import Image, ImageFile
    old = ImageFile.MAXBLOCK
    ImageFile.MAXBLOCK = max(old, 4 * x.shape[0] * x.shape[1] * 3 + 65536)
    try:
        buf = io.BytesIO()
        Image.fromarray(np.ascontiguousarray(x), 'RGB').save(buf, 'JPEG', quality=quality, subsampling=subsampling, progressive=True,
                                                              **kw)
        return buf.getvalue()
    finally:
        ImageFile.MAXBLOCK = old


def grids(h, w, subsampling):
    """[(blocks wide, blocks high)] of each component's own grid, and of its MCU-padded grid."""
    hs, vs = {'4:4:4': (1, 1), '4:2:2': (2, 1), '4:2:0': (2, 2)}[subsampling]
    mx, my = -(-w // (8 * hs)), -(-h // (8 * vs))
    own = [(-(-w // 8), -(-h // 8))] + [(-(-w // (8 * hs)), -(-h // (8 * vs)))] * 2
    mcu = [(mx * hs, my * vs)] + [(mx, my)] * 2
    return own, mcu


def scan_events(blocks, ss, se, ah, al):
    """The events of one AC scan over blocks (int [n][64], zig-zag order, the component's raster
    order), as libjpeg's encoder meets them: 'eobrun n' per EOB run emitted with n extra bits,
    'run 0x7fff' and 'be > 937' per forced emission, 'zrl' per ZRL, 'zrl with corrections' per ZRL
    that flushes buffered correction bits, 'new' per newly nonzero coefficient."""
    ev = collections.Counter()
    mag = np.abs(blocks[:, ss:se + 1].astype(np.int64)) >> al
    run = be = 0

    def eobrun():
        nonlocal run, be
        if run:
            ev[f'eobrun {run.bit_length() - 1}'] += 1
        run = be = 0
    for b in range(len(blocks)):
        m = mag[b]
        nz = np.flatnonzero(m)
        if not len(nz):
            run += 1
            if run == 0x7FFF:
                ev['run 0x7fff'] += 1
                eobrun()
            continue
        if ah == 0:                                     # AC first
            eobrun()
            prev = -1
            for k in nz:
                ev['zrl'] += (k - prev - 1) // 16
                prev = k
            trailing = m[-1] == 0
            tail = 0
        else:                                           # AC refine
            ones = np.flatnonzero(m == 1)
            eob = ones[-1] if len(ones) else -1
            r = br = 0
            for k in range(len(m)):
                if m[k] == 0:
                    r += 1
                    continue
                while r > 15 and k <= eob:
                    eobrun()
                    ev['zrl'] += 1
                    if br:
                        ev['zrl with corrections'] += 1
                    br = 0
                    r -= 16
                if m[k] > 1:
                    br += 1
                    continue
                eobrun()
                ev['new'] += 1
                br = r = 0
            trailing = r > 0 or br > 0
            tail = br
        if trailing:
            run += 1
            be += tail
            if run == 0x7FFF or be > 937:
                ev['run 0x7fff' if run == 0x7FFF else 'be > 937'] += 1
                eobrun()
    eobrun()
    return ev


def all_events(planes, h, w, subsampling):
    """scan_events summed over the AC scans of the script, for the coefficient planes of a file the
    reader takes (int16 [blocks][64] in natural order, raster order, each component's grid)."""
    own, _ = grids(h, w, subsampling)
    ev = collections.Counter()
    for comp, ss, se, ah, al in SCRIPT:
        if comp == 'all':
            continue
        zz = planes[comp].reshape(-1, 64)[:, NATURAL]
        assert len(zz) == own[comp][0] * own[comp][1]
        ev += scan_events(zz, ss, se, ah, al)
    return ev


@functools.lru_cache(maxsize=None)
def crafted():
    """name -> (h, w, 3) uint8 pixels, quality, subsampling, the events it must reach."""
    from tests import jpegenc_cases as JC
    out = {}
    # 40000 luma blocks: a run reaches 0x7FFF, and is then emitted with 14 extra bits
    out['flat 1600x1600'] = (np.full((1600, 1600, 3), 90, np.uint8), 75, '4:2:0', ('run 0x7fff', 'eobrun 14'))
    # one 8 x 8 tile of noise repeated: every luma block the same, no new coefficient in the last
    # luma refine and some 60 correction bits each, so BE passes 937 after 16 blocks
    rng = np.random.default_rng(2024)
    tile = rng.integers(0, 256, (8, 8, 3), dtype=np.uint8)
    out['repeated noise tile'] = (np.tile(tile, (16, 16, 1)), 100, '4:4:4', ('be > 937',))
    # large smooth shapes at high quality: ZRLs in refine scans while correction bits are buffered
    out['cartoon 256x256'] = (JC.content('cartoon', 256, 256, 31), 95, '4:4:4', ('zrl with corrections',))
    return out


def partial_mcu():
    """(h, w, subsampling) whose AC scans' raster grids differ from the MCU grid."""
    return [(33, 17, '4:2:0'), (9, 17, '4:2:2'), (47, 65, '4:2:0'), (40, 24, '4:2:0')]
