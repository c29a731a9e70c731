"""decode_jpeg(..., apply_exif_orientation=True) against the rotate-and-copy it replaces: prints one
JSON line.

usage: python tools/orientation_bench.py [--device D] [--files N] [--iterations I] [--reps R]

The files: N x 1920x1080 Q75 4:2:0 JPEGs (N = 64 by default) of synth.cartoon_image (seeded,
distinct images) written by Pillow once; each scenario splices an EXIF APP1 segment carrying its
orientations after SOI, so every scenario decodes the same coefficients.  uint8 CHW, I = 10
iterations.  Per scenario:
  export_ms   the export of the whole chunk (all N frames): CUDA events around 20 repetitions of the
              export call decode_jpeg makes, mean per call, on the current stream after the solve
  wall_ms     decode_jpeg wall clock from the bytes to the tensors, ending in a device synchronise,
              best of R after a warm-up
Scenarios: 'all_1' (the plain export), 'all_3', 'all_6', 'mix' (orientations 1..8 in turn), and
'torch_rotate_mix' / 'torch_rotate_6': apply_exif_orientation=False, then torch.rot90 / flip +
.contiguous() per frame; its export_ms is the plain export plus the rotate-and-copy of the chunk
(CUDA events, mean of 20), its wall_ms the decode plus that loop.  Checked: the torch results equal
the oriented tensors.  The card's name, power limit and clocks come from a read-only nvidia-smi
query in the same run.  Writes nothing to disk.
"""
import argparse
import io
import json
import os
import struct
import subprocess
import sys
import time

import numpy as np
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jpeg2png_b200 import abi, decode_jpeg, synth  # noqa: E402

EXPORTS = ('j2p_session_export', 'j2p_session_export_oriented')
REPEAT = 20


def card(device):
    q = 'name,power.limit,clocks.max.sm,clocks.sm,clocks.max.mem'
    try:
        out = subprocess.run(['nvidia-smi', f'--id={device}', f'--query-gpu={q}', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=20).stdout.strip().split(', ')
        return {'name': out[0], 'power_limit_w': float(out[1]), 'max_sm_mhz': int(out[2]), 'sm_mhz_idle': int(out[3]),
                'max_mem_mhz': int(out[4])}
    except Exception:
        return {'name': None}


def with_orientation(data, k):
    e = Image.Exif()
    e[0x0112] = k
    payload = e.tobytes()
    return data[:2] + b'\xff\xe1' + struct.pack('>H', len(payload) + 2) + payload + data[2:]


def rotate(t, k):
    """Orientation k of a (c, h, w) tensor with torch, as a new contiguous tensor."""
    hw = (-2, -1)
    return {1: lambda x: x, 2: lambda x: x.flip(-1), 3: lambda x: x.flip(hw), 4: lambda x: x.flip(-2),
            5: lambda x: x.transpose(-2, -1), 6: lambda x: torch.rot90(x, -1, hw), 7: lambda x: x.transpose(-2, -1).flip(hw),
            8: lambda x: torch.rot90(x, 1, hw)}[k](t).contiguous()


class ExportTimer:
    """Wraps the export calls of the product library: after the real call, the device is
    synchronised and the same call is repeated REPEAT times between CUDA events."""

    def __init__(self):
        self.lib = abi.load_product()
        self.ms = []
        self.saved = {name: getattr(self.lib, name) for name in EXPORTS}

    def __enter__(self):
        for name, fn in self.saved.items():
            setattr(self.lib, name, self._wrap(fn))
        return self

    def __exit__(self, *exc):
        for name, fn in self.saved.items():
            setattr(self.lib, name, fn)

    def _wrap(self, fn):
        def call(*args):
            rc = fn(*args)
            if rc != 0:
                return rc
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(REPEAT):
                fn(*args)
            b.record()
            b.synchronize()
            self.ms.append(a.elapsed_time(b) / REPEAT)
            return rc
        return call


def best_wall(fn, reps):
    fn()
    best = None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) * 1e3
        best = dt if best is None else min(best, dt)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--device', type=int, default=0)
    ap.add_argument('--files', type=int, default=64)
    ap.add_argument('--iterations', type=int, default=10)
    ap.add_argument('--reps', type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(args.device)
    w, h, n = 1920, 1080, args.files
    base = []
    for k in range(n):
        buf = io.BytesIO()
        Image.fromarray(synth.cartoon_image(w, h, 9000 + k).astype(np.uint8), 'RGB').save(buf, 'JPEG', quality=75, subsampling='4:2:0')
        base.append(buf.getvalue())
    orients = {'all_1': [1] * n, 'all_3': [3] * n, 'all_6': [6] * n, 'mix': [1 + i % 8 for i in range(n)]}
    kw = dict(iterations=args.iterations, device=args.device)
    res = {}
    tensors = {}
    for name, ks in orients.items():
        files = [with_orientation(d, k) for d, k in zip(base, ks)]
        with ExportTimer() as t:
            tensors[name] = decode_jpeg(files, apply_exif_orientation=True, **kw)
        wall = best_wall(lambda: decode_jpeg(files, apply_exif_orientation=True, **kw), args.reps)
        res[name] = {'export_ms': round(sum(t.ms), 4), 'export_calls': len(t.ms), 'wall_ms': round(wall, 2)}
    plain = tensors['all_1']
    bytes_moved = n * w * h * (3 * 4 + 3)                   # three fp32 planes read, three uint8 samples written
    for name in res:
        res[name]['export_gb_s'] = round(bytes_moved / res[name]['export_ms'] / 1e6, 1)
    checked = True
    for scenario, ks in (('mix', orients['mix']), ('6', orients['all_6'])):
        want = tensors['mix' if scenario == 'mix' else 'all_6']
        got = [rotate(t, k) for t, k in zip(plain, ks)]
        checked &= all(torch.equal(a, b) for a, b in zip(got, want))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(REPEAT):
            got = [rotate(t, k) for t, k in zip(plain, ks)]
        b.record()
        b.synchronize()
        rot_ms = a.elapsed_time(b) / REPEAT
        files = [with_orientation(d, k) for d, k in zip(base, ks)]

        def alternative():
            return [rotate(t, k) for t, k in zip(decode_jpeg(files, **kw), ks)]
        wall = best_wall(alternative, args.reps)
        res[f'torch_rotate_{scenario}'] = {'export_ms': round(res['all_1']['export_ms'] + rot_ms, 4),
                                          'rotate_ms': round(rot_ms, 4), 'wall_ms': round(wall, 2)}
    print(json.dumps({'tool': 'orientation_bench', 'files': n, 'size': [w, h], 'quality': 75, 'sampling': '4:2:0',
                      'iterations': args.iterations, 'dtype': 'uint8', 'layout': 'CHW', 'card': card(args.device),
                      'torch_equals_oriented': bool(checked), 'results': res}))


if __name__ == '__main__':
    main()
