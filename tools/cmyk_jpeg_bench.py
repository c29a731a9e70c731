"""encode_jpeg on CMYK tensors against Pillow 'CMYK': prints one JSON line.

usage: python tools/cmyk_jpeg_bench.py [--device D] [--files N] [--reps R] [--calls C] [--procs P]
                                       [--ab DIR] [--ab-rounds K]

The tensors: N x 1920x1080 CMYK images (N = 64 by default, seeded, distinct: synth.cartoon_image's
RGB as C, M, Y and its green channel reversed as K, as tests/cmyk_jpeg_cases.py builds them), as
(4, h, w) uint8 CUDA tensors.  For each of the default, optimize=True and progressive=True files, at
q75 and subsampling='4:4:4' (Pillow's keyword-less CMYK file):
  cmyk        encode_jpeg(tensors, cmyk=True): wall clock until the files are bytes, ms per image,
              and the one library call (CUDA events around j2p_jpeg{enc,opt,prog}_encode, mean of C
              calls);
  pillow_cmyk the tensors copied to the host (counted) and Pillow's JPEG writer on 'CMYK' images,
              one file per task, in P worker processes (16 by default), started before the timing;
  identical   whether every file equals Pillow's, in the same run.
Wall-clock figures are the best of R after one warm-up.

With --ab DIR (a directory holding another build's libj2pjpegenc.so, libj2pjpegopt.so and
libj2pjpegprog.so), also the regression check of the other kinds: N x 1920x1080 Q75 4:2:0 files
decoded at 100 iterations, encoded at q90 4:2:0 as RGB and, their green channel, as gray, by each
encoder: one whole library call timed with CUDA events (mean of C), alternating DIR's library and
the tree's K times, and whether both write the same bytes.  Also the card's name and power limit
(read-only nvidia-smi query in the same run).  Writes nothing.
"""
import argparse
import dataclasses
import io
import json
import os
import sys
import multiprocessing as mp
from concurrent.futures import ProcessPoolExecutor
from multiprocessing import shared_memory

import numpy as np
import torch
from PIL import Image, ImageFile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from batch_bench import gpu_card  # noqa: E402
from decode_bench import jpeg_files  # noqa: E402
from gray_jpeg_bench import LIBS, MODES, call_ms  # noqa: E402
from png_bench import best_of, encoder_call  # noqa: E402
from jpeg2png_b200 import abi, decode_jpeg, encode_jpeg, synth  # noqa: E402
from jpeg2png_b200 import jpeg_encode as J  # noqa: E402

SUBSAMPLING = '4:4:4'


def library_ms(tensors, quality, mode, calls):
    call, _ = encoder_call(J.codec(J.params(quality, SUBSAMPLING, cmyk=True), **MODES[mode]), tensors)
    return call_ms(call, calls)


def pillow_cmyk(a, quality, optimize=False, progressive=False):
    if optimize or progressive:     # libjpeg cannot suspend in a multi-pass file's last pass: room for the whole file
        ImageFile.MAXBLOCK = max(ImageFile.MAXBLOCK, 4 * a.size + 65536)
    buf = io.BytesIO()
    Image.fromarray(a, 'CMYK').save(buf, 'JPEG', quality=quality, subsampling=SUBSAMPLING, optimize=optimize, progressive=progressive)
    return buf.getvalue()


_shm = {}


def _pillow_shared(name, size, offset, h, w, quality, optimize=False, progressive=False):
    """In a worker process: Pillow on the CMYK image (h, w, 4) at `offset` of the shared buffer `name`."""
    if name not in _shm:
        _shm[name] = shared_memory.SharedMemory(name=name)
    return pillow_cmyk(np.ndarray((h, w, 4), np.uint8, buffer=_shm[name].buf[:size], offset=offset), quality, optimize, progressive)


def pillow_arm(tensors, quality, mode, reps, procs):
    """Best-of-`reps` seconds and files of: the (4, h, w) tensors copied into one shared host buffer
    as (h, w, 4), then Pillow in `procs` worker processes."""
    shapes = [(t.shape[1], t.shape[2]) for t in tensors]
    offs = np.cumsum([0] + [4 * h * w for h, w in shapes]).tolist()
    shm = shared_memory.SharedMemory(create=True, size=offs[-1])
    kw = MODES[mode]
    try:
        buf = torch.from_numpy(np.ndarray((offs[-1],), np.uint8, buffer=shm.buf))
        views = [buf[offs[k]:offs[k + 1]].view(h, w, 4) for k, (h, w) in enumerate(shapes)]
        with ProcessPoolExecutor(procs, mp_context=mp.get_context('spawn')) as pool:
            list(pool.map(_pillow_shared, [shm.name] * procs, [offs[-1]] * procs, [0] * procs, [1] * procs, [1] * procs,
                          [quality] * procs))               # start and attach every worker

            def arm():
                for v, t in zip(views, tensors):
                    v.copy_(t.permute(1, 2, 0))
                m = len(shapes)
                return list(pool.map(_pillow_shared, [shm.name] * m, [offs[-1]] * m, offs[:-1], [h for h, _ in shapes],
                                     [w for _, w in shapes], [quality] * m, [kw.get('optimize', False)] * m,
                                     [kw.get('progressive', False)] * m))
            t, files = best_of(arm, reps)
        del buf, views
    finally:
        shm.close()
        shm.unlink()
    return t, files


def cmyk_workloads(tensors, args):
    n, q, out = len(tensors), 75, []
    for mode, kw in MODES.items():
        t_k, files = best_of(lambda: encode_jpeg(tensors, quality=q, subsampling=SUBSAMPLING, cmyk=True, **kw), args.reps)
        t_p, pfiles = pillow_arm(tensors, q, mode, args.reps, args.procs)
        out.append({'mode': mode, 'quality': q, 'subsampling': SUBSAMPLING,
                    'cmyk': {'encode_jpeg_ms_per_image': t_k / n * 1e3, 'library_call_ms_per_image': library_ms(tensors, q, mode, args.calls) / n,
                             'total_bytes': sum(map(len, files))},
                    'pillow_cmyk': {'ms_per_image': t_p / n * 1e3, 'processes': args.procs, 'copies_counted': True},
                    'identical_to_pillow': files == pfiles})
    return out


def kinds_ab(args):
    """The tree's three encoders against DIR's on decoded RGB and gray tensors at q90 4:2:0, alternated."""
    rgb = decode_jpeg(jpeg_files(1920, 1080, 75, args.files), iterations=100, dtype=torch.uint8)
    gray = [t[1:2].contiguous() for t in rgb]
    torch.cuda.synchronize()
    out = []
    for kind, tensors, comps in (('rgb', rgb, 3), ('gray', gray, 1)):
        for mode, (name, so, declare) in LIBS.items():
            new = J.codec(J.params(90, '4:2:0', components=comps), **MODES[mode])
            path = os.path.join(args.ab, so)
            old = dataclasses.replace(new, load=lambda path=path, name=name, declare=declare: abi.load_library(path, f'{name} (A/B)', declare))
            arms = {label: encoder_call(codec, tensors)[0] for label, codec in (('parent', old), ('tree', new))}
            times = {'parent': [], 'tree': []}
            for _ in range(args.ab_rounds):
                for label in ('parent', 'tree'):
                    times[label].append(call_ms(arms[label], args.calls))
            files = {label: J.B.encode_device(codec, J.B.descs(codec, tensors, 'CHW'), tensors[0].device)
                     for label, codec in (('parent', old), ('tree', new))}
            out.append({'kind': kind, 'mode': mode, 'workload': f'{len(tensors)} x 1920x1080 Q75 4:2:0, -i 100, encoded q90 4:2:0',
                        'whole_call_ms': {k: [round(v, 4) for v in vs] for k, vs in times.items()},
                        'identical': files['parent'] == files['tree']})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--device', type=int, default=0)
    ap.add_argument('--files', type=int, default=64)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--calls', type=int, default=20)
    ap.add_argument('--procs', type=int, default=16)
    ap.add_argument('--ab', default=None)
    ap.add_argument('--ab-rounds', type=int, default=5)
    args = ap.parse_args()
    if abi.load_product().j2p_device_count() <= 0 or not torch.cuda.is_available():
        raise SystemExit('cmyk_jpeg_bench.py: no CUDA device')
    torch.cuda.set_device(args.device)
    line = {'card': gpu_card(args.device),
            'workload': f'{args.files} x 1920x1080 CMYK (4, h, w) uint8 CUDA tensors (cartoon RGB as C, M, Y; its green reversed as K)',
            'timing': f'wall clock, one warm-up, best of {args.reps}; library call: CUDA events, mean of {args.calls} calls'}
    tensors = []
    for k in range(args.files):
        rgb = synth.cartoon_image(1920, 1080, 7000 + k).astype(np.uint8)
        tensors.append(torch.from_numpy(np.dstack([rgb, rgb[::-1, ::-1, 1]]).transpose(2, 0, 1).copy()).cuda())
    torch.cuda.synchronize()
    line['cmyk_encode'] = cmyk_workloads(tensors, args)
    if args.ab:
        del tensors
        line['kinds_ab'] = kinds_ab(args)
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
