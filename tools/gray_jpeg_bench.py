"""encode_jpeg on gray tensors against the same pixels as RGB and against Pillow 'L': prints one JSON line.

usage: python tools/gray_jpeg_bench.py [--device D] [--files N] [--reps R] [--calls C] [--procs P]
                                       [--ab DIR] [--ab-rounds K]

The tensors: N x 1920x1080 synth.cartoon_image images (N = 64 by default, seeded, distinct), as
(1, h, w) uint8 gray CUDA tensors (the green channel) and as (3, h, w) RGB.  For each of the
default, optimize=True and progressive=True files, at q75:
  gray      encode_jpeg(gray tensors): wall clock until the files are bytes, ms per image, and the
            one library call (CUDA events around j2p_jpeg{enc,opt,prog}_encode, mean of C calls);
  rgb_420   the same for the RGB tensors at 4:2:0;
  pillow_l  the tensors copied to the host (counted) and Pillow's JPEG writer on 'L' images with
            subsampling='4:2:0' (encode_jpeg's default, as the gray arm), one file per task, in P
            worker processes (16 by default), started before the timing;
  identical whether every gray file equals Pillow's, in the same run.
Wall-clock figures are the best of R after one warm-up.

With --ab DIR (a directory holding another build's libj2pjpegenc.so, libj2pjpegopt.so and
libj2pjpegprog.so), also the colour regression check: tools/jpegenc_bench.py's workload (a) (N x
1920x1080 Q75 4:2:0 files decoded at 100 iterations) encoded at q90 4:2:0 by each encoder, one
whole library call timed with CUDA events (mean of C), alternating DIR's library and the tree's K
times, and whether both write the same bytes.  Also the card's name and power limit (read-only
nvidia-smi query in the same run).  Writes nothing.
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
from png_bench import best_of, encoder_call  # noqa: E402
from jpeg2png_b200 import abi, decode_jpeg, encode_jpeg, synth  # noqa: E402
from jpeg2png_b200 import jpeg_encode as J  # noqa: E402

MODES = {'default': {}, 'optimize': {'optimize': True}, 'progressive': {'progressive': True}}
LIBS = {'default': ('jpegenc', 'libj2pjpegenc.so', J._declare),
        'optimize': ('jpegopt', 'libj2pjpegopt.so', J._declare_opt),
        'progressive': ('jpegprog', 'libj2pjpegprog.so', J._declare_prog)}


def call_ms(call, calls):
    """CUDA events around call(), mean of `calls` after one warm-up."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    call()
    times = []
    for _ in range(calls):
        e0.record()
        call()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.mean(times))


def library_ms(tensors, quality, subsampling, mode, calls, components=3):
    p = J.params(quality, subsampling, components=components)
    call, _ = encoder_call(J.codec(p, **MODES[mode]), tensors)
    return call_ms(call, calls)


def pillow_l(a, quality, optimize=False, progressive=False):
    if optimize or progressive:     # libjpeg cannot suspend in a multi-pass file's last pass: room for the whole file
        ImageFile.MAXBLOCK = max(ImageFile.MAXBLOCK, 4 * a.size + 65536)
    buf = io.BytesIO()
    # subsampling as encode_jpeg's default: it sets the SOF's sampling byte of a gray file
    Image.fromarray(a, 'L').save(buf, 'JPEG', quality=quality, subsampling='4:2:0', optimize=optimize, progressive=progressive)
    return buf.getvalue()


_shm = {}


def _pillow_shared(name, size, offset, h, w, quality, optimize=False, progressive=False):
    """In a worker process: Pillow on the gray image (h, w) at `offset` of the shared buffer `name`."""
    if name not in _shm:
        _shm[name] = shared_memory.SharedMemory(name=name)
    return pillow_l(np.ndarray((h, w), np.uint8, buffer=_shm[name].buf[:size], offset=offset), quality, optimize, progressive)


def pillow_arm(tensors, quality, mode, reps, procs):
    """Best-of-`reps` seconds and files of: the gray tensors copied into one shared host buffer, then
    Pillow in `procs` worker processes."""
    shapes = [(t.shape[1], t.shape[2]) for t in tensors]
    offs = np.cumsum([0] + [h * w for h, w in shapes]).tolist()
    shm = shared_memory.SharedMemory(create=True, size=offs[-1])
    kw = MODES[mode]
    try:
        buf = torch.from_numpy(np.ndarray((offs[-1],), np.uint8, buffer=shm.buf))
        views = [buf[offs[k]:offs[k + 1]].view(h, w) for k, (h, w) in enumerate(shapes)]
        with ProcessPoolExecutor(procs, mp_context=mp.get_context('spawn')) as pool:
            list(pool.map(_pillow_shared, [shm.name] * procs, [offs[-1]] * procs, [0] * procs, [1] * procs, [1] * procs,
                          [quality] * procs))               # start and attach every worker

            def arm():
                for v, t in zip(views, tensors):
                    v.copy_(t[0])
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


def gray_workloads(gray, rgb, args):
    n, q, out = len(gray), 75, []
    for mode, kw in MODES.items():
        row = {'mode': mode, 'quality': q}
        t_g, files = best_of(lambda: encode_jpeg(gray, quality=q, **kw), args.reps)
        t_c, cfiles = best_of(lambda: encode_jpeg(rgb, quality=q, subsampling='4:2:0', **kw), args.reps)
        t_p, pfiles = pillow_arm(gray, q, mode, args.reps, args.procs)
        row['gray'] = {'encode_jpeg_ms_per_image': t_g / n * 1e3, 'library_call_ms_per_image': library_ms(gray, q, '4:2:0', mode, args.calls, 1) / n,
                       'total_bytes': sum(map(len, files))}
        row['rgb_420'] = {'encode_jpeg_ms_per_image': t_c / n * 1e3, 'library_call_ms_per_image': library_ms(rgb, q, '4:2:0', mode, args.calls) / n,
                          'total_bytes': sum(map(len, cfiles))}
        row['pillow_l'] = {'ms_per_image': t_p / n * 1e3, 'processes': args.procs, 'copies_counted': True}
        row['identical_to_pillow'] = files == pfiles
        out.append(row)
    return out


def colour_ab(args):
    """The tree's three encoders against DIR's on workload (a) at q90 4:2:0, alternated."""
    big = decode_jpeg(jpeg_files(1920, 1080, 75, args.files), iterations=100, dtype=torch.uint8)
    torch.cuda.synchronize()
    out = []
    for mode, (name, so, declare) in LIBS.items():
        p = J.params(90, '4:2:0')
        new = J.codec(p, **MODES[mode])
        path = os.path.join(args.ab, so)
        old = dataclasses.replace(new, load=lambda path=path, name=name, declare=declare: abi.load_library(path, f'{name} (A/B)', declare))
        arms, files = {}, {}
        for label, codec in (('parent', old), ('tree', new)):
            arms[label] = encoder_call(codec, big)[0]
        times = {'parent': [], 'tree': []}
        for _ in range(args.ab_rounds):
            for label in ('parent', 'tree'):
                times[label].append(call_ms(arms[label], args.calls))
        for label, codec in (('parent', old), ('tree', new)):
            d = J.B.descs(codec, big, 'CHW')
            files[label] = J.B.encode_device(codec, d, big[0].device)
        out.append({'mode': mode, 'workload': f'{len(big)} x 1920x1080 Q75 4:2:0, -i 100, encoded q90 4:2:0',
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
        raise SystemExit('gray_jpeg_bench.py: no CUDA device')
    torch.cuda.set_device(args.device)
    line = {'card': gpu_card(args.device),
            'workload': f'{args.files} x 1920x1080 synth.cartoon_image, gray (1, h, w) and RGB (3, h, w) uint8 CUDA tensors',
            'timing': f'wall clock, one warm-up, best of {args.reps}; library call: CUDA events, mean of {args.calls} calls'}
    rgb = [torch.from_numpy(synth.cartoon_image(1920, 1080, 7000 + k).astype(np.uint8).transpose(2, 0, 1).copy()).cuda()
           for k in range(args.files)]
    gray = [t[1:2].contiguous() for t in rgb]
    torch.cuda.synchronize()
    line['gray_encode'] = gray_workloads(gray, rgb, args)
    if args.ab:
        del rgb, gray
        line['colour_ab'] = colour_ab(args)
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
