"""Grayscale decode and encode against the colour paths on the same pixels: prints one JSON line.

usage: python tools/gray_bench.py [--device D] [--files N] [--reps R]

The files: N x 1920x1080 Q75 JPEGs (N = 64 by default) of synth.cartoon_image (seeded, distinct
images), written by Pillow twice: as 'L' (one component) and as RGB 4:2:0.  Each figure is wall clock
from the JPEG bytes to uint8 CHW CUDA tensors, ending in torch.cuda.synchronize(), after one
warm-up run, best of R, in ms per image, at 10, 50 and 100 iterations (-w 0.3 -p 0.001):
  gray_device       decode_jpeg(gray files, mode='UNCHANGED'), device Huffman decoding
  gray_host         the same with the host front end (every file parsed by j2p_read_jpeg_mem)
  colour            decode_jpeg(colour files), the default mode (joint solve, RGB)
  colour_gray_sep   decode_jpeg(colour files, mode='GRAY', separate=True): the luma solve alone
Also encode_png of the 100-iteration gray tensors against the colour ones (ms per image, best of R),
with the files' total bytes, and the card's name and power limit (read-only nvidia-smi query in the
same run).  Checked: the two gray front ends give identical tensors.  Writes nothing to disk.
"""
import argparse
import io
import json
import os
import sys
import time

import numpy as np
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from batch_bench import gpu_card  # noqa: E402
from jpeg2png_b200 import abi, decode as D, encode_png, synth  # noqa: E402


def files(w, h, n):
    gray, colour = [], []
    for k in range(n):
        rgb = Image.fromarray(synth.cartoon_image(w, h, 7000 + k).astype(np.uint8), 'RGB')
        for out, im, kw in ((gray, rgb.convert('L'), {}), (colour, rgb, {'subsampling': '4:2:0'})):
            buf = io.BytesIO()
            im.save(buf, 'JPEG', quality=75, **kw)
            out.append(buf.getvalue())
    return gray, colour


def best_of(fn, reps):
    fn()                                                    # warm-up
    best, result = None, None
    for _ in range(reps):
        result = None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        result = fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return best, result


def host_front_end(fn):
    def run():
        old = D._host_front_end
        D._host_front_end = True
        try:
            return fn()
        finally:
            D._host_front_end = old
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--device', type=int, default=0)
    ap.add_argument('--files', type=int, default=64)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    lib = abi.load_product()
    if lib.j2p_device_count() <= 0 or not torch.cuda.is_available():
        raise SystemExit('gray_bench.py: no CUDA device; the solver has no CPU fallback')
    torch.cuda.set_device(args.device)
    n, dev = args.files, args.device
    gray, colour = files(1920, 1080, n)
    line = {'card': gpu_card(dev),
            'workload': f'{n} x 1920x1080 Q75 (Pillow, synth.cartoon_image): L files and the same pixels as RGB 4:2:0; '
                        '-w 0.3 -p 0.001; uint8 CHW',
            'timing': f'wall clock from JPEG bytes to CUDA tensors, ending in torch.cuda.synchronize(), one warm-up, best of {args.reps}',
            'compressed_bytes': {'gray': sum(map(len, gray)), 'colour': sum(map(len, colour))},
            'decode_ms_per_image': {}}
    tensors = {}
    for it in (10, 50, 100):
        arms = {
            'gray_device': lambda: D.decode_jpeg(gray, mode='UNCHANGED', iterations=it, device=dev),
            'gray_host': host_front_end(lambda: D.decode_jpeg(gray, mode='UNCHANGED', iterations=it, device=dev)),
            'colour': lambda: D.decode_jpeg(colour, iterations=it, device=dev),
            'colour_gray_sep': lambda: D.decode_jpeg(colour, mode='GRAY', separate=True, iterations=it, device=dev),
        }
        row, out = {}, {}
        for name, fn in arms.items():
            t, out[name] = best_of(fn, args.reps)
            row[name] = t / n * 1e3
        row['gray_front_ends_identical'] = all(torch.equal(a, b) for a, b in zip(out['gray_device'], out['gray_host']))
        line['decode_ms_per_image'][f'iterations_{it}'] = row
        if it == 100:
            tensors = {'gray': out['gray_device'], 'colour': out['colour']}
        del out
    enc = {}
    for name, ts in tensors.items():
        t, pngs = best_of(lambda: encode_png(ts), args.reps)
        enc[name] = {'ms_per_image': t / n * 1e3, 'png_bytes': sum(map(len, pngs))}
    line['encode_png'] = enc
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
