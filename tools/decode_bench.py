"""decode_jpeg against what a Python user could do before it: prints one JSON line.

usage: python tools/decode_bench.py [--device D] [--files N] [--reps R]

Two workloads of JPEG files written with Pillow from synth.cartoon_image (seeded, distinct images):
  (a) N x 1920x1080 Q75 4:2:0, 100 iterations;
  (b) N x 256x256 Q10 4:2:0, 50 iterations  (N = 64 by default).
Two arms, each timed as wall clock from the JPEG bytes to RGB uint8 tensors on the device, ending
in torch.cuda.synchronize(), after one warm-up run, best of R:
  decode_jpeg   jpeg2png_b200.decode_jpeg(list of bytes): batch sessions, export into one tensor
  per_file      per file: parse, one session, upload, iterate, j2p_session_download_scanlines to
                the host, torch.from_numpy(...).cuda()
Both arms parse with the same reader.  Checked: every image is identical between the arms.  Also
reported: images/s and ms/image per arm; the host time of parsing alone; the device time of one
export launch per chunk (CUDA events around j2p_session_export of the whole batch, mean of 20);
the card's name and power limit (read-only nvidia-smi query in the same run).  Writes nothing to
disk.
"""
import argparse
import ctypes as C
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
from jpeg2png_b200 import abi, decode as D, synth  # noqa: E402


def jpeg_files(w, h, quality, n):
    out = []
    for k in range(n):
        buf = io.BytesIO()
        Image.fromarray(synth.cartoon_image(w, h, 7000 + k).astype(np.uint8), 'RGB').save(buf, 'JPEG', quality=quality, subsampling='4:2:0')
        out.append(buf.getvalue())
    return out


def per_file(lib, device, files, iterations):
    """One session per file, scanlines to the host, then to the device."""
    out = []
    for data in files:
        p = D.parse_jpeg(data)
        desc = abi.frame_desc(p, [0, 1, 2], 0.3, [0.001] * 3, iterations)
        with abi.Session(lib, desc, 1, device, batch=False) as s:
            s.upload([p], [0, 1, 2])
            s.iterate(0, iterations)
            raw = np.empty((p.h, p.w * 3 + 1), np.uint8)
            s._check(lib.j2p_session_download_scanlines(s.s, p.w, p.h, 8, raw.ctypes.data))
        out.append(torch.from_numpy(raw[:, 1:].reshape(p.h, p.w, 3)).cuda(device))
    return out


def best_of(fn, reps):
    fn()                                                    # warm-up
    best, result = None, None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        result = fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return best, result


def export_ms(lib, device, files, iterations):
    """Device time of one export of the whole batch (uint8 CHW), CUDA events, mean of 20."""
    parsed = [D.parse_jpeg(x) for x in files]
    desc = abi.frame_desc(parsed[0], [0, 1, 2], 0.3, [0.001] * 3, iterations)
    n, w, h = len(parsed), parsed[0].w, parsed[0].h
    with abi.Session(lib, desc, n, device) as s:
        s.upload(parsed, [0, 1, 2])
        s.iterate(0, iterations)
        dst = torch.empty((n, 3, h, w), dtype=torch.uint8, device=f'cuda:{device}')
        o = abi.ImageOut(w, h, 8, abi.LAYOUT_CHW, 3 * w * h)
        stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream or 1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s._check(lib.j2p_session_export(s.s, 0, n, C.byref(o), C.c_void_p(dst.data_ptr()), stream))    # waits for the solve
        torch.cuda.synchronize()
        times = []
        for _ in range(20):
            e0.record()
            s._check(lib.j2p_session_export(s.s, 0, n, C.byref(o), C.c_void_p(dst.data_ptr()), stream))
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        s.sync()
    return float(np.mean(times))


def run_workload(lib, device, w, h, quality, iterations, n, reps):
    files = jpeg_files(w, h, quality, n)
    t0 = time.perf_counter()
    for x in files:
        D.parse_jpeg(x)
    parse_s = time.perf_counter() - t0
    t_new, got = best_of(lambda: D.decode_jpeg(files, iterations=iterations, device=device), reps)
    t_old, want = best_of(lambda: per_file(lib, device, files, iterations), reps)
    same = all(torch.equal(a, b.permute(2, 0, 1)) for a, b in zip(got, want))
    out = {'workload': f'{n} x {w}x{h} Q{quality} 4:2:0 (Pillow, synth.cartoon_image), joint, -i {iterations} -w 0.3 -p 0.001',
           'files': n, 'parse_ms_per_image': parse_s / n * 1e3}
    for name, t in (('decode_jpeg', t_new), ('per_file', t_old)):
        out[name] = {'images_per_s': n / t, 'ms_per_image': t / n * 1e3}
    out['decode_jpeg_speedup'] = t_old / t_new
    out['identical'] = bool(same)
    out['export_kernel_ms_per_chunk'] = export_ms(lib, device, files, iterations)
    out['chunk_frames'] = n
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--device', type=int, default=0)
    ap.add_argument('--files', type=int, default=64)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    lib = abi.load_product()
    if lib.j2p_device_count() <= 0 or not torch.cuda.is_available():
        raise SystemExit('decode_bench.py: no CUDA device; the solver has no CPU fallback')
    torch.cuda.set_device(args.device)
    line = {'card': gpu_card(args.device),
            'timing': 'wall clock from JPEG bytes to uint8 CUDA tensors, ending in torch.cuda.synchronize(), one warm-up, best of '
                      f'{args.reps}',
            'workloads': [run_workload(lib, args.device, 1920, 1080, 75, 100, args.files, args.reps),
                          run_workload(lib, args.device, 256, 256, 10, 50, args.files, args.reps)]}
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
