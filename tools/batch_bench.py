"""Batch sessions against one session per frame: prints one JSON line.

usage: python tools/batch_bench.py [--device D] [--frames-1080p N] [--frames-256 N]

Two workloads of many frames of one geometry (j2p_session_create_batch, DESIGN.md §7b):
  (a) BASELINE config 5's frame, 1920x1080 Q75 4:2:0 x 100 iterations, 64 frames by default (config
      5 on N GPUs is 64/N frames per GPU: run with --frames-1080p 64/N on each of them);
  (b) 256x256 Q10 4:2:0 x 50 iterations (config 1's size), 64 frames.
Each workload is timed three ways on the same frames, with the coefficient planes already resident
in HBM: one batch session; one single-frame session per frame driven round-robin from one host
thread, each on its own stream; the single-frame sessions one after another.  Reported per way:
wall time per frame of the resident solves (device bound: the host only queues and waits), best
of three; Gpixel-iterations/s; kernel launches per iteration.  Per workload: whether every frame of
the batch is bit-identical to its single-frame result (full planes).  The card's name and power
limit are read with a read-only nvidia-smi query in the same run.  Writes nothing to disk.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jpeg2png_b200 import abi, synth  # noqa: E402

WEIGHT, PWEIGHT = 0.3, 0.001


def gpu_card(device):
    """Card name and enforced power limit (W) as nvidia-smi reports them."""
    try:
        out = subprocess.run(['nvidia-smi', f'--id={device}', '--query-gpu=name,power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=20).stdout.strip().split(', ')
        return {'name': out[0], 'power_limit_w': float(out[1])}
    except Exception:
        return {'name': None, 'power_limit_w': None}


def run_workload(lib, device, width, height, quality, iterations, n, distinct):
    # `distinct` frames with their own seeds, repeated to n (synthesising 64 1080p frames takes a minute)
    base = [synth.synth_coefs(width, height, quality, '4:2:0', 5000 + k) for k in range(distinct)]
    frames = [base[k % len(base)] for k in range(n)]
    desc = abi.frame_desc(frames[0], [0, 1, 2], WEIGHT, [PWEIGHT] * 3, iterations)
    bs = abi.Session(lib, desc, n, device)
    bs.upload(frames, [0, 1, 2])
    singles = [abi.Session(lib, desc, 1, device, batch=False) for _ in range(n)]
    for s1, img in zip(singles, frames):
        s1.upload([img], [0, 1, 2])

    def way_batch():
        bs.iterate(0, iterations)
        bs.sync()

    def way_round_robin():
        for i in range(iterations):
            for s1 in singles:
                s1.iterate(i, 1)
        for s1 in singles:
            s1.sync()

    def way_sequential():
        for s1 in singles:
            s1.iterate(0, iterations)
            s1.sync()

    out = {'workload': f'{width}x{height} Q{quality} 4:2:0 synthetic, joint 3 planes, -i {iterations} -w {WEIGHT} -p {PWEIGHT}',
           'frames': n}
    nplanes = len(frames[0].planes)
    for name, fn, counted in (('batch', way_batch, bs), ('round_robin', way_round_robin, singles[0]),
                              ('sequential', way_sequential, singles[0])):
        fn()                                                   # warm-up (and the first re-arm)
        best = None
        for _ in range(3):
            l0 = counted.launches
            t0 = time.perf_counter()
            fn()
            dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
            rearm = nplanes * (n if name == 'batch' else 1)     # k_init_plane launches of the re-arm
            per_it = (counted.launches - l0 - rearm) / iterations
        out[name] = {'ms_per_frame': best / n * 1e3, 'gpix_it_s': n * width * height * iterations / best / 1e9,
                     'launches_per_iteration': per_it}
    out['batch_speedup_vs_round_robin'] = out['round_robin']['ms_per_frame'] / out['batch']['ms_per_frame']
    out['batch_speedup_vs_sequential'] = out['sequential']['ms_per_frame'] / out['batch']['ms_per_frame']
    got = bs.download()
    same = True
    for k, s1 in enumerate(singles):
        want = s1.download()[0]
        same = same and all((np.ascontiguousarray(a).view(np.uint32) == np.ascontiguousarray(b).view(np.uint32)).all()
                            for a, b in zip(got[k], want))
    out['bit_identical_to_single_sessions'] = bool(same)
    bs.close()
    for s1 in singles:
        s1.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--device', type=int, default=0)
    ap.add_argument('--frames-1080p', type=int, default=64)
    ap.add_argument('--frames-256', type=int, default=64)
    args = ap.parse_args()
    lib = abi.load_product()
    if lib.j2p_device_count() <= 0:
        raise SystemExit('batch_bench.py: no CUDA device; the solver has no CPU fallback')
    line = {'card': gpu_card(args.device),
            'timing': 'wall clock around queueing + sync of resident solves (coefficients already in HBM, re-arm included), best of 3',
            'workloads': [run_workload(lib, args.device, 1920, 1080, 75, 100, args.frames_1080p, 4),
                          run_workload(lib, args.device, 256, 256, 10, 50, args.frames_256, 8)]}
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
