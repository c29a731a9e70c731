"""The front end of decode_jpeg for progressive files: Huffman decoding on the device
(progressive_on_device=True, libj2pprogressive.so) against the host reader.  Prints one JSON line.

usage: python tools/progressive_bench.py [--device D] [--files N] [--reps R] [--iterations 10,50,100]

Workloads, N progressive files each (64 by default; Pillow, synth.cartoon_image seeds 7000+k):
  1080p_q75_420      1920x1080 Q75 4:2:0, Pillow's standard 10-scan script
  1080p_q75_420_opt  the same with optimize=True (optimised Huffman tables)
  1080p_q75_420_rst  the same with restart_marker_rows=1 (one segment per MCU row)
  256_q10            256x256 Q10 4:2:0
For each:
  host_reader_ms_per_file     j2p_read_jpeg_mem, one thread and the thread pool of decode_jpeg
  layout_ms_per_file          j2p_read_jpeg_prog_layout, one thread and the pool
  decoder                     the device decoder on all N files in one call: CUDA events around
                              j2p_progressive_decode (host round trips included), mean of R; sync
                              rounds, round trips and launches; and from one torch.profiler run of its
                              own, the kernel time of the sync phase (sync rounds, scans, DC
                              differences), of the steps' stores and DC refine, and of the AC refine
                              masks and walkers
  decode_jpeg_ms_per_image    wall clock from bytes to uint8 CUDA tensors (ending in a synchronise),
                              best of R after one warm-up, at each iteration count, with the device
                              front end and with the host reader; every image is checked identical
The card's name and power limit are read (read-only nvidia-smi query) in the same run.  Writes
nothing to disk.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from batch_bench import gpu_card  # noqa: E402
from entropy_bench import per_file_ms, timed  # noqa: E402
from jpeg2png_b200 import decode as D, decode_jpeg  # noqa: E402
from tests import entropy_cases as E  # noqa: E402
from tests import progressive_cases as P  # noqa: E402

PHASES = {'sync': ('k_pg_sync', 'k_pg_scan', 'k_pg_dcdiff', 'k_pg_zero'), 'store_dc_refine': ('k_pg_store', 'k_pg_dcref'),
          'refine_walker': ('k_pg_mask', 'k_pg_refine')}


def workloads(n):
    return {
        '1080p_q75_420': [E.pillow(1920, 1080, 75, '4:2:0', progressive=True, seed=7000 + k) for k in range(n)],
        '1080p_q75_420_opt': [E.pillow(1920, 1080, 75, '4:2:0', optimize=True, progressive=True, seed=7000 + k) for k in range(n)],
        '1080p_q75_420_rst': [P.pillow_restarts(1920, 1080, 75, '4:2:0', seed=7000 + k) for k in range(n)],
        '256_q10': [E.pillow(256, 256, 10, '4:2:0', progressive=True, seed=7000 + k) for k in range(n)],
    }


def decoder(device, files, reps):
    lays = [D.ProgFileLayout(f) for f in files]
    stream = torch.cuda.Stream(device)
    D._ProgCoefs(device, lays, stream)                         # warm-up
    lib = D.load_progressive()
    sizes = [p.w * p.h for lay in lays for p in lay.planes]
    offs = np.concatenate([[0], np.cumsum(sizes)])

    def call(profile=False):
        # the decoder alone: the plan is packed and uploaded outside the events
        with torch.cuda.stream(stream):
            coefs = torch.empty(int(sum(sizes)), dtype=torch.int16, device=device)
            plan, addr, plan_bytes, work_bytes = D.progressive_plan(lays, [coefs.data_ptr() + 2 * int(o) for o in offs[:-1]], pinned=True)
            plan_dev = torch.empty(plan_bytes, dtype=torch.uint8, device=device)
            plan_dev.copy_(plan, non_blocking=True)
            work = torch.empty(work_bytes, dtype=torch.uint8, device=device)
            status = torch.empty(len(lays), dtype=torch.int32, device=device)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            stats = D.ProgressiveStats()
            stream.synchronize()
            e0.record(stream)
            assert lib.j2p_progressive_decode(addr, plan_dev.data_ptr(), work.data_ptr(), status.data_ptr(), stream.cuda_stream,
                                              D.C.byref(stats)) == 0
            e1.record(stream)
            e1.synchronize()
            assert (status.cpu() == 0).all()
            return e0.elapsed_time(e1), stats

    times = [call()[0] for _ in range(reps)]
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        _, stats = call()
        torch.cuda.synchronize()
    kernel_ms = {k: 0.0 for k in PHASES}
    for ev in prof.key_averages():
        for phase, names in PHASES.items():
            if any(n in ev.key for n in names):
                kernel_ms[phase] += ev.device_time_total / 1e3
    ms = float(np.mean(times))
    mb = sum(lay.compressed for lay in lays) / 1e6
    return {'ms_per_chunk': round(ms, 3), 'compressed_mb': round(mb, 2), 'mb_per_s': round(mb / ms * 1e3, 1),
            'kernel_ms': {k: round(v, 3) for k, v in kernel_ms.items()},
            'sync_rounds': stats.rounds, 'round_trips': stats.round_trips, 'launches': stats.launches, 'steps': stats.steps,
            'subsequences': stats.subsequences, 'refine_segments': stats.refine_segments}


def decode_arms(device, files, iterations, reps):
    res = {}
    for it in iterations:
        t_dev, a = timed(lambda: decode_jpeg(files, iterations=it, device=device, progressive_on_device=True), reps)
        t_host, b = timed(lambda: decode_jpeg(files, iterations=it, device=device), reps)
        assert all(torch.equal(x, y) for x, y in zip(a, b)), 'the two front ends disagree'
        res[str(it)] = {'device_front_end': round(t_dev * 1e3 / len(files), 3), 'host_front_end': round(t_host * 1e3 / len(files), 3)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--device', type=int, default=0)
    ap.add_argument('--files', type=int, default=64)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--iterations', default='10,50,100')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('progressive_bench: no CUDA device')
    iterations = [int(x) for x in a.iterations.split(',')]
    out = {'card': gpu_card(a.device), 'files': a.files, 'subseq_bits': D.SUBSEQ_BITS, 'workloads': {}}
    for name, files in workloads(a.files).items():
        w = {'mean_file_kb': round(sum(map(len, files)) / len(files) / 1e3, 1),
             'host_reader_ms_per_file': {'one_thread': round(per_file_ms(D.parse_jpeg, files, False), 3),
                                         'pool': round(per_file_ms(D.parse_jpeg, files, True), 3)},
             'layout_ms_per_file': {'one_thread': round(per_file_ms(D.ProgFileLayout, files, False), 3),
                                    'pool': round(per_file_ms(D.ProgFileLayout, files, True), 3)},
             'decoder': decoder(a.device, files, a.reps),
             'decode_jpeg_ms_per_image': decode_arms(a.device, files, iterations, a.reps)}
        out['workloads'][name] = w
    print(json.dumps(out))


if __name__ == '__main__':
    main()
