"""The front end of decode_jpeg: Huffman decoding on the device against the host reader.  Prints one
JSON line.

usage: python tools/entropy_bench.py [--device D] [--files N] [--reps R] [--iterations 10,50,100]

Workloads, N files each (64 by default):
  1080p_q75_420      1920x1080 Q75 4:2:0 (Pillow, synth.cartoon_image seeds 7000+k, as decode_bench.py)
  1080p_q90_444_opt  1920x1080 Q90 4:4:4, optimize=True (optimised Huffman tables)
  256_q10            256x256 Q10 4:2:0: small files, a few KB each
  1080p_ri8          1920x1080 4:2:0 with a restart interval of 8 MCUs (tests/jpeg_synth.py, random
                     coefficients; 4 distinct files repeated: synthesising one takes seconds)
For each:
  host_reader_ms_per_file     j2p_read_jpeg_mem, one thread and the thread pool of decode_jpeg
  layout_ms_per_file          j2p_read_jpeg_layout, one thread and the pool
  decoder_ms_per_chunk        the device decoder on all N files in one call: CUDA events around
                              j2p_entropy_decode (host round trips included), mean of R; with the
                              compressed (unstuffed) MB/s, sync rounds and host round trips
  decode_jpeg_ms_per_image    wall clock from bytes to uint8 CUDA tensors (ending in a synchronise),
                              best of R after one warm-up, at each iteration count, with the device
                              front end and with the host front end (the internal routing hook);
                              every image is checked identical between the two
The card's name and power limit are read (read-only nvidia-smi query) in the same run.  Writes
nothing to disk.
"""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from batch_bench import gpu_card  # noqa: E402
from jpeg2png_b200 import decode as D, decode_jpeg  # noqa: E402
from tests import entropy_cases as E  # noqa: E402


def workloads(n):
    synth = [E.synth_file(1920, 1080, [(2, 2), (1, 1), (1, 1)], 8, seed=k) for k in range(4)]
    return {
        '1080p_q75_420': [E.pillow(1920, 1080, 75, '4:2:0', seed=7000 + k) for k in range(n)],
        '1080p_q90_444_opt': [E.pillow(1920, 1080, 90, '4:4:4', optimize=True, seed=7000 + k) for k in range(n)],
        '256_q10': [E.pillow(256, 256, 10, '4:2:0', seed=7000 + k) for k in range(n)],
        '1080p_ri8': [synth[k % 4] for k in range(n)],
    }


def per_file_ms(fn, files, pool):
    t0 = time.perf_counter()
    if pool:
        with ThreadPoolExecutor(min(len(files), os.cpu_count() or 1, 16)) as ex:
            list(ex.map(fn, files))
    else:
        for f in files:
            fn(f)
    return (time.perf_counter() - t0) * 1e3 / len(files)


def decoder(device, files, reps):
    lays = [D.FileLayout(f) for f in files]
    stream = torch.cuda.Stream(device)
    D._DeviceCoefs(device, lays, stream)                       # warm-up
    lib = D.load_entropy()
    times = []
    for _ in range(reps):
        # time the decoder alone: the plan is packed and uploaded outside the events
        sizes = [p.w * p.h for lay in lays for p in lay.planes]
        with torch.cuda.stream(stream):
            coefs = torch.empty(int(sum(sizes)), dtype=torch.int16, device=device)
            offs = np.concatenate([[0], np.cumsum(sizes)])
            plan, addr, plan_bytes, work_bytes = D.entropy_plan(lays, [coefs.data_ptr() + 2 * int(o) for o in offs[:-1]], pinned=True)
            plan_dev = torch.empty(plan_bytes, dtype=torch.uint8, device=device)
            plan_dev.copy_(plan, non_blocking=True)
            work = torch.empty(work_bytes, dtype=torch.uint8, device=device)
            status = torch.empty(len(lays), dtype=torch.int32, device=device)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            stats = D.EntropyStats()
            e0.record(stream)
            assert lib.j2p_entropy_decode(addr, plan_dev.data_ptr(), work.data_ptr(), status.data_ptr(), stream.cuda_stream,
                                          D.C.byref(stats)) == 0
            e1.record(stream)
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
            assert (status.cpu() == 0).all()
    ms = float(np.mean(times))
    mb = sum(lay.compressed for lay in lays) / 1e6
    return {'ms_per_chunk': round(ms, 3), 'compressed_mb': round(mb, 2), 'mb_per_s': round(mb / ms * 1e3, 1),
            'sync_rounds': stats.rounds, 'round_trips': stats.round_trips, 'launches': stats.launches,
            'subsequences': stats.subsequences}


def timed(fn, reps):
    fn()
    best, out = None, None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return best, out


def decode_arms(device, files, iterations, reps):
    res = {}
    for it in iterations:
        t_dev, a = timed(lambda: decode_jpeg(files, iterations=it, device=device), reps)
        D._host_front_end = True
        try:
            t_host, b = timed(lambda: decode_jpeg(files, iterations=it, device=device), reps)
        finally:
            D._host_front_end = False
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
        raise SystemExit('entropy_bench: no CUDA device')
    iterations = [int(x) for x in a.iterations.split(',')]
    out = {'card': gpu_card(a.device), 'files': a.files, 'subseq_bits': D.SUBSEQ_BITS, 'workloads': {}}
    for name, files in workloads(a.files).items():
        parse = lambda f: D.parse_jpeg(f)                       # noqa: E731
        w = {'mean_file_kb': round(sum(map(len, files)) / len(files) / 1e3, 1),
             'host_reader_ms_per_file': {'one_thread': round(per_file_ms(parse, files, False), 3),
                                         'pool': round(per_file_ms(parse, files, True), 3)},
             'layout_ms_per_file': {'one_thread': round(per_file_ms(D.FileLayout, files, False), 3),
                                    'pool': round(per_file_ms(D.FileLayout, files, True), 3)},
             'decoder': decoder(a.device, files, a.reps),
             'decode_jpeg_ms_per_image': decode_arms(a.device, files, iterations, a.reps)}
        out['workloads'][name] = w
    print(json.dumps(out))


if __name__ == '__main__':
    main()
