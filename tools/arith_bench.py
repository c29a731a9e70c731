"""Arithmetic-coded (SOF9) files in decode_jpeg: the device decoder (libj2parith.so) against the host
reader, on each side of the routing rule.  Prints one JSON line.

usage: python tools/arith_bench.py [--device D] [--files N] [--reps R] [--iterations 10,50,100]

Workloads of N files (64 by default), 4 files and 1 file each, the arithmetic twins
tests/arith_synth.py writes of Pillow files (4 distinct files repeated: transcoding one 1080p file
takes seconds in Python):
  1080p_q75_420        1920x1080 Q75 4:2:0, no restart interval (one segment per file)
  1080p_q75_420_row    the same with one restart interval per MCU row (68 segments per file)
  256_q10              256x256 Q10 4:2:0, no restart interval
For each:
  longest_segment_kb          the longest segment of the workload, and whether the routing rule
                              (decode.arith_on_device, with decode_jpeg's thread count) sends it to
                              the device
  host_reader_ms_per_file     j2p_read_jpeg_mem, one thread and the thread pool of decode_jpeg
  layout_ms_per_file          j2p_read_jpeg_arith_layout, one thread and the pool
  decoder_ms_per_chunk        j2p_arith_decode on all N files in one call: CUDA events around it,
                              mean of R
  decode_jpeg_ms_per_image    wall clock from bytes to uint8 CUDA tensors (ending in a synchronise),
                              best of R after one warm-up, at each iteration count, with every file
                              on the device decoder and with the host front end; every image is
                              checked identical between the two
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
from tests import arith_synth as A  # noqa: E402
from tests import entropy_cases as E  # noqa: E402


def workloads(n):
    hd = [E.pillow(1920, 1080, 75, '4:2:0', seed=7000 + k) for k in range(4)]
    kinds = {'1080p_q75_420': [A.transcode(f) for f in hd], '1080p_q75_420_row': [A.transcode(f, 'sequential', 'row') for f in hd],
             '256_q10': [A.transcode(E.pillow(256, 256, 10, '4:2:0', seed=7000 + k)) for k in range(4)]}
    out = {}
    for name, files in kinds.items():
        for m in (n, 4, 1):
            out[f'{name}_x{m}'] = [files[k % 4] for k in range(m)]
    return out


def decoder(device, files, reps):
    lays = [D.ArithFileLayout(f) for f in files]
    stream = torch.cuda.Stream(device)
    D._ArithCoefs(device, lays, stream)                        # warm-up
    lib = D.load_arith()
    times = []
    for _ in range(reps):
        # time the decoder alone: the plan is packed and uploaded outside the events
        sizes = [p.w * p.h for lay in lays for p in lay.planes]
        with torch.cuda.stream(stream):
            coefs = torch.empty(int(sum(sizes)), dtype=torch.int16, device=device)
            offs = np.concatenate([[0], np.cumsum(sizes)])
            plan, addr, plan_bytes, _ = D.arith_plan(lays, [coefs.data_ptr() + 2 * int(o) for o in offs[:-1]], pinned=True)
            plan_dev = torch.empty(plan_bytes, dtype=torch.uint8, device=device)
            plan_dev.copy_(plan, non_blocking=True)
            status = torch.empty(len(lays), dtype=torch.int32, device=device)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            stats = D.ArithStats()
            e0.record(stream)
            assert lib.j2p_arith_decode(addr, plan_dev.data_ptr(), None, status.data_ptr(), stream.cuda_stream, D.C.byref(stats)) == 0
            e1.record(stream)
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
            assert (status.cpu() == 0).all()
    ms = float(np.mean(times))
    mb = sum(lay.compressed for lay in lays) / 1e6
    return {'ms_per_chunk': round(ms, 3), 'ms_per_file': round(ms / len(files), 3), 'compressed_mb': round(mb, 2),
            'launches': stats.launches, 'segments': stats.segments}


def decode_arms(device, files, iterations, reps):
    res = {}
    rule = D.arith_on_device
    for it in iterations:
        D.arith_on_device = lambda lays, workers: True
        try:
            t_dev, a = timed(lambda: decode_jpeg(files, iterations=it, device=device), reps)
        finally:
            D.arith_on_device = rule
        D._host_front_end = True
        try:
            t_host, b = timed(lambda: decode_jpeg(files, iterations=it, device=device), reps)
        finally:
            D._host_front_end = False
        assert all(torch.equal(x, y) for x, y in zip(a, b)), 'the two front ends disagree'
        res[str(it)] = {'device_decoder': round(t_dev * 1e3 / len(files), 3), 'host_front_end': round(t_host * 1e3 / len(files), 3)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--device', type=int, default=0)
    ap.add_argument('--files', type=int, default=64)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--iterations', default='10,50,100')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('arith_bench: no CUDA device')
    iterations = [int(x) for x in a.iterations.split(',')]
    out = {'card': gpu_card(a.device), 'files': a.files, 'cpus': os.cpu_count(), 'arith_device_ns_per_byte': D.ARITH_DEVICE_NS_PER_BYTE,
           'arith_host_ns_per_byte': D.ARITH_HOST_NS_PER_BYTE, 'workloads': {}}
    for name, files in workloads(a.files).items():
        parse = lambda f: D.parse_jpeg(f)                       # noqa: E731
        lays = [D.ArithFileLayout(f) for f in files]
        workers = min(len(files), os.cpu_count() or 1, 16)             # decode_jpeg's thread count
        w = {'mean_file_kb': round(sum(map(len, files)) / len(files) / 1e3, 1),
             'longest_segment_kb': round(max(lay.longest_segment for lay in lays) / 1e3, 2),
             'routed_to_device': D.arith_on_device(lays, workers),
             'host_reader_ms_per_file': {'one_thread': round(per_file_ms(parse, files, False), 3),
                                         'pool': round(per_file_ms(parse, files, True), 3)},
             'layout_ms_per_file': {'one_thread': round(per_file_ms(D.ArithFileLayout, files, False), 3),
                                    'pool': round(per_file_ms(D.ArithFileLayout, files, True), 3)},
             'decoder': decoder(a.device, files, a.reps),
             'decode_jpeg_ms_per_image': decode_arms(a.device, files, iterations, a.reps)}
        out['workloads'][name] = w
        print(json.dumps({name: w}), flush=True)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
