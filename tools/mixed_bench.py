#!/usr/bin/env python
"""mixed_bench.py — lists of JPEG files of distinct sizes, two measurements per workload.

decode: decode_jpeg from bytes to uint8 CHW tensors with grouping on (decode._group_chunks, the
        default) against grouping off, host clock around the call and a device synchronise; every
        image must be identical between the arms, or the tool fails.  Frames over
        decode.GROUP_MAX_PIXELS are not grouped, so there the two arms run the same calls.
device: the solve alone, planes resident: one group (j2p_session_iterate_group) against the sum of
        each session solved on its own (j2p_session_iterate, synchronised after each), per iteration.
        This arm groups whatever the frame size, to show where the size limit comes from.

Workloads: 64 distinct 4:2:0 sizes around 256² (Q10, 50 iterations), 64 distinct 4:2:0 sizes around
1080p (Q75, 100 iterations), 32 distinct 4:4:4 sizes around 256² and around 512² (Q50, 50 iterations).
Prints one JSON line.
"""
import argparse
import ctypes as C
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jpeg2png_b200 import abi, decode, decode_jpeg, synth  # noqa: E402

WORKLOADS = {   # name: (count, w0, h0, step, quality, subsampling, iterations)
    '256_420': (64, 256, 256, 8, 10, '4:2:0', 50),
    '1080p_420': (64, 1920, 1080, 16, 75, '4:2:0', 100),
    '256_444': (32, 256, 256, 8, 50, '4:4:4', 50),
    '512_444': (32, 512, 512, 8, 50, '4:4:4', 50),
}


def sizes(n, w0, h0, step, seed):
    rng = np.random.default_rng(seed)
    out = set()
    while len(out) < n:
        out.add((int(w0 + step * rng.integers(-8, 9)), int(h0 + step * rng.integers(-8, 9))))
    return sorted(out)


def files(name):
    n, w0, h0, step, q, sub, iters = WORKLOADS[name]
    out = []
    for k, (w, h) in enumerate(sizes(n, w0, h0, step, sorted(WORKLOADS).index(name) + 1)):
        buf = io.BytesIO()
        Image.fromarray(synth.cartoon_image(w, h, k).astype(np.uint8), 'RGB').save(buf, 'JPEG', quality=q, subsampling=sub)
        out.append(buf.getvalue())
    return out, iters


def decode_arms(data, iters, reps):
    out, res = {}, {}
    for arm, on in (('grouped', True), ('chunks', False), ('grouped_again', True), ('chunks_again', False)):
        decode._group_chunks = on
        got = decode_jpeg(data, iterations=iters)         # warm-up (and the images compared)
        torch.cuda.synchronize()
        t = []
        for _ in range(reps):
            t0 = time.perf_counter()
            decode_jpeg(data, iterations=iters)
            torch.cuda.synchronize()
            t.append(time.perf_counter() - t0)
        out[arm] = {'ms_per_file_median': 1e3 * float(np.median(t)) / len(data), 'ms_per_file_min': 1e3 * min(t) / len(data)}
        res[arm.split('_')[0]] = got
    decode._group_chunks = True
    for a, b in zip(res['grouped'], res['chunks']):
        assert torch.equal(a, b), 'the arms differ'
    return out


def device_arms(data, iters, reps):
    """Per iteration: the group against the sum of the sessions solved one by one."""
    lib = abi.load_product()
    ss = []
    for d in data:
        img = decode.parse_jpeg(d)
        desc = decode._frame_desc(img, [0, 1, 2], 0.3, [0.001] * 3, iters)
        s = abi.Session(lib, desc, batch=False)
        for c, p in enumerate(img.planes):
            s._check(lib.j2p_session_upload(s.s, c, p.data.ctypes.data, p.quant.ctypes.data, None))
        ss.append(s)
    arr = (C.c_void_p * len(ss))(*[s.s.value for s in ss])

    def grouped():
        assert lib.j2p_session_iterate_group(arr, len(ss), 0, iters) == 0, lib.j2p_last_error().decode()
        for s in ss:
            s.sync()

    def one_by_one():
        for s in ss:
            s.iterate(0, iters)
            s.sync()

    out, res = {}, {}
    for arm, fn in (('group', grouped), ('sum_of_sessions', one_by_one), ('group_again', grouped), ('sum_of_sessions_again', one_by_one)):
        fn()
        t = []
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()
            t.append(time.perf_counter() - t0)
        out[arm] = {'us_per_iteration_median': 1e6 * float(np.median(t)) / iters}
        res[arm.split('_again')[0]] = [s.download()[0] for s in ss]
    for a, b in zip(res['group'], res['sum_of_sessions']):
        for x, y in zip(a, b):
            assert np.array_equal(x.view(np.int32), y.view(np.int32)), 'the device arms differ'
    for s in ss:
        s.close()
    return out


def run(name, reps):
    data, iters = files(name)
    px = [decode.parse_jpeg(d).w * decode.parse_jpeg(d).h for d in data]
    return {'files': len(data), 'iterations': iters, 'mean_pixels': float(np.mean(px)),
            'grouped_by_decode_jpeg': max(px) <= decode.GROUP_MAX_PIXELS,
            'decode': decode_arms(data, iters, reps), 'device': device_arms(data, iters, reps), 'identical': True}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--workloads', default=','.join(WORKLOADS))
    a = ap.parse_args()
    lib = abi.load_product()
    if lib.j2p_device_count() <= 0:
        raise SystemExit('mixed_bench: no CUDA device (there is no CPU fallback)')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({'gpu': gpu, **{n: run(n, a.reps) for n in a.workloads.split(',')}}))


if __name__ == '__main__':
    main()
