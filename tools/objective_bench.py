#!/usr/bin/env python
"""objective_bench.py — what recording the objective costs, three arms per workload.

plain:    decode_jpeg(files) from bytes to uint8 CHW tensors, objective not recorded
recorded: decode_jpeg(files, return_objective=True): the recording kernels, one history read per batch
cli_path: the command line's -c path for the same files: one single-frame logging session per file
          (j2p_session_set_logging), iterated one step at a time, j2p_session_objective after each

Host clock around each call with a device synchronise; the median of --reps runs, arms alternated.
The recorded images must equal the plain ones, or the tool fails.  Workloads: 64 x 1080p Q75 4:2:0 x
100 iterations, 64 x 256² Q10 4:2:0 x 50 iterations.  Prints one JSON line with the card's name and
power limit read in the same run.
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

WORKLOADS = {'1080p_q75': (64, 1920, 1080, 75, 100), '256_q10': (64, 256, 256, 10, 50)}   # count, w, h, quality, iterations


def files(name):
    n, w, h, q, _ = WORKLOADS[name]
    out = []
    for k in range(n):
        buf = io.BytesIO()
        Image.fromarray(synth.cartoon_image(w, h, k).astype(np.uint8), 'RGB').save(buf, 'JPEG', quality=q, subsampling='4:2:0')
        out.append(buf.getvalue())
    return out


def cli_path(lib, data, iters):
    """The command line's logging loop (cli/main.c) on the host-parsed files."""
    for d in data:
        p = decode.parse_jpeg(d)
        desc = decode._frame_desc(p, [0, 1, 2], 0.3, [0.001] * 3, iters)
        s = C.c_void_p()
        assert lib.j2p_session_create(C.byref(s), 0, C.byref(desc)) == 0, lib.j2p_last_error()
        try:
            assert lib.j2p_session_set_logging(s, 1) == 0
            for c in range(3):
                pl = p.planes[c]
                assert lib.j2p_session_upload(s, c, pl.data.ctypes.data, pl.quant.ctypes.data, None) == 0, lib.j2p_last_error()
            o = (C.c_double * 4)()
            for i in range(iters):
                assert lib.j2p_session_iterate(s, i, 1) == 0, lib.j2p_last_error()
                assert lib.j2p_session_objective(s, o) == 0, lib.j2p_last_error()
        finally:
            lib.j2p_session_destroy(s)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--workloads', default=','.join(WORKLOADS))
    a = ap.parse_args()
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    lib = abi.load_product()
    result = {'tool': 'objective_bench', 'gpu': smi.splitlines()[0] if smi else 'unknown'}
    for name in a.workloads.split(','):
        data = files(name)
        iters = WORKLOADS[name][4]
        plain_img = decode_jpeg(data, iterations=iters)                        # warm-up of every shape
        rec_img, logs = decode_jpeg(data, iterations=iters, return_objective=True)
        for x, y in zip(plain_img, rec_img):
            if not torch.equal(x, y):
                raise SystemExit('recorded images differ from the plain ones')
        t = {'plain': [], 'recorded': [], 'cli_path': []}
        for _ in range(a.reps):
            t['plain'].append(timed(lambda: decode_jpeg(data, iterations=iters))[0])
            t['recorded'].append(timed(lambda: decode_jpeg(data, iterations=iters, return_objective=True))[0])
        t['cli_path'].append(timed(lambda: cli_path(lib, data, iters))[0])       # slow: one run
        med = {k: float(np.median(v)) for k, v in t.items()}
        n = len(data)
        result[name] = {'files': n, 'iterations': iters,
                        'ms_per_file': {k: round(1e3 * v / n, 3) for k, v in med.items()},
                        'recorded_over_plain': round(med['recorded'] / med['plain'], 4),
                        'runs_s': {k: [round(x, 4) for x in v] for k, v in t.items()}}
    print(json.dumps(result))


if __name__ == '__main__':
    main()
