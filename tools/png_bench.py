"""encode_png against the command line's host PNG writer: prints one JSON line.

usage: python tools/png_bench.py [--device D] [--files N] [--reps R] [--calls C]

Workloads (JPEG files written with Pillow from synth.cartoon_image, as tools/decode_bench.py):
  (a) N x 1920x1080 Q75 4:2:0, 100 iterations, uint8;
  (b) the same files as uint16 (16-bit PNG);
  (c) N x 256x256 Q10 4:2:0, 50 iterations, uint8                   (N = 64 by default).
For each, the decoded tensors (decode_jpeg, CHW) are the input, and reported are:
  encoder       CUDA events on the stream around one whole j2p_png_encode call on all N images
                (the host's plan, the pageable plan upload, the four kernels with their launch
                gaps and the read-back of the offsets; mean of C calls) and GB/s of filtered bytes
                (the PNG scanlines with their filter bytes);
  kernels       device time of each of the four kernels per call (torch.profiler, C calls);
  encode_png    wall clock of encode_png(list of tensors) until the bytes are Python objects;
  host_writer   wall clock of: tensors to the host (HWC), then j2p_write_png_scanlines from
                libj2pcodecs.so into memory, one file per host thread, as many threads as the
                command line uses (the affinity mask capped by the cgroup CPU quota), each thread
                with an OpenMP team of one, as in the command line's file loop (where nested
                parallelism is off, so a file's pieces are deflated one after another);
  total bytes of both arms, and whether every file's pixels equal the tensor.
For (a) and (c), end to end from JPEG bytes to PNG bytes: decode_jpeg + encode_png against the
command line (`jpeg2png -q -f -o` into a temporary directory, all files in one invocation).
Also the kernel times of one 7680x4320 uint16 image (a synthetic gradient), where one image has
~3000 pieces.  Every wall-clock figure is the best of R after one warm-up.  Also the card's name and power limit
(read-only nvidia-smi query in the same run).  Writes only into a temporary directory.
"""
import argparse
import ctypes as C
import io
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from batch_bench import gpu_card  # noqa: E402
from decode_bench import jpeg_files  # noqa: E402
from jpeg2png_b200 import abi, decode_jpeg, encode_png  # noqa: E402
from jpeg2png_b200 import batch_encode as B  # noqa: E402
from jpeg2png_b200 import encode as E  # noqa: E402
from jpeg2png_b200.pngcheck import holds_pixels  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, 'jpeg2png_b200', 'cli', 'jpeg2png')
CODECS = os.path.join(ROOT, 'jpeg2png_b200', 'cli', 'libj2pcodecs.so')
KERNELS = ('k_png_filter', 'k_png_piece', 'k_png_assemble', 'k_png_copy')


def host_threads():
    """The command line's thread count: CPUs in the affinity mask, capped by the cgroup quota."""
    n = len(os.sched_getaffinity(0))
    try:
        quota, period = open('/sys/fs/cgroup/cpu.max').read().split()
        if quota != 'max':
            n = min(n, max(1, -(-int(quota) // int(period))))
    except (OSError, ValueError):
        pass
    return n


class HostWriter:
    """j2p_write_png_scanlines into memory (open_memstream), one file per call."""

    def __init__(self):
        self.codecs = C.CDLL(CODECS)
        self.codecs.j2p_write_png_scanlines.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_void_p]
        self.libc = C.CDLL(None)
        self.libc.open_memstream.restype = C.c_void_p
        self.libc.open_memstream.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
        self.libc.fclose.argtypes = [C.c_void_p]
        self.libc.free.argtypes = [C.c_void_p]
        self.gomp = C.CDLL('libgomp.so.1')         # the OpenMP runtime libj2pcodecs.so links

    def serial_team(self):
        """Thread-pool initializer: this thread's OpenMP regions run with one thread, as inside
        the command line's file loop."""
        self.gomp.omp_set_num_threads(1)

    def write(self, hwc):
        hwc = np.ascontiguousarray(hwc)
        h, w, _ = hwc.shape
        bits = 8 * hwc.itemsize
        raw = np.zeros((h, w * 3 * hwc.itemsize + 1), np.uint8)
        raw[:, 1:] = (hwc.astype('>u2') if bits == 16 else hwc).view(np.uint8).reshape(h, -1)
        buf, size = C.c_void_p(), C.c_size_t()
        f = self.libc.open_memstream(C.byref(buf), C.byref(size))
        rc = self.codecs.j2p_write_png_scanlines(f, w, h, bits, raw.ctypes.data)
        self.libc.fclose(f)
        out = C.string_at(buf, size.value)
        self.libc.free(buf)
        if rc != 0:
            raise RuntimeError('j2p_write_png_scanlines failed')
        return out


def best_of(fn, reps):
    fn()
    best, result = None, None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        result = fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return best, result


def encoder_call(codec, tensors):
    """One whole device encode call of codec's library on all tensors (CHW), with its work area
    allocated once; and the work area's size."""
    d = B.descs(codec, tensors, 'CHW')
    n, _ = codec.plan(d)
    work = torch.empty(n, dtype=torch.uint8, device=tensors[0].device)
    offs = (C.c_uint64 * (len(tensors) + 1))()
    stream = torch.cuda.current_stream()
    return lambda: codec.call('encode', d, work.data_ptr(), n, stream.cuda_stream, offs, None, 0, None), n


def encoder_ms(call, kernel_names, calls):
    """CUDA events around call() (host plan, plan upload, kernels, offset read-back), mean of
    `calls`; and the device time per call of each kernel in kernel_names from torch.profiler over
    `calls` more calls."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    call()
    times = []
    for _ in range(calls):
        e0.record()
        call()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            call()
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        name = next((k for k in kernel_names if k in ev.key), None)
        if name:
            us = getattr(ev, 'device_time_total', None) or getattr(ev, 'cuda_time_total', 0)
            kernels[name] = kernels.get(name, 0.0) + us / 1e3 / calls
    return {'ms_per_call': float(np.mean(times)), 'kernel_ms_per_call': kernels}


def png_encoder_ms(tensors, calls):
    """encoder_ms of one j2p_png_encode call on all images, and GB/s of filtered bytes."""
    out = encoder_ms(encoder_call(E.CODEC, tensors)[0], KERNELS, calls)
    filtered = sum(t.shape[1] * (1 + t.shape[2] * 3 * t.element_size()) for t in tensors)
    return {'ms_per_call': out['ms_per_call'], 'filtered_bytes': filtered, 'GB_per_s': filtered / out['ms_per_call'] / 1e6,
            'kernel_ms_per_call': out['kernel_ms_per_call']}


def run_workload(files, label, iterations, dtype, reps, calls, writer, threads, e2e):
    tensors = decode_jpeg(files, iterations=iterations, dtype=dtype)
    torch.cuda.synchronize()
    out = {'workload': label, 'files': len(files), 'dtype': str(dtype).replace('torch.', '')}
    out['encoder'] = png_encoder_ms(tensors, calls)

    t_gpu, pngs = best_of(lambda: encode_png(tensors), reps)

    def host_arm():
        hwc = [t.permute(1, 2, 0).cpu().numpy() for t in tensors]
        with ThreadPoolExecutor(threads, initializer=writer.serial_team) as pool:
            return list(pool.map(writer.write, hwc))
    t_host, host_pngs = best_of(host_arm, reps)
    same = True
    for t, a, b in zip(tensors, pngs, host_pngs):
        want = t.permute(1, 2, 0).cpu().numpy()
        same &= holds_pixels(a, want) and holds_pixels(b, want)
    out['encode_png'] = {'wall_ms': t_gpu * 1e3, 'ms_per_image': t_gpu / len(files) * 1e3, 'total_bytes': sum(map(len, pngs))}
    out['host_writer'] = {'wall_ms': t_host * 1e3, 'ms_per_image': t_host / len(files) * 1e3,
                          'total_bytes': sum(map(len, host_pngs)), 'threads': threads}
    out['encode_png_speedup'] = t_host / t_gpu
    out['size_ratio_vs_host_writer'] = out['encode_png']['total_bytes'] / out['host_writer']['total_bytes']
    if e2e:
        with tempfile.TemporaryDirectory() as tmp:
            paths, outs = [], []
            for k, data in enumerate(files):
                p = os.path.join(tmp, f'{k}.jpg')
                with open(p, 'wb') as f:
                    f.write(data)
                paths.append(p)
                outs += ['-o', os.path.join(tmp, f'{k}.png')]
            cmd = [CLI, '-q', '-f', '-i', str(iterations)] + outs + paths

            def cli():
                subprocess.run(cmd, check=True)
                return [open(os.path.join(tmp, f'{k}.png'), 'rb').read() for k in range(len(files))]
            t_cli, cli_pngs = best_of(cli, reps)
            t_new, new_pngs = best_of(lambda: encode_png(decode_jpeg(files, iterations=iterations, dtype=dtype)), reps)
            same_e2e = all(holds_pixels(a, want) and holds_pixels(b, want) for a, b, want in
                           zip(new_pngs, cli_pngs, (np.asarray(Image.open(io.BytesIO(x)).convert('RGB')) for x in cli_pngs)))
        out['end_to_end'] = {'decode_jpeg_encode_png_ms': t_new * 1e3, 'cli_ms': t_cli * 1e3, 'speedup': t_cli / t_new,
                             'identical_pixels_to_cli': bool(same_e2e)}
    out['identical_pixels'] = same
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--device', type=int, default=0)
    ap.add_argument('--files', type=int, default=64)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--calls', type=int, default=20)
    args = ap.parse_args()
    if abi.load_product().j2p_device_count() <= 0 or not torch.cuda.is_available():
        raise SystemExit('png_bench.py: no CUDA device')
    torch.cuda.set_device(args.device)
    writer, threads = HostWriter(), host_threads()
    big = jpeg_files(1920, 1080, 75, args.files)
    small = jpeg_files(256, 256, 10, args.files)
    n = args.files
    line = {'card': gpu_card(args.device),
            'timing': f'wall clock, one warm-up, best of {args.reps}; encoder: CUDA events, mean of {args.calls} calls',
            'workloads': [
                run_workload(big, f'{n} x 1920x1080 Q75 4:2:0, -i 100', 100, torch.uint8, args.reps, args.calls, writer, threads, True),
                run_workload(big, f'{n} x 1920x1080 Q75 4:2:0, -i 100', 100, torch.uint16, args.reps, args.calls, writer, threads, False),
                run_workload(small, f'{n} x 256x256 Q10 4:2:0, -i 50', 50, torch.uint8, args.reps, args.calls, writer, threads, True)]}
    yy = torch.arange(4320, device='cuda', dtype=torch.int32)[:, None]
    xx = torch.arange(7680, device='cuda', dtype=torch.int32)[None, :]
    img8k = (torch.stack([yy * 7 + xx * 3, yy * 13 + xx, xx * 5 + yy]) % 65536).to(torch.uint16)
    line['one_8k_uint16_image'] = png_encoder_ms([img8k], args.calls)
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
