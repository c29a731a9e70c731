"""encode_jpeg against Pillow on the host: prints one JSON line.

usage: python tools/jpegenc_bench.py [--device D] [--files N] [--reps R] [--calls C]

Workloads:
  (a) N x 1920x1080 Q75 4:2:0 files (tools/decode_bench.py's), decoded by decode_jpeg at 100
      iterations to uint8 CHW tensors, then encoded at q95 4:4:4, q90 4:2:0 and q75 4:2:0;
  (b) N x 256x256 Q10 4:2:0 files, decoded at 50 iterations, encoded at q75 4:2:0;
  (c) one 7680x4320 image (synth.cartoon_image), encoded at q90 4:2:0    (N = 64 by default).
For each, reported are:
  encoder       CUDA events around one whole j2p_jpegenc_encode call on all images (the host's
                plan, the plan upload, the clearing of the bit stream, the seven kernels and the
                read-back of the offsets), mean of C calls;
  kernels       device time of each kernel per call (torch.profiler, C more calls);
  encode_jpeg   wall clock of encode_jpeg(list of tensors) until the files are bytes;
  host          wall clock of: tensors made contiguous HWC on the device and copied into one
                shared-memory buffer on the host, then Pillow's JPEG writer, one file per task, in
                as many worker processes as the process may use CPUs (png_bench.host_threads).
                Processes, not threads: Pillow holds the GIL while it encodes, so a thread pool runs
                the files one after another.  The workers are started before the timing.  With,
                apart, the copies alone and Pillow on the first image alone in this process;
  total bytes against encode_png's files for the same tensors, and whether every file equals the
  host arm's byte for byte.
Under "optimize_workloads", the same figures for encode_jpeg(..., optimize=True) (libj2pjpegopt.so,
nine kernels) against Pillow with optimize=True, on (a) at q90 4:2:0 and q95 4:4:4, (b) at q75
4:2:0 and (c), with the total bytes over the default files' bytes for the same tensors.
Under "progressive_workloads", the same figures for encode_jpeg(..., progressive=True)
(libj2pjpegprog.so, ten kernels) against Pillow with progressive=True, on (a) at q90 4:2:0 and q95
4:4:4, (b) at q75 4:2:0, (c), and one flat 7680x4320 image at q90 4:2:0 (every AC scan one EOB-run
segment, walked by one thread of k_jp_runs).  --progressive-only measures only these.
Under "restart_workloads" (last in the full run), for each of the three encoders on (a) at q90 4:2:0: restart_marker_rows=1
(the encoder call against the same mode without restarts, and encode_jpeg against Pillow with the
same options), and restart_marker_blocks=1, one stream per MCU, the worst case (the encoder call
alone); and the flat 7680x4320 image, progressive, restart_marker_rows=1, against the same without
restarts.  --restart-only measures only these.
Wall-clock figures are the best of R after one warm-up.  Also the card's name and power limit
(read-only nvidia-smi query in the same run).  Writes nothing.
"""
import argparse
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
from png_bench import best_of, encoder_call, encoder_ms, host_threads  # noqa: E402
from jpeg2png_b200 import abi, decode_jpeg, encode_jpeg, encode_png, synth  # noqa: E402
from jpeg2png_b200 import jpeg_encode as J  # noqa: E402

KERNELS = ('k_je_blocks', 'k_je_sizes', 'k_je_scan', 'k_je_emit', 'k_je_ffcount', 'k_je_offsets', 'k_je_stuff')
KERNELS_OPT = ('k_jo_blocks', 'k_jo_hist', 'k_jo_tables', 'k_jo_sizes', 'k_jo_scan', 'k_jo_emit', 'k_jo_ffcount', 'k_jo_offsets',
               'k_jo_stuff')
KERNELS_PROG = ('k_jp_blocks', 'k_jp_runs', 'k_jp_hist', 'k_jp_tables', 'k_jp_sizes', 'k_jp_scan', 'k_jp_emit', 'k_jp_ffcount',
                'k_jp_offsets', 'k_jp_stuff')


def jpeg_encoder_ms(tensors, quality, subsampling, calls, optimize=False, progressive=False, **restart):
    """encoder_ms of one j2p_jpegenc_encode (or j2p_jpegopt_encode, j2p_jpegprog_encode) call on all
    images, and the size of its work area; restart: the restart keywords."""
    call, work_bytes = encoder_call(J.codec(J.params(quality, subsampling, **restart), optimize, progressive), tensors)
    out = encoder_ms(call, KERNELS_PROG if progressive else KERNELS_OPT if optimize else KERNELS, calls)
    return {'ms_per_call': out['ms_per_call'], 'work_bytes': work_bytes, 'kernel_ms_per_call': out['kernel_ms_per_call']}


def pillow(hwc, quality, subsampling, optimize=False, progressive=False, restart=(0, 0)):
    buf = io.BytesIO()
    if optimize or progressive:     # libjpeg cannot suspend in a multi-pass file's last pass: room for the whole file
        ImageFile.MAXBLOCK = max(ImageFile.MAXBLOCK, 4 * hwc.shape[0] * hwc.shape[1] * 3 + 65536)
    kw = dict(restart_marker_blocks=restart[0], restart_marker_rows=restart[1]) if any(restart) else {}
    Image.fromarray(hwc, 'RGB').save(buf, 'JPEG', quality=quality, subsampling=subsampling, optimize=optimize, progressive=progressive, **kw)
    return buf.getvalue()


_shm = {}


def _pillow_shared(name, size, offset, h, w, quality, subsampling, optimize=False, progressive=False, restart=(0, 0)):
    """In a worker process: Pillow on image (h, w, 3) at `offset` of the shared buffer `name`."""
    if name not in _shm:
        _shm[name] = shared_memory.SharedMemory(name=name)
    hwc = np.ndarray((h, w, 3), np.uint8, buffer=_shm[name].buf[:size], offset=offset)
    return pillow(hwc, quality, subsampling, optimize, progressive, restart)


def host_arm(tensors, quality, subsampling, reps, procs, optimize=False, progressive=False, restart=(0, 0)):
    """Best-of-`reps` seconds and files of the host arm (copies, then Pillow in `procs` worker
    processes), and apart the copies alone and Pillow on the first image in this process."""
    shapes = [(t.shape[1], t.shape[2]) for t in tensors]
    offs = np.cumsum([0] + [h * w * 3 for h, w in shapes]).tolist()
    shm = shared_memory.SharedMemory(create=True, size=offs[-1])
    try:
        buf = torch.from_numpy(np.ndarray((offs[-1],), np.uint8, buffer=shm.buf))
        views = [buf[offs[k]:offs[k + 1]].view(h, w, 3) for k, (h, w) in enumerate(shapes)]

        def copies():
            for v, t in zip(views, tensors):
                v.copy_(t.permute(1, 2, 0).contiguous())
        with ProcessPoolExecutor(procs, mp_context=mp.get_context('spawn')) as pool:
            list(pool.map(_pillow_shared, [shm.name] * procs, [offs[-1]] * procs, [0] * procs, [1] * procs, [1] * procs,
                          [quality] * procs, [subsampling] * procs))        # start and attach every worker

            def arm():
                copies()
                return list(pool.map(_pillow_shared, [shm.name] * len(shapes), [offs[-1]] * len(shapes), offs[:-1],
                                     [h for h, _ in shapes], [w for _, w in shapes], [quality] * len(shapes),
                                     [subsampling] * len(shapes), [optimize] * len(shapes), [progressive] * len(shapes),
                                     [restart] * len(shapes)))
            t_host, host_files = best_of(arm, reps)
        t_copy, _ = best_of(copies, reps)
        t_one, _ = best_of(lambda: pillow(views[0].numpy(), quality, subsampling, optimize, progressive, restart), reps)
        del buf, views
    finally:
        shm.close()
        shm.unlink()
    return t_host, host_files, t_copy, t_one


def run(tensors, label, quality, subsampling, reps, calls, threads, png_bytes):
    out = {'workload': label, 'images': len(tensors), 'quality': quality, 'subsampling': subsampling}
    out['encoder'] = jpeg_encoder_ms(tensors, quality, subsampling, calls)
    t_gpu, files = best_of(lambda: encode_jpeg(tensors, quality=quality, subsampling=subsampling), reps)

    t_host, host_files, t_copy, t_one = host_arm(tensors, quality, subsampling, reps, threads)
    total = sum(map(len, files))
    out['encode_jpeg'] = {'wall_ms': t_gpu * 1e3, 'ms_per_image': t_gpu / len(tensors) * 1e3, 'total_bytes': total}
    out['host_pillow'] = {'wall_ms': t_host * 1e3, 'ms_per_image': t_host / len(tensors) * 1e3, 'processes': threads,
                          'copies_alone_ms': t_copy * 1e3, 'one_image_one_thread_ms': t_one * 1e3}
    out['speedup_vs_host'] = t_host / t_gpu
    out['bytes_vs_encode_png'] = total / png_bytes
    out['identical_to_host'] = files == host_files
    return out


def run_optimized(tensors, label, quality, subsampling, reps, calls, threads):
    """run's figures for optimize=True, with the bytes over the default files' bytes."""
    out = {'workload': label, 'images': len(tensors), 'quality': quality, 'subsampling': subsampling, 'optimize': True}
    out['encoder'] = jpeg_encoder_ms(tensors, quality, subsampling, calls, optimize=True)
    out['encoder_default_ms_per_call'] = jpeg_encoder_ms(tensors, quality, subsampling, calls)['ms_per_call']
    t_gpu, files = best_of(lambda: encode_jpeg(tensors, quality=quality, subsampling=subsampling, optimize=True), reps)
    default_bytes = sum(map(len, encode_jpeg(tensors, quality=quality, subsampling=subsampling)))
    t_host, host_files, t_copy, t_one = host_arm(tensors, quality, subsampling, reps, threads, optimize=True)
    total = sum(map(len, files))
    out['encode_jpeg'] = {'wall_ms': t_gpu * 1e3, 'ms_per_image': t_gpu / len(tensors) * 1e3, 'total_bytes': total}
    out['host_pillow'] = {'wall_ms': t_host * 1e3, 'ms_per_image': t_host / len(tensors) * 1e3, 'processes': threads,
                          'copies_alone_ms': t_copy * 1e3, 'one_image_one_thread_ms': t_one * 1e3}
    out['speedup_vs_host'] = t_host / t_gpu
    out['bytes_vs_default'] = total / default_bytes
    out['identical_to_host'] = files == host_files
    return out


def run_progressive(tensors, label, quality, subsampling, reps, calls, threads):
    """run's figures for progressive=True, with the bytes over the default files' bytes."""
    out = {'workload': label, 'images': len(tensors), 'quality': quality, 'subsampling': subsampling, 'progressive': True}
    out['encoder'] = jpeg_encoder_ms(tensors, quality, subsampling, calls, progressive=True)
    out['encoder_default_ms_per_call'] = jpeg_encoder_ms(tensors, quality, subsampling, calls)['ms_per_call']
    t_gpu, files = best_of(lambda: encode_jpeg(tensors, quality=quality, subsampling=subsampling, progressive=True), reps)
    default_bytes = sum(map(len, encode_jpeg(tensors, quality=quality, subsampling=subsampling)))
    t_host, host_files, t_copy, t_one = host_arm(tensors, quality, subsampling, reps, threads, progressive=True)
    total = sum(map(len, files))
    out['encode_jpeg'] = {'wall_ms': t_gpu * 1e3, 'ms_per_image': t_gpu / len(tensors) * 1e3, 'total_bytes': total}
    out['host_pillow'] = {'wall_ms': t_host * 1e3, 'ms_per_image': t_host / len(tensors) * 1e3, 'processes': threads,
                          'copies_alone_ms': t_copy * 1e3, 'one_image_one_thread_ms': t_one * 1e3}
    out['speedup_vs_host'] = t_host / t_gpu
    out['bytes_vs_default'] = total / default_bytes
    out['identical_to_host'] = files == host_files
    return out


def run_restart(tensors, label, quality, subsampling, mode, restart, reps, calls, threads, host=True):
    """For one encoder (mode: {} or optimize= or progressive=) and the restart keywords: the encoder
    call with and without them and, with host, encode_jpeg against Pillow with the same options."""
    out = {'workload': label, 'images': len(tensors), 'quality': quality, 'subsampling': subsampling, **mode, **restart}
    out['encoder'] = jpeg_encoder_ms(tensors, quality, subsampling, calls, **mode, **restart)
    out['encoder_without_restarts'] = jpeg_encoder_ms(tensors, quality, subsampling, calls, **mode)
    if not host:
        return out
    t_gpu, files = best_of(lambda: encode_jpeg(tensors, quality=quality, subsampling=subsampling, **mode, **restart), reps)
    t_host, host_files, t_copy, t_one = host_arm(tensors, quality, subsampling, reps, threads, mode.get('optimize', False),
                                                 mode.get('progressive', False),
                                                 (restart.get('restart_marker_blocks', 0), restart.get('restart_marker_rows', 0)))
    out['encode_jpeg'] = {'wall_ms': t_gpu * 1e3, 'ms_per_image': t_gpu / len(tensors) * 1e3, 'total_bytes': sum(map(len, files))}
    out['host_pillow'] = {'wall_ms': t_host * 1e3, 'ms_per_image': t_host / len(tensors) * 1e3, 'processes': threads,
                          'copies_alone_ms': t_copy * 1e3, 'one_image_one_thread_ms': t_one * 1e3}
    out['speedup_vs_host'] = t_host / t_gpu
    out['identical_to_host'] = files == host_files
    return out


def restart_workloads(big, flat8k, n, args, threads):
    """The restart figures: each encoder on (a) at q90 4:2:0 with one interval per MCU row (against
    Pillow too) and per MCU, and the flat 8K image, progressive, one interval per MCU row."""
    out, label = [], f'{n} x 1920x1080 Q75 4:2:0, -i 100'
    for mode in ({}, {'optimize': True}, {'progressive': True}):
        out.append(run_restart(big, label, 90, '4:2:0', mode, {'restart_marker_rows': 1}, args.reps, args.calls, threads))
        out.append(run_restart(big, label, 90, '4:2:0', mode, {'restart_marker_blocks': 1}, args.reps, args.calls, threads, host=False))
    out.append(run_restart([flat8k], '1 x 7680x4320 flat', 90, '4:2:0', {'progressive': True}, {'restart_marker_rows': 1}, args.reps, args.calls,
                           threads, host=False))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--device', type=int, default=0)
    ap.add_argument('--files', type=int, default=64)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--calls', type=int, default=20)
    ap.add_argument('--progressive-only', action='store_true')
    ap.add_argument('--restart-only', action='store_true')
    args = ap.parse_args()
    if abi.load_product().j2p_device_count() <= 0 or not torch.cuda.is_available():
        raise SystemExit('jpegenc_bench.py: no CUDA device')
    torch.cuda.set_device(args.device)
    threads, n = host_threads(), args.files
    line = {'card': gpu_card(args.device),
            'timing': f'wall clock, one warm-up, best of {args.reps}; encoder: CUDA events, mean of {args.calls} calls',
            'workloads': []}
    big = decode_jpeg(jpeg_files(1920, 1080, 75, n), iterations=100, dtype=torch.uint8)
    small = decode_jpeg(jpeg_files(256, 256, 10, n), iterations=50, dtype=torch.uint8)
    img8k = torch.from_numpy(synth.cartoon_image(7680, 4320, 9).round().astype(np.uint8).transpose(2, 0, 1).copy()).cuda()
    flat8k = torch.full((3, 4320, 7680), 77, dtype=torch.uint8, device='cuda')
    torch.cuda.synchronize()
    if args.restart_only:
        line['restart_workloads'] = restart_workloads(big, flat8k, n, args, threads)
        print(json.dumps(line), flush=True)
        return
    line['progressive_workloads'] = []
    for tensors, label, cases in ((big, f'{n} x 1920x1080 Q75 4:2:0, -i 100', ((90, '4:2:0'), (95, '4:4:4'))),
                                  (small, f'{n} x 256x256 Q10 4:2:0, -i 50', ((75, '4:2:0'),)),
                                  ([img8k], '1 x 7680x4320 cartoon', ((90, '4:2:0'),)),
                                  ([flat8k], '1 x 7680x4320 flat', ((90, '4:2:0'),))):
        for q, s in cases:
            line['progressive_workloads'].append(run_progressive(tensors, label, q, s, args.reps, args.calls, threads))
    if args.progressive_only:
        print(json.dumps(line), flush=True)
        return
    for tensors, label, cases in ((big, f'{n} x 1920x1080 Q75 4:2:0, -i 100', ((95, '4:4:4'), (90, '4:2:0'), (75, '4:2:0'))),
                                  (small, f'{n} x 256x256 Q10 4:2:0, -i 50', ((75, '4:2:0'),)),
                                  ([img8k], '1 x 7680x4320 cartoon', ((90, '4:2:0'),))):
        png_bytes = sum(map(len, encode_png(tensors)))
        for q, s in cases:
            line['workloads'].append(run(tensors, label, q, s, args.reps, args.calls, threads, png_bytes))
    line['optimize_workloads'] = []
    for tensors, label, cases in ((big, f'{n} x 1920x1080 Q75 4:2:0, -i 100', ((90, '4:2:0'), (95, '4:4:4'))),
                                  (small, f'{n} x 256x256 Q10 4:2:0, -i 50', ((75, '4:2:0'),)),
                                  ([img8k], '1 x 7680x4320 cartoon', ((90, '4:2:0'),))):
        for q, s in cases:
            line['optimize_workloads'].append(run_optimized(tensors, label, q, s, args.reps, args.calls, threads))
    line['restart_workloads'] = restart_workloads(big, flat8k, n, args, threads)
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
