"""decode_jpeg on four-component (CMYK) JPEGs against the same pixels as RGB: prints one JSON line.

usage: python tools/cmyk_bench.py [--device D] [--files N] [--reps R] [--ab LIB]

The files: N x 1920x1080 Q75 CMYK JPEGs from Pillow (N = 64 by default; four distinct seeded images
repeated), and the same pixels (Pillow's convert('RGB') of the CMYK image) saved as RGB 4:4:4 Q75.
At 10 and 50 iterations, wall clock of one decode_jpeg call on the list until the device is idle,
best of R after a warm-up, ms per image:
  cmyk_unchanged   mode='UNCHANGED' (four uint8 channels), CMYK files;
  cmyk_rgb         mode='RGB' uint8, CMYK files (Pillow's CMYK -> RGB on the device);
  rgb444_device    the RGB files, device entropy decoder (the default);
  rgb444_host      the RGB files through the host reader (the front end every CMYK file takes).
single_table_routing: the same files (no restart interval, and one per MCU row) with every file on
the device decoder and with every file on the host reader, 10 iterations (four_on_device's rule).
export_us: the export launches' device time per image (torch.profiler, k_scanlines), CMYK in both
modes and the RGB files.  With --ab LIB (another build's libjpeg2png_b200.so), also the colour
export's own device time with LIB's k_scanlines and with the tree's, on one 64-frame 1080p joint
session each, alternating, CUDA events around 20 exports.  The card's name, power limit and SM clock
are read (read-only nvidia-smi query) in the same run.  Writes nothing.
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
from jpeg2png_b200 import abi, decode_jpeg, synth  # noqa: E402
from jpeg2png_b200 import decode as D  # noqa: E402


def card(device):
    try:
        out = subprocess.run(['nvidia-smi', f'--id={device}', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                              '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=20).stdout.strip().split(', ')
        return {'name': out[0], 'power_limit_w': float(out[1]), 'sm_clock_mhz': int(out[2]), 'sm_clock_max_mhz': int(out[3])}
    except Exception:
        return {'name': None}


def files(n):
    cmyk, rgb = [], []
    for k in range(4):
        im = synth.cartoon_image(1920, 1080, 700 + k).astype(np.uint8)
        kk = ((np.add.outer(np.arange(1080), np.arange(1920)) + 40 * k) % 256).astype(np.uint8)
        c = Image.fromarray(np.dstack([im, kk]), 'CMYK')
        b = io.BytesIO()
        c.save(b, 'JPEG', quality=75)
        cmyk.append(b.getvalue())
        b = io.BytesIO()
        c.convert('RGB').save(b, 'JPEG', quality=75, subsampling='4:4:4')
        rgb.append(b.getvalue())
    return [cmyk[i % 4] for i in range(n)], [rgb[i % 4] for i in range(n)]


def _pillow_cmyk_rst(k):
    im = synth.cartoon_image(1920, 1080, 700 + k).astype(np.uint8)
    kk = ((np.add.outer(np.arange(1080), np.arange(1920)) + 40 * k) % 256).astype(np.uint8)
    b = io.BytesIO()
    Image.fromarray(np.dstack([im, kk]), 'CMYK').save(b, 'JPEG', quality=75, restart_marker_rows=1)
    return b.getvalue()


def best(fn, reps, n):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3 / n)
    return round(min(times), 3)


def export_us(fn, n):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if 'k_scanlines' in e.key)
    return round(us / n, 2)


def export_ab(path, device, reps=5):
    """The colour export's device time (us per 1080p frame), LIB's and the tree's k_scanlines."""
    tree, parent = abi.load_product(), C.CDLL(path, mode=C.RTLD_LOCAL)
    for name in ('j2p_last_error', 'j2p_session_create_batch', 'j2p_session_width', 'j2p_session_height', 'j2p_session_upload',
                 'j2p_session_iterate', 'j2p_session_destroy', 'j2p_session_export'):
        getattr(parent, name).restype, getattr(parent, name).argtypes = getattr(tree, name).restype, getattr(tree, name).argtypes
    libs = {'parent': parent, 'tree': tree}
    img = synth.synth_coefs(1920, 1080, 75, '4:2:0', 11)
    n = 64
    out = torch.empty((n, 3, 1080, 1920), dtype=torch.uint8, device='cuda')
    o = abi.ImageOut(1920, 1080, 8, abi.LAYOUT_CHW, 3 * 1080 * 1920)
    sessions = {}
    for name, lib in libs.items():
        s = abi.Session(lib, abi.frame_desc(img, [0, 1, 2], 0.3, [0.001] * 3, 1), n, device)
        s.upload([img] * n, [0, 1, 2])
        s.iterate(0, 1)
        sessions[name] = s
    res = {k: [] for k in libs}
    st = torch.cuda.current_stream().cuda_stream or 1
    for _ in range(reps):
        for name, lib in libs.items():
            s = sessions[name]
            lib.j2p_session_export(s.s, 0, n, C.byref(o), C.c_void_p(out.data_ptr()), C.c_void_p(st))
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(20):
                lib.j2p_session_export(s.s, 0, n, C.byref(o), C.c_void_p(out.data_ptr()), C.c_void_p(st))
            b.record()
            b.synchronize()
            res[name].append(a.elapsed_time(b) * 1e3 / 20 / n)
    same = []
    for name, lib in libs.items():
        lib.j2p_session_export(sessions[name].s, 0, n, C.byref(o), C.c_void_p(out.data_ptr()), C.c_void_p(st))
        torch.cuda.synchronize()
        same.append(out.clone())
    for s in sessions.values():
        s.close()
    return {k: round(min(v), 3) for k, v in res.items()} | {'identical': bool(torch.equal(same[0], same[1]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--device', type=int, default=0)
    ap.add_argument('--files', type=int, default=64)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--ab')
    a = ap.parse_args()
    torch.cuda.set_device(a.device)
    cmyk, rgb = files(a.files)
    n = a.files
    res = {'card': card(a.device), 'files': n, 'size': '1920x1080', 'quality': 75}
    for it in (10, 50):
        r = {}
        r['cmyk_unchanged'] = best(lambda: decode_jpeg(cmyk, mode='UNCHANGED', iterations=it), a.reps, n)
        r['cmyk_rgb'] = best(lambda: decode_jpeg(cmyk, iterations=it), a.reps, n)
        r['rgb444_device'] = best(lambda: decode_jpeg(rgb, iterations=it), a.reps, n)
        old = D._host_front_end
        D._host_front_end = True
        try:
            r['rgb444_host'] = best(lambda: decode_jpeg(rgb, iterations=it), a.reps, n)
        finally:
            D._host_front_end = old
        res[f'ms_per_image_{it}it'] = r
    # the routing rule of single-table four-component files (four_on_device): every such file on the
    # device decoder against every one on the host reader, without and with one restart interval per
    # MCU row, 10 iterations
    rst = [files_rst[i % 4] for i in range(n)] if (files_rst := [
        _pillow_cmyk_rst(k) for k in range(4)]) else []
    route = {}
    for name, fs in (('no_restart', cmyk), ('restart_rows1', rst)):
        for side, limit in (('device', 1 << 30), ('host', -1)):
            old = D.FOUR_SYNC_SUBSEQ
            D.FOUR_SYNC_SUBSEQ = limit
            try:
                route[f'{name}_{side}'] = best(lambda: decode_jpeg(fs, mode='UNCHANGED', iterations=10), a.reps, n)
            finally:
                D.FOUR_SYNC_SUBSEQ = old
    res['single_table_routing_ms_per_image_10it'] = route
    res['export_us_per_image'] = {
        'cmyk_unchanged': export_us(lambda: decode_jpeg(cmyk, mode='UNCHANGED', iterations=1), n),
        'cmyk_rgb': export_us(lambda: decode_jpeg(cmyk, iterations=1), n),
        'rgb444': export_us(lambda: decode_jpeg(rgb, iterations=1), n),
    }
    if a.ab:
        res['colour_export_us_per_frame'] = export_ab(a.ab, a.device)
    res['card_after'] = card(a.device)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
