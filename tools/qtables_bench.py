"""Cost of given quantisation tables in the JPEG encoders, on 64 1080p images (cartoon content, 4:2:0)
in one call, baseline / optimize / progressive, in three variants:

  quality90    quality=90 (the IJG tables: one set built from the quality);
  qtables_q90  qtables= the IJG tables of q90 (one given set; the same bytes);
  sets64       64 distinct given sets, one per image;

each alternated, round by round, with the same call of a reference build of the three libraries
(--parent DIR holding libj2pjpegenc.so, libj2pjpegopt.so and libj2pjpegprog.so of the commit
before given tables, driven through its own struct layout).  A call is the library's plan and encode
on a preallocated work area, ending when the offsets are on the host.  Also the end-to-end re-encode
of 64 files: decode_jpeg(mode='UNCHANGED') then encode_jpeg(**keep_settings(files)), against
Pillow's quality='keep' (decode and save) in 16 processes.  Prints one JSON line, with the card's
name and power limit read in the same run; --out also writes it to a file.

    python tools/qtables_bench.py --parent DIR --out results/qtables_bench.json
"""
import argparse
import ctypes as C
import io
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
from multiprocessing import Pool

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from jpeg2png_b200 import batch_encode as B  # noqa: E402
from jpeg2png_b200 import decode_jpeg, encode_jpeg, keep_settings  # noqa: E402
from jpeg2png_b200 import jpeg_encode as J  # noqa: E402
from jpeg2png_b200 import synth  # noqa: E402

MODES = {'baseline': ('jpegenc', False, False), 'optimize': ('jpegopt', True, False), 'progressive': ('jpegprog', False, True)}


class ParentImage(C.Structure):
    _fields_ = [('data', C.c_void_p), ('width', C.c_uint32), ('height', C.c_uint32),
                ('row_stride', C.c_int64), ('col_stride', C.c_int64), ('chan_stride', C.c_int64)]


class ParentParams(C.Structure):
    _fields_ = [('quality', C.c_int), ('sampling', C.c_int), ('restart_marker_blocks', C.c_int), ('restart_marker_rows', C.c_int),
                ('components', C.c_int)]


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown'


class Call:
    """One library's plan + encode of a fixed list, on a preallocated work area."""

    def __init__(self, lib, name, descs, params):
        self.lib, self.name, self.descs, self.params = lib, name, descs, params
        n, o = C.c_size_t(), C.c_size_t()
        self._check(getattr(lib, f'j2p_{name}_plan')(descs, len(descs), C.byref(params), C.byref(n), C.byref(o)))
        self.work = torch.empty(n.value, dtype=torch.uint8, device='cuda')
        self.base = o.value
        self.offs = (C.c_uint64 * (len(descs) + 1))()

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(getattr(self.lib, f'j2p_{self.name}_last_error')().decode())

    def __call__(self):
        n, o = C.c_size_t(), C.c_size_t()
        self._check(getattr(self.lib, f'j2p_{self.name}_plan')(self.descs, len(self.descs), C.byref(self.params), C.byref(n), C.byref(o)))
        st = J.Stats()
        self._check(getattr(self.lib, f'j2p_{self.name}_encode')(self.descs, len(self.descs), C.byref(self.params), C.c_void_p(self.work.data_ptr()),
                                                              C.c_size_t(n.value), C.c_void_p(torch.cuda.current_stream().cuda_stream),
                                                              self.offs, None, C.c_size_t(0), C.byref(st)))
        return st.launches

    def files(self):
        host = self.work[self.base:self.base + self.offs[len(self.descs)]].cpu().numpy()
        return [host[self.offs[i]:self.offs[i + 1]].tobytes() for i in range(len(self.descs))]


def new_call(ts, mode, sets):
    name, opt, prog = MODES[mode]
    codec = J.codec(J.params(90, '4:2:0'), opt, prog, sets)
    d = B.placed(codec, B.descs(codec, ts, 'CHW'))
    return Call(codec.load(), name, d, codec.params[0]._obj)


def parent_call(ts, mode, parent):
    name, _, _ = MODES[mode]
    lib = C.CDLL(os.path.join(parent, f'libj2p{name}.so'))
    d = (ParentImage * len(ts))()
    for x, t in zip(d, ts):
        x.data, x.width, x.height = t.data_ptr(), t.shape[2], t.shape[1]
        x.row_stride, x.col_stride, x.chan_stride = t.stride(1), t.stride(2), t.stride(0)
    getattr(lib, f'j2p_{name}_last_error').restype = C.c_char_p
    return Call(lib, name, d, ParentParams(90, 2, 0, 0, 3))


def timed(call):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    call()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def _pillow_keep(path):
    from PIL import Image
    buf = io.BytesIO()
    Image.open(path).save(buf, 'JPEG', quality='keep')
    return len(buf.getvalue())


def end_to_end(ts, rounds):
    """decode_jpeg + encode_jpeg(**keep_settings) of 64 files against Pillow's 'keep' in 16 processes."""
    from PIL import Image
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for k, t in enumerate(ts):
            p = os.path.join(tmp, f'{k}.jpg')
            Image.fromarray(t.permute(1, 2, 0).cpu().numpy()).save(p, 'JPEG', quality=90)
            paths.append(p)

        def ours():
            return encode_jpeg(decode_jpeg(paths, mode='UNCHANGED'), **keep_settings(paths))
        ours()
        dev = []
        for _ in range(rounds):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ours()
            dev.append(time.perf_counter() - t0)
        with Pool(16) as pool:
            pool.map(_pillow_keep, paths)
            cpu = []
            for _ in range(rounds):
                t0 = time.perf_counter()
                pool.map(_pillow_keep, paths)
                cpu.append(time.perf_counter() - t0)
    return {'decode_jpeg_plus_encode_keep_ms': round(1e3 * statistics.median(dev), 1),
            'pillow_keep_16proc_ms': round(1e3 * statistics.median(cpu), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=64)
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--parent', default=None, help='directory of the reference build of the three encoder libraries')
    ap.add_argument('--out', default=None)
    ap.add_argument('--no-e2e', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('qtables_bench needs a CUDA device')
    ts = [torch.from_numpy(synth.cartoon_image(1920, 1080, k).round().astype(np.uint8)).permute(2, 0, 1).contiguous().cuda()
          for k in range(a.images)]
    q90 = J.scaled_tables(J.IJG_TABLES, 90)
    sets = [J.scaled_tables(np.random.default_rng(k).integers(1, 60 + k, (2, 64)).tolist(), None) for k in range(a.images)]
    out = {'bench': 'qtables', 'card': card(), 'images': f'{a.images} x 1920x1080 4:2:0', 'rounds': a.rounds, 'modes': {}}
    for mode in MODES:
        calls = {'quality90': new_call(ts, mode, None), 'qtables_q90': new_call(ts, mode, [q90] * a.images),
                 'sets64': new_call(ts, mode, sets)}
        if a.parent:
            calls['parent_quality90'] = parent_call(ts, mode, a.parent)
        launches = {k: c() for k, c in calls.items()}
        files = {k: c.files() for k, c in calls.items()}
        assert files['qtables_q90'] == files['quality90'], mode
        if a.parent:
            assert files['parent_quality90'] == files['quality90'], mode
        times = {k: [] for k in calls}
        for r in range(a.rounds):
            order = list(calls) if r % 2 == 0 else list(calls)[::-1]
            for k in order:
                times[k].append(timed(calls[k]))
        res = {k: {'median_ms': round(1e3 * statistics.median(v), 2), 'min_ms': round(1e3 * min(v), 2), 'max_ms': round(1e3 * max(v), 2),
                   'launches': launches[k]} for k, v in times.items()}
        out['modes'][mode] = res
        del calls
        torch.cuda.empty_cache()
    if not a.no_e2e:
        out['end_to_end'] = end_to_end(ts, max(2, a.rounds // 3))
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
