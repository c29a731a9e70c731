"""What the gray JPEG encoder tests share (tests/test_gray_jpeg_host.py, tests/test_gpu_gray_jpeg.py):
the gray corpus, Pillow's 'L' file of a gray image, the scans and headers of a file, and the child
process that counts a gray call's kernel launches with the profiler."""
import ctypes as C
import io
import json

import numpy as np

from tests import jpegenc_cases as JC

MODES = {'baseline': {}, 'optimize': {'optimize': True}, 'progressive': {'progressive': True}}
QUALITIES = [1, 50, 75, 90, 100]
KINDS = ['cartoon', 'noise', 'flat128']
SOF_SAMPLING = {'4:4:4': 0x11, '4:2:2': 0x21, '4:2:0': 0x22}
# libjpeg's progression for one component: (Ss, Se, Ah, Al) of each scan
GRAY_SCRIPT = [(0, 0, 0, 1), (1, 5, 0, 2), (6, 63, 0, 2), (1, 63, 2, 1), (0, 0, 1, 0), (1, 63, 1, 0)]
NAMES = {'baseline': ('k_je_blocks', 'k_je_sizes', 'k_je_scan', 'k_je_emit', 'k_je_ffcount', 'k_je_offsets', 'k_je_stuff'),
         'optimize': ('k_jo_blocks', 'k_jo_hist', 'k_jo_tables', 'k_jo_sizes', 'k_jo_scan', 'k_jo_emit', 'k_jo_ffcount', 'k_jo_offsets',
                      'k_jo_stuff'),
         'progressive': ('k_jp_blocks', 'k_jp_runs', 'k_jp_hist', 'k_jp_tables', 'k_jp_sizes', 'k_jp_scan', 'k_jp_emit', 'k_jp_ffcount',
                         'k_jp_offsets', 'k_jp_stuff')}


def gray(kind, h, w, seed):
    """(h, w, 1) uint8 pixels of one kind: the green channel of jpegenc_cases' content."""
    return np.ascontiguousarray(JC.content(kind, h, w, seed)[..., 1:2])


def corpus(max_pixels=None):
    """name -> (h, w, 1) pixels: every JC.SIZES size in cartoon, noise and flat content (cartoon and
    noise only above JC.SMALL pixels), up to max_pixels."""
    out = {}
    for k, (h, w) in enumerate(JC.SIZES):
        if max_pixels and h * w > max_pixels:
            continue
        for kind in KINDS:
            if h * w > JC.SMALL and kind == 'flat128':
                continue
            out[f'{h}x{w}_{kind}'] = gray(kind, h, w, 700 + k)
    return out


def pillow_l(x, quality=75, subsampling='4:2:0', **kw):
    """Pillow's file of the gray pixels x ((h, w, 1) or (h, w)) as an 'L' image with the save options
    kw.  Its output buffer must hold the whole file when the tables are optimized; its size changes
    no byte."""
    from PIL import Image, ImageFile
    a = np.ascontiguousarray(x.reshape(x.shape[0], x.shape[1]))
    old = ImageFile.MAXBLOCK
    ImageFile.MAXBLOCK = max(old, 4 * a.size + 65536)
    try:
        buf = io.BytesIO()
        Image.fromarray(a, 'L').save(buf, 'JPEG', quality=quality, subsampling=subsampling, **kw)
        return buf.getvalue()
    finally:
        ImageFile.MAXBLOCK = old


def restart_settings(h, w):
    """The restart keywords for a gray image (its MCU is one block): blocks around the block count,
    rows around the block rows, both, and the cap."""
    bx, by = -(-w // 8), -(-h // 8)
    m = bx * by
    out = [dict(restart_marker_blocks=b) for b in sorted({1, 2, 3, 7, m - 1, m, m + 1, 65535}) if b > 0]
    out += [dict(restart_marker_rows=r) for r in sorted({1, 2, 5, by, by + 1})]
    out.append(dict(restart_marker_blocks=3, restart_marker_rows=2))
    out.append(dict(restart_marker_rows=65535))
    return out


def segments(data):
    """[(marker, offset, payload)] of the marker segments before and between a file's scans (RSTm,
    SOI and EOI have an empty payload; entropy-coded data is skipped)."""
    out, i = [], 2
    while i < len(data) - 1:
        if data[i] != 0xFF or data[i + 1] in (0x00, 0xFF):
            i += 1
            continue
        m = data[i + 1]
        if 0xD0 <= m <= 0xD9:
            out.append((m, i, b''))
            i += 2
            continue
        n = data[i + 2] << 8 | data[i + 3]
        out.append((m, i, data[i + 4:i + 2 + n]))
        i += 2 + n
    return out


def launch_counts(mode):
    """Child process of the launch-count test: prints, as JSON, per gray call its shapes, the
    profiler's count of each kernel of the mode, and the call's stats fields."""
    import torch

    from jpeg2png_b200 import batch_encode as B
    from jpeg2png_b200 import jpeg_encode as J
    p = J.params(75, '4:2:0', components=1)
    codec = J.codec(p, mode == 'optimize', mode == 'progressive')
    names = NAMES[mode]
    out = []
    for shapes in ([(1, 1)], [(300, 200)] * 5 + [(1, 1), (2000, 3000)]):
        ts = [torch.zeros(h, w, 1, dtype=torch.uint8, device='cuda') for h, w in shapes]
        d = B.descs(codec, ts, 'HWC')
        n, _ = codec.plan(d)
        work = torch.empty(n, dtype=torch.uint8, device='cuda')
        offs = (C.c_uint64 * (len(ts) + 1))()
        st = J.Stats()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            codec.call('encode', d, work.data_ptr(), n, torch.cuda.current_stream().cuda_stream, offs, None, 0, C.byref(st))
            torch.cuda.synchronize()
        ran = {k: 0 for k in names}
        for ev in prof.key_averages():
            k = next((k for k in names if k in ev.key), None)
            if k:
                ran[k] += ev.count
        out.append((shapes, ran, {'launches': st.launches, 'blocks': st.blocks}))
    print(json.dumps(out))
