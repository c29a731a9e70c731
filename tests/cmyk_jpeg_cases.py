"""What the CMYK JPEG encoder tests share (tests/test_cmyk_jpeg_host.py, tests/test_gpu_cmyk_jpeg.py):
the CMYK corpus, Pillow's 'CMYK' file of an image, libjpeg's four-component progression, the restart
settings of a CMYK image and the child process that counts a CMYK call's kernel launches."""
import ctypes as C
import io
import json

import numpy as np

from tests import gray_jpeg_cases as G
from tests import jpegenc_cases as JC

MODES = G.MODES
QUALITIES = [1, 50, 75, 90, 100]
KINDS = ['cartoon', 'noise', 'flat128']
FACTORS = {'4:4:4': (1, 1), '4:2:2': (2, 1), '4:2:0': (2, 2)}
IDS = b'CMYK'                       # the SOF's and SOS's component identifiers (67, 77, 89, 75)
APP14 = b'\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00'      # transform 0: CMYK
HEADER = 341                        # bytes up to the end of the SOS of the quality tables' baseline file
# libjpeg's generic progression for four components: (Ss, Se, Ah, Al) of each scan, and its components
SCRIPT = ([(0, 0, 0, 1)] + [(1, 5, 0, 2)] * 4 + [(6, 63, 0, 2)] * 4 + [(1, 63, 2, 1)] * 4 + [(0, 0, 1, 0)] + [(1, 63, 1, 0)] * 4)
SCRIPT_COMPS = [IDS] + [IDS[c:c + 1] for c in range(4)] * 3 + [IDS] + [IDS[c:c + 1] for c in range(4)]
# the per-scan work-area bounds of a block, bits (jpegprog_core.h): the gray script's, per component
PROG_BITS = [27] + [160] * 4 + [1538] * 4 + [1101] * 4 + [1] + [1101] * 4


def cmyk(kind, h, w, seed):
    """(h, w, 4) uint8 pixels of one kind, four planes that differ: jpegenc_cases' RGB content as C,
    M, Y, and for K its green channel reversed along both axes (a flat image stays flat)."""
    rgb = JC.content(kind, h, w, seed)
    return np.ascontiguousarray(np.dstack([rgb, rgb[::-1, ::-1, 1]]))


def corpus(max_pixels=None):
    """name -> (h, w, 4) pixels: every JC.SIZES size in cartoon, noise and flat content (cartoon and
    noise only above JC.SMALL pixels), up to max_pixels."""
    out = {}
    for k, (h, w) in enumerate(JC.SIZES):
        if max_pixels and h * w > max_pixels:
            continue
        for kind in KINDS:
            if h * w > JC.SMALL and kind == 'flat128':
                continue
            out[f'{h}x{w}_{kind}'] = cmyk(kind, h, w, 900 + k)
    return out


def pillow_cmyk(x, quality=75, subsampling='4:2:0', **kw):
    """Pillow's file of the pixels x ((h, w, 4)) as a 'CMYK' image with the save options kw (quality
    None: Pillow's default).  Its output buffer must hold the whole file when the tables are
    optimized; its size changes no byte."""
    from PIL import Image, ImageFile
    a = np.ascontiguousarray(x)
    old = ImageFile.MAXBLOCK
    ImageFile.MAXBLOCK = max(old, 4 * a.size + 65536)
    if quality is not None:
        kw['quality'] = quality
    try:
        buf = io.BytesIO()
        Image.fromarray(a, 'CMYK').save(buf, 'JPEG', subsampling=subsampling, **kw)
        return buf.getvalue()
    finally:
        ImageFile.MAXBLOCK = old


def restart_settings(h, w, subsampling):
    """The restart keywords for a CMYK image: blocks around the MCU count, rows around the MCU rows,
    both, and the cap."""
    hs, vs = FACTORS[subsampling]
    mx, my = -(-w // (8 * hs)), -(-h // (8 * vs))
    m = mx * my
    out = [dict(restart_marker_blocks=b) for b in sorted({1, 2, 3, 7, m - 1, m, m + 1, 65535}) if b > 0]
    out += [dict(restart_marker_rows=r) for r in sorted({1, 2, my, my + 1})]
    out.append(dict(restart_marker_blocks=3, restart_marker_rows=2))
    out.append(dict(restart_marker_rows=65535))
    return out


def launch_counts(mode):
    """Child process of the launch-count test: prints, as JSON, per CMYK call its shapes, the
    profiler's count of each kernel of the mode, and the call's stats fields."""
    import torch

    from jpeg2png_b200 import batch_encode as B
    from jpeg2png_b200 import jpeg_encode as J
    p = J.params(75, '4:2:0', cmyk=True)
    codec = J.codec(p, mode == 'optimize', mode == 'progressive')
    names = G.NAMES[mode]
    out = []
    for shapes in ([(1, 1)], [(300, 200)] * 5 + [(1, 1), (2000, 3000)]):
        ts = [torch.zeros(h, w, 4, dtype=torch.uint8, device='cuda') for h, w in shapes]
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


def blocks(h, w, subsampling):
    """The blocks a CMYK image codes: its MCUs times hs vs + 3."""
    hs, vs = FACTORS[subsampling]
    return -(-w // (8 * hs)) * -(-h // (8 * vs)) * (hs * vs + 3)
