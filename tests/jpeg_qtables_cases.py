"""Given quantisation tables (encode_jpeg's qtables, keep_settings): the cases shared by the CPU
tests (host driver against Pillow) and the GPU tests (device against host driver): tables drawn at
random and with edge entries, every form Pillow takes, the modes, and a corpus of source files for
quality='keep'."""
import io

import numpy as np

from tests import jpeg_synth as S
from tests import jpegenc_cases as JC

SIZES = [(1, 1), (9, 8), (17, 13), (97, 61), (200, 300)]      # (h, w): edges, dummies, several MCUs
MODES = {'default': {}, 'optimize': {'optimize': True}, 'progressive': {'progressive': True},
         'restart': {'restart_marker_rows': 1}, 'restart_progressive': {'progressive': True, 'restart_marker_blocks': 7}}
EDGE = [0, 1, 255, 256, 8191]


def tables(n, seed, hi=300, edge=False):
    """n tables of 64 entries in 0..hi - 1 (natural order); with edge, each also holds 0, 1, 255,
    256 and 8191 somewhere."""
    rng = np.random.default_rng(seed)
    out = [rng.integers(0, hi, 64).tolist() for _ in range(n)]
    if edge:
        for k, t in enumerate(out):
            for j, v in enumerate(EDGE):
                t[(7 * j + 11 * k) % 64] = v
    return out


def forms(ts):
    """ts in each of Pillow's forms: list, tuple, dict, and a gapped dict that keeps only table 0
    ({0: a, 2: b} is [a])."""
    return {'list': list(ts), 'tuple': tuple(ts), 'dict': dict(enumerate(ts)), 'gapped': {0: ts[0], 2: ts[-1]}}


def rgb(h, w, seed):
    """Pixels of one kind: noise for small even sizes, else cartoon (a large noise image at quality 100
    outgrows the buffer Pillow gives an optimized or progressive file, and Pillow fails)."""
    return JC.content('noise' if (h * w) % 2 == 0 and h * w < 10000 else 'cartoon', h, w, seed)


def pillow(x, **kw):
    """Pillow's file for the (h, w, 3) RGB or (h, w) / (h, w, 1) gray uint8 pixels; quality=None is
    Pillow's default (no quality keyword)."""
    from PIL import Image
    kw = {k: v for k, v in kw.items() if not (k == 'quality' and v is None)}
    x = np.ascontiguousarray(x)
    im = Image.fromarray(x[..., 0] if x.ndim == 3 and x.shape[2] == 1 else x, 'L' if x.ndim == 2 or x.shape[2] == 1 else 'RGB')
    buf = io.BytesIO()
    im.save(buf, 'JPEG', **kw)
    return buf.getvalue()


def markers(data):
    """[(marker, segment bytes after the length)] of the headers up to the first SOS."""
    out, i = [], 2
    while True:
        m = data[i + 1]
        n = data[i + 2] << 8 | data[i + 3]
        out.append((m, data[i + 4:i + 2 + n]))
        if m == 0xDA:
            return out
        i += 2 + n


def ijg(q):
    """Pillow's tables for quality q, as Image.quantization reads them from its file."""
    from PIL import Image
    return [list(t) for t in Image.open(io.BytesIO(pillow(np.zeros((8, 8, 3), np.uint8), quality=q))).quantization.values()]


def keep_sources():
    """name -> JPEG bytes whose settings quality='keep' re-uses: IJG files at several qualities in
    all three samplings, files with one and with three tables, a 16-bit table, gray files, a
    progressive file and a 4:4:0 file (which Pillow's get_sampling maps to libjpeg's default)."""
    out = {}
    for k, (h, w) in enumerate([(62, 96), (30, 46)]):      # sizes whose chroma grids the reader's geometry check accepts
        x = rgb(h, w, 50 + k)
        for q in (30, 75, 95):
            for s in JC.SAMPLINGS:
                out[f'ijg_q{q}_{s}_{h}x{w}'] = pillow(x, quality=q, subsampling=s)
        out[f'one_table_{h}x{w}'] = pillow(x, qtables=tables(1, 60 + k, 120))
        out[f'sixteen_bit_{h}x{w}'] = pillow(x, qtables=[[v + 200 for v in t] for t in tables(2, 70 + k, 200)], subsampling='4:2:2')
        out[f'gray_q80_{h}x{w}'] = pillow(x[..., 1], quality=80)
        out[f'gray_two_tables_{h}x{w}'] = pillow(x[..., 2], qtables=tables(2, 80 + k, 90), subsampling='4:2:0')
        out[f'progressive_{h}x{w}'] = pillow(x, quality=85, progressive=True, subsampling='4:4:4')
    for name, sampling in (('three_tables_420', [(2, 2), (1, 1), (1, 1)]), ('three_tables_444', [(1, 1)] * 3),
                           ('sampling_440', [(1, 2), (1, 1), (1, 1)])):
        planes, quants = S.random_planes(40, 24, sampling, seed=len(out))
        quants[2] = np.random.default_rng(len(out)).integers(1, 100, 64)
        out[name] = S.encode_baseline(40, 24, sampling, planes, quants)
    return out


def pillow_keep(src, pixels=None):
    """Pillow's quality='keep' re-save of the JPEG bytes src: of its own decode, or of the given
    (h, w, 3) or (h, w, 1) pixels with src's tables and sampling (what 'keep' takes from the file)."""
    from PIL import Image, JpegImagePlugin
    im = Image.open(io.BytesIO(src))
    buf = io.BytesIO()
    if pixels is None:
        im.save(buf, 'JPEG', quality='keep')
    else:
        x = np.ascontiguousarray(pixels)
        out = Image.fromarray(x[..., 0] if x.shape[2] == 1 else x, 'L' if x.shape[2] == 1 else 'RGB')
        out.save(buf, 'JPEG', qtables=im.quantization, subsampling=JpegImagePlugin.get_sampling(im))
    return buf.getvalue()


def pillow_pixels(src):
    """Pillow's decode of the JPEG bytes src: (h, w, 3) RGB or (h, w, 1) gray uint8."""
    from PIL import Image
    im = Image.open(io.BytesIO(src))
    x = np.asarray(im)
    return x[..., None] if x.ndim == 2 else x
