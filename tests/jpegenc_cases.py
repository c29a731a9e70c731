"""The JPEG encoder's test corpus, shared by the CPU tests (host driver against Pillow) and the GPU
tests (device against host driver): sizes that reach edge replication and dummy blocks in every
sampling, several kinds of content, and HWC, CHW and strided views."""
import io

import numpy as np

from jpeg2png_b200 import synth

SIZES = [(1, 1), (7, 9), (8, 8), (9, 8), (16, 16), (17, 13), (31, 33), (97, 61), (200, 300), (1023, 769)]   # (h, w)
QUALITIES = [1, 10, 50, 75, 90, 95, 100]
SAMPLINGS = ['4:4:4', '4:2:2', '4:2:0']
SMALL = 97 * 61                      # every content up to this many pixels; above it cartoon and noise


def content(kind, h, w, seed):
    """(h, w, 3) uint8 pixels of one kind."""
    if kind == 'cartoon':
        return synth.cartoon_image(w, h, seed).round().astype(np.uint8)
    if kind == 'noise':
        return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind.startswith('flat'):
        return np.full((h, w, 3), int(kind[4:]), np.uint8)
    if kind == 'primaries':             # stripes of saturated R, G, B, C, M, Y, K, W
        cols = np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255], [0, 255, 255], [255, 0, 255], [255, 255, 0], [0, 0, 0],
                         [255, 255, 255]], np.uint8)
        yy, xx = np.mgrid[0:h, 0:w]
        return cols[((xx // 3) + (yy // 5)) % 8]
    raise ValueError(kind)


KINDS = ['cartoon', 'noise', 'flat0', 'flat128', 'flat255', 'primaries']


def view(x, how, seed):
    """x (h, w, 3) as ('HWC' | 'CHW', array): contiguous HWC, contiguous CHW, or a strided view
    (a step-sliced, channel-reversed window of a larger array) holding the same pixels."""
    if how == 'HWC':
        return 'HWC', x
    if how == 'CHW':
        return 'CHW', np.ascontiguousarray(x.transpose(2, 0, 1))
    h, w, _ = x.shape
    big = np.random.default_rng(seed).integers(0, 256, (2 * h + 3, 3 * w + 2, 3), dtype=np.uint8)
    big[1:1 + 2 * h:2, 2:2 + 3 * w:3] = x[:, :, ::-1]
    return 'HWC', big[1:1 + 2 * h:2, 2:2 + 3 * w:3, ::-1]


def corpus():
    """name -> (layout, array, hwc): every size with every kind (cartoon and noise only above
    SMALL pixels), cycling through the three views."""
    out, k = {}, 0
    for h, w in SIZES:
        for kind in KINDS:
            if h * w > SMALL and kind not in ('cartoon', 'noise'):
                continue
            x = content(kind, h, w, seed=1000 + k)
            how = ['HWC', 'CHW', 'strided'][k % 3]
            lay, a = view(x, how, seed=k)
            out[f'{h}x{w}_{kind}_{how}'] = (lay, a, x)
            k += 1
    return out


def pillow(x, quality, subsampling):
    """Pillow's file for the (h, w, 3) uint8 pixels."""
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(x), 'RGB').save(buf, 'JPEG', quality=quality, subsampling=subsampling)
    return buf.getvalue()


def turbo_version():
    from PIL import features
    return f"libjpeg-turbo {features.version('libjpeg_turbo')}"
