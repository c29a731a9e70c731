"""A numpy restatement of PNG row filtering, for checking encoded files without a PNG decoder
(16-bit RGB and gray included): the scanlines of an image, the five filters' residuals, the filter
heuristic of encode_png, and whether a file's inflated scanlines are an image's pixels filtered as
the file's filter bytes say (filtering is invertible, so that is pixel equality)."""
import zlib

import numpy as np


def scanlines(x):
    """(h, row bytes) uint8: the unfiltered PNG samples of an (h, w, c) uint8 / uint16 array (c = 3
    for RGB, 1 for gray), 16-bit samples big-endian."""
    h, w, c = x.shape
    if x.dtype == np.uint16:
        return np.ascontiguousarray(x).astype('>u2').view(np.uint8).reshape(h, w * c * 2)
    return np.ascontiguousarray(x).reshape(h, w * c)


def residuals(raw, bpp):
    """(5, h, row bytes) int32: every byte of the scanlines under filters None, Sub, Up, Average
    and Paeth (mod 256); row 0's row above is zero."""
    h, rb = raw.shape
    x = raw.astype(np.int32)
    up = np.vstack([np.zeros((1, rb), np.int32), x[:-1]])
    left = np.hstack([np.zeros((h, bpp), np.int32), x[:, :-bpp]]) if rb > bpp else np.zeros_like(x)
    ul = np.hstack([np.zeros((h, bpp), np.int32), up[:, :-bpp]]) if rb > bpp else np.zeros_like(x)
    p = left + up - ul
    pa, pb, pc = np.abs(p - left), np.abs(p - up), np.abs(p - ul)
    paeth = np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, up, ul))
    return np.stack([x, x - left, x - up, x - (left + up) // 2, x - paeth]) & 255


def filtered(res, types):
    """The filtered stream (bytes) of residuals `res` with filter types[y] on row y."""
    _, h, rb = res.shape
    out = np.empty((h, rb + 1), np.uint8)
    out[:, 0] = types
    out[:, 1:] = res[types, np.arange(h)]
    return out.reshape(-1).tobytes()


def filter_rows(raw, bpp):
    """encode_png's heuristic: per row the filter with the smallest sum of |residual| (bytes read
    as signed), the lower type on a tie.  Returns (filter types, filtered stream)."""
    res = residuals(raw, bpp)
    cost = np.where(res < 128, res, 256 - res).sum(axis=2)
    types = np.argmin(cost, axis=0)                    # first minimum: the lower type wins a tie
    return types, filtered(res, types)


def idat(png):
    """The concatenated IDAT data of a PNG file."""
    z, i = b'', 8
    while i < len(png):
        n = int.from_bytes(png[i:i + 4], 'big')
        if png[i + 4:i + 8] == b'IDAT':
            z += png[i + 8:i + 8 + n]
        i += 12 + n
    return z


def holds_pixels(png, x, bpp=None):
    """Whether the non-interlaced PNG file `png` holds the (h, w, c) uint8 / uint16 array x.  bpp:
    the filters' bytes per pixel, by default c times the sample size (3 or 6 for RGB, 1 or 2 for
    gray)."""
    raw = scanlines(x)
    h = raw.shape[0]
    s = np.frombuffer(zlib.decompress(idat(png)), np.uint8)
    if s.size != h * (raw.shape[1] + 1):
        return False
    s = s.reshape(h, -1)
    types = s[:, 0].astype(np.int64)
    if types.max() > 4:
        return False
    if bpp is None:
        bpp = x.shape[2] * x.itemsize
    return filtered(residuals(raw, bpp), types) == s.tobytes()
