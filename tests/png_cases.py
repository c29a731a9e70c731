"""The images of the PNG encoder tests and the checks they share: a chunk walker that checks every
CRC, the numpy restatement of the filter heuristic (jpeg2png_b200.pngcheck), a row unfilter, and a
reader of deflate block headers (types and code lengths)."""
import struct
import zlib

import numpy as np

from jpeg2png_b200.pngcheck import filter_rows, scanlines  # noqa: F401  (the tests use them from here)

PIECE = 65536


def _fib_row():
    """One row of bytes 0..18 with Fibonacci frequencies (4181, 2584, ..., 1, 1), no two adjacent
    bytes equal (so no matches): a Huffman code over them is 18 bits deep, so the 15-bit limit has
    to act.  Filter None wins on it."""
    fib = [1, 1]
    while len(fib) < 19:
        fib.append(fib[-1] + fib[-2])
    left = {k: c for k, c in enumerate(reversed(fib))}
    out, prev = [], -1
    while any(left.values()):
        k = -max((c, -k) for k, c in left.items() if c and k != prev)[1]   # most left, not the previous
        out.append(k)
        left[k] -= 1
        prev = k
    out = np.array(out[:len(out) // 3 * 3], np.uint8)
    return out.reshape(1, len(out) // 3, 3)


def _smooth(h, w, dtype=np.uint8, seed=0):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    top = 255 if dtype == np.uint8 else 65535
    base = np.stack([(yy * 3 + xx) % 97, (yy + 2 * xx) % 61, (xx * yy) % 37], -1) * (top // 97)
    return np.clip(base + rng.integers(0, 3, base.shape), 0, top).astype(dtype)


def _noise(h, w, dtype=np.uint8, seed=0):
    top = 256 if dtype == np.uint8 else 65536
    return np.random.default_rng(seed).integers(0, top, (h, w, 3)).astype(dtype)


def cases():
    """name -> (array, layout): HWC or CHW numpy arrays, some of them strided views."""
    c = {
        '1x1': _noise(1, 1), '1x1_u16': _noise(1, 1, np.uint16),
        '1x300': _smooth(1, 300), '300x1': _smooth(300, 1), '1x1000_u16': _noise(1, 1000, np.uint16, 3),
        'stride_below_piece': _smooth(3, 21844), 'stride_at_piece': _smooth(3, 21845), 'stride_above_piece': _smooth(3, 21846),
        'one_piece_exact': _smooth(1, 21845, seed=1), 'one_piece_minus_1': _smooth(15, 1456),
        'two_pieces_exact': _smooth(2, 21845, seed=2), 'two_pieces_minus_1': _noise(1, 43690),
        'three_pieces_exact': _smooth(3, 21845, seed=3), 'three_pieces_plus_1': _smooth(1, 65536),
        'three_pieces_minus_1_u16': _smooth(467, 70, np.uint16),
        'noise_stored': _noise(64, 200), 'noise_u16': _noise(40, 90, np.uint16, 5),
        'fibonacci': _fib_row(),
        'smooth_200x300': _smooth(200, 300, seed=4), 'smooth_u16': _smooth(120, 77, np.uint16, 6),
    }
    for r, (h, w) in enumerate([(7, 98), (2, 129), (3, 86), (4, 86), (5, 86)]):       # run remainders 0..4
        c[f'constant_rem{r}'] = np.zeros((h, w, 3), np.uint8)
    c['constant_7'] = np.full((50, 400, 3), 7, np.uint8)
    c['constant_big'] = np.full((400, 700, 3), 200, np.uint8)
    out = {k: (v, 'HWC') for k, v in c.items()}
    out['chw'] = (np.ascontiguousarray(_smooth(60, 70, seed=8).transpose(2, 0, 1)), 'CHW')
    out['chw_u16'] = (np.ascontiguousarray(_smooth(33, 45, np.uint16, 9).transpose(2, 0, 1)), 'CHW')
    big = _smooth(90, 130, seed=10)
    out['strided_hwc'] = (big[5:80:2, 7:120:3], 'HWC')
    out['hwc_as_chw_view'] = (big.transpose(2, 0, 1), 'CHW')
    out['strided_u16'] = (_smooth(70, 90, np.uint16, 12)[::3, ::2], 'HWC')
    return out


def random_cases(n=100, seed=1234):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        h, w = int(rng.integers(1, 301)), int(rng.integers(1, 301))
        dt = np.uint16 if k % 4 == 3 else np.uint8
        kind = k % 3
        x = _noise(h, w, dt, k) if kind == 0 else _smooth(h, w, dt, k)
        if kind == 2:
            x = (x // (64 if dt == np.uint8 else 16384)).astype(dt)
        out.append((x, 'HWC'))
    return out


def hwc(x, layout):
    return x.transpose(1, 2, 0) if layout == 'CHW' else x


def chunks(png):
    """[(type, data)], every CRC checked with zlib.crc32."""
    assert png[:8] == b'\x89PNG\r\n\x1a\n'
    i, out = 8, []
    while i < len(png):
        n, = struct.unpack('>I', png[i:i + 4])
        t, d = png[i + 4:i + 8], png[i + 8:i + 8 + n]
        crc, = struct.unpack('>I', png[i + 8 + n:i + 12 + n])
        assert zlib.crc32(t + d) == crc, f'CRC of {t}'
        out.append((t, d))
        i += 12 + n
    assert i == len(png)
    return out


def unfilter(stream, h, rb, bpp):
    """Pure-Python PNG unfiltering: (h, rb) uint8."""
    rows, prev = [], [0] * rb
    for y in range(h):
        t, r = stream[y * (rb + 1)], stream[y * (rb + 1) + 1:(y + 1) * (rb + 1)]
        cur = [0] * rb
        for i in range(rb):
            a = cur[i - bpp] if i >= bpp else 0
            b = prev[i]
            c = prev[i - bpp] if i >= bpp else 0
            if t == 0:
                q = 0
            elif t == 1:
                q = a
            elif t == 2:
                q = b
            elif t == 3:
                q = (a + b) >> 1
            else:
                pp = a + b - c
                pa, pb, pc = abs(pp - a), abs(pp - b), abs(pp - c)
                q = a if pa <= pb and pa <= pc else (b if pb <= pc else c)
            cur[i] = (r[i] + q) & 255
        rows.append(cur)
        prev = cur
    return np.array(rows, np.uint8).reshape(h, rb)


class Bits:
    def __init__(self, data):
        self.d, self.p = data, 0

    def get(self, n):
        v = 0
        for k in range(n):
            v |= ((self.d[self.p >> 3] >> (self.p & 7)) & 1) << k
            self.p += 1
        return v


def _decoder(lengths):
    """Canonical Huffman decoding table: {(length, code): symbol}."""
    count = [0] * 16
    for l in lengths:
        count[l] += 1
    count[0] = 0
    code, nxt = 0, [0] * 16
    for l in range(1, 16):
        code = (code + count[l - 1]) << 1
        nxt[l] = code
    table = {}
    for s, l in enumerate(lengths):
        if l:
            table[(l, nxt[l])] = s
            nxt[l] += 1
    return table


def _decode(bits, table):
    code, l = 0, 0
    while True:
        code = code << 1 | bits.get(1)
        l += 1
        if (l, code) in table:
            return table[(l, code)]
        assert l <= 15, 'bad code'


def first_block(zdata):
    """The first deflate block of a zlib stream: (BTYPE, literal/length lengths, distance lengths)
    (lengths None unless the block is dynamic)."""
    bits = Bits(zdata[2:])
    bits.get(1)
    btype = bits.get(2)
    if btype != 2:
        return btype, None, None
    hlit, hdist, hclen = bits.get(5) + 257, bits.get(5) + 1, bits.get(4) + 4
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
    bl = [0] * 19
    for k in range(hclen):
        bl[order[k]] = bits.get(3)
    table, lens = _decoder(bl), []
    while len(lens) < hlit + hdist:
        s = _decode(bits, table)
        if s < 16:
            lens.append(s)
        elif s == 16:
            lens += [lens[-1]] * (3 + bits.get(2))
        elif s == 17:
            lens += [0] * (3 + bits.get(3))
        else:
            lens += [0] * (11 + bits.get(7))
    return btype, lens[:hlit], lens[hlit:]


def check_png(png, x, layout):
    """Container, checksums, filtering and round trip of one file against its input array.
    Returns the filtered stream."""
    x = hwc(x, layout)
    h, w, _ = x.shape
    sb = x.itemsize
    ch = chunks(png)
    assert [t for t, _ in ch] == [b'IHDR', b'IDAT', b'IEND']
    assert ch[0][1] == struct.pack('>IIBBBBB', w, h, 8 * sb, 2, 0, 0, 0)
    z = ch[1][1]
    assert z[:2] == b'\x78\x01'
    stream = zlib.decompress(z)                         # checks the Adler-32 too
    raw = scanlines(x)
    types, want = filter_rows(raw, 3 * sb)
    assert stream == want
    return stream
