"""Arithmetic-coded twins of Huffman JPEGs (test infrastructure), as `jpegtran -arithmetic` makes them.

transcode() takes a file's quantised coefficients (j2p_read_jpeg_mem on the Huffman file), its
quantisation tables, frame components and APPn/COM segments, and writes the SOF9 (sequential) or
SOF10 (progressive) file that codes the same coefficients: one interleaved scan, one scan per
component, or a progressive script with successive approximation, with an optional restart interval
and DAC conditioning.  The coder is the QM encoder of T.81 Annex D with the statistical models of
T.81 F.1.4.4 and G.1.3 as libjpeg's jcarith.c has them, flush included (trailing zero bytes are not
written; the decoder reads zeros past a segment's end).

The encoder is checked against libjpeg-turbo through Pillow: Pillow's pixels for each twin equal its
pixels for the Huffman original (tests/test_arith_host.py), before anything of ours is compared with it.
"""
import io
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jpeg2png_b200 import decode as D  # noqa: E402


def _qm(qe, nmps, nlps, sw):
    return (qe << 16) | (nmps << 8) | (sw << 7) | nlps


# T.81 table D.2 (Qe, NMPS, NLPS, SWITCH), and state 113: the fixed bin
QM = [_qm(*e) for e in [
    (0x5a1d, 1, 1, 1), (0x2586, 2, 14, 0), (0x1114, 3, 16, 0), (0x080b, 4, 18, 0), (0x03d8, 5, 20, 0), (0x01da, 6, 23, 0),
    (0x00e5, 7, 25, 0), (0x006f, 8, 28, 0), (0x0036, 9, 30, 0), (0x001a, 10, 33, 0), (0x000d, 11, 35, 0), (0x0006, 12, 9, 0),
    (0x0003, 13, 10, 0), (0x0001, 13, 12, 0), (0x5a7f, 15, 15, 1), (0x3f25, 16, 36, 0), (0x2cf2, 17, 38, 0), (0x207c, 18, 39, 0),
    (0x17b9, 19, 40, 0), (0x1182, 20, 42, 0), (0x0cef, 21, 43, 0), (0x09a1, 22, 45, 0), (0x072f, 23, 46, 0), (0x055c, 24, 48, 0),
    (0x0406, 25, 49, 0), (0x0303, 26, 51, 0), (0x0240, 27, 52, 0), (0x01b1, 28, 54, 0), (0x0144, 29, 56, 0), (0x00f5, 30, 57, 0),
    (0x00b7, 31, 59, 0), (0x008a, 32, 60, 0), (0x0068, 33, 62, 0), (0x004e, 34, 63, 0), (0x003b, 35, 32, 0), (0x002c, 9, 33, 0),
    (0x5ae1, 37, 37, 1), (0x484c, 38, 64, 0), (0x3a0d, 39, 65, 0), (0x2ef1, 40, 67, 0), (0x261f, 41, 68, 0), (0x1f33, 42, 69, 0),
    (0x19a8, 43, 70, 0), (0x1518, 44, 72, 0), (0x1177, 45, 73, 0), (0x0e74, 46, 74, 0), (0x0bfb, 47, 75, 0), (0x09f8, 48, 77, 0),
    (0x0861, 49, 78, 0), (0x0706, 50, 79, 0), (0x05cd, 51, 48, 0), (0x04de, 52, 50, 0), (0x040f, 53, 50, 0), (0x0363, 54, 51, 0),
    (0x02d4, 55, 52, 0), (0x025c, 56, 53, 0), (0x01f8, 57, 54, 0), (0x01a4, 58, 55, 0), (0x0160, 59, 56, 0), (0x0125, 60, 57, 0),
    (0x00f6, 61, 58, 0), (0x00cb, 62, 59, 0), (0x00ab, 63, 61, 0), (0x008f, 32, 61, 0), (0x5b12, 65, 65, 1), (0x4d04, 66, 80, 0),
    (0x412c, 67, 81, 0), (0x37d8, 68, 82, 0), (0x2fe8, 69, 83, 0), (0x293c, 70, 84, 0), (0x2379, 71, 86, 0), (0x1edf, 72, 87, 0),
    (0x1aa9, 73, 87, 0), (0x174e, 74, 72, 0), (0x1424, 75, 72, 0), (0x119c, 76, 74, 0), (0x0f6b, 77, 74, 0), (0x0d51, 78, 75, 0),
    (0x0bb6, 79, 77, 0), (0x0a40, 48, 77, 0), (0x5832, 81, 80, 1), (0x4d1c, 82, 88, 0), (0x438e, 83, 89, 0), (0x3bdd, 84, 90, 0),
    (0x34ee, 85, 91, 0), (0x2eae, 86, 92, 0), (0x299a, 87, 93, 0), (0x2516, 71, 86, 0), (0x5570, 89, 88, 1), (0x4ca9, 90, 95, 0),
    (0x44d9, 91, 96, 0), (0x3e22, 92, 97, 0), (0x3824, 93, 99, 0), (0x32b4, 94, 99, 0), (0x2e17, 86, 93, 0), (0x56a8, 96, 95, 1),
    (0x4f46, 97, 101, 0), (0x47e5, 98, 102, 0), (0x41cf, 99, 103, 0), (0x3c3d, 100, 104, 0), (0x375e, 93, 99, 0),
    (0x5231, 102, 105, 0), (0x4c0f, 103, 106, 0), (0x4639, 104, 107, 0), (0x415e, 99, 103, 0), (0x5627, 106, 105, 1),
    (0x50e7, 107, 108, 0), (0x4b85, 103, 109, 0), (0x5597, 109, 110, 0), (0x504f, 107, 111, 0), (0x5a10, 111, 110, 1),
    (0x5522, 109, 112, 0), (0x59eb, 111, 112, 1), (0x5a1d, 113, 113, 0)]]

ZZ = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
      35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63]


class QMEncoder:
    """T.81 D.1 with libjpeg's byte output (carry over stacked FF bytes, FF 00 stuffing) and flush."""

    def __init__(self):
        self.out = bytearray()
        self.c, self.a, self.ct, self.buffer, self.sc, self.zc = 0, 0x10000, 11, -1, 0, 0

    def _zeros(self):
        if self.zc:
            self.out += bytes(self.zc)
            self.zc = 0

    def encode(self, st, i, val):
        """One decision `val` with the adaptive state st[i]."""
        sv = st[i]
        e = QM[sv & 0x7f]
        qe, nm, nl = e >> 16, (e >> 8) & 0xff, e & 0xff
        a = self.a - qe
        if val != (sv >> 7):
            if a >= qe:
                self.c += a
                a = qe
            st[i] = (sv & 0x80) ^ nl
        else:
            if a >= 0x8000:
                self.a = a
                return
            if a < qe:
                self.c += a
                a = qe
            st[i] = (sv & 0x80) ^ nm
        c, ct = self.c, self.ct
        while True:
            a <<= 1
            c <<= 1
            ct -= 1
            if ct == 0:
                temp = c >> 19
                if temp > 0xff:
                    if self.buffer >= 0:
                        self._zeros()
                        self.out.append(self.buffer + 1)
                        if self.buffer + 1 == 0xff:
                            self.out.append(0)
                    self.zc += self.sc
                    self.sc = 0
                    self.buffer = temp & 0xff
                elif temp == 0xff:
                    self.sc += 1
                else:
                    self._flush_stacked()
                    self.buffer = temp & 0xff
                c &= 0x7ffff
                ct += 8
            if a >= 0x8000:
                break
        self.a, self.c, self.ct = a, c, ct

    def _flush_stacked(self):
        if self.buffer == 0:
            self.zc += 1
        elif self.buffer >= 0:
            self._zeros()
            self.out.append(self.buffer)
        if self.sc:
            self._zeros()
            self.out += b'\xff\x00' * self.sc
            self.sc = 0

    def finish(self):
        """T.81 D.1.8 as libjpeg: the value in the interval with the most trailing zeros, then the
        pending bytes; final zero bytes are not written.  Returns the segment's bytes."""
        temp = (self.a - 1 + self.c) & 0xffff0000
        self.c = temp + 0x8000 if temp < self.c else temp
        self.c <<= self.ct
        if self.c & 0xf8000000:
            if self.buffer >= 0:
                self._zeros()
                self.out.append(self.buffer + 1)
                if self.buffer + 1 == 0xff:
                    self.out.append(0)
            self.zc += self.sc
            self.sc = 0
        else:
            self._flush_stacked()
        if self.c & 0x7fff800:
            self._zeros()
            self.out.append((self.c >> 19) & 0xff)
            if ((self.c >> 19) & 0xff) == 0xff:
                self.out.append(0)
            if self.c & 0x7f800:
                self.out.append((self.c >> 11) & 0xff)
                if ((self.c >> 11) & 0xff) == 0xff:
                    self.out.append(0)
        return bytes(self.out)


# ---- the statistical models (jcarith.c) --------------------------------------------------------
def _magnitude(enc, stats, st, v, x1):
    """v - 1 >= 0 coded from bin st: the category (its further decisions from bin x1) and the bits."""
    m = 0
    if v:
        enc.encode(stats, st, 1)
        m = 1
        v2 = v >> 1
        if x1 is None:                      # DC: bins 20.. after the first decision
            st = 20
            while v2:
                enc.encode(stats, st, 1)
                m <<= 1
                st += 1
                v2 >>= 1
        elif v2:                            # AC: a second decision on st, then bins 189 or 217
            enc.encode(stats, st, 1)
            m = 2
            st = x1
            v2 >>= 1
            while v2:
                enc.encode(stats, st, 1)
                m <<= 1
                st += 1
                v2 >>= 1
    enc.encode(stats, st, 0)
    st += 14
    m >>= 1
    while m:
        enc.encode(stats, st, 1 if m & v else 0)
        m >>= 1


def encode_dc(enc, dcst, ctx, ci, v, L, U):
    """A DC difference v of component slot ci (F.1.4.4.1); ctx: the slots' conditioning categories."""
    st = ctx[ci]
    if v == 0:
        enc.encode(dcst, st, 0)
        ctx[ci] = 0
        return
    enc.encode(dcst, st, 1)
    if v > 0:
        enc.encode(dcst, st + 1, 0)
        st += 2
        new = 4
    else:
        v = -v
        enc.encode(dcst, st + 1, 1)
        st += 3
        new = 8
    v -= 1
    m = 1 << (v.bit_length() - 1) if v else 0
    _magnitude(enc, dcst, st, v, None)
    if m < (1 << L) >> 1:
        new = 0
    elif m > (1 << U) >> 1:
        new += 8
    ctx[ci] = new


def encode_ac(enc, acst, fixed, vals, ss, se, kx):
    """AC values vals[k] (zig-zag order, point transform applied) for k = ss..se (F.1.4.4.2, G.1.3.2)."""
    ke = 0
    for k in range(se, 0, -1):
        if vals[k]:
            ke = k
            break
    k = ss
    while k <= ke:
        st = 3 * (k - 1)
        enc.encode(acst, st, 0)
        while vals[k] == 0:
            enc.encode(acst, st + 1, 0)
            st += 3
            k += 1
        enc.encode(acst, st + 1, 1)
        v = vals[k]
        enc.encode(fixed, 0, 1 if v < 0 else 0)
        _magnitude(enc, acst, st + 2, abs(v) - 1, 189 if k <= kx else 217)
        k += 1
    if k <= se:
        enc.encode(acst, 3 * (k - 1), 1)


def encode_ac_refine(enc, acst, fixed, blk, ss, se, al):
    """The bit al of the AC coefficients ss..se of blk (zig-zag order, full values), G.1.3.3."""
    def pt(v, s):
        return v >> s if v >= 0 else -((-v) >> s)
    ke = 0
    for k in range(se, 0, -1):
        if pt(blk[k], al):
            ke = k
            break
    kex = 0
    for k in range(ke, 0, -1):
        if pt(blk[k], al + 1):
            kex = k
            break
    k = ss
    while k <= ke:
        st = 3 * (k - 1)
        if k > kex:
            enc.encode(acst, st, 0)
        while True:
            v = abs(pt(blk[k], al))
            if v:
                if v >> 1:
                    enc.encode(acst, st + 2, v & 1)
                else:
                    enc.encode(acst, st + 1, 1)
                    enc.encode(fixed, 0, 1 if blk[k] < 0 else 0)
                break
            enc.encode(acst, st + 1, 0)
            st += 3
            k += 1
        k += 1
    if k <= se:
        enc.encode(acst, 3 * (k - 1), 1)


# ---- files ---------------------------------------------------------------------------------------
def _seg(marker, body):
    return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, 'big') + bytes(body)


def parse_headers(data):
    """(APPn/COM/DQT segments before the frame, [(id, h, v, tq)], [scan (component indices, ss, se, ah, al)])."""
    keep, comps, scans, pos = [], [], [], 2
    while pos + 4 <= len(data):
        if data[pos] != 0xFF:
            pos += 1
            continue
        m = data[pos + 1]
        if m == 0xFF or m == 0x00 or 0xD0 <= m <= 0xD7:
            pos += 1 if m == 0xFF else 2
            continue
        if m == 0xD9:
            break
        ln = int.from_bytes(data[pos + 2:pos + 4], 'big')
        body = data[pos + 4:pos + 2 + ln]
        if m in (0xDB, 0xFE) or 0xE0 <= m <= 0xEF:
            if not comps:
                keep.append(data[pos:pos + 2 + ln])
        elif m in (0xC0, 0xC1, 0xC2):
            comps = [(body[6 + 3 * i], body[7 + 3 * i] >> 4, body[7 + 3 * i] & 15, body[8 + 3 * i]) for i in range(body[5])]
        elif m == 0xDA:
            ns = body[0]
            ids = [body[1 + 2 * i] for i in range(ns)]
            idx = [next(k for k, c in enumerate(comps) if c[0] == x) for x in ids]
            scans.append((idx, body[1 + 2 * ns], body[2 + 2 * ns], body[3 + 2 * ns] >> 4, body[3 + 2 * ns] & 15))
        pos += 2 + ln
    return keep, comps, scans


# libjpeg's jpeg_simple_progression for three components (and its one-component script)
SIMPLE_PROGRESSION_3 = [([0, 1, 2], 0, 0, 0, 1), ([0], 1, 5, 0, 2), ([2], 1, 63, 0, 1), ([1], 1, 63, 0, 1),
                        ([0], 6, 63, 0, 2), ([0], 1, 63, 2, 1), ([0, 1, 2], 0, 0, 1, 0), ([2], 1, 63, 1, 0),
                        ([1], 1, 63, 1, 0), ([0], 1, 63, 1, 0)]
SIMPLE_PROGRESSION_1 = [([0], 0, 0, 0, 1), ([0], 1, 5, 0, 2), ([0], 6, 63, 0, 2), ([0], 1, 63, 2, 1), ([0], 0, 0, 1, 0),
                        ([0], 1, 63, 1, 0)]


def transcode(data, script='sequential', restart_interval=0, dac=None, tables=None):
    """The arithmetic-coded twin of the Huffman JPEG `data`.

    script: 'sequential' (SOF9, one interleaved scan; one scan for a gray file), 'components' (SOF9,
    one scan per component), 'own' (SOF10 with the file's own progressive scans; the file must be
    progressive), 'progressive' (SOF10 with libjpeg's simple progression) or a list of
    (component indices, ss, se, ah, al) for SOF10.  restart_interval: MCUs per segment (DRI), or
    'row' for one MCU row of the frame.  dac: {table index (0..15 DC, 16..31 AC): value}, written
    before the first scan.  tables: the DC/AC table selector of each component (default luma 0,
    chroma 1)."""
    keep, comps, own = parse_headers(data)
    p = D.parse_jpeg(data, D.READ_GRAY)
    planes = [pl.data.reshape(pl.h // 8, pl.w // 8, 64) for pl in p.planes]
    return write(p.w, p.h, keep, comps, planes, own if script == 'own' else script, restart_interval, dac, tables)


def write(w, h, keep, comps, planes, script='sequential', restart_interval=0, dac=None, tables=None):
    """The SOF9/SOF10 file of the given coefficients: planes[c] int [hb][wb][64] in natural order on the
    component's real block grid; keep: segments (DQT, APPn, ...) written before the frame header;
    comps: (id, h, v, tq) per component; the other arguments as transcode's."""
    nc = len(comps)
    maxh, maxv = max(c[1] for c in comps), max(c[2] for c in comps)
    mcux, mcuy = -(-w // (8 * maxh)), -(-h // (8 * maxv))
    planes = [np.asarray(pl).astype(np.int64)[:, :, ZZ] for pl in planes]     # zig-zag order
    if script == 'sequential':
        scans, progressive = [(list(range(nc)), 0, 63, 0, 0)], False
    elif script == 'components':
        scans, progressive = [([c], 0, 63, 0, 0) for c in range(nc)], False
    elif script == 'progressive':
        scans, progressive = (SIMPLE_PROGRESSION_3 if nc == 3 else SIMPLE_PROGRESSION_1), True
    else:
        scans, progressive = list(script), True
    tables = tables or [0] + [1] * (nc - 1)
    L, U, K = [0] * 16, [1] * 16, [5] * 16
    for idx, val in (dac or {}).items():
        if idx < 16:
            L[idx], U[idx] = val & 15, val >> 4
        else:
            K[idx - 16] = val
    ri = mcux if restart_interval == 'row' else restart_interval

    out = bytearray(b'\xff\xd8')
    for s in keep:
        out += s
    sof = bytearray([8]) + h.to_bytes(2, 'big') + w.to_bytes(2, 'big') + bytes([nc])
    for cid, ch, cv, tq in comps:
        sof += bytes([cid, (ch << 4) | cv, tq])
    out += _seg(0xCA if progressive else 0xC9, sof)
    if dac:
        out += _seg(0xCC, b''.join(bytes([i, v]) for i, v in sorted(dac.items())))
    if ri:
        out += _seg(0xDD, ri.to_bytes(2, 'big'))
    for idx, ss, se, ah, al in scans:
        ns = len(idx)
        body = bytearray([ns])
        for c in idx:
            body += bytes([comps[c][0], (tables[c] << 4) | tables[c]])
        body += bytes([ss, se, (ah << 4) | al])
        out += _seg(0xDA, body)
        if ns > 1:
            units = [[(c, my * comps[idx[c]][2] + y, mx * comps[idx[c]][1] + x) for c in range(ns)
                      for y in range(comps[idx[c]][2]) for x in range(comps[idx[c]][1])]
                     for my in range(mcuy) for mx in range(mcux)]
        else:
            hb, wb = planes[idx[0]].shape[:2]
            units = [[(0, by, bx)] for by in range(hb) for bx in range(wb)]
        enc = None
        rst = 0
        for n, unit in enumerate(units):
            if enc is None or (ri and n % ri == 0):
                if enc is not None:
                    out += enc.finish() + bytes([0xFF, 0xD0 + (rst & 7)])
                    rst += 1
                enc = QMEncoder()
                dcst = [bytearray(64) for _ in range(4)]
                acst = [bytearray(256) for _ in range(4)]
                fixed = bytearray([113])
                pred, ctx = [0] * ns, [0] * ns
            for s, by, bx in unit:
                c = idx[s]
                pl = planes[c]
                blk = pl[by, bx] if by < pl.shape[0] and bx < pl.shape[1] else np.zeros(64, np.int64)
                td = ta = tables[c]
                if ss == 0 and ah == 0:
                    dc = int(blk[0]) >> al
                    encode_dc(enc, dcst[td], ctx, s, dc - pred[s], L[td], U[td])
                    pred[s] = dc
                elif ss == 0:
                    enc.encode(fixed, 0, (int(blk[0]) >> al) & 1)
                if not progressive:
                    encode_ac(enc, acst[ta], fixed, [int(x) for x in blk], 1, 63, K[ta])
                elif ss > 0 and ah == 0:
                    vals = [int(x) >> al if x >= 0 else -((-int(x)) >> al) for x in blk]
                    encode_ac(enc, acst[ta], fixed, vals, ss, se, K[ta])
                elif ss > 0:
                    encode_ac_refine(enc, acst[ta], fixed, [int(x) for x in blk], ss, se, al)
        out += enc.finish()
    return bytes(out + b'\xff\xd9')


def dqt(tables):
    """A DQT segment of 8-bit tables (natural order), ids 0, 1, ..."""
    body = bytearray()
    for t, q in enumerate(tables):
        body += bytes([t]) + bytes(int(q[z]) for z in ZZ)
    return _seg(0xDB, body)


def raw_scan(width, height, decisions, dac=None):
    """A one-component gray SOF9 file (quantisation 1) whose single scan codes `decisions`: a list of
    (bins, index, bit) with bins 'dc', 'ac' or 'fixed' (table 0): crafted streams for the reader's
    refusals."""
    enc = QMEncoder()
    bins = {'dc': bytearray(64), 'ac': bytearray(256), 'fixed': bytearray([113])}
    for b, i, v in decisions:
        enc.encode(bins[b], i, v)
    out = bytearray(b'\xff\xd8') + _seg(0xDB, bytes([0]) + bytes([1] * 64))
    out += _seg(0xC9, bytes([8]) + height.to_bytes(2, 'big') + width.to_bytes(2, 'big') + bytes([1, 1, 0x11, 0]))
    if dac:
        out += _seg(0xCC, b''.join(bytes([i, v]) for i, v in sorted(dac.items())))
    out += _seg(0xDA, bytes([1, 1, 0x00, 0, 63, 0]))
    return bytes(out + enc.finish() + b'\xff\xd9')


def pillow_pixels(data):
    """Pillow's (libjpeg-turbo's) decode of JPEG bytes as an array."""
    from PIL import Image
    im = Image.open(io.BytesIO(data))
    im.load()
    return np.asarray(im)
