"""Four-component JPEG fixtures (test infrastructure): Pillow's CMYK files, the same files with their
Adobe APP14 segment removed or rewritten, YCCK files written from known coefficients (Pillow cannot
write YCCK), and arithmetic-coded twins; plus numpy restatements of decode_jpeg's four-component
samples (DESIGN §7q)."""
import io

import numpy as np
from PIL import Image

from jpeg2png_b200 import decode as D
from jpeg2png_b200 import synth
from tests import arith_synth
from tests import jpeg_synth as J


def cmyk_array(w, h, seed):
    """(h, w, 4) uint8: the synthetic cartoon's RGB as C, M, Y and a smooth K ramp."""
    rgb = synth.cartoon_image(w, h, seed).astype(np.uint8)
    k = (np.add.outer(np.arange(h) * 3, np.arange(w) * 2) + seed * 17) % 256
    return np.dstack([rgb, k.astype(np.uint8)])


def pillow_cmyk(w, h, quality=75, seed=1, **kw):
    """Pillow's CMYK JPEG (Adobe APP14, transform 0) of cmyk_array."""
    buf = io.BytesIO()
    Image.fromarray(cmyk_array(w, h, seed), 'CMYK').save(buf, 'JPEG', quality=quality, **kw)
    return buf.getvalue()


def segments(data):
    """[(marker, start, end)] of the marker segments before the first SOS."""
    out, pos = [], 2
    while pos + 4 <= len(data):
        assert data[pos] == 0xFF
        m = data[pos + 1]
        n = int.from_bytes(data[pos + 2:pos + 4], 'big')
        out.append((m, pos, pos + 2 + n))
        if m == 0xDA:
            break
        pos += 2 + n
    return out


def strip_app14(data):
    """data without its APP14 segments."""
    out = bytearray(data[:2])
    last = 2
    for m, a, b in segments(data):
        if m == 0xEE:
            out += data[last:a]
            last = b
    return bytes(out + data[last:])


def app14(transform, body=None):
    """An APP14 segment: "Adobe", version 100, flags 0 and 0, transform (12 data bytes), or `body`."""
    if body is None:
        body = b'Adobe' + bytes([0, 100, 0, 0, 0, 0, transform])
    return bytes([0xFF, 0xEE]) + (len(body) + 2).to_bytes(2, 'big') + body


def exif_segment(k):
    """An APP1 Exif segment carrying Orientation k."""
    e = Image.Exif()
    e[0x0112] = k
    body = e.tobytes()
    return b'\xff\xe1' + (len(body) + 2).to_bytes(2, 'big') + body


def with_app14(data, *segs):
    """data with its APP14 segments replaced by `segs`, right after SOI."""
    d = strip_app14(data)
    return d[:2] + b''.join(segs) + d[2:]


def encode_four(width, height, sampling, planes, quants, restart_interval=0, transform=2, interleaved=True):
    """A baseline four-component JPEG of given coefficients (jpeg_synth.encode_baseline for four
    components): sampling [(h, v)] * 4, planes[c] int [padded blocks y][padded blocks x][64] natural
    order on the MCU-padded grid, quants[c] 64 natural-order values (tables per component).  One
    interleaved scan, or with interleaved=False one scan per component over its real block grid;
    components 0 and 3 use the luma Huffman tables, 1 and 2 the chroma ones, as libjpeg writes YCCK.
    transform: the APP14 transform, None for no APP14 segment."""
    tabs = J.standard_huffman_tables()
    dc = [J._codes(*tabs[(0, 0)]), J._codes(*tabs[(0, 1)])]
    ac = [J._codes(*tabs[(1, 0)]), J._codes(*tabs[(1, 1)])]
    ht = [0, 1, 1, 0]
    maxh, maxv = max(h for h, _ in sampling), max(v for _, v in sampling)
    mcux, mcuy = -(-width // (8 * maxh)), -(-height // (8 * maxv))
    out = bytearray(b'\xff\xd8')
    if transform is not None:
        out += app14(transform)
    for c, q in enumerate(quants):
        out += b'\xff\xdb' + (67).to_bytes(2, 'big') + bytes([c]) + bytes(int(q[J.ZZ[k]]) for k in range(64))
    out += b'\xff\xc0' + (20).to_bytes(2, 'big') + b'\x08' + height.to_bytes(2, 'big') + width.to_bytes(2, 'big') + b'\x04'
    for c in range(4):
        out += bytes([c + 1, (sampling[c][0] << 4) | sampling[c][1], c])
    for (tc, th), (bits, vals) in tabs.items():
        out += b'\xff\xc4' + (19 + len(vals)).to_bytes(2, 'big') + bytes([(tc << 4) | th]) + bytes(bits) + bytes(vals)
    if restart_interval:
        out += b'\xff\xdd\x00\x04' + restart_interval.to_bytes(2, 'big')

    def block(bw, b, c, pred):
        t = ht[c]
        s, bits = J._size_bits(int(b[0]) - pred[c])
        pred[c] = int(b[0])
        bw.put(*dc[t][s])
        if s:
            bw.put(bits, s)
        run = 0
        last = max([k for k in range(1, 64) if b[J.ZZ[k]] != 0], default=0)
        for k in range(1, last + 1):
            val = int(b[J.ZZ[k]])
            if val == 0:
                run += 1
                continue
            while run > 15:
                bw.put(*ac[t][0xF0])
                run -= 16
            s, bits = J._size_bits(val)
            bw.put(*ac[t][(run << 4) | s])
            bw.put(bits, s)
            run = 0
        if last < 63:
            bw.put(*ac[t][0x00])

    if interleaved:
        scans = [(list(range(4)), [[(c, my * sampling[c][1] + y, mx * sampling[c][0] + x) for c in range(4)
                                    for y in range(sampling[c][1]) for x in range(sampling[c][0])]
                                   for my in range(mcuy) for mx in range(mcux)])]
    else:
        scans = []
        for c, (h, v) in enumerate(sampling):
            wb, hb = -(-(-(-width * h // maxh)) // 8), -(-(-(-height * v // maxv)) // 8)
            scans.append(([c], [[(c, by, bx)] for by in range(hb) for bx in range(wb)]))
    for comps, units in scans:
        body = bytes([len(comps)]) + b''.join(bytes([c + 1, 0x00 if ht[c] == 0 else 0x11]) for c in comps) + b'\x00\x3f\x00'
        out += b'\xff\xda' + (len(body) + 2).to_bytes(2, 'big') + body
        bw = J._Bits()
        pred = [0] * 4
        rst = 0
        for n, unit in enumerate(units):
            if restart_interval and n and n % restart_interval == 0:
                bw.flush()
                out += bw.out + bytes([0xFF, 0xD0 + (rst & 7)])
                bw = J._Bits()
                rst += 1
                pred = [0] * 4
            for c, by, bx in unit:
                block(bw, planes[c][by][bx], c, pred)
        bw.flush()
        out += bw.out
    return bytes(out + b'\xff\xd9')


def random_four(width, height, sampling, seed):
    """Coefficients for encode_four: planes as jpeg_synth.random_planes, four quantisation tables."""
    planes, _ = J.random_planes(width, height, sampling, seed)
    rng = np.random.default_rng(seed + 1)
    return planes, [rng.integers(1, 100, 64) for _ in range(4)]


def real_grid(planes, width, height, sampling):
    """The planes of random_four cut to each component's real block grid, flattened as the reader
    returns them (int16 [blocks * 64])."""
    maxh, maxv = max(h for h, _ in sampling), max(v for _, v in sampling)
    out = []
    for p, (h, v) in zip(planes, sampling):
        wb, hb = -(-(-(-width * h // maxh)) // 8), -(-(-(-height * v // maxv)) // 8)
        out.append(np.ascontiguousarray(p[:hb, :wb]).reshape(-1).astype(np.int16))
    return out


def ycck_file(w, h, sampling, seed, restart_interval=0, transform=2, interleaved=True):
    """(bytes, real-grid planes) of a YCCK (or, with transform 0 / None, CMYK) file of random coefficients."""
    planes, quants = random_four(w, h, sampling, seed)
    return (encode_four(w, h, sampling, planes, quants, restart_interval, transform, interleaved),
            real_grid(planes, w, h, sampling))


def arith_twin(data, restart_interval=0):
    """The SOF9 twin of a four-component Huffman file (arith_synth.write on its coefficients)."""
    keep, comps, _ = arith_synth.parse_headers(data)
    p = D.parse_jpeg4(data)
    planes = [pl.data.reshape(pl.h // 8, pl.w // 8, 64) for pl in p.planes]
    return arith_synth.write(p.w, p.h, keep, comps, planes, 'sequential', restart_interval)


def corpus():
    """{name: (bytes, kind)}: kind D.CMYK or D.YCCK, as libjpeg decides it."""
    files = {
        'pillow_q10_61x37': (pillow_cmyk(61, 37, 10, seed=2), D.CMYK),
        'pillow_q75_97x61': (pillow_cmyk(97, 61, 75, seed=3), D.CMYK),
        'pillow_q95_40x24': (pillow_cmyk(40, 24, 95, seed=4), D.CMYK),
        'pillow_progressive_q50_97x61': (pillow_cmyk(97, 61, 50, seed=5, progressive=True), D.CMYK),
    }
    files['no_app14_q75_97x61'] = (strip_app14(files['pillow_q75_97x61'][0]), D.CMYK)
    files['no_app14_progressive'] = (strip_app14(files['pillow_progressive_q50_97x61'][0]), D.CMYK)
    files['ycck_444_53x29'] = (ycck_file(53, 29, [(1, 1)] * 4, 7)[0], D.YCCK)
    files['ycck_2211_45x35'] = (ycck_file(45, 35, [(2, 2), (1, 1), (1, 1), (2, 2)], 8)[0], D.YCCK)
    files['ycck_444_restart3'] = (ycck_file(53, 29, [(1, 1)] * 4, 9, restart_interval=3)[0], D.YCCK)
    files['ycck_2211_restart2'] = (ycck_file(45, 35, [(2, 2), (1, 1), (1, 1), (2, 2)], 10, restart_interval=2)[0], D.YCCK)
    files['cmyk_2211_t0'] = (ycck_file(45, 35, [(2, 2), (1, 1), (1, 1), (2, 2)], 11, transform=0)[0], D.CMYK)
    files['ycck_2211_components'] = (ycck_file(45, 35, [(2, 2), (1, 1), (1, 1), (2, 2)], 12, interleaved=False)[0], D.YCCK)
    files['cmyk_444_components_restart5'] = (ycck_file(53, 29, [(1, 1)] * 4, 13, restart_interval=5, transform=0,
                                                       interleaved=False)[0], D.CMYK)
    files['arith_cmyk'] = (arith_twin(files['pillow_q75_97x61'][0]), D.CMYK)
    files['arith_ycck_2211'] = (arith_twin(files['ycck_2211_restart2'][0], restart_interval=2), D.YCCK)
    return files


def pillow_opens_as_cmyk(data):
    im = Image.open(io.BytesIO(data))
    im.load()
    return im.mode == 'CMYK'


def pillow_rgb(cmyk):
    """Pillow's Image.convert('RGB') of (..., 4) uint8 CMYK samples, restated in numpy."""
    x = cmyk[..., :3].astype(np.int32)
    nk = 255 - cmyk[..., 3:4].astype(np.int32)
    t = x * nk + 128
    return np.clip(nk - ((t + (t >> 8)) >> 8), 0, 255).astype(np.uint8)


def invert(g):
    """The inversion of gray samples g (uint8, uint16 or float32) into Pillow's CMYK polarity."""
    if g.dtype == np.uint8:
        return (255 - g).astype(np.uint8)
    if g.dtype == np.uint16:
        return (65535 - g.astype(np.int64)).astype(np.uint16)
    return (np.float32(255.0) - g).astype(np.float32)
