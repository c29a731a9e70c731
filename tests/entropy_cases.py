"""Test files for the entropy decoder (test infrastructure, shared by test_entropy_host.py and
test_gpu_entropy.py): a sequential encoder with a free choice of scans (three non-interleaved scans,
a component scanned twice or never), a raw-bit-stream writer with custom Huffman tables for crafted
streams, and helpers that decode a list of files through libj2pentropy.so (host driver or device)
and through the host reader."""
import ctypes as C
import io

import numpy as np
from PIL import Image

from jpeg2png_b200 import decode as D
from jpeg2png_b200 import synth
from tests import jpeg_synth as J


def _header(width, height, sampling, quants, tables, restart_interval):
    out = bytearray(b'\xff\xd8')
    for c in range(3):
        out += b'\xff\xdb' + (67).to_bytes(2, 'big') + bytes([c]) + bytes(int(quants[c][J.ZZ[k]]) for k in range(64))
    out += b'\xff\xc0' + (17).to_bytes(2, 'big') + b'\x08' + height.to_bytes(2, 'big') + width.to_bytes(2, 'big') + b'\x03'
    for c in range(3):
        out += bytes([c + 1, (sampling[c][0] << 4) | sampling[c][1], c])
    for (tc, th), (bits, vals) in tables.items():
        out += b'\xff\xc4' + (19 + len(vals)).to_bytes(2, 'big') + bytes([(tc << 4) | th]) + bytes(bits) + bytes(vals)
    if restart_interval:
        out += b'\xff\xdd\x00\x04' + restart_interval.to_bytes(2, 'big')
    return out


def _sos(comps, tab):
    return b'\xff\xda' + (6 + 2 * len(comps)).to_bytes(2, 'big') + bytes([len(comps)]) + b''.join(
        bytes([c + 1, (tab[c] << 4) | tab[c]]) for c in comps) + b'\x00\x3f\x00'


def _put_block(bw, b, pred, dc, ac):
    s, bits = J._size_bits(int(b[0]) - pred)
    bw.put(*dc[s])
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
            bw.put(*ac[0xF0])
            run -= 16
        s, bits = J._size_bits(val)
        bw.put(*ac[(run << 4) | s])
        bw.put(bits, s)
        run = 0
    if last < 63:
        bw.put(*ac[0x00])
    return int(b[0])


def encode_scans(width, height, sampling, planes, quants, scans, restart_interval=0):
    """Sequential JPEG with the given scans (lists of component indices, in scan order): a scan of
    one component is non-interleaved (its real block grid), one of several is interleaved.
    planes/quants as jpeg_synth.encode_baseline (MCU-padded grids, natural order)."""
    tabs = J.standard_huffman_tables()
    dc = [J._codes(*tabs[(0, 0)]), J._codes(*tabs[(0, 1)])]
    ac = [J._codes(*tabs[(1, 0)]), J._codes(*tabs[(1, 1)])]
    maxh, maxv = max(h for h, _ in sampling), max(v for _, v in sampling)
    mcux, mcuy = -(-width // (8 * maxh)), -(-height // (8 * maxv))
    tab = [0, 1, 1]
    out = _header(width, height, sampling, quants, tabs, restart_interval)
    for comps in scans:
        out += _sos(comps, tab)
        if len(comps) > 1:
            units = [[(c, my * sampling[c][1] + y, mx * sampling[c][0] + x) for c in comps
                      for y in range(sampling[c][1]) for x in range(sampling[c][0])]
                     for my in range(mcuy) for mx in range(mcux)]
        else:
            c = comps[0]
            wb = -(-(-(-width * sampling[c][0] // maxh)) // 8)
            hb = -(-(-(-height * sampling[c][1] // maxv)) // 8)
            units = [[(c, by, bx)] for by in range(hb) for bx in range(wb)]
        bw, pred, rst = J._Bits(), [0, 0, 0], 0
        for n, unit in enumerate(units):
            if restart_interval and n and n % restart_interval == 0:
                bw.flush()
                out += bw.out + bytes([0xFF, 0xD0 + (rst & 7)])
                bw, pred, rst = J._Bits(), [0, 0, 0], rst + 1
            for c, by, bx in unit:
                pred[c] = _put_block(bw, planes[c][by][bx], pred[c], dc[tab[c]], ac[tab[c]])
        bw.flush()
        out += bw.out
    return bytes(out + b'\xff\xd9')


def encode_raw(width, height, dc_table, ac_table, bits, restart_interval=0):
    """A 4:4:4 sequential file whose one interleaved scan is the raw bit string `bits` ('0'/'1',
    byte-stuffed here), every component on the tables (bits[16], vals) given."""
    tables = {(0, 0): dc_table, (1, 0): ac_table}
    q = [np.ones(64, np.int64)] * 3
    out = _header(width, height, [(1, 1)] * 3, q, tables, restart_interval)
    out += _sos([0, 1, 2], [0, 0, 0])
    bw = J._Bits()
    for ch in bits:
        bw.put(int(ch), 1)
    bw.flush()
    return bytes(out + bw.out + b'\xff\xd9')


def code_bits(table, sym):
    code, n = J._codes(*table)[sym]
    return format(code, f'0{n}b')


def pillow(w, h, q, ss, optimize=False, progressive=False, seed=1):
    rgb = synth.cartoon_image(w, h, seed).astype(np.uint8)
    buf = io.BytesIO()
    Image.fromarray(rgb, 'RGB').save(buf, 'JPEG', quality=q, subsampling=ss, optimize=optimize, progressive=progressive)
    return buf.getvalue()


def synth_file(w, h, sampling, ri, seed=None, scans=None):
    planes, quants = J.random_planes(w, h, sampling, seed=w * 7 + h if seed is None else seed)
    if scans is None:
        return J.encode_baseline(w, h, sampling, planes, quants, restart_interval=ri)
    return encode_scans(w, h, sampling, planes, quants, scans, restart_interval=ri)


STD = J.standard_huffman_tables()
DC0, AC0 = STD[(0, 0)], STD[(1, 0)]


def crafted():
    """name -> bytes: streams that exercise one rule of the reader each."""
    cases = {}
    good = synth_file(64, 48, [(1, 1)] * 3, 0, seed=3)
    sos = good.rfind(b'\xff\xda')
    body = good[sos + 14:-2]
    cases['truncated_zero_padding'] = good[:sos + 14] + body[:len(body) // 3] + b'\xff\xd9'
    cases['truncated_no_eoi'] = good[:sos + 14] + body[:len(body) // 2]
    ri = synth_file(70, 50, [(2, 2), (1, 1), (1, 1)], 2, seed=4)
    fill = bytearray()
    i = 0
    while i < len(ri):                  # fill bytes and junk before every RSTn
        if ri[i] == 0xFF and i + 1 < len(ri) and 0xD0 <= ri[i + 1] <= 0xD7:
            fill += (b'\x12\x34' if ri[i + 1] & 1 else b'') + b'\xff\xff\xff'
            i += 1
            continue
        fill.append(ri[i])
        i += 1
    cases['fill_and_junk_before_rst'] = bytes(fill)
    cases['extra_rst_after_last_interval'] = ri[:-2] + b'\xff\xd0\xff\xd1\x00\xff\xd9'
    rst = ri.find(b'\xff\xd1')
    cases['rst_out_of_sequence'] = ri[:rst] + b'\xff\xd5' + ri[rst + 2:]
    cases['missing_rst'] = ri[:rst] + b'\xff\xc8' + ri[rst + 2:]
    cases['truncated_at_rst'] = ri[:rst]
    eob, zrl = code_bits(AC0, 0x00), code_bits(AC0, 0xF0)
    dc0 = code_bits(DC0, 0)
    one = code_bits(AC0, 0x01) + '1'
    blk = dc0 + one + zrl * 4                   # k=1 then four ZRL: k runs past 63, the block ends without EOB
    cases['zrl_past_63'] = encode_raw(8, 8, DC0, AC0, blk + (dc0 + eob) * 2)
    cases['bad_code'] = encode_raw(8, 8, DC0, AC0, dc0 + eob + '1' * 16 + '0' * 32)
    cases['bad_index'] = encode_raw(8, 8, DC0, AC0, dc0 + zrl * 3 + code_bits(AC0, 0xF1) + '1' + (dc0 + eob) * 2)
    big_dc = ([1, 2] + [0] * 14, [0, 17, 3])      # codes '0' -> 0, '10' -> 17, '11' -> 3
    cases['bad_magnitude'] = encode_raw(8, 8, big_dc, AC0, '0' + eob + '10' + '1' * 17 + eob + '0' + eob)
    cases['dc_category_16'] = encode_raw(8, 8, ([0, 2] + [0] * 14, [0, 16]), AC0,
                                         ('01' + '1' * 16 + eob) + ('00' + eob) + ('01' + '0' * 16 + eob))
    # one-bit codes: blocks of two bits that look the same at every offset, so a guessed block index
    # within the MCU is only corrected round by round
    tiny_dc, tiny_ac = ([1, 1] + [0] * 14, [0, 1]), ([1] + [0] * 15, [0])      # DC '0' -> 0, '10' -> 1; AC '0' -> EOB
    rng = np.random.default_rng(9)
    bits = ''.join('00' if rng.random() < 0.995 else '10' + str(int(rng.integers(0, 2))) + '0' for _ in range(96 * 64 * 3))
    cases['late_sync_one_bit_codes'] = encode_raw(768, 64, tiny_dc, tiny_ac, bits)
    return cases


# ---- decoding through the library ------------------------------------------------------------
def reader(data):
    """(planes as int16 arrays, '') or (None, message) from j2p_read_jpeg_mem."""
    try:
        p = D.parse_jpeg(data)
    except ValueError as e:
        return None, str(e)
    return [x.data for x in p.planes], ''


def entropy_host(layouts, subseq_bits):
    """Decode FileLayouts with the serial host driver: ([per file: 3 int16 arrays], statuses, stats)."""
    arrs, outs = [], []
    for lay in layouts:
        planes = []
        for p in lay.planes:
            a = np.full(p.w * p.h, 0x5a5a, np.int16)      # the decoder writes every coefficient
            planes.append(a)
            outs.append(a.ctypes.data)
        arrs.append(planes)
    buf, addr, _, work_bytes = D.entropy_plan(layouts, outs, subseq_bits)
    work = np.zeros(work_bytes + 16, np.uint8)
    status = np.zeros(max(len(layouts), 1), np.uint32)
    stats = D.EntropyStats()
    lib = D.load_entropy()
    assert lib.j2p_entropy_decode_host(addr, (work.ctypes.data + 15) & ~15, status.ctypes.data, C.byref(stats)) == 0, \
        lib.j2p_entropy_last_error()
    return arrs, status[:len(layouts)], stats
