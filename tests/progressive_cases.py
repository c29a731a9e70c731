"""Test files for the progressive decoder (shared by test_progressive_host.py, test_gpu_progressive.py
and fuzz_progressive.py): Pillow progressive files, a small progressive writer for scan scripts Pillow
cannot produce, and helpers that decode layouts through libj2pprogressive.so (host driver or device).

The writer codes each scan's segments as raw symbol streams under complete Huffman codes, so random
bits always decode: DC categories 0..15 and an AC alphabet of EOB runs (EOB0..EOB14), ZRL and runs of
up to 10 zeros before a value.  Bits past a segment's end read as zero, which is code 0: category 0 or
EOB.  What a file means is whatever the host reader makes of it; the decoder must agree."""
import ctypes as C

import numpy as np

from jpeg2png_b200 import decode as D
from tests import entropy_cases as E

DC_SYMS = list(range(16))                                  # categories 0..15, 4 bits each
AC_SYMS = [0x00, 0x01, 0x11, 0x21, 0x51, 0xF0, 0x10, 0x20, 0xE0, 0x02, 0x31, 0xA1, 0x03, 0x41, 0x71, 0xC0]
TABLE = [0, 0, 0, 16] + [0] * 12                           # bits[1..16]: 16 codes of length 4


def _table(tc, th, syms, bits=TABLE):
    return b'\xff\xc4' + (19 + len(syms)).to_bytes(2, 'big') + bytes([(tc << 4) | th]) + bytes(bits) + bytes(syms)


def _stuff(raw: bytes) -> bytes:
    return raw.replace(b'\xff', b'\xff\x00')


def _sym_bits(syms, sym):
    return format(syms.index(sym), '04b')


def bits_to_bytes(bits: str) -> bytes:
    bits += '0' * (-len(bits) % 8)
    return bytes(int(bits[i:i + 8], 2) for i in range(0, len(bits), 8))


def write(width, height, sampling, scans, ri=0, seed=0, ac_syms=AC_SYMS, ac_bits=TABLE):
    """A progressive file.  scans: (components, Ss, Se, Ah, Al, data) with data None (random
    segments about as long as the scan's blocks need), an int (that many random bytes per
    segment) or a bit string (the one segment's bits)."""
    rng = np.random.default_rng(seed)
    maxh, maxv = max(h for h, _ in sampling), max(v for _, v in sampling)
    mcux, mcuy = -(-width // (8 * maxh)), -(-height // (8 * maxv))
    out = bytearray(b'\xff\xd8')
    for c in range(3):
        out += b'\xff\xdb\x00\x43' + bytes([c]) + bytes([1 + (k % 7) for k in range(64)])
    out += b'\xff\xc2' + (17).to_bytes(2, 'big') + b'\x08' + height.to_bytes(2, 'big') + width.to_bytes(2, 'big') + b'\x03'
    for c in range(3):
        out += bytes([c + 1, (sampling[c][0] << 4) | sampling[c][1], c])
    out += _table(0, 0, DC_SYMS) + _table(1, 0, ac_syms, ac_bits)
    if ri:
        out += b'\xff\xdd\x00\x04' + ri.to_bytes(2, 'big')
    for comps, ss, se, ah, al, data in scans:
        out += b'\xff\xda' + (6 + 2 * len(comps)).to_bytes(2, 'big') + bytes([len(comps)])
        out += b''.join(bytes([c + 1, 0x00]) for c in comps) + bytes([ss, se, (ah << 4) | al])
        if len(comps) > 1:
            units = mcux * mcuy
            bpm = sum(sampling[c][0] * sampling[c][1] for c in comps)
        else:
            c = comps[0]
            units = -(-(-(-width * sampling[c][0] // maxh)) // 8) * -(-(-(-height * sampling[c][1] // maxv)) // 8)
            bpm = 1
        nseg = -(-units // ri) if ri else 1
        for k in range(nseg):
            if isinstance(data, str):
                raw = bits_to_bytes(data)
            else:
                blocks = (min(ri, units - k * ri) if ri else units) * bpm
                n = data if isinstance(data, int) else max(1, blocks * (1 if ss == 0 else 2) * int(rng.integers(1, 4)) // 4)
                raw = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
            out += _stuff(raw)
            if k + 1 < nseg:
                out += bytes([0xFF, 0xD0 + (k & 7)])
    return bytes(out + b'\xff\xd9')


ALL3 = [0, 1, 2]
# libjpeg's standard script (what Pillow writes for progressive=True, 4:2:0 or 4:4:4)
STANDARD = [(ALL3, 0, 0, 0, 1, None), ([0], 1, 5, 0, 2, None), ([2], 1, 63, 0, 1, None), ([1], 1, 63, 0, 1, None),
            ([0], 6, 63, 0, 2, None), ([0], 1, 63, 2, 1, None), (ALL3, 0, 0, 1, 0, None), ([2], 1, 63, 1, 0, None),
            ([1], 1, 63, 1, 0, None), ([0], 1, 63, 1, 0, None)]
# non-interleaved DC scans and successive approximation from Al = 13 down to 0, in narrow bands
DEEP = ([([c], 0, 0, 0, 13, None) for c in ALL3] + [(ALL3, 0, 0, a + 1, a, None) for a in (12, 9, 5, 0)]
        + [([c], lo, hi, 0, 13, None) for c in ALL3 for lo, hi in ((1, 1), (2, 3), (4, 9), (10, 20), (21, 63))]
        + [([c], lo, hi, a + 1, a, None) for c in (0, 1) for a in (12, 7, 0) for lo, hi in ((1, 2), (3, 63))])
# a refine scan of a band no first scan coded, a component never scanned
ODD = [([0, 1], 0, 0, 0, 0, None), ([0], 1, 10, 3, 2, None), ([1], 5, 63, 0, 0, None), ([1], 1, 63, 1, 0, None),
       ([0], 11, 63, 0, 0, None), ([0], 11, 63, 5, 4, None)]

S420, S444, S422 = [(2, 2), (1, 1), (1, 1)], [(1, 1)] * 3, [(2, 1), (1, 1), (1, 1)]


def eob_bits(r, extra):
    """The AC symbol EOBr (r 0..14) followed by its r extra bits (the run is 2^r + extra)."""
    return _sym_bits(AC_SYMS, r << 4) + (format(extra, f'0{r}b') if r else '')


def crafted():
    """name -> bytes: scripts Pillow cannot write and one file per quirk of the reader."""
    cases = {}
    for k, (w, h, s) in enumerate([(64, 48, S420), (97, 61, S444), (32, 70, S422), (8, 8, S444), (16, 16, S420)]):
        cases[f'standard_random_{k}'] = write(w, h, s, STANDARD, seed=k)
        cases[f'deep_{k}'] = write(w, h, s, DEEP, seed=10 + k)
        cases[f'odd_{k}'] = write(w, h, s, ODD, seed=20 + k)
        for ri in (1, 3):
            cases[f'standard_ri{ri}_{k}'] = write(w, h, s, STANDARD, ri=ri, seed=30 + k)
    cases['deep_ri2'] = write(80, 48, S420, DEEP, ri=2, seed=40)
    # an EOB run of 32767 in AC first and AC refine scans, past the scan's end; across restarts
    run = eob_bits(14, (1 << 14) - 1)
    first_dc = (ALL3, 0, 0, 0, 0, None)
    cases['eob_32767'] = write(256, 256, S444, [first_dc, ([0], 1, 63, 0, 1, '0001' * 40 + run), ([0], 1, 63, 1, 0, '0001' * 40 + run)], seed=50)
    cases['eob_runs_cross_restarts'] = write(64, 64, S444, [first_dc, ([0], 1, 63, 0, 1, None), ([0], 1, 63, 1, 0, None)], ri=5, seed=51,
                                             ac_syms=[0x00, 0x10, 0x20, 0x30, 0x40, 0x50, 0x60, 0x70, 0x01, 0x11, 0x21, 0x02, 0xF0, 0x03, 0x31, 0x12])
    # a run landing past Se: Se = 5, the symbol (r = 10, s = 1) at k = 1 stores at k = 11
    cases['run_past_se'] = write(8, 8, S444, [first_dc, ([0], 1, 5, 0, 0, _sym_bits(AC_SYMS, 0xA1) + '1' + '0000')], seed=52)
    # a refine symbol of size 2 and 3 places +-1 all the same
    cases['refine_size_2_3'] = write(8, 8, S444, [first_dc, ([0], 1, 63, 1, 0, _sym_bits(AC_SYMS, 0x02) + '1' + _sym_bits(AC_SYMS, 0x03) + '0'
                                                             + '0000')], seed=53)
    # failures: k > 63 after a run; a code no table has; a DC category of 17
    cases['bad_index'] = write(8, 8, S444, [first_dc, ([0], 60, 63, 0, 0, _sym_bits(AC_SYMS, 0x71) + '1')], seed=54)
    short = [0, 0, 0, 15] + [0] * 12                    # 15 codes of 4 bits: 1111 is no code
    cases['bad_code'] = write(16, 16, S444, [first_dc, ([0], 1, 63, 0, 0, '1111' * 8)], seed=55, ac_syms=AC_SYMS[:15], ac_bits=short)
    cases['bad_code_refine'] = write(16, 16, S444, [first_dc, ([0], 1, 63, 1, 0, '1111' * 8)], seed=56, ac_syms=AC_SYMS[:15], ac_bits=short)
    big = bytearray(write(8, 8, S444, [(ALL3, 0, 0, 0, 0, '0001' + '1' * 8)], seed=57))
    i = big.index(b'\xff\xc4\x00\x23\x00') + 5 + 16           # the DC table's symbols: make category 1 read 17
    big[i + 1] = 17
    cases['dc_category_17'] = bytes(big)
    return cases


def pillow_grid(sizes=((1, 1), (7, 9), (64, 48), (97, 61), (1023, 769)), qualities=(5, 20, 50, 75, 90, 100)):
    """Pillow progressive files at every sampling, with and without optimize."""
    out = {}
    for w, h in sizes:
        for q in qualities:
            for ss in ('4:4:4', '4:2:2', '4:2:0'):
                for opt in (False, True):
                    if (w, h) == (1023, 769) and (q not in (20, 90) or ss == '4:2:2'):
                        continue                            # keep the big size to a few
                    out[f'pillow_{w}x{h}_q{q}_{ss}_{"opt" if opt else "std"}'] = E.pillow(w, h, q, ss, optimize=opt, progressive=True,
                                                                                             seed=w + q)
    return out


def pillow_restarts(w, h, q, ss, optimize=False, seed=1, rows=1):
    """A Pillow progressive file with a restart marker every `rows` MCU rows."""
    import io
    from PIL import Image
    from jpeg2png_b200 import synth
    buf = io.BytesIO()
    Image.fromarray(synth.cartoon_image(w, h, seed).astype(np.uint8), 'RGB').save(
        buf, 'JPEG', quality=q, subsampling=ss, optimize=optimize, progressive=True, restart_marker_rows=rows)
    return buf.getvalue()


# ---- decoding through the library ------------------------------------------------------------
def prog_host(layouts, subseq_bits):
    """Decode ProgFileLayouts with the serial host driver: ([per file: 3 int16 arrays], statuses, stats)."""
    arrs, outs = [], []
    for lay in layouts:
        planes = [np.full(p.w * p.h, 0x5a5a, np.int16) for p in lay.planes]      # the decoder zeroes them
        arrs.append(planes)
        outs += [a.ctypes.data for a in planes]
    buf, addr, _, work_bytes = D.progressive_plan(layouts, outs, subseq_bits)
    work = np.zeros(work_bytes + 16, np.uint8)
    status = np.zeros(max(len(layouts), 1), np.uint32)
    stats = D.ProgressiveStats()
    lib = D.load_progressive()
    assert lib.j2p_progressive_decode_host(addr, (work.ctypes.data + 15) & ~15, status.ctypes.data, C.byref(stats)) == 0, \
        lib.j2p_progressive_last_error()
    return arrs, status[:len(layouts)], stats


def layout(data):
    """The progressive layout of data, or None when the layout pass rejects it."""
    try:
        return D.ProgFileLayout(data)
    except ValueError:
        return None
