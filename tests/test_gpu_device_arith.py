"""The device arithmetic of the solver and the device-only paths of the codec cores, run on the GPU
through tests/device_probe (libj2pprobe.so), which includes the real headers and is compiled with
the solver's floating-point flags.

- numerics.cuh: the IEEE instructions themselves against numpy; sqrt_core / rcp_core and their
  packed forms over every fp32 in [2^-80, 2^80]; the gradient's divisor pipeline; every division
  sequence over its whole guard box; the guards and keys at their endpoints.
- project_common.cuh: the 8-lane 8x8 transforms bit for bit against the reference's own transforms
  and within an fp32 rounding bound of the orthonormal DCT-II; the steppers against IEEE division.
- jpegopt_core.h's WarpLanes table builder, progressive_core.h's j2p_pg_nth and entropy_core.h's
  j2p_ent_word, which the device compiles differently from their host twins.

Results are compared bit for bit.  The one exclusion is the sign of a zero quotient, which the
fast division sequences do not keep (numerics.cuh; no such zero reaches a pixel, DESIGN.md §5)."""
import ctypes as C
import os
import time
import zlib

import numpy as np
import pytest

from jpeg2png_b200 import jpeg_encode as J
from tests import helpers as H
from tests import jpegopt_cases as OC

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE = os.path.join(ROOT, 'tests', 'device_probe', 'libj2pprobe.so')
P = C.c_void_p
U32MAX = 0xffffffff


class Tally(C.Structure):
    _fields_ = [('checked', C.c_uint64), ('bad', C.c_uint64 * 8), ('nex', C.c_uint), ('ex', (C.c_uint * 5) * 8)]


_lib = None


def probe():
    global _lib
    if _lib is None:
        lib = C.CDLL(PROBE)
        for name, args in (('probe_ieee', [P, P, C.c_size_t, P, P, P]), ('probe_guards', [P, C.c_size_t, P, P]),
                           ('probe_roots', [C.c_uint32, C.c_uint32, P]), ('probe_div', [P, P, C.c_size_t, P]),
                           ('probe_grad_div', [P, P, P, C.c_size_t, P]), ('probe_dct', [C.c_int, P, C.c_uint32, P, P]),
                           ('probe_stepper', [C.c_float, C.c_float, C.c_float, C.c_int, P, P, P, C.c_size_t, P, P, P, P, P]),
                           ('probe_jo_tables', [P, C.c_uint32, P, P, P, P, P, P]), ('probe_pg_nth', [P, C.c_size_t, P, P]),
                           ('probe_ent_word', [P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, P]),
                           ('probe_ent_word_host', [P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, P])):
            getattr(lib, name).argtypes = args
            getattr(lib, name).restype = C.c_int
        lib.probe_pg_nth_host.argtypes = [P, C.c_size_t, P, P]
        lib.probe_pg_nth_host.restype = None
        lib.probe_constants.argtypes = [P]
        lib.probe_constants.restype = None
        lib.probe_last_error.restype = C.c_char_p
        _lib = lib
    return _lib


def call(name, *args):
    lib = probe()
    assert getattr(lib, name)(*[a.ctypes.data if isinstance(a, np.ndarray) else a for a in args]) == 0, lib.probe_last_error().decode()


def f32(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def run_tally(name, *args):
    t = Tally()
    call(name, *args, C.addressof(t))
    return t


def check_tally(t, names, n, what):
    """The kernels ran all n arguments and no sequence mismatched; else the counts and the first
    mismatches, as hex floats."""
    hexf = lambda b: float(f32(b)).hex()
    assert t.checked == n, f'{what}: the probe checked {t.checked} of {n}'
    if any(t.bad[k] for k in range(len(names))):
        lines = [f'{what}: mismatches ' + ', '.join(f'{n} {t.bad[k]}' for k, n in enumerate(names) if t.bad[k])]
        for e in list(t.ex)[:min(t.nex, 8)]:
            lines.append(f'  {names[e[0]]}: operands {hexf(e[1])}, {hexf(e[2])}: got {hexf(e[3])}, IEEE {hexf(e[4])}')
        pytest.fail('\n'.join(lines))


# ---- the IEEE instructions are IEEE in this build ----------------------------------------------
def test_ieee_instructions_equal_numpy():
    """__fdiv_rn / __fsqrt_rn / __frcp_rn, the references of every check below, against numpy's
    float32 `/`, sqrt and 1/x on four million random bit patterns (every class: subnormals, zeros,
    infinities, NaNs) and the boundary values.  NaN results compare as NaN: the device writes the
    canonical NaN and the CPU propagates an operand's payload, and no payload is part of IEEE 754's
    result."""
    rng = np.random.default_rng(1)
    n = 1 << 22
    special = f32([0, 0x80000000, 1, 0x80000001, 0x007fffff, 0x00800000, 0x7f7fffff, 0x7f800000, 0xff800000, 0x7fc00000,
                   0x3f800000, 0xbf800000, 0x17800000, 0x67800000, 0x2b800000, 0x53800000, 0x21800000, 0x5d800000])
    a = np.concatenate([np.repeat(special, special.size), f32(rng.integers(0, 1 << 32, n, dtype=np.uint64))])
    b = np.concatenate([np.tile(special, special.size), f32(rng.integers(0, 1 << 32, n, dtype=np.uint64))])
    q, s, r = (np.empty_like(a) for _ in range(3))
    call('probe_ieee', a, b, a.size, q, s, r)
    with np.errstate(all='ignore'):
        want = {'div': a / b, 'sqrt': np.sqrt(a), 'rcp': np.float32(1) / a}
    for name, got in (('div', q), ('sqrt', s), ('rcp', r)):
        w = want[name]
        bad = (bits(got) != bits(w)) & ~(np.isnan(got) & np.isnan(w))
        assert not bad.any(), f'{name}: {bad.sum()} differ from numpy, first at a={a[bad][0]!r} b={b[bad][0]!r}: {got[bad][0]!r} vs {w[bad][0]!r}'


# ---- guards and keys ---------------------------------------------------------------------------
def _edges():
    """Every guard endpoint, its neighbours, and the special classes."""
    pts = [2.0 ** -80, 2.0 ** 80, 2.0 ** -60, 2.0 ** 60, 2.0 ** -40, 2.0 ** 40, 2.0 ** -35, 1.0]
    out = []
    for p in pts:
        p = np.float32(p)
        out += [p, np.nextafter(p, np.float32(0)), np.nextafter(p, np.float32(np.inf))]
    out = np.array(out, np.float32)
    out = np.concatenate([out, -out, f32([0, 0x80000000, 1, 0x80000001, 0x007fffff, 0x807fffff, 0x00800000, 0x7f7fffff,
                                          0x7f800000, 0xff800000, 0x7fc00000, 0xffc00000])])
    rng = np.random.default_rng(2)
    return np.concatenate([out, f32(rng.integers(0, 1 << 32, 1 << 20, dtype=np.uint64))])


def test_guards_accept_exactly_their_intervals():
    """root_arg_ok: [2^-80, 2^80]; qdiv_divisor_ok: [2^-40, 2^40]; qdiv_fast's ok for a numerator:
    0, -0 or |a| in [2^-60, 2^60].  Endpoints in, their nextafters out, subnormals, inf and NaN out."""
    x = _edges()
    flags, keys = np.empty(x.size, np.uint32), np.empty(x.size, np.uint32)
    call('probe_guards', x, x.size, flags, keys)
    with np.errstate(invalid='ignore'):
        want = {'root_arg_ok': (x >= 2.0 ** -80) & (x <= 2.0 ** 80), 'qdiv_divisor_ok': (x >= 2.0 ** -40) & (x <= 2.0 ** 40),
                'qdiv_fast ok': ((np.abs(x) >= 2.0 ** -60) & (np.abs(x) <= 2.0 ** 60)) | (x == 0)}
    for bit, (name, w) in enumerate(want.items()):
        got = (flags >> bit & 1).astype(bool)
        bad = got != w
        assert not bad.any(), f'{name} wrong on {[float(v).hex() for v in x[bad][:8]]}'
    # the endpoints themselves are in and their outer neighbours out
    for name, lo, hi in (('root_arg_ok', -80, 80), ('qdiv_divisor_ok', -40, 40)):
        g = dict(zip(('root_arg_ok', 'qdiv_divisor_ok'), (flags & 1, flags >> 1 & 1)))[name]
        at = lambda v: int(g[np.flatnonzero(bits(x) == bits(np.float32(v)))[0]])
        assert at(2.0 ** lo) == 1 and at(2.0 ** hi) == 1, name
        assert at(np.nextafter(np.float32(2.0 ** lo), np.float32(0))) == 0, name
        assert at(np.nextafter(np.float32(2.0 ** hi), np.float32(np.inf))) == 0, name


def test_qdiv_key_orders_magnitudes_and_constants_are_the_documented_keys():
    """key(a) = 2 bits(a) - 1: +-0 go to UINT_MAX, finite nonzero magnitudes keep their order (and
    equal magnitudes of either sign share a key), and QDIV_KEY_MIN / QDIV_YKEY_MIN are the keys the
    device computes for 2^-60 and 2^-35."""
    x = _edges()
    x = x[np.isfinite(x)]
    flags, keys = np.empty(x.size, np.uint32), np.empty(x.size, np.uint32)
    call('probe_guards', x, x.size, flags, keys)
    assert np.array_equal(keys, (bits(x).astype(np.uint64) * 2 - 1).astype(np.uint32))        # key(a) = 2*bits(a) - 1
    zero = x == 0
    assert (keys[zero] == U32MAX).all()
    nz = ~zero
    order = np.argsort(np.abs(x[nz]).astype(np.float64), kind='stable')
    k = keys[nz][order].astype(np.int64)
    m = np.abs(x[nz][order]).astype(np.float64)
    assert (np.diff(k) >= 0).all() and ((np.diff(k) == 0) == (np.diff(m) == 0)).all()       # strictly with |a|
    assert (keys[nz] < U32MAX).all()
    const = np.empty(2, np.uint32)
    probe().probe_constants(const.ctypes.data)
    kk = np.empty(2, np.uint32)
    call('probe_guards', np.array([2.0 ** -60, 2.0 ** -35], np.float32), 2, np.empty(2, np.uint32), kk)
    assert list(const) == list(kk), (const, kk)                                          # QDIV_KEY_MIN, QDIV_YKEY_MIN


# ---- square root and reciprocal, exhaustively ----------------------------------------------------
ROOT_LO, ROOT_HI = 0x17800000, 0x67800000                  # 2^-80, 2^80


def test_roots_over_every_fp32_in_the_guard():
    """sqrt_core, rcp_core, rcp_core(sqrt_core(s)) and both halves of sqrt2_core / rcp2_core equal
    sqrt.rn / rcp.rn on every fp32 in [2^-80, 2^80], both endpoints included.  The hi half of the
    packed forms walks the same range in reverse."""
    assert float(f32(ROOT_LO)) == 2.0 ** -80 and float(f32(ROOT_HI)) == 2.0 ** 80
    n = ROOT_HI - ROOT_LO + 1
    assert n == 160 * (1 << 23) + 1
    t0 = time.perf_counter()
    t = run_tally('probe_roots', ROOT_LO, ROOT_HI)
    names = ['sqrt_core', 'rcp_core', 'rcp_core(sqrt_core)', 'sqrt2_core lo', 'sqrt2_core hi', 'rcp2_core lo', 'rcp2_core hi']
    check_tally(t, names, n, 'roots')
    print(f'\nroots: {n:,} arguments x {len(names)} sequences, 0 mismatches ({time.perf_counter() - t0:.2f} s)')


# ---- division --------------------------------------------------------------------------------
A_LO, A_HI, B_LO, B_HI = 2.0 ** -60, 2.0 ** 60, 2.0 ** -40, 2.0 ** 40
DIV_SEQS = ['qdiv_fast', 'qdiv_fast ok', 'qdiv_core', 'qdiv2 lo', 'qdiv2 hi', 'qdiv4_core', 'qdiv2x lo', 'qdiv2x hi']


def _mk(sign, e, m):
    return f32((np.asarray(sign, np.uint32) << 31) | ((np.asarray(e, np.int64) + 127).astype(np.uint32) << 23) | np.asarray(m, np.uint32))


def in_guard(a, b):
    aa = np.abs(a)
    return (b >= B_LO) & (b <= B_HI) & ((a == 0) | ((aa >= A_LO) & (aa <= A_HI)))


def _nudge(a, rng):
    """a moved by up to two ulps either way (on the bit pattern of |a|)."""
    return f32((bits(a).astype(np.int64) + rng.integers(-2, 3, a.size)).astype(np.uint32))


def div_operands(kind, n, rng):
    """n (a, b) pairs of one distribution, all inside the guard."""
    sa = rng.integers(0, 2, n)
    ma, mb = rng.integers(0, 1 << 23, n), rng.integers(0, 1 << 23, n)
    ea, eb = rng.integers(-60, 60, n), rng.integers(-40, 40, n)      # |a| in [2^-60, 2^60), b in [2^-40, 2^40)
    if kind == 'uniform':
        a, b = _mk(sa, ea, ma), _mk(0, eb, mb)
    elif kind == 'corners':                                          # both from the outermost binades: quotients near 2^+-100
        a, b = _mk(sa, rng.choice([-60, 59], n), ma), _mk(0, rng.choice([-40, 39], n), mb)
    elif kind == 'endpoints':                                        # a = +-2^-60, +-2^60 or b = 2^-40, 2^40, the other random
        ends_a = np.array([A_LO, -A_LO, A_HI, -A_HI], np.float32)
        ends_b = np.array([B_LO, B_HI], np.float32)
        a, b = _mk(sa, ea, ma), _mk(0, eb, mb)
        pick = rng.integers(0, 3, n)
        a = np.where(pick != 1, ends_a[rng.integers(0, 4, n)], a)
        b = np.where(pick != 0, ends_b[rng.integers(0, 2, n)], b)
        a[:8] = np.repeat(ends_a, 2)
        b[:8] = np.tile(ends_b, 4)
    elif kind == 'divisor significands':                              # near all-ones / all-zeros, numerators random or extreme
        r = rng.integers(0, 64, n)
        mb = np.where(rng.integers(0, 2, n) == 1, (1 << 23) - 1 - r, r)
        ext = rng.integers(0, 3, n)
        ma = np.where(ext == 1, (1 << 23) - 1 - rng.integers(0, 256, n), np.where(ext == 2, rng.integers(0, 256, n), ma))
        a, b = _mk(sa, ea, ma), _mk(0, eb, mb)
    elif kind in ('midpoints', 'exact'):
        b = _mk(0, eb, mb if kind == 'midpoints' else rng.integers(0, 1 << 11, n) << 12)
        k = rng.integers(-60 - eb, 59 - eb)                           # the quotient's binade: a lands in [2^-60, 2^60]
        if kind == 'midpoints':                                       # quotient next to halfway between two floats
            m = ((1 << 23) + rng.integers(0, 1 << 23, n) + 0.5) * 2.0 ** -23
            a = _nudge((b.astype(np.float64) * m * np.exp2(k)).astype(np.float32), rng)
        else:                                                         # 12-bit significands: the product is exact
            m = ((1 << 11) + rng.integers(0, 1 << 11, n)) * 2.0 ** -11
            a = (b.astype(np.float64) * m * np.exp2(k)).astype(np.float32)
            assert (a.astype(np.float64) == b.astype(np.float64) * m * np.exp2(k)).all()
        a = np.where(sa == 1, -a, a)
    elif kind == 'hard midpoints':
        # a/b within |t| 2^-48 (relative) of the midpoint M 2^-s of two floats: the divisor's significand
        # B is odd, M is an odd 25-bit significand with B M = t (mod 2^25) for a small odd t, and
        # a = A = round(B M / 2^s) is a float.  Only such quotients tell a faithful rounding from the
        # correct one: random pairs come this close about once in ten million.
        B = rng.integers(1 << 22, 1 << 23, 2 * n).astype(np.uint64) * np.uint64(2) + np.uint64(1)
        inv = B.copy()                                                # B^-1 mod 2^64 (Newton: 3 -> 96 correct bits)
        for _ in range(5):
            inv = inv * (np.uint64(2) - B * inv)
        t = (rng.integers(1, 3, 2 * n) * 2 - 1) * rng.choice([-1, 1], 2 * n)          # +-1, +-3
        M = (t.astype(np.int64).astype(np.uint64) * inv) & np.uint64((1 << 25) - 1)
        use = np.flatnonzero(M >= np.uint64(1 << 24))[:n]
        B, M = B[use], M[use]
        P = B * M
        s = np.where(P >= np.uint64(1 << 48), np.uint64(25), np.uint64(24))
        A = (P + (np.uint64(1) << (s - np.uint64(1)))) >> s
        assert ((P - (A << s)).astype(np.int64) == t[use]).all()
        m = use.size
        a = (A.astype(np.float64) * np.exp2(rng.integers(-83, 37, m))).astype(np.float32)
        b = (B.astype(np.float64) * np.exp2(rng.integers(-63, 17, m))).astype(np.float32)
        a = np.where(sa[:m] == 1, -a, a)
    elif kind == 'a = 0':
        a, b = np.where(sa == 1, np.float32(-0.0), np.float32(0.0)), _mk(0, eb, mb)
    else:
        raise ValueError(kind)
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    keep = in_guard(a, b)
    assert keep.mean() > 0.99, (kind, keep.mean())
    return a[keep], b[keep]


# (distribution, calls of 2^22 pairs)
DIV_PLAN = (('uniform', 16), ('corners', 8), ('endpoints', 4), ('divisor significands', 8), ('midpoints', 12), ('hard midpoints', 8),
            ('exact', 4), ('a = 0', 2))


def test_division_sequences_equal_div_rn_over_the_guard():
    """qdiv_fast (and its ok), qdiv_core, qdiv2, qdiv4_core with rcp_low and qdiv2x with rcp2_low equal
    div.rn.f32 on seeded pairs over the whole guard box |a| in [2^-60, 2^60] or 0, b in [2^-40, 2^40]."""
    rng = np.random.default_rng(3)
    total, t0 = {}, time.perf_counter()
    for kind, calls in DIV_PLAN:
        for _ in range(calls):
            a, b = div_operands(kind, 1 << 22, rng)
            t = run_tally('probe_div', a, b, a.size)
            check_tally(t, DIV_SEQS, a.size, kind)
            total[kind] = total.get(kind, 0) + a.size
    n = sum(total.values())
    print(f'\ndivision: {n:,} pairs checked per sequence ({", ".join(DIV_SEQS)}); '
          + ', '.join(f'{k} {v:,}' for k, v in total.items()) + f' ({time.perf_counter() - t0:.1f} s)')


def test_gradient_divisor_pipeline():
    """As k_gradient runs it: n = sqrt2_core(ss), y = rcp2_core(n, -n), yl = rcp2_low, qdiv2x(a, ...)
    equals RN(a / RN(sqrt(ss))) for ss in [2^-80, 2^80]; a dead source (ss = 1, y = 0) gives a zero
    quotient for every a."""
    rng = np.random.default_rng(4)
    n, done = 1 << 22, 0
    for rep in range(4):
        ss = _mk(0, rng.integers(-80, 80, n), rng.integers(0, 1 << 23, n))
        ss[:2] = [2.0 ** -80, 2.0 ** 80]
        a, _ = div_operands(('uniform', 'corners', 'midpoints', 'a = 0')[rep], n, rng)
        ss = ss[:a.size].copy()
        live = (rng.random(a.size) < 0.9).astype(np.uint8)
        if rep == 0:                                             # dead sources see every kind of numerator
            a[:64] = [0.0, -0.0, A_LO, -A_LO, A_HI, -A_HI, 1.0, -1.0] * 8
            live[:64] = 0
        ss[live == 0] = 1.0
        assert ((ss >= 2.0 ** -80) & (ss <= 2.0 ** 80)).all()
        t = run_tally('probe_grad_div', ss, a, live, a.size)
        check_tally(t, ['qdiv2x lo', 'qdiv2x hi'], a.size, 'gradient pipeline')
        done += a.size
    print(f'\ngradient divisor pipeline: {done:,} (ss, a) pairs, both halves')


# ---- the 8x8 transforms ------------------------------------------------------------------------
def _aligned(n):
    raw = np.empty(n + 16, np.float32)
    off = (-raw.ctypes.data % 64) // 4
    return raw[off:off + n]


def reference_transform(kind, blocks):
    """dct8x8s / idct8x8s of the reference where it is built, else the oracle's restatement."""
    if H.have_ref():
        lib = H.load_ref()
        fn = lib.dct8x8s if kind == 'fdct' else lib.idct8x8s
    else:
        lib = H.load_oracle()
        fn = lib.oracle_dct8x8 if kind == 'fdct' else lib.oracle_idct8x8
    buf = _aligned(64)
    out = np.empty_like(blocks)
    for i in range(blocks.shape[0]):
        buf[:] = blocks[i].ravel()
        fn(buf.ctypes.data)
        out[i] = buf.reshape(8, 8)
    return out


def transform_inputs(kind, n, rng):
    """n 8x8 float32 blocks."""
    sgn = np.where(rng.integers(0, 2, (n, 8, 8)) == 1, -1, 1).astype(np.float32)
    if kind == 'pixels':
        x = rng.uniform(-128, 128, (n, 8, 8)).astype(np.float32)
        x[::2] = np.round(x[::2])
    elif kind == 'dequantised':                                   # int16 coefficient x a 16-bit table entry, as fp32
        d = rng.integers(-32768, 32768, (n, 8, 8)).astype(np.float32)
        q = rng.integers(1, 65536, (n, 8, 8)).astype(np.float32)
        x = d * q
        x[0::4, 0, 0] = np.float32(-32768) * np.float32(65535)
        x[1::4, 0, 0] = np.float32(32767) * np.float32(65535)
        x[2::4] = np.float32(-32768) * np.float32(65535) * sgn[2::4]
    elif kind == 'mixed magnitudes':                              # 2^-149 .. 2^31 in one block
        e = rng.uniform(-149, 31, (n, 8, 8))
        x = (np.exp2(np.floor(e)) * rng.uniform(1, 2, (n, 8, 8))).astype(np.float32) * sgn
    elif kind == 'subnormals and zeros':
        x = f32(rng.integers(1, 1 << 23, (n, 8, 8))) * sgn
        z = rng.random((n, 8, 8))
        x = np.where(z < 0.3, np.float32(0) * sgn, x)              # +0 and -0
        x[1::4] = np.float32(0) * sgn[1::4]                        # blocks of signed zeros only
        x[2::8] = np.float32(-0.0)
        x[3::8] = np.float32(0.0)
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(x, np.float32)


TRANSFORM_INPUTS = ('pixels', 'dequantised', 'mixed magnitudes', 'subnormals and zeros')


def _dct_matrix():
    k, m = np.meshgrid(np.arange(8), np.arange(8), indexing='ij')
    c = np.cos(np.pi * (2 * m + 1) * k / 16) * np.where(k == 0, np.sqrt(1 / 8), np.sqrt(2 / 8))
    return c


@pytest.mark.parametrize('inputs', TRANSFORM_INPUTS)
@pytest.mark.parametrize('kind', ['fdct8x8_rows', 'idct8x8_rows', 'idct8x8_rows_x2'])
def test_transforms_equal_the_reference(kind, inputs):
    """The 8-lane transforms (lane j holds row j, four blocks per warp, tiles TILE_STRIDE apart) equal
    the reference's dct8x8s / idct8x8s bit for bit, signed zeros included: once with every group
    active and, for the masked forms, once with partial group masks in which some groups idle (an
    idle group's block is left as it was)."""
    rng = np.random.default_rng(zlib.crc32(f'{kind} {inputs}'.encode()))
    n = 2048
    x = transform_inputs(inputs, n, rng)
    want = reference_transform('fdct' if kind == 'fdct8x8_rows' else 'idct', x)
    code = {'fdct8x8_rows': 0, 'idct8x8_rows': 1, 'idct8x8_rows_x2': 2}[kind]
    runs = [None] if code == 2 else [None, rng.integers(0, 16, n // 4).astype(np.uint8)]
    if code != 2:
        runs[1][:16] = np.arange(16)                              # every pattern of idle groups
    for active in runs:
        sentinel = np.full_like(x, f32(0x7fc0dead))
        out = sentinel.copy()
        call('probe_dct', code, x, n, active, out)
        on = np.ones(n, bool) if active is None else ((active[:, None] >> np.arange(4)) & 1).astype(bool).ravel()
        assert (bits(out[~on]) == bits(sentinel[~on])).all(), 'an idle group wrote its block'
        diff = bits(out[on]) != bits(want[on])
        if diff.any():
            i = np.argwhere(diff)[0]
            g, w = out[on][tuple(i)], want[on][tuple(i)]
            pytest.fail(f'{kind} on {inputs} ({"all groups" if active is None else "partial masks"}): {diff.sum()} of {diff.size} '
                        f'values differ; block {i[0]} ({i[1]}, {i[2]}): {float(g).hex()} against {float(w).hex()}')
    print(f'\n{kind} on {inputs}: {n * len(runs)} blocks')


@pytest.mark.parametrize('inputs', ['pixels', 'dequantised'])
@pytest.mark.parametrize('kind', ['fdct8x8_rows', 'idct8x8_rows'])
def test_transforms_compute_the_orthonormal_dct(kind, inputs):
    """The same wiring computes the orthonormal 8x8 DCT-II (C x C^T, C[k, n] = s_k cos(pi (2n + 1) k / 16))
    and its inverse in float64 to within fp32 rounding, u = 2^-24.  A 1-D pass rounds at most six times
    on the way to an output, and every intermediate is at most 1.5 times the sum of its |inputs|, so
    it adds at most 9u times that sum.  The first pass's outputs sum to at most 4 sum|x| (|C| <= 1/2),
    and the second pass amplifies their errors by at most max_k sum_n |C[k, n]| < 2 sqrt(2).  So per
    block |error| <= (9 * 2 sqrt(2) + 9 * 4) u sum|x| < 64u sum|x|; the test allows twice that,
    2^-17 sum|x|.  A transform wired wrongly is off by about the values themselves."""
    rng = np.random.default_rng(7)
    n = 1024
    x = transform_inputs(inputs, n, rng)
    code = 0 if kind == 'fdct8x8_rows' else 1
    out = np.zeros_like(x)
    call('probe_dct', code, x, n, None, out)
    c = _dct_matrix()
    xd = x.astype(np.float64)
    want = c @ xd @ c.T if code == 0 else c.T @ xd @ c
    err = np.abs(out.astype(np.float64) - want).max(axis=(1, 2))
    bound = 2.0 ** -17 * np.abs(xd).sum(axis=(1, 2))
    assert (err <= bound).all(), f'{kind}: error {err.max()} against bound {bound[np.argmax(err - bound)]}'


# ---- the steppers ------------------------------------------------------------------------------
def _stepper_values(rng, n):
    """Pixel values with +-0, subnormals and the guard's edges mixed in."""
    x = rng.uniform(-300, 600, n).astype(np.float32)
    sp = np.array([0.0, -0.0, 2.0 ** -149, -(2.0 ** -149), 2.0 ** -126, 1e-30, -1e-30, 255.0], np.float32)
    pick = rng.random(n) < 0.2
    x[pick] = sp[rng.integers(0, sp.size, pick.sum())]
    return x


def _gradients(rng, n):
    """Gradient values: ordinary, tiny (below 2^-60, outside the guard), +0 and large; never -0, which
    the gradient kernel does not produce (project_common.cuh, Stepper2)."""
    e = rng.integers(-70, 30, n)
    g = _mk(rng.integers(0, 2, n), e, rng.integers(0, 1 << 23, n))
    g[rng.random(n) < 0.05] = 0.0
    g[rng.random(n) < 0.01] = np.float32(2.0 ** -149)
    return g


def _run_stepper(factor, step, norm, stepping, x, xp, g):
    n = x.size
    ieee, fast, fast2 = (np.empty(n, np.float32) for _ in range(3))
    key, key2 = np.empty(n, np.uint32), np.empty(n // 2, np.uint32)
    call('probe_stepper', float(factor), float(step), float(norm), int(stepping), x, xp, g, n, ieee, fast, key, fast2, key2)
    return ieee, fast, key, fast2, key2


def _keys(g):
    return (bits(g).astype(np.uint64) * 2 - 1).astype(np.uint32)


@pytest.mark.parametrize('norm', [123.456, 2.0 ** -40, 2.0 ** 40, 0.0371, 2.0 ** -41, 2.0 ** 41])
def test_steppers_equal_ieee_inside_the_guard(norm):
    """Stepper::fast and both halves of Stepper2::fast equal Stepper::operator() (IEEE division) bit
    for bit wherever the guard holds (qdiv_divisor_ok(norm), key >= QDIV_KEY_MIN); the keys are the
    minimum of qdiv_key(g); and operator() is y = x + f (x - xp) - step (g / norm) in float32 as numpy
    computes it."""
    rng = np.random.default_rng(int(np.float32(norm).view(np.uint32)))
    n = 1 << 20
    x, xp, g = _stepper_values(rng, n), _stepper_values(rng, n), _gradients(rng, n)
    factor, step = np.float32(0.6180339), np.float32(0.3719)
    ieee, fast, key, fast2, key2 = _run_stepper(factor, step, norm, True, x, xp, g)
    with np.errstate(all='ignore'):
        y = x + factor * (x - xp)
        want = y - step * (g / np.float32(norm))
    assert (bits(ieee) == bits(want)).all(), 'Stepper::operator() is not the float32 formula'
    kmin = np.empty(2, np.uint32)
    probe().probe_constants(kmin.ctypes.data)
    k = _keys(g)
    assert (key == k).all() and (key2 == np.minimum(k[0::2], k[1::2])).all()
    norm_ok = 2.0 ** -40 <= norm <= 2.0 ** 40
    if not norm_ok:
        return
    ok1 = key >= kmin[0]
    ok2 = np.repeat(key2 >= kmin[0], 2)
    assert ok1.mean() > 0.8 and ok2.mean() > 0.6
    assert (bits(fast[ok1]) == bits(ieee[ok1])).all(), 'Stepper::fast differs from IEEE division inside the guard'
    bad = ok2 & (bits(fast2) != bits(ieee))
    assert not bad.any(), f'Stepper2::fast differs inside the guard: x={x[bad][0]!r} xp={xp[bad][0]!r} g={g[bad][0]!r}'


def test_stepper2_leaves_y_untouched_when_not_stepping():
    """With stepping false (a zero norm) and g = +0, Stepper2::fast returns x + f (x - xp) exactly for
    every x and xp, +-0 and subnormals included, as Stepper does."""
    rng = np.random.default_rng(9)
    n = 1 << 20
    x, xp = _stepper_values(rng, n), _stepper_values(rng, n)
    sp = np.array([0.0, -0.0, 2.0 ** -149, -(2.0 ** -149), 2.0 ** -130], np.float32)
    m = np.array(np.meshgrid(sp, sp)).reshape(2, -1)               # every pair of the special values
    x[:m.shape[1]], xp[:m.shape[1]] = m[0], m[1]
    g = np.zeros(n, np.float32)
    factor = np.float32(0.75)
    ieee, fast, key, fast2, key2 = _run_stepper(factor, 0.5, 0.0, False, x, xp, g)
    want = x + factor * (x - xp)
    assert (bits(ieee) == bits(want)).all()
    assert (bits(fast) == bits(want)).all()
    assert (bits(fast2) == bits(want)).all(), 'Stepper2 changed y on a zero norm'
    assert (key == U32MAX).all() and (key2 == U32MAX).all()


# ---- the warp table builder ----------------------------------------------------------------------
def _table_cases():
    out = dict(OC.crafted())
    rng = np.random.default_rng(12)
    for s in range(12):                                             # tied least counts in lanes with different residues mod 32
        c = rng.integers(2, 5000, 256) * (rng.random(256) < 0.7)
        lanes = rng.choice(32, size=int(rng.integers(2, 9)), replace=False)
        for ln in lanes:
            c[int(ln + 32 * rng.integers(0, 8))] = 1 + s % 2        # count 1 ties with the pseudo-symbol too
        out[f'ties across lanes {s}'] = [int(v) for v in c]
    for s in range(6):                                               # at and above 2^32, mixed with ones
        c = rng.integers(1 << 32, 1 << 40, 256)
        c[rng.random(256) < 0.3] = 1
        c[rng.random(256) < 0.1] = 1 << 32
        out[f'2^32 and ones {s}'] = [int(v) for v in c]
    out['257-way tie'] = [1] * 256                                   # every symbol and the pseudo-symbol at count 1
    out['257-way tie at 2^32'] = [1 << 32] * 256
    return out


def _annex_c(bits16, vals):
    code, size, c, p = [0] * 256, [0] * 256, 0, 0
    for length in range(1, 17):
        for _ in range(bits16[length - 1]):
            code[vals[p]], size[vals[p]] = c, length
            c += 1
            p += 1
        c <<= 1
    return code, size


def test_warp_table_builder_equals_serial_and_restatement():
    """j2p_jo_table on WarpLanes (one warp per table, four per CTA, scratch in shared memory, as
    k_jo_tables runs it) gives the serial builder's and the restatement's bits and vals, and Annex C's
    canonical codes of them.  The LONG cases make K.3 run on the device."""
    cases = _table_cases()
    names = list(cases)
    n = len(names)
    counts = np.array([cases[k] for k in names], np.uint64)
    bits16, vals, nvals = np.empty((n, 16), np.uint8), np.empty((n, 256), np.uint8), np.empty(n, np.uint32)
    code, size, top = np.empty((n, 256), np.uint16), np.empty((n, 256), np.uint8), np.empty(n, np.uint32)
    call('probe_jo_tables', counts, n, bits16, vals, nvals, code, size, top)
    for i, name in enumerate(names):
        got_bits, got_vals = list(bits16[i]), list(vals[i][:nvals[i]])
        want_bits, want_vals, longest = OC.restated_table(cases[name])
        got_bits, got_vals = [int(v) for v in got_bits], [int(v) for v in got_vals]
        assert (got_bits, got_vals) == (want_bits, want_vals), f'{name}: warp builder differs from the restatement'
        assert (got_bits, got_vals) == J.build_table(cases[name]), f'{name}: warp builder differs from the serial builder'
        want_code, want_size = _annex_c(got_bits, got_vals)
        assert list(code[i]) == want_code and list(size[i]) == want_size, f'{name}: codes'
        assert top[i] == longest, name
        if name in OC.LONG:
            assert top[i] > 16, f'{name}: K.3 did not run'
    assert sum(top[i] > 16 for i in range(n)) >= len(OC.LONG)
    print(f'\nwarp table builder: {n} tables')


# ---- j2p_pg_nth, J2P_PG_CTZ64 ---------------------------------------------------------------------
def test_pg_nth_and_ctz64():
    """Every n from 0 to 64 on 0, ~0, every single bit, low-word-only and high-word-only masks and
    seeded masks of every popcount, against a Python restatement (64: no such bit), on the device and
    through the host twin.  J2P_PG_CTZ64 on every nonzero mask."""
    rng = np.random.default_rng(13)
    ms = [0, (1 << 64) - 1] + [1 << b for b in range(64)]
    ms += [int(v) for v in rng.integers(1, 1 << 32, 64, dtype=np.uint64)]
    ms += [int(v) << 32 for v in rng.integers(1, 1 << 32, 64, dtype=np.uint64)]
    ms += [0xffffffff, 0xffffffff << 32, 0x80000000, 1 << 32, 0x80000001 << 31]
    for pc in range(65):
        for _ in range(8):
            ms.append(sum(1 << int(b) for b in rng.choice(64, pc, replace=False)))
    m = np.array(ms, np.uint64)
    want = np.full((m.size, 65), 64, np.int32)
    for i, v in enumerate(ms):
        pos = [b for b in range(64) if v >> b & 1]
        want[i, :len(pos)] = pos
    for entry in ('probe_pg_nth', 'probe_pg_nth_host'):
        nth, ctz = np.empty((m.size, 65), np.int32), np.empty(m.size, np.int32)
        if entry == 'probe_pg_nth':
            call(entry, m, m.size, nth, ctz)
        else:
            probe().probe_pg_nth_host(m.ctypes.data, m.size, nth.ctypes.data, ctz.ctypes.data)
        bad = np.argwhere(nth != want)
        assert bad.size == 0, f'{entry}: mask {ms[bad[0][0]]:#018x} n={bad[0][1]}: {nth[tuple(bad[0])]} against {want[tuple(bad[0])]}'
        nz = m != 0
        assert (ctz[nz] == want[nz, 0]).all(), entry


# ---- j2p_ent_word ----------------------------------------------------------------------------------
def test_ent_word_at_the_end_of_a_padded_segment():
    """Segments of 1 to 16 bytes at the end of a buffer, padded to 4 bytes with nonzero bytes as the
    packed plan pads them: every word, up to three wholly past the end (which read 0), equals the host
    twin and a big-endian restatement with the bytes past the segment zeroed."""
    rng = np.random.default_rng(14)
    for nbytes in range(1, 17):
        for rep in range(4):
            seg = rng.integers(0, 256, nbytes).astype(np.uint8)
            if rep == 1:
                seg[:] = 0xff
            pad = (-nbytes) % 4
            buf = np.concatenate([rng.integers(0, 256, 8).astype(np.uint8), seg, np.full(pad, 0xa5, np.uint8)])
            nwords = (nbytes + 3) // 4 + 3
            padded = np.concatenate([seg, np.zeros(4 * nwords - nbytes, np.uint8)])
            want = [int.from_bytes(bytes(padded[4 * w:4 * w + 4]), 'big') for w in range(nwords)]
            for entry in ('probe_ent_word', 'probe_ent_word_host'):
                out = np.empty(nwords, np.uint32)
                call(entry, buf, buf.size, 8, nbytes, nwords, out)
                assert list(out) == want, f'{entry}, {nbytes} bytes: {[hex(v) for v in out]} against {[hex(v) for v in want]}'
