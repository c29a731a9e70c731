"""CPU tests: the oracle restatement against the golden vectors and against the compiled reference.
Bit-exact everywhere: the path is fp32/fp64 arithmetic in a fixed IEEE operation order, so "equal"
means equal bit patterns.

The reference comparisons run everywhere: each one checks the oracle against the digests of what
the reference returned for the same solve (tests/golden/reference_digests.json, recorded by
tests/golden/make_golden.py), and, where the reference is built under oracle/_ref, against the
reference itself as well."""
import ctypes as C

import numpy as np
import pytest

from jpeg2png_b200 import synth
from tests import helpers as H
from tests.golden_io import golden_cases, load_case, plane_digests, reference_digests


def check_reference(key, got, run_ref):
    """`got` (list of arrays) must be bit-identical to what the reference returns: run_ref() where
    the reference is built, and the digests recorded from it in any case."""
    if H.have_ref():
        H.assert_bit_identical(got, run_ref(), f'{key} vs reference')
    assert plane_digests(got) == reference_digests(key), f'{key}: differs from the recorded reference result'


# parameters of the reference comparisons; tests/golden/make_golden.py records the reference's
# results for exactly these
CONFIGS = [
    (256, 256, 10, '4:2:0', [0, 1, 2], 0.3, [0.001] * 3, 50),      # BASELINE config 1
    (256, 256, 10, '4:2:0', [2], 0.3, [0.001], 50),                # config 1, separate mode, chroma
    (200, 120, 30, '4:2:0', [0, 1, 2], 0.3, [0.001] * 3, 30),      # luma grid narrower/shorter than the frame
    (136, 72, 50, '4:4:4', [0, 1, 2], 0.7, [0.001, 0.0, 0.01], 40),
    (64, 64, 90, '4:4:4', [0, 1, 2], 0.0, [0.0] * 3, 20),          # TV only
]


def config_key(w, h, q, ss, channels, weight, pw, iters):
    return f'config/{w}x{h}-q{q}-{ss}-c{"".join(map(str, channels))}-w{weight}-p{",".join(map(str, pw))}-i{iters}'


def config_case(w, h, q, ss, channels, weight, pw, iters):
    img = synth.synth_coefs(w, h, q, ss, seed=1234 + w + h)
    return img, channels, weight, pw, iters, H.decode_planes(img, channels)


def simd_case():
    img = synth.synth_coefs(96, 64, 10, '4:2:0', 11)
    return img, [0, 1, 2], 0.3, [0.001] * 3, 25, H.decode_planes(img)


def random_planes_case(seed):
    img = synth.random_coefs([(40, 24), (24, 16), (16, 8)], [(1, 1), (2, 2), (3, 4)], seed)
    return img, [0, 1, 2], 0.4, [0.001] * 3, 12, H.decode_planes(img)


def sweep_case(seed):
    """Randomised configuration `seed`: plane sizes, sampling factors up to 3x4, zero and non-zero
    weights, single-plane and joint mode, planes smaller than the frame."""
    rng = np.random.default_rng(1000 + seed)
    nplanes = 3
    samp = [(1, 1)] + [(int(rng.integers(1, 4)), int(rng.integers(1, 5))) for _ in range(2)]
    fw, fh = 8 * int(rng.integers(2, 9)), 8 * int(rng.integers(2, 7))
    dims = []
    for (sw, sh) in samp:
        cw, ch = -(-fw // sw), -(-fh // sh)
        cw, ch = -(-cw // 8) * 8, -(-ch // 8) * 8
        if rng.random() < 0.3 and cw > 8:
            cw -= 8                                               # a plane that does not cover the frame
        dims.append((cw, ch))
    img = synth.random_coefs(dims, samp, seed=seed, amplitude=int(rng.integers(5, 60)), qmax=int(rng.integers(2, 80)))
    joint = rng.random() < 0.6
    channels = [0, 1, 2] if joint else [int(rng.integers(0, nplanes))]
    weight = float(rng.choice([0.0, 0.1, 0.3, 1.0]))
    pw = [float(rng.choice([0.0, 0.001, 0.05])) for _ in channels]
    iters = int(rng.integers(1, 25))
    return img, channels, weight, pw, iters, H.decode_planes(img, channels)


def transform_blocks():
    """Random and extreme 8x8 blocks for the DCT / IDCT comparison."""
    rng = np.random.default_rng(5)
    blocks = [rng.normal(0, s, 64).astype(np.float32) for s in (1e-3, 1.0, 50.0, 1e4, 1e-30) for _ in range(40)]
    blocks += [np.zeros(64, np.float32), np.full(64, 127.5, np.float32), -np.ones(64, np.float32) * 1e-42]
    return blocks


def apply_transform(fn, block):
    """fn (an 8x8 in-place transform taking a float pointer) applied to a copy of block."""
    a = np.array(block, dtype=np.float32)
    pa = H.abi.alloc_floats(64)
    C.memmove(pa, a.ctypes.data, 256)
    fn(pa)
    C.memmove(a.ctypes.data, pa, 256)
    H.abi.free_ptr(pa)
    return a


def solve(kind, case):
    img, channels, weight, pw, iters, f = case
    return H.run_compute(kind, img, channels, weight, pw, iters, [p.copy() for p in f])


@pytest.fixture(scope='module', autouse=True)
def _build():
    H.build_oracle_libs()


@pytest.mark.parametrize('name', golden_cases())
def test_oracle_matches_golden(name):
    g = load_case(name)
    out = H.run_compute('oracle', g['img'], g['channels'], g['weight'], g['pweight'], g['iterations'], g['fdata'])
    H.assert_bit_identical(out, g['out'], f'golden {name}')


@pytest.mark.parametrize('name', golden_cases())
def test_oracle_decode_matches_golden(name):
    """The conventional decode (jpeg.c:83-92 + unbox) that produced the fixtures' fdata."""
    g = load_case(name)
    dec = H.decode_planes(g['img'], g['channels'])
    H.assert_bit_identical(dec, g['fdata'], f'decode {name}')


@pytest.mark.parametrize('name', golden_cases())
def test_reference_reproduces_golden(name):
    """Guards the fixtures themselves: the reference build still returns what was recorded."""
    g = load_case(name)
    check_reference(f'golden/{name}', g['out'],
                    lambda: H.run_compute('ref', g['img'], g['channels'], g['weight'], g['pweight'], g['iterations'], g['fdata']))


def test_reference_simd_equals_scalar():
    """The reference's own invariant (compute_simd_step.c:103-104, :223-224): its SIMD and scalar
    builds agree bit for bit, and the oracle agrees with both."""
    case = simd_case()
    assert reference_digests('simd_vs_c/simd') == reference_digests('simd_vs_c/c')
    if H.have_ref():
        H.assert_bit_identical(solve('ref', case), solve('ref_c', case), 'simd vs c')
    check_reference('simd_vs_c/simd', solve('oracle', case), lambda: solve('ref', case))


@pytest.mark.skipif(not H.have_ref(), reason='needs both reference builds under oracle/_ref')
def test_tables_above_32767_follow_the_scalar_reference():
    """The one place the reference's two builds disagree: its SIMD step converts the quantisation
    tables with _mm_cvtpi16_ps (compute_simd_step.c:17, :160), a signed 16-bit conversion, so a
    16-bit table entry above 32767 turns negative there.  The scalar build reads struct coef's
    uint16_t, and so do the oracle and the library (tests/test_gpu_kernel_matrix.py, 'u16')."""
    img = synth.random_coefs([(48, 32), (24, 16), (24, 16)], [(1, 1), (2, 2), (2, 2)], 5)
    rng = np.random.default_rng(5)
    for p in img.planes:
        p.quant[:] = rng.integers(1, 65536, size=64).astype(np.uint16)
        p.quant[0] = 65535
    f = H.decode_planes(img)
    args = (img, [0, 1, 2], 0.3, [0.001] * 3, 4)
    want = H.run_compute('ref_c', *args, [p.copy() for p in f])
    H.assert_bit_identical(H.run_compute('oracle', *args, [p.copy() for p in f]), want, 'oracle vs scalar reference')
    simd = H.run_compute('ref', *args, [p.copy() for p in f])
    assert any((H.bits(a) != H.bits(b)).any() for a, b in zip(simd, want)), 'the SIMD reference now reads the tables unsigned'


@pytest.mark.parametrize('w,h,q,ss,channels,weight,pw,iters', CONFIGS)
def test_oracle_matches_reference(w, h, q, ss, channels, weight, pw, iters):
    case = config_case(w, h, q, ss, channels, weight, pw, iters)
    check_reference(config_key(w, h, q, ss, channels, weight, pw, iters), solve('oracle', case), lambda: solve('ref', case))


def test_oracle_matches_reference_random_planes():
    for seed in range(5):
        case = random_planes_case(seed)
        check_reference(f'random_planes/{seed}', solve('oracle', case), lambda: solve('ref', case))


def test_transforms_match_reference():
    """8x8 DCT / IDCT restatement vs ooura/dct.c on random and extreme blocks."""
    ora = H.load_oracle()
    blocks = transform_blocks()
    for name, fn in (('dct', ora.oracle_dct8x8), ('idct', ora.oracle_idct8x8)):
        got = [np.stack([apply_transform(fn, b) for b in blocks])]
        check_reference(f'transforms/{name}', got,
                        lambda: [np.stack([apply_transform(getattr(H.load_ref(), name + '8x8s'), b) for b in blocks])])


def test_oracle_objective_log_decreases():
    """Sanity of the logged objective (compute.c:271-272): finite, and lower at the end than at the start."""
    img = synth.synth_coefs(64, 64, 10, '4:2:0', 3)
    _, log = H.run_compute('oracle', img, [0, 1, 2], 0.3, [0.001] * 3, 30, want_log=True)
    assert np.isfinite(log).all()
    assert log[-1, 0] < log[0, 0]
    assert log[0, 1] == 0.0           # first step: DCT distance is exactly zero (cos == data*q)


def test_rgb_conversion_restatement():
    """png.c:39-62 restatement: truncation, clamping, 8 and 16 bit packing."""
    ora = H.load_oracle()
    y = np.array([[0.0, 255.0, 128.4, 300.0, -5.0, 16.999]], np.float32)
    cb = np.array([[0.0, 0.0, 10.0, 0.0, 0.0, -20.5]], np.float32)
    cr = np.array([[0.0, 0.0, -10.0, 0.0, 0.0, 30.25]], np.float32)
    out8 = np.zeros(6 * 3, np.uint8)
    ora.oracle_ycc_to_rgb(6, 1, 8, y.ctypes.data, 6, cb.ctypes.data, 6, cr.ctypes.data, 6, out8.ctypes.data)
    out8 = out8.reshape(6, 3)
    assert tuple(out8[0]) == (0, 0, 0) and tuple(out8[1]) == (255, 255, 255)
    assert tuple(out8[3]) == (255, 255, 255) and tuple(out8[4]) == (0, 0, 0)
    r = min(255.0, max(0.0, float(np.float32(128.4)) + 1.402 * -10.0))
    assert out8[2, 0] == int(np.float32(r))
    out16 = np.zeros(6 * 6, np.uint8)
    ora.oracle_ycc_to_rgb(6, 1, 16, y.ctypes.data, 6, cb.ctypes.data, 6, cr.ctypes.data, 6, out16.ctypes.data)
    v = out16.reshape(6, 3, 2)
    assert (int(v[1, 0, 0]) << 8 | int(v[1, 0, 1])) == 255 * 256


@pytest.mark.parametrize('seed', range(16))
def test_oracle_matches_reference_random_sweep(seed):
    """Randomised configurations (sweep_case): restatement == compiled reference."""
    case = sweep_case(seed)
    check_reference(f'sweep/{seed}', solve('oracle', case), lambda: solve('ref', case))
