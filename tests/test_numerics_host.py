"""The exact shared-reciprocal division of numerics.cuh, restated for the host and checked against
IEEE division on the CPU (tests/qdiv_check.c); tests/test_gpu_device_arith.py checks the device
sequences themselves on the GPU."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def test_shared_reciprocal_division_is_correctly_rounded(tmp_path):
    exe = tmp_path / 'qdiv_check'
    cc = '/usr/bin/gcc' if os.path.exists('/usr/bin/gcc') else 'gcc'
    subprocess.run([cc, '-O2', '-std=c11', '-ffp-contract=off', '-msse2', '-mfpmath=sse', '-o', str(exe),
                    os.path.join(HERE, 'qdiv_check.c'), '-lm'], check=True)
    r = subprocess.run([str(exe), '30000000'], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert ' 0 mismatches' in r.stdout


def test_row_guard_property(tmp_path):
    """One magnitude test per loaded value implies the per-numerator guard (tests/rowguard_check.c)."""
    exe = tmp_path / 'rowguard_check'
    cc = '/usr/bin/gcc' if os.path.exists('/usr/bin/gcc') else 'gcc'
    subprocess.run([cc, '-O2', '-std=c11', '-ffp-contract=off', '-msse2', '-mfpmath=sse', '-o', str(exe),
                    os.path.join(HERE, 'rowguard_check.c'), '-lm'], check=True)
    r = subprocess.run([str(exe), '5000000'], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert ' 0 below 2^-60' in r.stdout


def test_packed_products_are_not_contracted(tmp_path):
    """A product followed by a sum must stay two roundings, as in the reference: one fused
    multiply-add where the reference has a mul and an add moves pixels.  The pair operations of
    numerics.cuh are explicitly rounded scalar PTX (.rn), which the PTX ISA exempts from contraction
    whatever --fmad says.  Two tripwires on the sm_90a build: (1) a probe kernel that writes
    add2 / sub2 over the result of a mul2 must come out of ptxas as FMUL + FADD, never FFMA;
    (2) the PTX of the paired-pixel kernels carries no fp32 add / sub / mul / fma without an
    explicit rounding mode, i.e. nothing ptxas would be allowed to fuse."""
    import collections
    import re
    import shutil
    import subprocess
    nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not (os.path.exists(nvcc) and os.path.exists(cuobjdump)):
        import pytest
        pytest.skip('CUDA toolkit not installed')
    arch = ['-gencode', 'arch=compute_90a,code=sm_90a']
    flags = ['-O3', '-std=c++17', '-fmad=false', '-prec-div=true', '-prec-sqrt=true', '-ftz=false']
    csrc = os.path.join(ROOT, 'jpeg2png_b200', 'csrc')
    probe = tmp_path / 'probe.cu'
    probe.write_text('#include "numerics.cuh"\nusing namespace j2p;\n'
                     '__global__ void p_add(f2 *o, const f2 *a, const f2 *b, const f2 *c) { o[0] = add2(mul2(a[0], b[0]), c[0]); }\n'
                     '__global__ void p_sub(f2 *o, const f2 *a, const f2 *b, const f2 *c) { o[0] = sub2(c[0], mul2(a[0], b[0])); }\n'
                     '__global__ void p_rev(f2 *o, const f2 *a, const f2 *b, const f2 *c) { o[0] = add2(c[0], mul2(a[0], b[0])); }\n')
    cubin = str(tmp_path / 'probe.cubin')
    subprocess.run([nvcc, *arch, *flags, '-I', csrc, '-cubin', '-o', cubin, str(probe)], check=True, capture_output=True)
    sass = subprocess.run([cuobjdump, '-sass', cubin], check=True, capture_output=True, text=True).stdout
    funs = re.split(r'\n\s+Function : ', sass)[1:]
    assert len(funs) == 3
    for fun in funs:
        c = collections.Counter(re.findall(r'\b(FFMA|FMUL|FADD)\b', fun))
        assert (c['FFMA'], c['FMUL'], c['FADD']) == (0, 2, 2), f"{fun.split(chr(10))[0]}: {dict(c)}"
    # (source, kernels expected): the gradient kernel and the projection kernels whose stepper /
    # clamp sections run on pixel pairs
    for base, min_kernels in (('kernels_gradient_packed', 12), ('kernels_project_tma', 2)):
        ptx = str(tmp_path / (base + '.ptx'))
        subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=compute_90a', *flags, '-ptx', '-o', ptx,
                        os.path.join(csrc, base + '.cu')], check=True, capture_output=True)
        entries = re.split(r'\n\.visible \.entry ', open(ptx).read())[1:]
        assert len(entries) >= min_kernels, base
        for entry in entries:
            name = entry.split('(')[0].strip()
            loose = re.findall(r'\b(?:add|sub|mul|fma)(?:\.ftz)?(?:\.sat)?\.f32\b', entry)
            assert not loose, f'{name}: fp32 arithmetic without explicit rounding: {loose[:4]}'
            assert len(re.findall(r'\bfma\.rn\.f32\b', entry)) > 20, f'{name} no longer works on pixel pairs?'


def test_small_int_to_float_trick():
    """project_common.cuh small_int_to_float: (float)d for a quantised coefficient without the
    conversion pipe — integer add on the bit pattern of 1.5 * 2^23, then an exact fp32 subtraction.
    Exhaustive over int16 (the coefficient type) and beyond, against numpy's conversion."""
    import numpy as np
    d = np.arange(-(1 << 22) + 1, 1 << 22, dtype=np.int64)
    bits = (np.int64(0x4B400000) + d).astype(np.uint32)
    got = bits.view(np.float32) - np.float32(12582912.0)
    assert got.dtype == np.float32
    assert (got == d.astype(np.float32)).all()
    assert (np.signbit(got) == (d < 0)).all()          # and +0 for d == 0, like (float)0


def test_product_sum_through_fma_with_one():
    """numerics.cuh addm2: fma(m, 1, b) == RN(m + b) bit for bit (the form that keeps ptxas from
    contracting a packed product into the sum that follows it).  fp64 has fp32's exact products
    and sums to spare, so RN32 of the exact value is one cast away."""
    import numpy as np
    rng = np.random.default_rng(3)
    m = (rng.standard_normal(2_000_000) * np.exp2(rng.integers(-40, 40, 2_000_000))).astype(np.float32)
    b = (rng.standard_normal(2_000_000) * np.exp2(rng.integers(-40, 40, 2_000_000))).astype(np.float32)
    b[::7] = -m[::7]                                     # exact cancellations
    b[::11] = 0.0
    m[::13] = 0.0
    fma = (m.astype(np.float64) * 1.0 + b.astype(np.float64)).astype(np.float32)   # exact in fp64, one rounding
    add = m + b
    assert (fma.view(np.uint32) == add.view(np.uint32)).all()
