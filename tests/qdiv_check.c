/* Host restatement of the shared-reciprocal division of jpeg2png_b200/csrc/numerics.cuh
 * (qdiv_core and qdiv4_core + their guard), checked against IEEE float division on this CPU.  The GPU-side twin is
 * tests/test_gpu_device_arith.py; this one runs in the CPU suite and pins the ALGORITHM (Markstein's sequence
 * with y = RN(1/b)) independently of any GPU.  fmaf() is the correctly rounded fused multiply-add
 * of C99; the file is compiled with -ffp-contract=off so nothing else is fused. */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

static float qdiv_core(float a, float b, float y) {
        const float q0 = a * y;
        const float r0 = fmaf(-b, q0, a);
        const float q1 = fmaf(r0, y, q0);
        const float r1 = fmaf(-b, q1, a);
        return fmaf(r1, y, q1);
}
/* the four-operation sequence on a two-term reciprocal (numerics.cuh rcp_low / qdiv4_core, round 2) */
static float rcp_low(float b, float y) { return fmaf(-b, y, 1.0f) * y; }
static float qdiv4_core(float a, float b, float y, float yl) {
        const float p = a * yl;
        const float q = fmaf(a, y, p);
        const float r = fmaf(-b, q, a);
        return fmaf(r, y, q);
}
static int divisor_ok(float b) { return b >= 9.094947017729282e-13f && b <= 1.099511627776e12f; }            /* [2^-40, 2^40] */
static int numerator_ok(float a) { const float m = fabsf(a); return a == 0.f || (m >= 8.673617379884035e-19f && m <= 1.152921504606847e18f); } /* 0 or [2^-60, 2^60] */

static uint64_t rng = 88172645463325252ull;
static uint64_t next(void) { rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17; return rng; }
static float from_bits(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static uint32_t bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

int main(int argc, char **argv) {
        const long n = argc > 1 ? atol(argv[1]) : 20000000;
        long tested = 0, bad = 0;
        for (long i = 0; i < n; i++) {
                const uint64_t r = next();
                /* divisor: random significand, exponent in [-40, 40) */
                float b = from_bits(((uint32_t)(127 - 40 + (r % 80)) << 23) | (uint32_t)((r >> 8) & 0x7fffff));
                float a;
                switch ((r >> 40) & 7) {
                case 0: a = b * (float)((int)((r >> 44) % 2001) - 1000); break;                         /* exact multiples */
                case 1: a = nextafterf(b * (float)(1 + (r >> 44) % 97), (r & 1) ? INFINITY : -INFINITY); break; /* one ulp off a multiple */
                case 2: a = from_bits(((uint32_t)(127 - 60 + ((r >> 44) % 120)) << 23) | (uint32_t)(next() & 0x7fffff)); break; /* anything in range */
                case 3: a = from_bits(((uint32_t)(127 - 60 + ((r >> 44) % 120)) << 23)); break;        /* powers of two */
                case 4: a = 0.f; break;
                case 5: {                                                                                /* next to the midpoint of two floats: a = RN(b * (m + 1/2 ulp)) +- a few ulps */
                        const double m = ((double)(0x800000u | (uint32_t)(next() & 0x7fffff)) + 0.5) * 1.1920928955078125e-07;
                        a = (float)((double)b * m);
                        a = from_bits(bits(a) + (uint32_t)((r >> 44) % 5) - 2u);
                        break;
                }
                default: {                                                                               /* same magnitude as b, random sign */
                        const int e = (int)((r >> 44) % 9) - 4;
                        a = ldexpf(from_bits((bits(b) & 0xff800000u) | (uint32_t)(next() & 0x7fffff)), e);
                        if (r & 2) a = -a;
                }
                }
                if (!divisor_ok(b) || !numerator_ok(a) || !isfinite(a)) continue;
                const float y = (float)(1.0 / (double)b);          /* RN(1/b): the double quotient narrowed once is correctly rounded */
                const float q = qdiv_core(a, b, y), want = a / b;
                const float q4 = qdiv4_core(a, b, y, rcp_low(b, y));
                tested++;
                if (!(q4 == want)) {
                        if (bad < 10) printf("MISMATCH (four operations) a=%a b=%a got %a want %a\n", a, b, q4, want);
                        bad++;
                }
                if (!(q == want)) {                                /* value comparison: the sign of a zero quotient is not preserved by design */
                        if (bad < 10) printf("MISMATCH a=%a b=%a got %a want %a\n", a, b, q, want);
                        bad++;
                }
        }
        printf("qdiv_check: %ld quotients inside the guard, %ld mismatches\n", tested, bad);
        return bad ? 1 : 0;
}
