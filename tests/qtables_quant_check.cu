// The encoder's quantiser (j2p_je_quant with the reciprocals of jpegenc_plan.h) against x / (8q)
// rounded half away from zero, for every table entry q in 1 .. 8191 and every |x| < 2^15: the range
// given quantisation tables reach.  Host code, built with nvcc (the header is __host__ __device__).
#include <stdio.h>

#include "../jpeg2png_b200/jpegenc/jpegenc_plan.h"

int main() {
    static struct j2p_je_tables t;
    long bad = 0, tested = 0;
    for (uint32_t q = 1; q <= 8191; q++) {
        reciprocal(q << 3, &t.recip[0][0], &t.corr[0][0], &t.shift[0][0]);
        const int d = (int)(q << 3);
        for (int x = -32767; x <= 32767; x++) {
            const int a = x < 0 ? -x : x, want = (x < 0 ? -1 : 1) * ((a + d / 2) / d);
            tested++;
            if (j2p_je_quant(&t, 0, 0, x) != want && bad++ < 10) printf("q %u x %d: %d, want %d\n", q, x, j2p_je_quant(&t, 0, 0, x), want);
        }
    }
    printf("qtables_quant_check: %ld quotients, %ld mismatches\n", tested, bad);
    return bad != 0;
}
