/* arith_core.h — the QM decoder of T.81 Annex D and the sequential block step of T.81 F.1.4.4 (the
 * DC and AC statistical models of arithmetic-coded JPEG), written once for the host reader
 * (jpeg_reader.c, C11), the serial host driver and the kernel of libj2parith.so (arith.cu, CUDA).
 *
 * The rules are libjpeg's jdarith.c, which is what decodes these files elsewhere:
 *   - a segment (a scan, or one restart interval of it) starts with C = A = 0, CT = -16, zeroed
 *     statistics, a zero DC prediction and a zero DC context (j2p_qm_start, the caller's zeroing);
 *   - the decoder reads the segment's unstuffed bytes (FF 00 already FF) and zero bytes past its
 *     end, which is where the reader's and the layout pass's segments stop: at the first marker;
 *   - a magnitude category reaching 2^15, or a zero run past the last coefficient, is
 *     J2P_ARITH_BAD_CODE (libjpeg's JWRN_ARITH_BAD_CODE, where it stops decoding the segment).
 * State 113 of the probability table is libjpeg's fixed bin: Qe = 0x5A1D for every decision, used
 * for AC signs and the bits of successive-approximation refinements.
 */
#ifndef J2P_ARITH_CORE_H
#define J2P_ARITH_CORE_H

#include <stdint.h>

#ifdef __CUDACC__
#define J2P_AHD __host__ __device__ __forceinline__
#else
#define J2P_AHD static inline
#endif

enum { J2P_ARITH_OK = 0, J2P_ARITH_BAD_CODE = 1 };
enum { J2P_ARITH_DC_BINS = 64, J2P_ARITH_AC_BINS = 256, J2P_ARITH_FIXED_STATE = 113 };

/* T.81 table D.2 and the fixed state: (Qe << 16) | (NMPS << 8) | (SWITCH << 7) | NLPS */
#define J2P_QM(qe, nmps, nlps, sw) (((uint32_t)(qe) << 16) | ((uint32_t)(nmps) << 8) | ((uint32_t)(sw) << 7) | (uint32_t)(nlps))
#define J2P_QM_TABLE                                                                                                           \
        {J2P_QM(0x5a1d, 1, 1, 1),     J2P_QM(0x2586, 2, 14, 0),    J2P_QM(0x1114, 3, 16, 0),    J2P_QM(0x080b, 4, 18, 0),      \
         J2P_QM(0x03d8, 5, 20, 0),    J2P_QM(0x01da, 6, 23, 0),    J2P_QM(0x00e5, 7, 25, 0),    J2P_QM(0x006f, 8, 28, 0),      \
         J2P_QM(0x0036, 9, 30, 0),    J2P_QM(0x001a, 10, 33, 0),   J2P_QM(0x000d, 11, 35, 0),   J2P_QM(0x0006, 12, 9, 0),      \
         J2P_QM(0x0003, 13, 10, 0),   J2P_QM(0x0001, 13, 12, 0),   J2P_QM(0x5a7f, 15, 15, 1),   J2P_QM(0x3f25, 16, 36, 0),     \
         J2P_QM(0x2cf2, 17, 38, 0),   J2P_QM(0x207c, 18, 39, 0),   J2P_QM(0x17b9, 19, 40, 0),   J2P_QM(0x1182, 20, 42, 0),     \
         J2P_QM(0x0cef, 21, 43, 0),   J2P_QM(0x09a1, 22, 45, 0),   J2P_QM(0x072f, 23, 46, 0),   J2P_QM(0x055c, 24, 48, 0),     \
         J2P_QM(0x0406, 25, 49, 0),   J2P_QM(0x0303, 26, 51, 0),   J2P_QM(0x0240, 27, 52, 0),   J2P_QM(0x01b1, 28, 54, 0),     \
         J2P_QM(0x0144, 29, 56, 0),   J2P_QM(0x00f5, 30, 57, 0),   J2P_QM(0x00b7, 31, 59, 0),   J2P_QM(0x008a, 32, 60, 0),     \
         J2P_QM(0x0068, 33, 62, 0),   J2P_QM(0x004e, 34, 63, 0),   J2P_QM(0x003b, 35, 32, 0),   J2P_QM(0x002c, 9, 33, 0),      \
         J2P_QM(0x5ae1, 37, 37, 1),   J2P_QM(0x484c, 38, 64, 0),   J2P_QM(0x3a0d, 39, 65, 0),   J2P_QM(0x2ef1, 40, 67, 0),     \
         J2P_QM(0x261f, 41, 68, 0),   J2P_QM(0x1f33, 42, 69, 0),   J2P_QM(0x19a8, 43, 70, 0),   J2P_QM(0x1518, 44, 72, 0),     \
         J2P_QM(0x1177, 45, 73, 0),   J2P_QM(0x0e74, 46, 74, 0),   J2P_QM(0x0bfb, 47, 75, 0),   J2P_QM(0x09f8, 48, 77, 0),     \
         J2P_QM(0x0861, 49, 78, 0),   J2P_QM(0x0706, 50, 79, 0),   J2P_QM(0x05cd, 51, 48, 0),   J2P_QM(0x04de, 52, 50, 0),     \
         J2P_QM(0x040f, 53, 50, 0),   J2P_QM(0x0363, 54, 51, 0),   J2P_QM(0x02d4, 55, 52, 0),   J2P_QM(0x025c, 56, 53, 0),     \
         J2P_QM(0x01f8, 57, 54, 0),   J2P_QM(0x01a4, 58, 55, 0),   J2P_QM(0x0160, 59, 56, 0),   J2P_QM(0x0125, 60, 57, 0),     \
         J2P_QM(0x00f6, 61, 58, 0),   J2P_QM(0x00cb, 62, 59, 0),   J2P_QM(0x00ab, 63, 61, 0),   J2P_QM(0x008f, 32, 61, 0),     \
         J2P_QM(0x5b12, 65, 65, 1),   J2P_QM(0x4d04, 66, 80, 0),   J2P_QM(0x412c, 67, 81, 0),   J2P_QM(0x37d8, 68, 82, 0),     \
         J2P_QM(0x2fe8, 69, 83, 0),   J2P_QM(0x293c, 70, 84, 0),   J2P_QM(0x2379, 71, 86, 0),   J2P_QM(0x1edf, 72, 87, 0),     \
         J2P_QM(0x1aa9, 73, 87, 0),   J2P_QM(0x174e, 74, 72, 0),   J2P_QM(0x1424, 75, 72, 0),   J2P_QM(0x119c, 76, 74, 0),     \
         J2P_QM(0x0f6b, 77, 74, 0),   J2P_QM(0x0d51, 78, 75, 0),   J2P_QM(0x0bb6, 79, 77, 0),   J2P_QM(0x0a40, 48, 77, 0),     \
         J2P_QM(0x5832, 81, 80, 1),   J2P_QM(0x4d1c, 82, 88, 0),   J2P_QM(0x438e, 83, 89, 0),   J2P_QM(0x3bdd, 84, 90, 0),     \
         J2P_QM(0x34ee, 85, 91, 0),   J2P_QM(0x2eae, 86, 92, 0),   J2P_QM(0x299a, 87, 93, 0),   J2P_QM(0x2516, 71, 86, 0),     \
         J2P_QM(0x5570, 89, 88, 1),   J2P_QM(0x4ca9, 90, 95, 0),   J2P_QM(0x44d9, 91, 96, 0),   J2P_QM(0x3e22, 92, 97, 0),     \
         J2P_QM(0x3824, 93, 99, 0),   J2P_QM(0x32b4, 94, 99, 0),   J2P_QM(0x2e17, 86, 93, 0),   J2P_QM(0x56a8, 96, 95, 1),     \
         J2P_QM(0x4f46, 97, 101, 0),  J2P_QM(0x47e5, 98, 102, 0),  J2P_QM(0x41cf, 99, 103, 0),  J2P_QM(0x3c3d, 100, 104, 0),   \
         J2P_QM(0x375e, 93, 99, 0),   J2P_QM(0x5231, 102, 105, 0), J2P_QM(0x4c0f, 103, 106, 0), J2P_QM(0x4639, 104, 107, 0),   \
         J2P_QM(0x415e, 99, 103, 0),  J2P_QM(0x5627, 106, 105, 1), J2P_QM(0x50e7, 107, 108, 0), J2P_QM(0x4b85, 103, 109, 0),   \
         J2P_QM(0x5597, 109, 110, 0), J2P_QM(0x504f, 107, 111, 0), J2P_QM(0x5a10, 111, 110, 1), J2P_QM(0x5522, 109, 112, 0),   \
         J2P_QM(0x59eb, 111, 112, 1), J2P_QM(0x5a1d, 113, 113, 0)}

#ifdef __CUDACC__
__device__ const uint32_t j2p_qm_table_dev[114] = J2P_QM_TABLE;
__device__ const uint8_t j2p_arith_zz_dev[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                                 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                                 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                                 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
#endif
static const uint32_t j2p_qm_table_host[114] = J2P_QM_TABLE;
static const uint8_t j2p_arith_zz_host[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                              12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                              35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                              58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

J2P_AHD uint32_t j2p_qm_entry(unsigned s) {
#ifdef __CUDA_ARCH__
        return __ldg(&j2p_qm_table_dev[s]);
#else
        return j2p_qm_table_host[s];
#endif
}
J2P_AHD unsigned j2p_arith_zz(unsigned k) {
#ifdef __CUDA_ARCH__
        return __ldg(&j2p_arith_zz_dev[k]);
#else
        return j2p_arith_zz_host[k];
#endif
}

/* the decoder of one segment: its unstuffed bytes [p, p + n) */
struct j2p_qm {
        const uint8_t *p;
        uint32_t n, pos;
        int32_t c, a;
        int ct;
};

J2P_AHD void j2p_qm_start(struct j2p_qm *q, const uint8_t *p, uint32_t n) {
        q->p = p;
        q->n = n;
        q->pos = 0;
        q->c = 0;
        q->a = 0;
        q->ct = -16;            /* the first decision reads two bytes into C */
}

/* one binary decision with the adaptive state *st (bit 7: the MPS, bits 0..6: the table index), D.2 */
J2P_AHD int j2p_qm_decode(struct j2p_qm *q, uint8_t *st) {
        while (q->a < 0x8000) {
                if (--q->ct < 0) {
                        const int32_t byte = q->pos < q->n ? q->p[q->pos++] : 0;
                        q->c = (q->c << 8) | byte;
                        if ((q->ct += 8) < 0) {
                                if (++q->ct == 0) q->a = 0x8000;     /* the second of the two start bytes */
                        }
                }
                q->a <<= 1;
        }
        const unsigned sv = *st;
        const uint32_t e = j2p_qm_entry(sv & 0x7f);
        const int32_t qe = (int32_t)(e >> 16);
        const unsigned nm = (e >> 8) & 0xff, nl = e & 0xff;
        int32_t t = q->a - qe;
        q->a = t;
        t <<= q->ct;
        unsigned bit = sv >> 7;
        if (q->c >= t) {
                q->c -= t;
                if (q->a < qe) {                        /* conditional exchange: the MPS */
                        q->a = qe;
                        *st = (uint8_t)((sv & 0x80) ^ nm);
                } else {                                /* the LPS */
                        q->a = qe;
                        *st = (uint8_t)((sv & 0x80) ^ nl);
                        bit ^= 1;
                }
        } else if (q->a < 0x8000) {
                if (q->a < qe) {                        /* conditional exchange: the LPS */
                        *st = (uint8_t)((sv & 0x80) ^ nl);
                        bit ^= 1;
                } else {
                        *st = (uint8_t)((sv & 0x80) ^ nm);
                }
        }
        return (int)bit;
}

/* A DC difference (F.1.4.4.1, the DC first scans of G.1.3.1 too).  dcst: the table's 64 bins;
 * *ctx: the component's conditioning category; L, U: its DAC bounds.  *diff = the difference. */
J2P_AHD int j2p_arith_dc_diff(struct j2p_qm *q, uint8_t *dcst, int *ctx, int L, int U, int *diff) {
        uint8_t *st = dcst + *ctx;
        if (j2p_qm_decode(q, st) == 0) {
                *ctx = 0;
                *diff = 0;
                return J2P_ARITH_OK;
        }
        const int sign = j2p_qm_decode(q, st + 1);
        st += 2 + sign;
        int m = j2p_qm_decode(q, st);
        if (m) {                                        /* further categories on bins 20.. */
                st = dcst + 20;
                while (j2p_qm_decode(q, st)) {
                        if ((m <<= 1) == 0x8000) return J2P_ARITH_BAD_CODE;
                        st++;
                }
        }
        if (m < (int)((1u << L) >> 1)) *ctx = 0;
        else if (m > (int)((1u << U) >> 1)) *ctx = 12 + 4 * sign;
        else *ctx = 4 + 4 * sign;
        int v = m;
        st += 14;
        while (m >>= 1)
                if (j2p_qm_decode(q, st)) v |= m;
        v += 1;
        *diff = sign ? -v : v;
        return J2P_ARITH_OK;
}

/* One nonzero AC value after its zero run (F.1.4.4.2): the sign on the fixed bin, then the category
 * starting at st (= bin 3(k-1) + 2) and the bins 189 (k <= Kx) or 217.  *val = the value. */
J2P_AHD int j2p_arith_ac_value(struct j2p_qm *q, uint8_t *acst, uint8_t *st, int k, int Kx, uint8_t *fixed, int *val) {
        const int sign = j2p_qm_decode(q, fixed);
        int m = j2p_qm_decode(q, st);
        if (m && j2p_qm_decode(q, st)) {
                m <<= 1;
                st = acst + (k <= Kx ? 189 : 217);
                while (j2p_qm_decode(q, st)) {
                        if ((m <<= 1) == 0x8000) return J2P_ARITH_BAD_CODE;
                        st++;
                }
        }
        int v = m;
        st += 14;
        while (m >>= 1)
                if (j2p_qm_decode(q, st)) v |= m;
        v += 1;
        *val = sign ? -v : v;
        return J2P_ARITH_OK;
}

/* AC values ss..se of one block (F.1.4.4.2, and the AC first scans of G.1.3.2 with al): zero runs,
 * EOB, values stored at b[natural] << al when b is not NULL (b: zero on entry where nothing is decoded). */
J2P_AHD int j2p_arith_ac(struct j2p_qm *q, uint8_t *acst, int Kx, uint8_t *fixed, int ss, int se, int al, int16_t *b) {
        for (int k = ss; k <= se; k++) {
                uint8_t *st = acst + 3 * (k - 1);
                if (j2p_qm_decode(q, st)) break;                /* EOB */
                while (j2p_qm_decode(q, st + 1) == 0) {
                        st += 3;
                        if (++k > se) return J2P_ARITH_BAD_CODE;      /* a zero run past the band */
                }
                int v;
                if (j2p_arith_ac_value(q, acst, st + 2, k, Kx, fixed, &v) != J2P_ARITH_OK) return J2P_ARITH_BAD_CODE;
                if (b) b[j2p_arith_zz((unsigned)k)] = (int16_t)(int)((unsigned)v << al);
        }
        return J2P_ARITH_OK;
}

/* One block of a sequential scan (F.1.4.4): *pred, *ctx: the component's DC prediction and
 * conditioning category.  b: the block (natural order, zero on entry), or NULL to decode without
 * storing (MCU padding). */
J2P_AHD int j2p_arith_block_seq(struct j2p_qm *q, uint8_t *dcst, uint8_t *acst, int *pred, int *ctx, int L, int U, int Kx,
                                uint8_t *fixed, int16_t *b) {
        int diff;
        if (j2p_arith_dc_diff(q, dcst, ctx, L, U, &diff) != J2P_ARITH_OK) return J2P_ARITH_BAD_CODE;
        *pred += diff;
        if (b) b[0] = (int16_t)*pred;
        return j2p_arith_ac(q, acst, Kx, fixed, 1, 63, 0, b);
}

#endif
