// jpegopt_core.h — the optimized Huffman tables of one image, written once as __host__ __device__
// code for the kernels of jpegopt.cu and its serial host driver.  The steps are libjpeg's
// jpeg_gen_optimal_table, as its compressor runs it with optimize_coding:
//
//   counts     per image and table, the symbols j2p_je_symbols walks (dummy blocks included): table
//              0 counts the luma DC categories, 1 the luma AC symbols, 2 and 3 those of Cb and Cr
//              together (a gray image has tables 0 and 1 only, and its header DHTs 0x00 and 0x10;
//              so has a CMYK image, whose four components all count into them);
//              a pseudo-symbol 256 with count 1 keeps any real code from being all 1-bits;
//   lengths    T.81 Annex K.2: merge the two least counts until one node is left, lengthening both
//              chains through others[].  V1 is the highest-numbered symbol among those of least
//              nonzero count (a `<=` scan from 0 to 256), V2 the same without V1;
//   limit      K.3: while a length i > 16 has codes, move two of them up and take the longest
//              shorter length j that has codes; then drop one code of the longest length, which
//              removes the pseudo-symbol;
//   symbols    HUFFVAL sorted by the K.2 code length, then by symbol value;
//   codes      canonical codes from the counts per length (Annex C, j2p_je_derive).
//
// Two departures, both beyond what libjpeg can code: libjpeg starts its scans at 10^9, so a node
// whose count exceeds that is never merged; here every nonzero count takes part (counts are 64-bit).
// The two agree while a table codes fewer than 10^9 symbols (about a gigapixel of noise); past that
// libjpeg's tables are not checked against these.  And libjpeg refuses a K.2 length above 32; here
// the K.3 limit brings any length down to 16.
//
// The lengths run on `Lanes`: a warp on the device (a shuffle argmin over the 257 counts, ballots
// for the sort) or one host thread, with the same results.
#ifndef J2P_JPEGOPT_CORE_H
#define J2P_JPEGOPT_CORE_H

#include "../jpegenc/jpegenc_plan.h"

// scratch of one table's build
struct j2p_jo_scratch {
        uint64_t freq[257];             // symbol 256 is the pseudo-symbol
        int16_t others[257];            // next symbol in the chain of a merged node, or -1
        uint16_t codesize[257];         // K.2 length, up to 256
        uint16_t bits[258];             // codes per K.2 length
        uint32_t top;                   // the longest K.2 length
};

// the DHT contents of an image's four tables: DC0, AC0, DC1, AC1
struct j2p_jo_dht {
        uint8_t bits[4][16];
        uint8_t vals[4][256];
        uint32_t nvals[4];
};

// one host thread as the lanes of a table build
struct j2p_jo_serial {
        uint32_t lane = 0, n = 1;
        J2P_HD void sync() const {}
        J2P_HD int least(uint64_t, int c) const { return c; }
        J2P_HD uint32_t ballot(bool p) const { return p ? 1u : 0u; }
};

#ifdef __CUDACC__
// a warp as the lanes of a table build
struct WarpLanes {
    uint32_t lane, n;
    __device__ void sync() const { __syncwarp(); }
    __device__ int least(uint64_t f, int c) const {
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const uint64_t f2 = __shfl_xor_sync(0xffffffffu, f, o);
            const int c2 = __shfl_xor_sync(0xffffffffu, c, o);
            if (c2 >= 0 && (c < 0 || f2 < f || (f2 == f && c2 > c))) {
                f = f2;
                c = c2;
            }
        }
        return c;
    }
    __device__ uint32_t ballot(bool p) const { return __ballot_sync(0xffffffffu, p); }
};
#endif

J2P_HD uint32_t j2p_jo_popc(uint32_t m) {
#ifdef __CUDA_ARCH__
        return __popc(m);
#else
        return (uint32_t)__builtin_popcount(m);
#endif
}

// the symbol of least nonzero count, the highest-numbered one among equals, skipping `skip`; -1 if none
template <class Lanes>
J2P_HD int j2p_jo_least(const uint64_t *freq, int skip, const Lanes &L) {
        uint64_t f = 0;
        int c = -1;
        for (int k = (int)L.lane; k < 257; k += (int)L.n) {
                const uint64_t v = freq[k];
                if (v && k != skip && (c < 0 || v <= f)) {
                        f = v;
                        c = k;
                }
        }
        return L.least(f, c);
}

// One table from its counts[256]: the DHT's code counts per length bits[16] and symbols vals; returns
// how many symbols.  Every lane returns the same.
template <class Lanes>
J2P_HD uint32_t j2p_jo_build(const uint64_t *counts, struct j2p_jo_scratch *s, uint8_t *bits, uint8_t *vals, const Lanes &L) {
        for (uint32_t k = L.lane; k < 258; k += L.n) {
                if (k < 257) {
                        s->freq[k] = k < 256 ? counts[k] : 1;
                        s->others[k] = -1;
                        s->codesize[k] = 0;
                }
                s->bits[k] = 0;
        }
        L.sync();
        for (;;) {                                              // K.2
                int c1 = j2p_jo_least(s->freq, -1, L);
                int c2 = j2p_jo_least(s->freq, c1, L);
                if (c2 < 0) break;
                if (L.lane == 0) {
                        s->freq[c1] += s->freq[c2];
                        s->freq[c2] = 0;
                        s->codesize[c1]++;
                        while (s->others[c1] >= 0) {
                                c1 = s->others[c1];
                                s->codesize[c1]++;
                        }
                        s->others[c1] = (int16_t)c2;
                        s->codesize[c2]++;
                        while (s->others[c2] >= 0) {
                                c2 = s->others[c2];
                                s->codesize[c2]++;
                        }
                }
                L.sync();
        }
        if (L.lane == 0) {                                      // K.3
                uint32_t top = 0;
                for (int k = 0; k < 257; k++) {
                        const uint32_t c = s->codesize[k];
                        if (c) {
                                s->bits[c]++;
                                top = c > top ? c : top;
                        }
                }
                for (uint32_t i = top; i > 16; i--) {
                        while (s->bits[i] > 0) {
                                uint32_t j = i - 2;
                                while (s->bits[j] == 0) j--;
                                s->bits[i] -= 2;
                                s->bits[i - 1]++;
                                s->bits[j + 1] += 2;
                                s->bits[j]--;
                        }
                }
                uint32_t i = 16;
                while (s->bits[i] == 0) i--;
                s->bits[i]--;
                for (int k = 0; k < 16; k++) bits[k] = (uint8_t)s->bits[k + 1];
                s->top = top;
        }
        L.sync();
        uint32_t p = 0;                                         // HUFFVAL
        for (uint32_t len = 1; len <= s->top; len++) {
                for (uint32_t v0 = 0; v0 < 256; v0 += L.n) {
                        const uint32_t v = v0 + L.lane;
                        const bool on = s->codesize[v] == len;
                        const uint32_t m = L.ballot(on);
                        if (on) vals[p + j2p_jo_popc(m & ((1u << L.lane) - 1))] = (uint8_t)v;
                        p += j2p_jo_popc(m);
                }
        }
        L.sync();
        return p;
}

// Table tb of an image from its counts: its DHT contents into d, its codes into h.
template <class Lanes>
J2P_HD void j2p_jo_table(const uint64_t *counts, struct j2p_jo_scratch *s, struct j2p_jo_dht *d, struct j2p_je_huff *h, int tb, const Lanes &L) {
        const uint32_t nv = j2p_jo_build(counts, s, d->bits[tb], d->vals[tb], L);
        if (L.lane == 0) d->nvals[tb] = nv;
        for (uint32_t k = L.lane; k < 256; k += L.n) {
                h->code[tb][k] = 0;
                h->size[tb][k] = 0;
        }
        L.sync();
        if (L.lane == 0) j2p_je_derive(d->bits[tb], d->vals[tb], h->code[tb], h->size[tb]);
}

// the tables of an image of the call: DC0, AC0, DC1, AC1, or a gray or CMYK image's DC0 and AC0
J2P_HD uint32_t j2p_jo_ntables(const struct j2p_je_tables *t) { return t->nc == 3 ? 4 : 2; }

J2P_HD uint32_t j2p_jo_head_len(const struct j2p_je_tables *t, const struct j2p_jo_dht *d) {
        uint32_t n = j2p_je_sof_end(t) + j2p_je_sos_len(t);
        for (uint32_t tb = 0; tb < j2p_jo_ntables(t); tb++) n += 21 + d->nvals[tb];
        return n;
}

// The header of an image whose set is t: the template's SOI .. SOF with the image's size (its length
// is the set's: j2p_je_sof_end), the image's own DHTs, the template's SOS.  An optimized table codes
// no more symbols than the Annex K one of its kind, so the header fits the template's room.
// byte k of it:
J2P_HD uint8_t j2p_jo_head_byte(const struct j2p_je_tables *t, const struct j2p_je_img *im, const struct j2p_jo_dht *d, uint32_t k) {
        const uint32_t pre = j2p_je_sof_end(t);
        if (k < pre) return j2p_je_head_byte(t, im, k);
        k -= pre;
        for (int tb = 0; tb < (int)j2p_jo_ntables(t); tb++) {
                const uint32_t nv = d->nvals[tb], len = 2 + 2 + 1 + 16 + nv;
                if (k < len) {
                        if (k < 2) return k ? 0xc4 : 0xff;
                        if (k < 4) return (uint8_t)(k == 2 ? (19 + nv) >> 8 : 19 + nv);
                        if (k == 4) return (uint8_t)((tb & 1) << 4 | tb >> 1);         // Tc, Th
                        if (k < 21) return d->bits[tb][k - 5];
                        return d->vals[tb][k - 21];
                }
                k -= len;
        }
        return t->head[t->head_len - j2p_je_sos_len(t) + k];
}

// an image's file header: j2p_jo_head_byte with the image's DRI before the SOS when it has restarts
J2P_HD uint32_t j2p_jo_file_head_len(const struct j2p_je_tables *t, const struct j2p_je_img *im, const struct j2p_jo_dht *d) {
        return j2p_jo_head_len(t, d) + (im->ri ? J2P_JE_DRI : 0);
}

J2P_HD uint8_t j2p_jo_file_head_byte(const struct j2p_je_tables *t, const struct j2p_je_img *im, const struct j2p_jo_dht *d, uint32_t k) {
        return j2p_je_dri_head(im->ri, j2p_jo_head_len(t, d), j2p_je_sos_len(t), k, [&](uint32_t k1) { return j2p_jo_head_byte(t, im, d, k1); });
}

#endif  // J2P_JPEGOPT_CORE_H
