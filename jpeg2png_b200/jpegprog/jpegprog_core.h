// jpegprog_core.h — the scans of a progressive JPEG file, written once as __host__ __device__ code
// for the kernels of jpegprog.cu and its serial host driver.  The file is libjpeg's progressive file
// as jpeg_simple_progression scripts it for YCbCr, Huffman-coded with a table per scan built from
// that scan's own symbol counts (jpegopt_core.h's builder):
//
//   scan  components  Ss..Se  Ah Al  tables (slot: DHT index)
//   0     Y Cb Cr     0..0    0  1   0: 0x00 (Y), 1: 0x01 (Cb, Cr)     DC first, interleaved
//   1     Y           1..5    0  2   2: 0x10
//   2     Cr          1..63   0  1   3: 0x11
//   3     Cb          1..63   0  1   4: 0x11
//   4     Y           6..63   0  2   5: 0x10
//   5     Y           1..63   2  1   6: 0x10                           AC refine
//   6     Y Cb Cr     0..0    1  0   none                              DC refine, interleaved
//   7     Cr          1..63   1  0   7: 0x11
//   8     Cb          1..63   1  0   8: 0x11
//   9     Y           1..63   1  0   9: 0x10
//
// and, for a gray call (j2p_je_tables.nc == 1), as jpeg_simple_progression scripts one component:
//
//   scan  components  Ss..Se  Ah Al  tables (slot: DHT index)
//   0     Y           0..0    0  1   0: 0x00                           DC first
//   1     Y           1..5    0  2   1: 0x10
//   2     Y           6..63   0  2   2: 0x10
//   3     Y           1..63   2  1   3: 0x10                           AC refine
//   4     Y           0..0    1  0   none                              DC refine
//   5     Y           1..63   1  0   4: 0x10
//
// Every gray scan is non-interleaved over the component's block grid, which is also its MCU grid,
// so the stored order is the raster and every scan has the same restart interval.
//
// and, for a CMYK call (nc == 4), as jpeg_simple_progression scripts any other colour space, its
// generic script for four components:
//
//   scan   components  Ss..Se  Ah Al  tables (slot: DHT index)
//   0      C M Y K     0..0    0  1   0: 0x00                          DC first, interleaved
//   1..4   C, M, Y, K  1..5    0  2   1..4: 0x10
//   5..8   C, M, Y, K  6..63   0  2   5..8: 0x10
//   9..12  C, M, Y, K  1..63   2  1   9..12: 0x10                      AC refine
//   13     C M Y K     0..0    1  0   none                             DC refine, interleaved
//   14..17 C, M, Y, K  1..63   1  0   13..16: 0x10
//
// Every CMYK table is DC0 or AC0 in the file (each scan's DHT replaces the last).  The kind is the
// call's, its component count nc: the kernels take it as a launch-uniform value.
//
// The coding is T.81 Annex G as libjpeg's progressive Huffman encoder applies it:
//
//   point      DC: arithmetic shift right by Al; AC: the magnitude shifted, the sign kept;
//   blocks     the DC scans walk the MCU grid with its dummy blocks (the stored order of the
//              coefficients); an AC scan walks only its component's own block grid, in raster order;
//   DC first   the difference of successive shifted DCs of a component, coded as in a baseline scan;
//   DC refine  one raw bit per block, (DC >> Al) & 1;
//   AC first   a block ending in zeros adds one to the pending EOB run; the run is emitted before the
//              next symbol, when it reaches 0x7FFF and at the end of the scan or of a restart
//              interval (the stream's last block, `last`), as the symbol n << 4
//              (n = floor(log2 run)) and the run's low n bits;
//   AC refine  a coefficient of shifted magnitude 1 is new: (r << 4) | 1, its sign, then the
//              correction bits (magnitude & 1 of the already nonzero coefficients) buffered since
//              the block's last emission.  A ZRL, only at or before the block's last new
//              coefficient, flushes the pending run and then the buffered bits.  After the last new
//              coefficient the block adds one to the EOB run and its correction bits to the run's
//              buffer, BE; the run and BE go out before the next emission of a block, when the run
//              reaches 0x7FFF, when BE exceeds 937 (libjpeg's 1000-bit buffer less 63) and at the
//              end of the scan or of a restart interval.
//
// A block of an AC scan takes the run state (EOB run, BE) left by the block before it.  A block with
// a nonzero coefficient (AC first) or a new one (AC refine) emits the incoming state before anything
// else and leaves a state that depends on itself alone, so the state is resolved by one serial walk
// per segment between such blocks, over one summary byte per block (j2p_jp_summary, j2p_jp_walk).
#ifndef J2P_JPEGPROG_CORE_H
#define J2P_JPEGPROG_CORE_H

#include "../jpegopt/jpegopt_core.h"
#include "jpegprog.h"

#define J2P_JP_SCANS 10u                // scans, and so bit streams, per colour image
#define J2P_JP_SCANS_GRAY 6u            // per gray image
#define J2P_JP_SCANS_CMYK 18u           // per CMYK image
#define J2P_JP_TABLES 10u               // Huffman table slots per colour image
#define J2P_JP_TABLES_GRAY 5u
#define J2P_JP_TABLES_CMYK 17u
#define J2P_JP_TABLES_MAX J2P_JP_TABLES_CMYK
#define J2P_JP_ALL 4u                   // j2p_jp_scan.comp of an interleaved scan: every component
#define J2P_JP_HEAD 1024u               // room for a scan's header: SOI .. SOF2, its DHTs, DRI, SOS
// scan 0's header is the longest: colour, three 16-bit DQTs and two DHTs; CMYK, four 16-bit DQTs and one
static_assert(J2P_JP_HEAD >= J2P_JE_PRE_MAX + 2 * (21 + 256) + J2P_JE_DRI + 14 && J2P_JP_HEAD % 16 == 0, "a scan's header fits");
static_assert(J2P_JP_HEAD >= J2P_JE_PRE_MAX_CMYK + (21 + 256) + J2P_JE_DRI + 16, "a CMYK scan's header fits");
#define J2P_JP_MAX_RUN 0x7fffu          // the longest EOB run
#define J2P_JP_MAX_BE 937u              // correction bits an EOB run may buffer before it is emitted
#define J2P_JP_RESET 0x80u              // summary: the block emits the incoming state and sets its own
#define J2P_JP_TRAIL 0x40u              // summary of such a block: it leaves a run of one behind

// Work-area bound of a block in each kind of scan, band of L coefficients: codes of up to 16 bits,
// AC magnitudes of up to 10 bits, DC differences of up to 11, one EOB-run emission (16 + 14 bits)
// per block amortised (a run covers at least one block), and each correction bit counted once, in
// the block it comes from.  An AC refine position costs at most 17 bits (a new coefficient with its
// sign), a ZRL 16 for 16 positions.
#define J2P_JP_DC_FIRST_BITS (16u + 11u)
#define J2P_JP_DC_REFINE_BITS 1u
#define J2P_JP_AC_FIRST_BITS(L) ((L) * (16u + 10u) + 16u + 14u)
#define J2P_JP_AC_REFINE_BITS(L) ((L) * (16u + 1u) + 16u + 14u)
static_assert(J2P_JP_AC_FIRST_BITS(63u) == J2P_JPEGPROG_BLOCK_BITS && J2P_JP_AC_REFINE_BITS(63u) < J2P_JPEGPROG_BLOCK_BITS &&
                  J2P_JP_DC_FIRST_BITS < J2P_JPEGPROG_BLOCK_BITS,
              "J2P_JPEGPROG_BLOCK_BITS is the worst scan's bound");
// With restart intervals each interval is a stream of its own, and its bound is still per block: its
// last EOB-run emission covers at least one of its blocks.  The byte padding at the interval's end
// costs no room: a stream of nb blocks gets nb x j2p_jp_bound_words(k) whole words, a multiple of 8
// bits that its coded bits never exceed, so rounding them up to a byte stays inside it, even where
// the bound fills its words exactly (scan 1: J2P_JP_AC_FIRST_BITS(5) is 160 bits, 5 words).  The RST
// is the stream's 2-byte header, counted in the output outside its words.
static_assert(J2P_JP_AC_FIRST_BITS(5u) == 5u * 32u && 32u % 8u == 0u, "a bound in whole words is whole bytes: padding stays inside it");
// The gray script's per-scan bounds: DC first 27, AC first over 1..5 160 and over 6..63 1538, AC
// refine over 1..63 1101, DC refine 1 bit a block.
static_assert(J2P_JP_AC_FIRST_BITS(58u) == 1538u && J2P_JP_AC_FIRST_BITS(58u) < J2P_JPEGPROG_BLOCK_BITS, "the gray scans are within the bound");
// The CMYK script's scans are the gray script's, per component: the same per-scan bounds.

struct j2p_jp_scan {
        uint32_t comp;                  // 0 Y, 1 Cb, 2 Cr (C, M, Y, K: 0 .. 3); J2P_JP_ALL: all, interleaved
        uint32_t ss, se, ah, al;
};

// the scans and the table slots of an image of a call of nc components
constexpr J2P_HD uint32_t j2p_jp_nscans(uint32_t nc) { return nc == 1 ? J2P_JP_SCANS_GRAY : nc == 4 ? J2P_JP_SCANS_CMYK : J2P_JP_SCANS; }
J2P_HD uint32_t j2p_jp_ntables(uint32_t nc) { return nc == 1 ? J2P_JP_TABLES_GRAY : nc == 4 ? J2P_JP_TABLES_CMYK : J2P_JP_TABLES; }

J2P_HD struct j2p_jp_scan j2p_jp_scan_of(uint32_t nc, uint32_t k) {
        if (nc == 4) {
                switch (k) {
                case 0: return {J2P_JP_ALL, 0, 0, 0, 1};
                case 1: return {0, 1, 5, 0, 2};
                case 2: return {1, 1, 5, 0, 2};
                case 3: return {2, 1, 5, 0, 2};
                case 4: return {3, 1, 5, 0, 2};
                case 5: return {0, 6, 63, 0, 2};
                case 6: return {1, 6, 63, 0, 2};
                case 7: return {2, 6, 63, 0, 2};
                case 8: return {3, 6, 63, 0, 2};
                case 9: return {0, 1, 63, 2, 1};
                case 10: return {1, 1, 63, 2, 1};
                case 11: return {2, 1, 63, 2, 1};
                case 12: return {3, 1, 63, 2, 1};
                case 13: return {J2P_JP_ALL, 0, 0, 1, 0};
                case 14: return {0, 1, 63, 1, 0};
                case 15: return {1, 1, 63, 1, 0};
                case 16: return {2, 1, 63, 1, 0};
                default: return {3, 1, 63, 1, 0};
                }
        }
        if (nc == 1) {
                switch (k) {
                case 0: return {0, 0, 0, 0, 1};
                case 1: return {0, 1, 5, 0, 2};
                case 2: return {0, 6, 63, 0, 2};
                case 3: return {0, 1, 63, 2, 1};
                case 4: return {0, 0, 0, 1, 0};
                default: return {0, 1, 63, 1, 0};
                }
        }
        switch (k) {
        case 0: return {J2P_JP_ALL, 0, 0, 0, 1};
        case 1: return {0, 1, 5, 0, 2};
        case 2: return {2, 1, 63, 0, 1};
        case 3: return {1, 1, 63, 0, 1};
        case 4: return {0, 6, 63, 0, 2};
        case 5: return {0, 1, 63, 2, 1};
        case 6: return {J2P_JP_ALL, 0, 0, 1, 0};
        case 7: return {2, 1, 63, 1, 0};
        case 8: return {1, 1, 63, 1, 0};
        default: return {0, 1, 63, 1, 0};
        }
}

// the DC refine scan: 6, a gray image's 4, a CMYK image's 13
J2P_HD bool j2p_jp_is_ac(uint32_t nc, uint32_t k) { return k != 0 && k != (nc == 1 ? 4u : nc == 4 ? 13u : 6u); }

// the table slot of scan k's first table (colour scan 0: luma 0, chroma 1); the DC refine has none
// (its slot is the next scan's, and it counts no symbols there)
J2P_HD uint32_t j2p_jp_slot(uint32_t nc, uint32_t k) {
        if (nc == 4) return k < 14 ? k : k - 1;
        return nc == 1 ? (k < 4 ? k : 4) : k == 0 ? 0 : k < 6 ? k + 1 : k;
}

// the tables scan k codes with: two for a colour DC first scan, none for the DC refine, else one
J2P_HD uint32_t j2p_jp_ntab(uint32_t nc, uint32_t k) { return j2p_jp_is_ac(nc, k) ? 1 : k ? 0 : nc == 3 ? 2 : 1; }

// the worst case of a block of scan k, in bits and in 32-bit words
J2P_HD uint32_t j2p_jp_bound_bits(uint32_t nc, uint32_t k) {
        const struct j2p_jp_scan s = j2p_jp_scan_of(nc, k);
        if (!j2p_jp_is_ac(nc, k)) return s.ah ? J2P_JP_DC_REFINE_BITS : J2P_JP_DC_FIRST_BITS;
        return s.ah ? J2P_JP_AC_REFINE_BITS(s.se - s.ss + 1) : J2P_JP_AC_FIRST_BITS(s.se - s.ss + 1);
}

J2P_HD uint32_t j2p_jp_bound_words(uint32_t nc, uint32_t k) { return (j2p_jp_bound_bits(nc, k) + 31) / 32; }

// the AC scans of component comp, q = 0, 1, ...; -1 past the last
J2P_HD int j2p_jp_comp_scan(uint32_t nc, uint32_t comp, uint32_t q) {
        if (nc == 4) return q < 3 ? (int)(1 + 4 * q + comp) : q == 3 ? (int)(14 + comp) : -1;
        if (nc == 1) return q == 0 ? 1 : q == 1 ? 2 : q == 2 ? 3 : q == 3 ? 5 : -1;
        if (comp == 0) return q == 0 ? 1 : q == 1 ? 4 : q == 2 ? 5 : q == 3 ? 9 : -1;
        if (comp == 1) return q == 0 ? 3 : q == 1 ? 8 : -1;
        return q == 0 ? 2 : q == 1 ? 7 : -1;
}

// ---- geometry -------------------------------------------------------------------------------------
// the block grid of a component: ceil(ceil(W h_c / h_max) / 8) x ceil(ceil(H v_c / v_max) / 8)
J2P_HD uint32_t j2p_jp_grid_w(const struct j2p_je_img *im, const struct j2p_je_tables *t, uint32_t comp) {
        return comp ? (im->w + 8 * t->hs - 1) / (8 * t->hs) : (im->w + 7) / 8;
}

J2P_HD uint32_t j2p_jp_grid_h(const struct j2p_je_img *im, const struct j2p_je_tables *t, uint32_t comp) {
        return comp ? (im->h + 8 * t->vs - 1) / (8 * t->vs) : (im->h + 7) / 8;
}

// block j of an AC scan over component comp (raster order, grid width bw) in the stored MCU order; a
// component has fewer than 2^26 blocks
J2P_HD uint64_t j2p_jp_stored(const struct j2p_je_img *im, const struct j2p_je_tables *t, uint32_t comp, uint32_t bw, uint32_t j) {
        const uint32_t row = j / bw, col = j % bw;
        const uint32_t cw = comp ? 1 : t->hs, ch = comp ? 1 : t->vs, nl = t->hs * t->vs;
        const uint64_t mcu = (uint64_t)(row / ch) * im->mcux + col / cw;
        const uint32_t k = comp ? nl + comp - 1 : (row % ch) * t->hs + col % cw;
        return mcu * j2p_je_bpm(t) + k;
}

// ---- run state ------------------------------------------------------------------------------------
// (EOB run, BE) packed as run | BE << 16

J2P_HD uint32_t j2p_jp_mag(const struct j2p_jp_scan &s, int v) { return (uint32_t)(v < 0 ? -v : v) >> s.al; }

// index of a refine block's last new coefficient, ss - 1 when it has none
J2P_HD int j2p_jp_eob(const struct j2p_jp_scan &s, const int16_t *c) {
        int eob = (int)s.ss - 1;
        for (int k = (int)s.ss; k <= (int)s.se; k++)
                if (j2p_jp_mag(s, c[k]) == 1) eob = k;
        return eob;
}

// A block of an AC scan in one byte: RESET when it emits the incoming state (a nonzero coefficient in
// AC first, a new one in AC refine), TRAIL when such a block then leaves a run of one, and the
// correction bits it adds to BE (all of them without RESET; those after its last new one with).
J2P_HD uint32_t j2p_jp_summary(const struct j2p_jp_scan &s, const int16_t *c) {
        if (!s.ah) {
                bool any = false;
                for (uint32_t k = s.ss; k <= s.se; k++) any |= j2p_jp_mag(s, c[k]) != 0;
                return any ? J2P_JP_RESET | (j2p_jp_mag(s, c[s.se]) == 0 ? J2P_JP_TRAIL : 0u) : 0u;
        }
        const int eob = j2p_jp_eob(s, c);
        uint32_t n = 0;
        for (int k = eob + 1; k <= (int)s.se; k++) n += j2p_jp_mag(s, c[k]) > 1;
        if (eob < (int)s.ss) return n;
        return J2P_JP_RESET | (eob < (int)s.se ? J2P_JP_TRAIL : 0u) | n;
}

// the state after a block of summary m, given the state before it
J2P_HD uint32_t j2p_jp_next(uint32_t st, uint32_t m) {
        if (m & J2P_JP_RESET) return m & J2P_JP_TRAIL ? 1u | (m & 63u) << 16 : 0u;
        const uint32_t run = (st & 0xffffu) + 1, be = (st >> 16) + (m & 63u);
        return run == J2P_JP_MAX_RUN || be > J2P_JP_MAX_BE ? 0u : run | be << 16;
}

// The walk of one segment: from block j, which starts the scan or follows a RESET block, to the next
// RESET block or the end, storing each block's incoming state with put(j, state).
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <class Summ, class Put>
J2P_HD void j2p_jp_walk(uint64_t j, uint64_t nb, Summ summ, Put put) {
        uint32_t st = j ? j2p_jp_next(0, summ(j - 1)) : 0u;
        for (; j < nb; j++) {
                put(j, st);
                const uint32_t m = summ(j);
                if (m & J2P_JP_RESET) break;
                st = j2p_jp_next(st, m);
        }
}

// ---- coding ---------------------------------------------------------------------------------------
// A block's emissions go to an Out with:
//   sym(tb, s)               a Huffman symbol of the stream's table tb (1 only for chroma in scan 0);
//   bits(v, n)               n raw bits, the low n of v;
//   deferred(first, n, be)   the be correction bits buffered by the EOB run of the n blocks from
//                            block `first`, in order (each block's j2p_jp_tail).

// the correction bits of a refine block's coefficients k0 .. k1 - 1
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <class Out>
J2P_HD void j2p_jp_corrections(const struct j2p_jp_scan &s, const int16_t *c, int k0, int k1, Out &o) {
        for (int k = k0; k < k1; k++) {
                const uint32_t a = j2p_jp_mag(s, c[k]);
                if (a > 1) o.bits(a & 1u, 1);
        }
}

// the correction bits a refine block adds to BE: those after its last new coefficient
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <class Out>
J2P_HD void j2p_jp_tail(const struct j2p_jp_scan &s, const int16_t *c, Out &o) {
        j2p_jp_corrections(s, c, j2p_jp_eob(s, c) + 1, (int)s.se + 1, o);
}

#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <class Out>
J2P_HD void j2p_jp_eobrun(Out &o, uint32_t run, uint32_t be, uint64_t first) {
        uint32_t n = 0;
        for (uint32_t t = run; t >>= 1;) n++;
        o.sym(0, (int)(n << 4));
        if (n) o.bits(run & ((1u << n) - 1), (int)n);
        if (be) o.deferred(first, run, be);
}

// Block j of scan s, coefficients c (zig-zag), of component comp, with the DC prediction pred (DC
// first) or the incoming run state st (AC scans); last: the last block of the scan or restart interval.
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <class Out>
J2P_HD void j2p_jp_code(const struct j2p_jp_scan &s, const int16_t *c, int pred, uint32_t comp, uint32_t st, uint64_t j, bool last, Out &o) {
        if (s.ss == 0) {
                if (s.ah) {                                     // DC refine
                        o.bits((uint32_t)(c[0] >> s.al) & 1u, 1);
                        return;
                }
                const int diff = (c[0] >> s.al) - (pred >> s.al), nb = j2p_je_nbits(diff);
                o.sym(comp ? 1 : 0, nb);
                if (nb) o.bits((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << nb) - 1), nb);
                return;
        }
        uint32_t run = st & 0xffffu, be = st >> 16;
        int r = 0;
        if (!s.ah) {                                            // AC first
                for (int k = (int)s.ss; k <= (int)s.se; k++) {
                        const int v = c[k];
                        const uint32_t a = j2p_jp_mag(s, v);
                        if (!a) {
                                r++;
                                continue;
                        }
                        if (run) j2p_jp_eobrun(o, run, 0, 0);
                        run = 0;
                        for (; r > 15; r -= 16) o.sym(0, 0xf0);
                        const int nb = j2p_je_nbits((int)a);
                        o.sym(0, (r << 4) + nb);
                        o.bits((v < 0 ? ~a : a) & ((1u << nb) - 1), nb);
                        r = 0;
                }
                if (r > 0 && ++run == J2P_JP_MAX_RUN) {
                        j2p_jp_eobrun(o, run, 0, 0);
                        run = 0;
                }
                if (last && run) j2p_jp_eobrun(o, run, 0, 0);
                return;
        }
        const int eob = j2p_jp_eob(s, c);                       // AC refine
        int kb = (int)s.ss;                                     // correction bits buffered from here
        for (int k = (int)s.ss; k <= (int)s.se; k++) {
                const uint32_t a = j2p_jp_mag(s, c[k]);
                if (!a) {
                        r++;
                        continue;
                }
                for (; r > 15 && k <= eob; r -= 16) {
                        if (run) j2p_jp_eobrun(o, run, be, j - run);
                        run = be = 0;
                        o.sym(0, 0xf0);
                        j2p_jp_corrections(s, c, kb, k, o);
                        kb = k;
                }
                if (a > 1) continue;
                if (run) j2p_jp_eobrun(o, run, be, j - run);
                run = be = 0;
                o.sym(0, (r << 4) + 1);
                o.bits(c[k] < 0 ? 0u : 1u, 1);
                j2p_jp_corrections(s, c, kb, k, o);
                kb = k + 1;
                r = 0;
        }
        uint32_t n = 0;
        for (int k = kb; k <= (int)s.se; k++) n += j2p_jp_mag(s, c[k]) > 1;
        if (r > 0 || n > 0) {
                run++;
                be += n;
                if (run == J2P_JP_MAX_RUN || be > J2P_JP_MAX_BE) {
                        j2p_jp_eobrun(o, run, be, j + 1 - run);
                        run = be = 0;
                }
        }
        if (last && run) j2p_jp_eobrun(o, run, be, j + 1 - run);
}

// ---- headers --------------------------------------------------------------------------------------
// the DHT contents of an image's tables (ten, five for gray, seventeen for CMYK)
struct j2p_jp_dht {
        uint8_t bits[J2P_JP_TABLES_MAX][16];
        uint8_t vals[J2P_JP_TABLES_MAX][256];
        uint32_t nvals[J2P_JP_TABLES_MAX];
};

// derived codes of one table
struct j2p_jp_huff {
        uint16_t code[256];
        uint8_t size[256];
};

// Table slot tb of an image from its counts: its DHT contents into d, its codes into h.
template <class Lanes>
J2P_HD void j2p_jp_table(const uint64_t *counts, struct j2p_jo_scratch *s, struct j2p_jp_dht *d, struct j2p_jp_huff *h, uint32_t tb,
                         const Lanes &L) {
        const uint32_t nv = j2p_jo_build(counts, s, d->bits[tb], d->vals[tb], L);
        if (L.lane == 0) d->nvals[tb] = nv;
        for (uint32_t k = L.lane; k < 256; k += L.n) {
                h->code[k] = 0;
                h->size[k] = 0;
        }
        L.sync();
        if (L.lane == 0) j2p_je_derive(d->bits[tb], d->vals[tb], h->code, h->size);
}

J2P_HD uint32_t j2p_jp_dht_len(const struct j2p_jp_dht *d, uint32_t tb) { return 21 + d->nvals[tb]; }

// the components of scan k's SOS, and its length
J2P_HD uint32_t j2p_jp_sos_ns(uint32_t nc, uint32_t k) { return j2p_jp_scan_of(nc, k).comp == J2P_JP_ALL ? nc : 1; }
J2P_HD uint32_t j2p_jp_sos_len(uint32_t nc, uint32_t k) { return 8 + 2 * j2p_jp_sos_ns(nc, k); }

// the header of scan k of an image whose set is t: SOI .. SOF2 (its set's DQTs) before scan 0, the
// DHTs of its tables, its SOS (without DRI)
J2P_HD uint32_t j2p_jp_head_len(const struct j2p_je_tables *t, const struct j2p_jp_dht *d, uint32_t k) {
        const uint32_t nc = t->nc;
        if (k == 0) return j2p_je_sof_end(t) + j2p_jp_dht_len(d, 0) + (nc == 3 ? j2p_jp_dht_len(d, 1) : 0) + j2p_jp_sos_len(nc, 0);
        return (j2p_jp_is_ac(nc, k) ? j2p_jp_dht_len(d, j2p_jp_slot(nc, k)) : 0) + j2p_jp_sos_len(nc, k);
}

J2P_HD uint8_t j2p_jp_dht_byte(const struct j2p_jp_dht *d, uint32_t tb, uint32_t index, uint32_t k) {
        const uint32_t nv = d->nvals[tb];
        if (k < 2) return k ? 0xc4 : 0xff;
        if (k < 4) return (uint8_t)(k == 2 ? (19 + nv) >> 8 : 19 + nv);
        if (k == 4) return (uint8_t)index;
        if (k < 21) return d->bits[tb][k - 5];
        return d->vals[tb][k - 21];
}

// SOS: the components with their table selectors (td << 4 | ta, 0 where the scan uses none), Ss,
// Se, Ah << 4 | Al
J2P_HD uint8_t j2p_jp_sos_byte(const struct j2p_je_tables *t, uint32_t k, uint32_t b) {
        const struct j2p_jp_scan s = j2p_jp_scan_of(t->nc, k);
        const uint32_t ns = j2p_jp_sos_ns(t->nc, k), len = 6 + 2 * ns;
        if (b < 2) return b ? 0xda : 0xff;
        if (b < 4) return (uint8_t)(b == 2 ? 0 : len);
        if (b == 4) return (uint8_t)ns;
        if (b < 5 + 2 * ns) {
                const uint32_t q = (b - 5) / 2, comp = s.comp == J2P_JP_ALL ? q : s.comp, h = j2p_je_htab(t, comp);
                if ((b - 5) % 2 == 0) return (uint8_t)j2p_je_comp_id(t, comp);
                if (s.ss == 0) return (uint8_t)(s.ah == 0 && h ? 0x10 : 0);
                return (uint8_t)(h ? 0x01 : 0);
        }
        b -= 5 + 2 * ns;
        return (uint8_t)(b == 0 ? s.ss : b == 1 ? s.se : s.ah << 4 | s.al);
}

J2P_HD uint8_t j2p_jp_head_byte(const struct j2p_je_tables *t, const struct j2p_je_img *im, const struct j2p_jp_dht *d, uint32_t k, uint32_t b) {
        const uint32_t nc = t->nc;
        if (k == 0) {
                const uint32_t pre = j2p_je_sof_end(t);
                if (b < pre) return b == t->sof_at + 1 ? 0xc2 : j2p_je_head_byte(t, im, b);
                b -= pre;
                for (uint32_t tb = 0; tb < j2p_jp_ntab(nc, 0); tb++) {
                        if (b < j2p_jp_dht_len(d, tb)) return j2p_jp_dht_byte(d, tb, tb, b);
                        b -= j2p_jp_dht_len(d, tb);
                }
                return j2p_jp_sos_byte(t, 0, b);
        }
        if (j2p_jp_is_ac(nc, k)) {
                const uint32_t tb = j2p_jp_slot(nc, k);
                if (b < j2p_jp_dht_len(d, tb)) return j2p_jp_dht_byte(d, tb, j2p_je_htab(t, j2p_jp_scan_of(nc, k).comp) ? 0x11 : 0x10, b);
                b -= j2p_jp_dht_len(d, tb);
        }
        return j2p_jp_sos_byte(t, k, b);
}

// scan k's header with DRI for dri (0: none) before its SOS
J2P_HD uint32_t j2p_jp_scan_head_len(const struct j2p_je_tables *t, const struct j2p_jp_dht *d, uint32_t k, uint32_t dri) {
        return j2p_jp_head_len(t, d, k) + (dri ? J2P_JE_DRI : 0);
}

J2P_HD uint8_t j2p_jp_scan_head_byte(const struct j2p_je_tables *t, const struct j2p_je_img *im, const struct j2p_jp_dht *d, uint32_t k,
                                     uint32_t dri, uint32_t b) {
        return j2p_je_dri_head(dri, j2p_jp_head_len(t, d, k), j2p_jp_sos_len(t->nc, k), b,
                               [&](uint32_t b1) { return j2p_jp_head_byte(t, im, d, k, b1); });
}

#endif  // J2P_JPEGPROG_CORE_H
