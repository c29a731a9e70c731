/* png_core.h — the steps of the PNG encoder, written once for the device kernels and the serial
 * host driver (png.cu).  Everything here is __host__ __device__ and takes its scratch from the
 * caller, so the kernels keep it in shared memory and the host driver on its stack.
 *
 * The encoding (DESIGN §7e):
 *   filtering  each row gets the PNG filter (None, Sub, Up, Average, Paeth) with the smallest sum of
 *              |residual| (residual bytes read as signed), ties to the lower type; row 0's row
 *              above is zero;
 *   pieces     the filtered stream of an image is cut into pieces of J2P_PNG_PIECE bytes;
 *   parse      zlib's run-length parse restarted at every piece: a run of L equal bytes is one
 *              literal, matches of 258 at distance 1, then a match for a remainder of 3 or more
 *              bytes or literals for 1 or 2;
 *   blocks     the symbols of a piece go in blocks of J2P_PNG_BLOCK_SYMS, each stored, fixed or
 *              dynamic, whichever is smallest (ties: fixed before dynamic, Huffman before stored);
 *   joining    every piece but an image's last ends with an empty stored block; the last block of
 *              the last piece has BFINAL.
 */
#ifndef J2P_PNG_CORE_H
#define J2P_PNG_CORE_H

#include <stdint.h>

#include "../common/codec_host.h"       /* J2P_HD */
#include "png.h"

#define J2P_PNG_PIECE 65536u              /* bytes of filtered stream per piece */
#define J2P_PNG_BLOCK_SYMS 16383u         /* symbols per deflate block (zlib's default) */
#define J2P_PNG_MAX_BLOCKS 5u             /* ceil(J2P_PNG_PIECE / J2P_PNG_BLOCK_SYMS) */
#define J2P_PNG_NLIT 286u                 /* literal/length symbols that can occur */
#define J2P_PNG_NBL 19u
#define J2P_PNG_SLOT 65600u               /* j2p_png_piece_bound(J2P_PNG_PIECE), rounded up to 16 */
#define J2P_PNG_MAX_IDAT 0x7fffffffu      /* PNG's largest chunk: bounds an image's IDAT (one per file) */
#define J2P_PNG_CRC_POLY 0xedb88320u

enum { J2P_BT_STORED = 0, J2P_BT_FIXED = 1, J2P_BT_DYNAMIC = 2 };

/* One image of a call, as the kernels see it. */
struct j2p_png_img {
        const uint8_t *src;
        int64_t s_row, s_col, s_chan;     /* element strides */
        uint32_t w, h, sb;                /* sample bytes: 1 or 2 */
        uint32_t nc;                      /* samples per pixel: 3 (RGB) or 1 (gray) */
        uint32_t piece0, npieces;
        uint64_t row0;                    /* first row among all rows of the call */
        uint64_t filt_off, filt_len;      /* the filtered stream in the filtered buffer */
        uint64_t file_off, file_len;      /* filled by the assembly step */
        uint32_t adler, crc;              /* of the filtered stream / of the IDAT type and data */
};

/* ---- filtering ------------------------------------------------------------------------------ */
/* The steps below take the image's channel count NC (im->nc: 3 or 1) as a template argument:
 * callers branch on it once per row, so each byte's address arithmetic has a constant divisor
 * (none for gray) and the RGB code is what it is with 3 written in. */
template <uint32_t NC> J2P_HD uint64_t j2p_png_row_bytes(const struct j2p_png_img *im) { return (uint64_t)im->w * NC * im->sb; }

/* Byte i of row y of the unfiltered scanline (16-bit samples big-endian); 0 outside the image. */
template <uint32_t NC> J2P_HD uint32_t j2p_png_raw(const struct j2p_png_img *im, int64_t y, int64_t i) {
        if (y < 0 || i < 0) return 0;
        /* a row holds fewer than J2P_PNG_MAX_IDAT bytes (the plan refuses larger images), so the
         * byte index fits 32 bits and its divisions are 32-bit ones */
        const uint32_t u = (uint32_t)i, s = im->sb == 2 ? u >> 1 : u, k = u - s * im->sb;
        const uint32_t x = s / NC, c = s - x * NC;
        const int64_t e = y * im->s_row + (int64_t)x * im->s_col + (int64_t)c * im->s_chan;
        if (im->sb == 1) return im->src[e];
        const uint16_t v = ((const uint16_t *)im->src)[e];
        return k == 0 ? (uint32_t)(v >> 8) : (uint32_t)(v & 0xff);
}

J2P_HD uint32_t j2p_png_paeth(uint32_t a, uint32_t b, uint32_t c) {
        const int p = (int)a + (int)b - (int)c;
        const int pa = p > (int)a ? p - (int)a : (int)a - p, pb = p > (int)b ? p - (int)b : (int)b - p,
                  pc = p > (int)c ? p - (int)c : (int)c - p;
        return pa <= pb && pa <= pc ? a : (pb <= pc ? b : c);
}

/* The residual byte of filter type t for x with left a, up b, up-left c. */
J2P_HD uint32_t j2p_png_residual(int t, uint32_t x, uint32_t a, uint32_t b, uint32_t c) {
        switch (t) {
        case 0: return x;
        case 1: return (x - a) & 0xff;
        case 2: return (x - b) & 0xff;
        case 3: return (x - ((a + b) >> 1)) & 0xff;
        default: return (x - j2p_png_paeth(a, b, c)) & 0xff;
        }
}

J2P_HD uint32_t j2p_png_cost(uint32_t r) { return r < 128 ? r : 256 - r; }

/* Adds byte i of row y to the five filter sums. */
template <uint32_t NC> J2P_HD void j2p_png_filter_sums(const struct j2p_png_img *im, int64_t y, int64_t i, uint64_t sum[5]) {
        const int64_t bpp = NC * (int64_t)im->sb;
        const uint32_t x = j2p_png_raw<NC>(im, y, i), a = j2p_png_raw<NC>(im, y, i - bpp), b = j2p_png_raw<NC>(im, y - 1, i),
                       c = j2p_png_raw<NC>(im, y - 1, i - bpp);
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
        for (int t = 0; t < 5; t++) sum[t] += j2p_png_cost(j2p_png_residual(t, x, a, b, c));
}

J2P_HD int j2p_png_pick(const uint64_t sum[5]) {
        int best = 0;
        uint64_t low = sum[0];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
        for (int t = 1; t < 5; t++)
                if (sum[t] < low) { low = sum[t]; best = t; }
        return best;
}

template <uint32_t NC> J2P_HD uint8_t j2p_png_filtered(const struct j2p_png_img *im, int t, int64_t y, int64_t i) {
        const int64_t bpp = NC * (int64_t)im->sb;
        return (uint8_t)j2p_png_residual(t, j2p_png_raw<NC>(im, y, i), j2p_png_raw<NC>(im, y, i - bpp), j2p_png_raw<NC>(im, y - 1, i),
                                         j2p_png_raw<NC>(im, y - 1, i - bpp));
}

/* ---- parse ---------------------------------------------------------------------------------- */
/* Within a run of L equal bytes: the first offset >= k where a symbol starts (L if none) and the
 * length in bytes of the symbol that starts at offset k. */
J2P_HD uint32_t j2p_png_next_sym(uint32_t k, uint32_t L) {
        if (k == 0) return 0;
        uint32_t m = k - 1;
        const uint32_t q = (L - 1) / 258, full = q * 258, rem = L - 1 - full;
        if (m < full) {
                const uint32_t t = (m + 257) / 258 * 258;
                if (t < full) return t + 1;
                m = full;
        }
        if (rem >= 3) return m == full ? full + 1 : L;
        return m + 1;
}

J2P_HD uint32_t j2p_png_sym_len(uint32_t k, uint32_t L) {
        if (k == 0) return 1;
        const uint32_t q = (L - 1) / 258, full = q * 258, rem = L - 1 - full;
        if (k - 1 < full) return 258;
        return rem >= 3 ? rem : 1;
}

/* Calls f(position, symbol) for every symbol that starts in [i0, i1) of the piece p[0, n): symbol
 * < 256 a literal, 256 + len a match of len bytes at distance 1.  r0: start of the run holding
 * byte i0; e1: end of the run holding byte i1 - 1 (n when i1 == n). */
#ifdef __CUDACC__
#pragma nv_exec_check_disable           /* f is a host lambda in the host driver, a device one in the kernels */
#endif
template <class F>
J2P_HD void j2p_png_walk(const uint8_t *p, uint32_t i0, uint32_t i1, uint32_t r0, uint32_t e1, F &&f) {
        uint32_t i = i0, r = r0, e = i0;
        bool first = true;
        while (i < i1) {
                if (first || i >= e) {
                        if (!first) r = i;
                        uint32_t j = i + 1;
                        while (j < i1 && p[j] == p[i]) j++;
                        e = j == i1 ? e1 : j;
                        first = false;
                }
                const uint32_t L = e - r, k = j2p_png_next_sym(i - r, L);
                if (k >= L) { i = e; continue; }
                const uint32_t s = r + k;
                if (s >= i1) break;
                const uint32_t len = j2p_png_sym_len(k, L);
                f(s, len == 1 ? (uint32_t)p[s] : 256u + len);
                i = s + len;
        }
}

/* Length symbol (257..285) and extra bits of a match of len bytes (3..258). */
J2P_HD uint32_t j2p_png_len_code(uint32_t len, uint32_t *ebits, uint32_t *eval) {
        if (len == 258) { *ebits = 0; *eval = 0; return 285; }
        const uint32_t l = len - 3;
        if (l < 8) { *ebits = 0; *eval = 0; return 257 + l; }
        uint32_t e = 0;
        while ((l >> (e + 3)) != 0) e++;          /* e = floor(log2 l) - 2 */
        *ebits = e;
        *eval = l & ((1u << e) - 1);
        return 257 + 4 * e + (l >> e);
}

/* ---- Huffman codes -------------------------------------------------------------------------- */
/* Sort key of a symbol: by frequency, then by symbol (unique, so every sort gives one order). */
J2P_HD uint32_t j2p_png_key(uint32_t freq, uint32_t sym) { return freq << 9 | sym; }

/* Scratch of the code construction of one block (shared memory in the kernel: dynamically
 * indexed arrays would otherwise go to local memory). */
struct j2p_png_scratch {
        uint32_t key[288];                /* sorted keys of the symbols that occur */
        uint32_t a[288];
        uint32_t count[34], next[16];
        uint32_t blf[J2P_PNG_NBL];
        uint8_t fl[288];
};

/* Code lengths, at most `limit` bits, for the m symbols of `key` (sorted ascending, m >= 2),
 * written to len[symbol].  Minimum-redundancy lengths by the in-place
 * method of Moffat and Katajainen; lengths over the limit are cut to it and the Kraft sum repaired
 * by lengthening the longest codes below the limit. */
J2P_HD void j2p_png_lengths(const uint32_t *key, uint32_t m, uint32_t limit, struct j2p_png_scratch *sc, uint8_t *len) {
        uint32_t *a = sc->a, *count = sc->count;
        for (uint32_t i = 0; i < m; i++) a[i] = key[i] >> 9;
        a[0] += a[1];
        int root = 0;
        uint32_t leaf = 2;
        for (uint32_t next = 1; next + 1 < m; next++) {
                if (leaf >= m || a[root] < a[leaf]) { a[next] = a[root]; a[root++] = next; }
                else a[next] = a[leaf++];
                if (leaf >= m || ((uint32_t)root < next && a[root] < a[leaf])) { a[next] += a[root]; a[root++] = next; }
                else a[next] += a[leaf++];
        }
        a[m - 2] = 0;
        for (int next = (int)m - 3; next >= 0; next--) a[next] = a[a[next]] + 1;
        int avail = 1, used = 0, depth = 0, next = (int)m - 1;
        root = (int)m - 2;
        while (avail > 0) {
                while (root >= 0 && a[root] == (uint32_t)depth) { used++; root--; }
                while (avail > used) { a[next--] = (uint32_t)depth; avail--; }
                avail = 2 * used;
                depth++;
                used = 0;
        }
        /* a[i]: length of sorted symbol i, non-increasing in i */
        for (int l = 0; l <= 32; l++) count[l] = 0;
        for (uint32_t i = 0; i < m; i++) count[a[i] > limit ? limit : a[i]]++;
        uint32_t kraft = 0;
        for (uint32_t l = 1; l <= limit; l++) kraft += count[l] << (limit - l);
        while (kraft > (1u << limit)) {
                count[limit]--;
                for (uint32_t l = limit - 1; l > 0; l--)
                        if (count[l]) { count[l]--; count[l + 1] += 2; break; }
                kraft--;
        }
        uint32_t j = 0;
        for (uint32_t l = limit; l > 0; l--)
                for (uint32_t c = count[l]; c > 0; c--) len[key[j++] & 511] = (uint8_t)l;
}

/* Canonical codes, bit-reversed for LSB-first output. */
J2P_HD void j2p_png_codes(const uint8_t *len, uint32_t n, uint16_t *code, struct j2p_png_scratch *sc) {
        uint32_t *count = sc->count, *next = sc->next;
        for (int l = 0; l < 16; l++) count[l] = 0;
        for (uint32_t s = 0; s < n; s++) count[len[s]]++;
        count[0] = 0;
        uint32_t c = 0;
        for (int l = 1; l < 16; l++) { c = (c + count[l - 1]) << 1; next[l] = c; }
        for (uint32_t s = 0; s < n; s++) {
                const uint32_t l = len[s];
                if (!l) { code[s] = 0; continue; }
                uint32_t v = next[l]++, r = 0;
                for (uint32_t b = 0; b < l; b++) { r = r << 1 | (v & 1); v >>= 1; }
                code[s] = (uint16_t)r;
        }
}

J2P_HD void j2p_png_fixed_lengths(uint8_t *len) {
        for (uint32_t s = 0; s < 288; s++) len[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
}

/* The code-length sequence (hlit literal/length lengths, then one distance length of 1) as
 * symbols of the code-length alphabet: f(symbol, extra bits, extra value). */
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <class F>
J2P_HD void j2p_png_rle_lengths(const uint8_t *lit, uint32_t hlit, F &&f) {
        uint32_t i = 0;
        const uint32_t n = hlit + 1;
        while (i < n) {
                const uint32_t v = i < hlit ? lit[i] : 1;
                uint32_t run = 1;
                while (i + run < n && (i + run < hlit ? lit[i + run] : 1u) == v) run++;
                i += run;
                if (v == 0) {
                        while (run >= 11) { const uint32_t r = run < 138 ? run : 138; f(18u, 7u, r - 11); run -= r; }
                        if (run >= 3) { f(17u, 3u, run - 3); run = 0; }
                        while (run) { f(0u, 0u, 0u); run--; }
                } else {
                        f(v, 0u, 0u);
                        run--;
                        while (run >= 3) { const uint32_t r = run < 6 ? run : 6; f(16u, 2u, r - 3); run -= r; }
                        while (run) { f(v, 0u, 0u); run--; }
                }
        }
}

J2P_HD uint32_t j2p_png_bl_order(uint32_t k) {
        /* 16 17 18 0 8 7 9 6 10 5 11 4 12 3 13 2 14 1 15 */
        if (k < 3) return 16 + k;
        if (k == 3) return 0;
        const uint32_t j = k - 4;                 /* 0..14 -> 8 7 9 6 10 5 11 4 12 3 13 2 14 1 15 */
        return (j & 1) ? 7 - (j >> 1) : 8 + (j >> 1);
}

/* Per block of a piece: the choice and the codes.  hist: literal/length frequencies (EOB
 * included); nmatch: how many matches (each one distance code). */
struct j2p_png_block {
        uint32_t byte0, byte1;            /* bytes of the piece the block covers */
        uint32_t type, hlit, hclen;
        uint32_t hdr_bits, data_bits;     /* after the 3 header bits; data excludes end-of-block */
        uint32_t bit0, data_bit0;         /* where the block starts, where its first symbol goes */
        uint8_t len[288];
        uint16_t code[288];
        uint8_t bl_len[J2P_PNG_NBL];
        uint16_t bl_code[J2P_PNG_NBL];
};

J2P_HD uint32_t j2p_png_len_extra(uint32_t s) { return s >= 265 && s < 285 ? (s - 261) / 4 : 0; }

/* Bits of the block's symbols under lengths len (distance code of dlen bits), end-of-block excluded. */
J2P_HD uint32_t j2p_png_data_bits(const uint32_t *hist, const uint8_t *len, uint32_t dlen) {
        uint32_t bits = 0, nmatch = 0;
        for (uint32_t s = 0; s < J2P_PNG_NLIT; s++) {
                if (s == 256 || !hist[s]) continue;
                bits += hist[s] * (len[s] + j2p_png_len_extra(s));
                if (s > 256) nmatch += hist[s];
        }
        return bits + nmatch * dlen;
}

J2P_HD uint32_t j2p_png_stored_subs(uint32_t nbytes) { return nbytes ? (nbytes + 65534) / 65535 : 1; }

/* Chooses the block's type and fills its codes, given its dynamic literal/length lengths in
 * b->len (from j2p_png_lengths). */
J2P_HD void j2p_png_choose(struct j2p_png_block *b, const uint32_t *hist, struct j2p_png_scratch *sc) {
        uint32_t *key = sc->key, *blf = sc->blf;
        uint32_t hlit = 257;
        for (uint32_t s = 257; s < J2P_PNG_NLIT; s++)
                if (b->len[s]) hlit = s + 1;
        b->hlit = hlit;
        for (uint32_t s = 0; s < J2P_PNG_NBL; s++) { blf[s] = 0; b->bl_len[s] = 0; }
        j2p_png_rle_lengths(b->len, hlit, [&](uint32_t s, uint32_t, uint32_t) { blf[s]++; });
        uint32_t m = 0;
        for (uint32_t s = 0; s < J2P_PNG_NBL; s++)
                if (blf[s]) {
                        const uint32_t k = j2p_png_key(blf[s], s);
                        uint32_t j = m++;
                        while (j > 0 && key[j - 1] > k) { key[j] = key[j - 1]; j--; }
                        key[j] = k;
                }
        if (m == 1) {                             /* a code-length code must be complete */
                b->bl_len[key[0] & 511] = 1;
                b->bl_len[(key[0] & 511) == 0 ? 1 : 0] = 1;
        } else {
                j2p_png_lengths(key, m, 7, sc, b->bl_len);
        }
        j2p_png_codes(b->bl_len, J2P_PNG_NBL, b->bl_code, sc);
        uint32_t hclen = 4;
        for (uint32_t k = 0; k < J2P_PNG_NBL; k++)
                if (b->bl_len[j2p_png_bl_order(k)]) hclen = k + 1 > 4 ? k + 1 : 4;
        b->hclen = hclen;
        uint32_t hdr = 5 + 5 + 4 + 3 * hclen;
        for (uint32_t s = 0; s < J2P_PNG_NBL; s++) hdr += blf[s] * (b->bl_len[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0));
        const uint32_t dyn = hdr + j2p_png_data_bits(hist, b->len, 1) + b->len[256];
        uint8_t *fl = sc->fl;
        j2p_png_fixed_lengths(fl);
        const uint32_t fixed = j2p_png_data_bits(hist, fl, 5) + 7;
        const uint32_t nbytes = b->byte1 - b->byte0;
        const uint32_t stored = j2p_png_stored_subs(nbytes) * (3 + 7 + 32) + 8 * nbytes - 3;   /* worst padding */
        if (fixed <= dyn && fixed <= stored) {
                b->type = J2P_BT_FIXED;
                for (uint32_t s = 0; s < 288; s++) b->len[s] = fl[s];
                b->hdr_bits = 0;
                b->data_bits = fixed - 7;
        } else if (dyn <= stored) {
                b->type = J2P_BT_DYNAMIC;
                b->hdr_bits = hdr;
                b->data_bits = dyn - hdr - b->len[256];
        } else {
                b->type = J2P_BT_STORED;
                b->hdr_bits = 0;
                b->data_bits = 0;
        }
        if (b->type != J2P_BT_STORED) j2p_png_codes(b->len, 288, b->code, sc);
}

/* ---- bits ----------------------------------------------------------------------------------- */
/* ORs the n low bits of v (n <= 25) into buf at bit position pos, LSB first. */
J2P_HD void j2p_png_put(uint32_t *buf, uint32_t pos, uint32_t v, uint32_t n) {
        if (!n) return;
        const uint32_t w = pos >> 5, o = pos & 31;
        const uint64_t x = (uint64_t)v << o;
#ifdef __CUDA_ARCH__
        atomicOr(&buf[w], (uint32_t)x);
        if ((uint32_t)(x >> 32)) atomicOr(&buf[w + 1], (uint32_t)(x >> 32));
#else
        buf[w] |= (uint32_t)x;
        if ((uint32_t)(x >> 32)) buf[w + 1] |= (uint32_t)(x >> 32);
#endif
}

/* Bits symbol sym takes in block b. */
J2P_HD uint32_t j2p_png_sym_bits(const struct j2p_png_block *b, uint32_t sym) {
        if (sym < 256) return b->len[sym];
        uint32_t eb, ev;
        const uint32_t s = j2p_png_len_code(sym - 256, &eb, &ev);
        return b->len[s] + eb + (b->type == J2P_BT_FIXED ? 5 : 1);
}

/* Writes symbol sym of block b at bit pos. */
J2P_HD void j2p_png_put_sym(uint32_t *buf, uint32_t pos, const struct j2p_png_block *b, uint32_t sym) {
        if (sym < 256) { j2p_png_put(buf, pos, b->code[sym], b->len[sym]); return; }
        uint32_t eb, ev;
        const uint32_t s = j2p_png_len_code(sym - 256, &eb, &ev);
        j2p_png_put(buf, pos, b->code[s], b->len[s]);
        j2p_png_put(buf, pos + b->len[s], ev, eb);
        /* distance 1: code 0 (5 bits fixed, 1 bit dynamic), no extra bits: zeros */
}

/* Lays out the blocks of a piece one after another from bit 0: block starts, stored padding, the
 * sync flush or BFINAL.  Returns the piece's length in bytes. */
J2P_HD uint32_t j2p_png_layout(struct j2p_png_block *blk, uint32_t nblocks, bool last_piece) {
        uint32_t pos = 0;
        for (uint32_t k = 0; k < nblocks; k++) {
                struct j2p_png_block *b = &blk[k];
                b->bit0 = pos;
                if (b->type == J2P_BT_STORED) {
                        const uint32_t subs = j2p_png_stored_subs(b->byte1 - b->byte0);
                        for (uint32_t s = 0; s < subs; s++) pos = ((pos + 3 + 7) & ~7u) + 32 + 8 * (s + 1 < subs ? 65535 : (b->byte1 - b->byte0) - 65535 * s);
                        b->data_bit0 = 0;
                } else {
                        b->data_bit0 = pos + 3 + b->hdr_bits;
                        pos = b->data_bit0 + b->data_bits + b->len[256];
                }
        }
        if (!last_piece) pos = ((pos + 3 + 7) & ~7u) + 32;
        return (pos + 7) / 8;
}

/* Block headers (and dynamic code descriptions), end-of-block codes, stored headers and the sync
 * flush of a laid-out piece; the stored bytes themselves are the caller's (j2p_png_stored_at). */
J2P_HD void j2p_png_put_block_frame(uint32_t *buf, const struct j2p_png_block *b, bool final_block) {
        uint32_t pos = b->bit0;
        if (b->type == J2P_BT_STORED) {
                const uint32_t nb = b->byte1 - b->byte0, subs = j2p_png_stored_subs(nb);
                for (uint32_t s = 0; s < subs; s++) {
                        const uint32_t len = s + 1 < subs ? 65535 : nb - 65535 * s;
                        j2p_png_put(buf, pos, (final_block && s + 1 == subs) ? 1 : 0, 3);
                        pos = (pos + 3 + 7) & ~7u;
                        j2p_png_put(buf, pos, len, 16);
                        j2p_png_put(buf, pos + 16, ~len & 0xffff, 16);
                        pos += 32 + 8 * len;
                }
                return;
        }
        j2p_png_put(buf, pos, (final_block ? 1 : 0) | b->type << 1, 3);
        pos += 3;
        if (b->type == J2P_BT_DYNAMIC) {
                j2p_png_put(buf, pos, b->hlit - 257, 5);
                j2p_png_put(buf, pos + 5, 0, 5);          /* one distance code */
                j2p_png_put(buf, pos + 10, b->hclen - 4, 4);
                pos += 14;
                for (uint32_t k = 0; k < b->hclen; k++, pos += 3) j2p_png_put(buf, pos, b->bl_len[j2p_png_bl_order(k)], 3);
                j2p_png_rle_lengths(b->len, b->hlit, [&](uint32_t s, uint32_t eb, uint32_t ev) {
                        j2p_png_put(buf, pos, b->bl_code[s], b->bl_len[s]);
                        j2p_png_put(buf, pos + b->bl_len[s], ev, eb);
                        pos += b->bl_len[s] + eb;
                });
        }
        j2p_png_put(buf, b->data_bit0 + b->data_bits, b->code[256], b->len[256]);
}

/* Byte offset in the piece's output of stored byte j (0-based within block b). */
J2P_HD uint32_t j2p_png_stored_at(const struct j2p_png_block *b, uint32_t j) {
        const uint32_t s = j / 65535;
        return ((b->bit0 + 3 + 7) & ~7u) / 8 + s * (65535 + 5) + 4 + (j - 65535 * s);
}

/* The sync flush after the last block of a piece that is not an image's last: an empty stored
 * block (header bits and padding are zero), then 00 00 ff ff. */
J2P_HD void j2p_png_put_flush(uint32_t *buf, uint32_t nbytes) { j2p_png_put(buf, (nbytes - 2) * 8, 0xffff, 16); }

/* ---- checksums ------------------------------------------------------------------------------ */
J2P_HD uint32_t j2p_png_crc(uint32_t crc, const uint8_t *p, uint64_t n, const uint32_t *table) {
        crc = ~crc;
        for (uint64_t i = 0; i < n; i++) crc = table[(crc ^ p[i]) & 0xff] ^ (crc >> 8);
        return ~crc;
}

/* a * b modulo the CRC polynomial (bit-reflected). */
J2P_HD uint32_t j2p_png_mulmod(uint32_t a, uint32_t b) {
        uint32_t p = 0;
        for (uint32_t m = 1u << 31; m; m >>= 1) {
                if (a & m) p ^= b;
                b = (b & 1) ? (b >> 1) ^ J2P_PNG_CRC_POLY : b >> 1;
        }
        return p;
}

/* x^(8n) modulo the polynomial; x2k[k] = x^(2^k). */
J2P_HD uint32_t j2p_png_shift(uint64_t n, const uint32_t *x2k) {
        uint32_t p = 1u << 31, k = 3;
        while (n) {
                if (n & 1) p = j2p_png_mulmod(x2k[k & 31], p);
                n >>= 1;
                k++;
        }
        return p;
}

/* CRC of A then B from crc(A), crc(B) and the operator j2p_png_shift(|B|). */
J2P_HD uint32_t j2p_png_crc_join(uint32_t ca, uint32_t cb, uint32_t op) { return j2p_png_mulmod(op, ca) ^ cb; }

J2P_HD uint32_t j2p_png_adler(uint32_t adler, const uint8_t *p, uint64_t n) {
        uint32_t a = adler & 0xffff, b = adler >> 16;
        while (n) {
                const uint32_t k = n < 5552 ? (uint32_t)n : 5552;
                for (uint32_t i = 0; i < k; i++) { a += p[i]; b += a; }
                a %= 65521;
                b %= 65521;
                p += k;
                n -= k;
        }
        return b << 16 | a;
}

/* Adler-32 of A then B (B of n bytes). */
J2P_HD uint32_t j2p_png_adler_join(uint32_t x, uint32_t y, uint64_t n) {
        const uint32_t BASE = 65521, r = (uint32_t)(n % BASE);
        const uint32_t a1 = x & 0xffff, b1 = x >> 16, a2 = y & 0xffff, b2 = y >> 16;
        const uint32_t a = (a1 + a2 + BASE - 1) % BASE;
        const uint32_t b = (uint32_t)(((uint64_t)b1 + b2 + (uint64_t)r * ((a1 + BASE - 1) % BASE)) % BASE);
        return b << 16 | a;
}

/* ---- container ------------------------------------------------------------------------------ */
#define J2P_PNG_HEAD 43u                  /* signature, IHDR, IDAT length and type, zlib header */
#define J2P_PNG_TAIL 20u                  /* Adler-32, IDAT CRC, IEND */

J2P_HD void j2p_png_be32(uint8_t *p, uint32_t v) {
        p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v;
}

/* Writes the head of a file whose IDAT holds idat_len bytes. */
J2P_HD void j2p_png_head(uint8_t *o, const struct j2p_png_img *im, uint32_t idat_len, const uint32_t *table) {
        o[0] = 0x89; o[1] = 'P'; o[2] = 'N'; o[3] = 'G'; o[4] = 0x0D; o[5] = 0x0A; o[6] = 0x1A; o[7] = 0x0A;
        j2p_png_be32(o + 8, 13);
        o[12] = 'I'; o[13] = 'H'; o[14] = 'D'; o[15] = 'R';
        j2p_png_be32(o + 16, im->w);
        j2p_png_be32(o + 20, im->h);
        o[24] = (uint8_t)(8 * im->sb); o[25] = im->nc == 1 ? 0 : 2; o[26] = 0; o[27] = 0; o[28] = 0;     /* colour type: gray or RGB */
        j2p_png_be32(o + 29, j2p_png_crc(0, o + 12, 17, table));
        j2p_png_be32(o + 33, idat_len);
        o[37] = 'I'; o[38] = 'D'; o[39] = 'A'; o[40] = 'T';
        o[41] = 0x78; o[42] = 0x01;
}

J2P_HD void j2p_png_tail(uint8_t *o, uint32_t adler, uint32_t crc) {
        j2p_png_be32(o, adler);
        j2p_png_be32(o + 4, crc);
        j2p_png_be32(o + 8, 0);
        o[12] = 'I'; o[13] = 'E'; o[14] = 'N'; o[15] = 'D';
        j2p_png_be32(o + 16, 0xae426082u);         /* CRC of "IEND" */
}

/* Upper bound of a piece's output (every block stored, worst padding, the sync flush). */
J2P_HD uint32_t j2p_png_piece_bound(uint32_t n) {
        return n + 6 * ((n + J2P_PNG_BLOCK_SYMS - 1) / J2P_PNG_BLOCK_SYMS + (n + 65534) / 65535 + 2) + 8;
}

#endif
