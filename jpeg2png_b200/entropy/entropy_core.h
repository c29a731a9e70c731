/* entropy_core.h — the per-block Huffman decode step and the three per-subsequence phases of the
 * device entropy decoder, written once for the device kernels (entropy.cu) and the serial host
 * driver (j2p_entropy_decode_host), which runs the same phases in order so that a machine without
 * a GPU can test them against jpeg_reader.c.
 *
 * Every rule here restates the sequential path of jpeg_reader.c (block_sequential, decode_huff,
 * getbits, extend) on one segment of unstuffed bytes:
 *   - bits past the segment's end read as zero;
 *   - a code matching no length <= 16 is J2P_ENT_BAD_CODE, a DC category > 16 J2P_ENT_BAD_MAGNITUDE,
 *     k > 63 after a run J2P_ENT_BAD_INDEX; a ZRL that runs past k = 63 ends the block silently;
 *   - the DC difference is summed per component over the segment in decode order (padding blocks
 *     included) and stored as (int16_t) of the sum, which wraps like the reader's int.
 *
 * Self-synchronising decode (Weißenberger & Schmidt): a segment's bits are cut into subsequences of
 * subseq_bits; a subsequence owns the blocks whose first bit lies in it, so a decoder state at a
 * boundary is (bit offset, block index within the MCU) and its zig-zag index is always 0.  Sync
 * round r decodes every subsequence from its start state (round 0: a guess at its first bit) and
 * makes each exit state the successor's start state; a subsequence whose start did not change keeps
 * its exit.  A round in which no start changed leaves every state exact.  Speculative decodes that
 * hit an invalid code stop at the subsequence's end; only the final pass records a failure.
 */
#ifndef J2P_ENTROPY_CORE_H
#define J2P_ENTROPY_CORE_H

#include <stdint.h>
#include <string.h>

#include "../cli/jpeg_reader.h"         /* struct j2p_jpeg_huff */
#include "../common/codec_host.h"       /* J2P_HD */
#include "entropy.h"

#define J2P_ENT_MAX_BPM 48      /* blocks per MCU: three components of up to 4x4 (the reader allows 4); a
                                   four-component file's interleaved scan has at most 10 (jpeg_reader.h) */
#define J2P_ENT_PLANES 4        /* planes per file: three (colour), one (gray) or four (CMYK, YCCK) used */

/* one Huffman table: T.81 F.2.2.3 as jpeg_reader.c's build_huff, plus a 9-bit first level */
struct j2p_ent_table {
        int32_t maxcode[17], mincode[17], valptr[17];   /* [l], l = 1..16 */
        uint16_t lut[512];      /* (length << 8) | value for codes of at most 9 bits; 0: longer */
        uint8_t vals[256];
};
struct j2p_ent_file {
        int16_t *out[J2P_ENT_PLANES];       /* int16 [hb][wb][64] per plane, natural order */
        uint32_t wb[J2P_ENT_PLANES], hb[J2P_ENT_PLANES];   /* real block grids */
};
struct j2p_ent_scan {
        uint32_t file, ncomp, bpm, mcux;
        uint32_t comp[J2P_ENT_PLANES], bw[J2P_ENT_PLANES], bh[J2P_ENT_PLANES], dctab[J2P_ENT_PLANES], actab[J2P_ENT_PLANES];
        uint32_t diff_base;     /* the scan's first block in the DC-difference array */
        uint8_t slot[J2P_ENT_MAX_BPM], dx[J2P_ENT_MAX_BPM], dy[J2P_ENT_MAX_BPM];   /* block r of an MCU */
};
struct j2p_ent_seg {
        uint64_t data_off;      /* 4-byte aligned */
        uint32_t nbytes, scan;
        uint32_t block0, nblocks;   /* its blocks in the scan's decode order */
        uint32_t sub0, nsub;    /* its subsequences */
};
struct j2p_ent_header {
        uint32_t magic, nfiles, nscan, nseg, ntab, nsub, subseq_bits;
        uint32_t nslot;         /* scan slots with DC sums: 3, or 4 when a scan has four components */
        uint64_t nblocks;       /* DC differences (all blocks of all scans, padding included) */
        uint64_t off_files, off_scans, off_segs, off_subs, off_tabs, off_data, total;
};

/* pointers into a packed plan (host or device copy) and the work area */
struct j2p_ent_view {
        const struct j2p_ent_file *files;
        const struct j2p_ent_scan *scans;
        const struct j2p_ent_seg *segs;
        const uint32_t *sub_seg;    /* subsequence -> segment */
        const struct j2p_ent_table *tabs;
        const uint8_t *data;
        uint32_t nsub, subseq_bits, nslot;
        /* work */
        uint64_t *exit_st[2];       /* exit state per subsequence, by round parity */
        uint64_t *start_st;         /* the start state of its last decode */
        uint32_t *cnt, *cnt_x;      /* blocks owned (sync), exclusive scan */
        uint32_t *fcnt;             /* blocks decoded by the final pass */
        uint32_t *dcs, *dcs_x;      /* [nslot][nsub] DC sums per scan slot, exclusive scan */
        int32_t *diff;              /* DC difference per block */
        uint32_t *changed;
        uint32_t *status;           /* per file */
};

/* build_huff of jpeg_reader.c, plus the 9-bit first level (host) */
static inline void j2p_ent_build_table(const struct j2p_jpeg_huff *src, struct j2p_ent_table *t) {
        memset(t, 0, sizeof *t);
        int code = 0, k = 0;
        for (int l = 1; l <= 16; l++) {
                t->valptr[l] = k;
                t->mincode[l] = code;
                code += src->bits[l];
                k += src->bits[l];
                t->maxcode[l] = src->bits[l] ? code - 1 : -1;
                code <<= 1;
        }
        memcpy(t->vals, src->vals, 256);
        for (int p = 0; p < 512; p++)
                for (int l = 1; l <= 9; l++) {
                        const int c = p >> (9 - l);
                        if (t->maxcode[l] >= 0 && c <= t->maxcode[l] && c >= t->mincode[l]) {
                                t->lut[p] = (uint16_t)((l << 8) | t->vals[t->valptr[l] + c - t->mincode[l]]);
                                break;
                        }
                }
}

#ifdef __CUDA_ARCH__
__constant__ uint8_t j2p_ent_zz[64] =
#else
static const uint8_t j2p_ent_zz[64] =
#endif
        {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
         41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
         30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

/* ---- bit reader over one segment: 64-bit window, big-endian 32-bit words, zero past the end ---- */
struct j2p_ent_bits {
        const uint8_t *base;    /* 4-byte aligned; the packed plan pads every segment to 4 bytes */
        uint32_t nbytes, wnext, pos;
        int nbuf;
        uint64_t buf;
};

J2P_HD uint32_t j2p_ent_word(const struct j2p_ent_bits *b, uint32_t w) {
        const uint32_t off = w * 4;
        if (off >= b->nbytes) return 0;
        uint32_t v;
#ifdef __CUDA_ARCH__
        v = __byte_perm(__ldg((const unsigned int *)(b->base + off)), 0, 0x0123);
#else
        memcpy(&v, b->base + off, 4);
        v = __builtin_bswap32(v);
#endif
        if (off + 4 > b->nbytes) v &= ~0u << (8 * (off + 4 - b->nbytes));
        return v;
}
J2P_HD void j2p_ent_refill(struct j2p_ent_bits *b) {
        while (b->nbuf <= 32) {
                b->buf |= (uint64_t)j2p_ent_word(b, b->wnext++) << (32 - b->nbuf);
                b->nbuf += 32;
        }
}
J2P_HD void j2p_ent_seek(struct j2p_ent_bits *b, const uint8_t *base, uint32_t nbytes, uint32_t pos) {
        b->base = base;
        b->nbytes = nbytes;
        b->wnext = pos >> 5;
        b->buf = 0;
        b->nbuf = 0;
        j2p_ent_refill(b);
        b->buf <<= (pos & 31);
        b->nbuf -= (int)(pos & 31);
        b->pos = pos;
}
J2P_HD void j2p_ent_skip(struct j2p_ent_bits *b, int n) {
        b->buf <<= n;
        b->nbuf -= n;
        b->pos += (uint32_t)n;
}
/* decode_huff; < 0: no code of length <= 16 matches.  Needs 16 bits in the window. */
J2P_HD int j2p_ent_huff(struct j2p_ent_bits *b, const struct j2p_ent_table *t) {
        const uint32_t p16 = (uint32_t)(b->buf >> 48);
        const uint32_t e = t->lut[p16 >> 7];
        if (e) {
                j2p_ent_skip(b, (int)(e >> 8));
                return (int)(e & 255);
        }
        for (int l = 10; l <= 16; l++) {
                const int32_t code = (int32_t)(p16 >> (16 - l));
                if (t->maxcode[l] >= 0 && code <= t->maxcode[l] && code >= t->mincode[l]) {
                        j2p_ent_skip(b, l);
                        return t->vals[t->valptr[l] + code - t->mincode[l]];
                }
        }
        return -1;
}
J2P_HD int j2p_ent_getbits(struct j2p_ent_bits *b, int n) {      /* 0 <= n <= 16 */
        if (n <= 0) return 0;
        const int v = (int)(b->buf >> (64 - n));
        j2p_ent_skip(b, n);
        return v;
}
J2P_HD int j2p_ent_extend(int v, int s) { return (s < 1 || s > 16) ? 0 : (v < (1 << (s - 1)) ? v - (1 << s) + 1 : v); }

/* One block (block_sequential).  out: the block's 64 coefficients in natural order, written whole
 * (zeros included), or NULL to decode without storing.  *diff: the DC difference. */
J2P_HD int j2p_ent_block(struct j2p_ent_bits *b, const struct j2p_ent_table *dc, const struct j2p_ent_table *ac, int16_t *out,
                         int32_t *diff) {
        j2p_ent_refill(b);
        int s = j2p_ent_huff(b, dc);
        if (s < 0) return J2P_ENT_BAD_CODE;
        if (s > 16) return J2P_ENT_BAD_MAGNITUDE;
        *diff = s ? j2p_ent_extend(j2p_ent_getbits(b, s), s) : 0;
        if (out) {
#ifdef __CUDA_ARCH__
                uint4 *o = (uint4 *)out;
#pragma unroll
                for (int i = 0; i < 8; i++) o[i] = make_uint4(0, 0, 0, 0);
#else
                memset(out, 0, 64 * sizeof(int16_t));
#endif
        }
        for (int k = 1; k < 64; k++) {
                j2p_ent_refill(b);
                const int rs = j2p_ent_huff(b, ac);
                if (rs < 0) return J2P_ENT_BAD_CODE;
                const int r = rs >> 4;
                s = rs & 15;
                if (s) {
                        k += r;
                        if (k > 63) return J2P_ENT_BAD_INDEX;
                        const int v = j2p_ent_extend(j2p_ent_getbits(b, s), s);
                        if (out) out[j2p_ent_zz[k]] = (int16_t)v;
                } else {
                        if (r != 15) break;     /* EOB */
                        k += 15;
                }
        }
        return J2P_ENT_OK;
}

J2P_HD uint64_t j2p_ent_state(uint32_t pos, uint32_t blk) { return ((uint64_t)pos << 8) | blk; }

/* the bit range [first, end) whose blocks subsequence j owns; end = UINT32_MAX for a segment's last */
J2P_HD const struct j2p_ent_seg *j2p_ent_range(const struct j2p_ent_view *v, uint32_t j, uint32_t *i, uint32_t *end) {
        const struct j2p_ent_seg *g = &v->segs[v->sub_seg[j]];
        *i = j - g->sub0;
        *end = *i + 1 == g->nsub ? 0xffffffffu : (*i + 1) * v->subseq_bits;
        return g;
}

/* phase 1, one sync round for subsequence j.  Returns 1 when its start state changed. */
J2P_HD int j2p_ent_sync_one(const struct j2p_ent_view *v, uint32_t j, uint32_t round) {
        uint32_t i, end;
        const struct j2p_ent_seg *g = j2p_ent_range(v, j, &i, &end);
        const uint64_t start = i == 0 ? 0 : round == 0 ? j2p_ent_state(i * v->subseq_bits, 0) : v->exit_st[(round - 1) & 1][j - 1];
        uint64_t *exit_now = v->exit_st[round & 1];
        if (round > 0 && start == v->start_st[j]) {
                exit_now[j] = v->exit_st[(round - 1) & 1][j];
                return 0;
        }
        v->start_st[j] = start;
        if (i + 1 == g->nsub) {             /* the last subsequence's exit and count are never used */
                exit_now[j] = start;
                v->cnt[j] = 0;
                return 0;
        }
        const struct j2p_ent_scan *sc = &v->scans[g->scan];
        struct j2p_ent_bits b;
        j2p_ent_seek(&b, v->data + g->data_off, g->nbytes, (uint32_t)(start >> 8));
        uint32_t blk = (uint32_t)(start & 255), n = 0;
        while (b.pos < end) {
                const uint32_t s = sc->slot[blk];
                int32_t diff;
                if (j2p_ent_block(&b, &v->tabs[sc->dctab[s]], &v->tabs[sc->actab[s]], 0, &diff) != J2P_ENT_OK) {
                        b.pos = end;        /* a guessed state ran into an invalid code: any fixed exit will do */
                        blk = 0;
                        break;
                }
                n++;
                blk = blk + 1 == sc->bpm ? 0 : blk + 1;
        }
        exit_now[j] = j2p_ent_state(b.pos, blk);
        v->cnt[j] = n;
        return round > 0;
}

/* phase 2 (after the exclusive scan of cnt): decode subsequence j from its exact start state, write
 * its whole blocks and DC differences, and sum the differences per scan slot.  Returns a failure
 * code of a block inside the segment's MCUs, J2P_ENT_OK otherwise. */
J2P_HD int j2p_ent_final_one(const struct j2p_ent_view *v, uint32_t j) {
        uint32_t i, end;
        const struct j2p_ent_seg *g = j2p_ent_range(v, j, &i, &end);
        const struct j2p_ent_scan *sc = &v->scans[g->scan];
        const struct j2p_ent_file *f = &v->files[sc->file];
        const uint64_t start = v->start_st[j];
        uint32_t gi = g->block0 + (v->cnt_x[j] - v->cnt_x[g->sub0]);
        const uint32_t limit = g->block0 + g->nblocks;
        uint32_t sum[4] = {0, 0, 0, 0}, n = 0;
        int rc = J2P_ENT_OK;
        struct j2p_ent_bits b;
        j2p_ent_seek(&b, v->data + g->data_off, g->nbytes, (uint32_t)(start >> 8));
        for (; gi < limit && b.pos < end; gi++, n++) {
                const uint32_t m = gi / sc->bpm, r = gi - m * sc->bpm, s = sc->slot[r], c = sc->comp[s];
                const uint32_t my = m / sc->mcux, mx = m - my * sc->mcux;
                const uint32_t bx = mx * sc->bw[s] + sc->dx[r], by = my * sc->bh[s] + sc->dy[r];
                int16_t *out = bx < f->wb[c] && by < f->hb[c] ? f->out[c] + ((size_t)by * f->wb[c] + bx) * 64 : 0;
                int32_t diff = 0;
                rc = j2p_ent_block(&b, &v->tabs[sc->dctab[s]], &v->tabs[sc->actab[s]], out, &diff);
                if (rc != J2P_ENT_OK) break;
                v->diff[sc->diff_base + gi] = diff;
                sum[0] += s == 0 ? (uint32_t)diff : 0;     /* no dynamic index: keeps the sums in registers */
                sum[1] += s == 1 ? (uint32_t)diff : 0;
                sum[2] += s == 2 ? (uint32_t)diff : 0;
                sum[3] += s == 3 ? (uint32_t)diff : 0;
        }
        v->fcnt[j] = n;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
        for (int s = 0; s < 4; s++)
                if ((uint32_t)s < v->nslot) v->dcs[(size_t)s * v->nsub + j] = sum[s];
        return rc;
}

/* phase 3 (after the exclusive scan of dcs): the DC predictions of subsequence j's blocks */
J2P_HD void j2p_ent_dc_one(const struct j2p_ent_view *v, uint32_t j) {
        uint32_t i, end;
        const struct j2p_ent_seg *g = j2p_ent_range(v, j, &i, &end);
        const struct j2p_ent_scan *sc = &v->scans[g->scan];
        const struct j2p_ent_file *f = &v->files[sc->file];
        uint32_t pred[4] = {0, 0, 0, 0};
        for (uint32_t s = 0; s < v->nslot; s++) pred[s] = v->dcs_x[(size_t)s * v->nsub + j] - v->dcs_x[(size_t)s * v->nsub + g->sub0];
        const uint32_t gi0 = g->block0 + (v->cnt_x[j] - v->cnt_x[g->sub0]), n = v->fcnt[j];
        for (uint32_t gi = gi0; gi < gi0 + n; gi++) {
                const uint32_t m = gi / sc->bpm, r = gi - m * sc->bpm, s = sc->slot[r], c = sc->comp[s];
                pred[s] += (uint32_t)v->diff[sc->diff_base + gi];
                const uint32_t my = m / sc->mcux, mx = m - my * sc->mcux;
                const uint32_t bx = mx * sc->bw[s] + sc->dx[r], by = my * sc->bh[s] + sc->dy[r];
                if (bx < f->wb[c] && by < f->hb[c]) f->out[c][((size_t)by * f->wb[c] + bx) * 64] = (int16_t)pred[s];
        }
}

#endif
