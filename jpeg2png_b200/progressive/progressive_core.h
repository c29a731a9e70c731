/* progressive_core.h — the per-block decode of each progressive scan kind and the per-subsequence,
 * per-block and per-segment passes of the progressive decoder, written once for the device kernels
 * (progressive.cu) and the serial host driver (j2p_progressive_decode_host).  The bit reader, the
 * Huffman step and the tables are entropy_core.h's.
 *
 * Every rule restates the progressive path of jpeg_reader.c (block_dc_first, block_dc_refine,
 * block_ac_first, block_ac_refine, decode_scan) on one segment of unstuffed bytes:
 *   - bits past the segment's end read as zero; EOB runs start at zero in every segment, and the
 *     blocks of a run that extends past the scan's last block are dropped;
 *   - a code matching no length <= 16 is J2P_ENT_BAD_CODE, a DC category > 16 J2P_ENT_BAD_MAGNITUDE,
 *     k > 63 after a run J2P_ENT_BAD_INDEX; a ZRL that runs past Se ends the block;
 *   - an AC first run may land past Se (up to 63), and the coefficient is stored there;
 *   - an AC refine symbol of any nonzero size places +-2^Al;
 *   - DC first stores (int16_t)(pred << Al), the prediction summed per component over the segment
 *     in decode order, padding blocks of interleaved scans included.
 *
 * DC first and AC first scans are decoded self-synchronising as in entropy_core.h.  The state at a
 * subsequence boundary is (bit offset, x): x is the block index within the MCU for DC first, and the
 * blocks left in the current EOB run for AC first (Ss > 0 scans are never interleaved).  A block that
 * starts inside an EOB run takes no bits and belongs to the subsequence whose bit range holds the
 * position it starts at.  AC refine scans cannot be synchronised that way (the bits a block takes
 * depend on which of its coefficients are already nonzero), so each (file, scan, segment) is walked
 * serially, with a 64-bit zig-zag mask of each block's nonzero coefficients computed before.
 */
#ifndef J2P_PROGRESSIVE_CORE_H
#define J2P_PROGRESSIVE_CORE_H

#include "../entropy/entropy_core.h"
#include "progressive.h"

enum { J2P_PG_DC_FIRST = 0, J2P_PG_DC_REFINE = 1, J2P_PG_AC_FIRST = 2, J2P_PG_AC_REFINE = 3 };

#define J2P_PG_CHUNK 256        /* blocks per chunk of the per-block passes (one CTA each) */

struct j2p_pg_scan {
        uint32_t file, kind, ss, se, al, ncomp, bpm, mcux;
        uint32_t comp[3], bw[3], bh[3], dctab[3], actab[3];
        uint32_t diff_base;     /* DC first: the scan's first block in the DC-difference array */
        uint32_t mask_base;     /* AC refine: the scan's first block in its step's mask array */
        uint8_t slot[J2P_ENT_MAX_BPM], dx[J2P_ENT_MAX_BPM], dy[J2P_ENT_MAX_BPM];   /* block r of an MCU */
};
/* J2P_PG_CHUNK blocks from `first` of a DC refine segment or an AC refine scan (`item`) */
struct j2p_pg_chunk {
        uint32_t item, first;
};
/* the work of one step: its subsequences (DC and AC first), refine segments, DC refine chunks and
 * mask chunks */
struct j2p_pg_step {
        uint32_t sub0, nsub, rseg0, nrseg, dchunk0, ndchunk, mchunk0, nmchunk;
};
struct j2p_pg_header {
        uint32_t magic, nfiles, nscan, nseg, ntab, nsub, subseq_bits, nsteps;
        uint32_t nrseg, nchunk, pad[2];
        uint64_t nblocks;       /* DC differences (all blocks of all DC first scans, padding included) */
        uint64_t nmask;         /* mask words: the most blocks of AC refine scans in one step */
        uint64_t off_files, off_scans, off_segs, off_subs, off_tabs, off_steps, off_rsegs, off_chunks, off_data, total;
};

/* pointers into a packed plan (host or device copy) and the work area */
struct j2p_pg_view {
        const struct j2p_ent_file *files;
        const struct j2p_pg_scan *scans;
        const struct j2p_ent_seg *segs;
        const uint32_t *sub_seg;    /* subsequence -> segment */
        const struct j2p_ent_table *tabs;
        const uint32_t *rsegs;      /* refine walker -> segment */
        const struct j2p_pg_chunk *chunks;
        const uint8_t *data;
        uint32_t nsub, subseq_bits;
        /* work */
        uint64_t *exit_st[2];       /* exit state per subsequence, by round parity */
        uint64_t *start_st;         /* the start state of its last decode */
        uint64_t *cnt, *cnt_x;      /* blocks owned (sync, at most the segment's), exclusive scan */
        uint32_t *fcnt;             /* blocks of a DC first subsequence decoded by the difference pass */
        uint64_t *dcs, *dcs_x;      /* [3][nsub] DC sums per scan slot, exclusive scan */
        int32_t *diff;              /* DC difference per block */
        uint64_t *mask;             /* zig-zag nonzero mask per block of the step's AC refine scans */
        uint32_t *changed;
        uint32_t *status;           /* per file */
};

#ifdef __CUDA_ARCH__
#define J2P_PG_POPC64(x) __popcll(x)
#define J2P_PG_CTZ64(x) (__ffsll((long long)(x)) - 1)
#else
#define J2P_PG_POPC64(x) __builtin_popcountll(x)
#define J2P_PG_CTZ64(x) __builtin_ctzll(x)
#endif

J2P_HD uint64_t j2p_pg_state(uint32_t pos, uint32_t x) { return ((uint64_t)pos << 32) | x; }
J2P_HD uint64_t j2p_pg_from(int k) { return k >= 64 ? 0 : ~0ull << k; }             /* positions >= k */
J2P_HD uint64_t j2p_pg_below(int k) { return k >= 64 ? ~0ull : (1ull << k) - 1; }  /* positions < k */

/* the position of set bit n (from 0, lowest first) of m; 64 when m has no more */
J2P_HD int j2p_pg_nth(uint64_t m, int n) {
#ifdef __CUDA_ARCH__
        const uint32_t lo = (uint32_t)m, hi = (uint32_t)(m >> 32);
        const int nlo = __popc(lo);
        if (n < nlo) return (int)__fns(lo, 0, n + 1);
        n -= nlo;
        return n < __popc(hi) ? 32 + (int)__fns(hi, 0, n + 1) : 64;
#else
        for (; m; m &= m - 1)
                if (n-- == 0) return __builtin_ctzll(m);
        return 64;
#endif
}

/* the bit range [first, end) whose blocks subsequence j owns; end = UINT32_MAX for a segment's last */
J2P_HD const struct j2p_ent_seg *j2p_pg_range(const struct j2p_pg_view *v, uint32_t j, uint32_t *i, uint32_t *end) {
        const struct j2p_ent_seg *g = &v->segs[v->sub_seg[j]];
        *i = j - g->sub0;
        *end = *i + 1 == g->nsub ? 0xffffffffu : (*i + 1) * v->subseq_bits;
        return g;
}

/* ---- one block of each kind ---------------------------------------------------------------- */
/* block_dc_first's bits: *diff, the DC difference */
J2P_HD int j2p_pg_dc_block(struct j2p_ent_bits *b, const struct j2p_ent_table *t, int32_t *diff) {
        j2p_ent_refill(b);
        const int s = j2p_ent_huff(b, t);
        if (s < 0) return J2P_ENT_BAD_CODE;
        if (s > 16) return J2P_ENT_BAD_MAGNITUDE;
        *diff = s ? j2p_ent_extend(j2p_ent_getbits(b, s), s) : 0;
        return J2P_ENT_OK;
}

/* block_ac_first for a block outside an EOB run: stores extend(v) << Al into out (natural order;
 * NULL: decode only) and sets *run to the blocks of the EOB run that follow the block */
J2P_HD int j2p_pg_acf_block(struct j2p_ent_bits *b, const struct j2p_ent_table *t, int ss, int se, int al, int16_t *out, uint32_t *run) {
        for (int k = ss; k <= se; k++) {
                j2p_ent_refill(b);
                const int rs = j2p_ent_huff(b, t);
                if (rs < 0) return J2P_ENT_BAD_CODE;
                const int r = rs >> 4, s = rs & 15;
                if (s) {
                        k += r;
                        if (k > 63) return J2P_ENT_BAD_INDEX;
                        const int v = j2p_ent_extend(j2p_ent_getbits(b, s), s);
                        if (out) out[j2p_ent_zz[k]] = (int16_t)(v * (1 << al));
                } else if (r == 15) {
                        k += 15;
                } else {
                        uint32_t n = 1u << r;
                        if (r) n += (uint32_t)j2p_ent_getbits(b, r);
                        *run = n - 1;
                        break;
                }
        }
        return J2P_ENT_OK;
}

/* the correction bits of the nonzero coefficients at the zig-zag positions in `corr`, lowest first:
 * a 1 adds 2^Al away from zero to a coefficient whose 2^Al bit is clear (G.1.2.3) */
J2P_HD void j2p_pg_correct(struct j2p_ent_bits *b, int16_t *blk, uint64_t corr, int p1) {
        while (corr) {
                const int pc = J2P_PG_POPC64(corr), take = pc < 16 ? pc : 16;
                j2p_ent_refill(b);
                const uint32_t bits = (uint32_t)j2p_ent_getbits(b, take);
                for (int i = take - 1; i >= 0; i--) {
                        const int pos = J2P_PG_CTZ64(corr);
                        corr &= corr - 1;
                        if ((bits >> i) & 1) {
                                int16_t *cf = &blk[j2p_ent_zz[pos]];
                                const int c = *cf;
                                if ((c & p1) == 0) *cf = (int16_t)(c + (c >= 0 ? p1 : -p1));
                        }
                }
        }
}

/* block_ac_refine on a block whose coefficients (natural order) were nonzero at the zig-zag
 * positions of nz before the scan.  Memory is touched only to place a new +-2^Al and to apply a
 * correction whose bit is 1. */
J2P_HD int j2p_pg_refine_block(struct j2p_ent_bits *b, const struct j2p_ent_table *t, int ss, int se, int al, int16_t *blk, uint64_t nz,
                               uint32_t *run) {
        const int p1 = 1 << al;
        const uint64_t band = j2p_pg_below(se + 1);
        int k = ss;
        if (*run == 0) {
                for (; k <= se; k++) {
                        j2p_ent_refill(b);
                        const int rs = j2p_ent_huff(b, t);
                        if (rs < 0) return J2P_ENT_BAD_CODE;
                        const int r = rs >> 4, s = rs & 15;
                        int val = 0;
                        if (s) {
                                val = j2p_ent_getbits(b, 1) ? p1 : -p1;
                        } else if (r != 15) {
                                uint32_t n = 1u << r;
                                if (r) n += (uint32_t)j2p_ent_getbits(b, r);
                                *run = n;
                                break;
                        }
                        /* skip r zero-history positions, correcting the nonzero ones passed, and stop
                         * on the next zero-history position (past Se when there is none) */
                        const uint64_t ahead = band & j2p_pg_from(k);
                        const int kz = j2p_pg_nth(~nz & ahead, r);
                        const int stop = kz < 64 ? kz : se + 1;
                        j2p_pg_correct(b, blk, nz & ahead & j2p_pg_below(stop), p1);
                        k = stop;
                        if (s && k <= se) blk[j2p_ent_zz[k]] = (int16_t)val;
                }
        }
        if (*run > 0) {
                j2p_pg_correct(b, blk, nz & band & j2p_pg_from(k), p1);
                (*run)--;
        }
        return J2P_ENT_OK;
}

/* ---- DC first and AC first: self-synchronising passes ------------------------------------- */
/* one sync round for subsequence j.  Returns 1 when its start state changed. */
J2P_HD int j2p_pg_sync_one(const struct j2p_pg_view *v, uint32_t j, uint32_t round) {
        uint32_t i, end;
        const struct j2p_ent_seg *g = j2p_pg_range(v, j, &i, &end);
        const uint64_t start = i == 0 ? 0 : round == 0 ? j2p_pg_state(i * v->subseq_bits, 0) : v->exit_st[(round - 1) & 1][j - 1];
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
        const struct j2p_pg_scan *sc = &v->scans[g->scan];
        struct j2p_ent_bits b;
        j2p_ent_seek(&b, v->data + g->data_off, g->nbytes, (uint32_t)(start >> 32));
        uint32_t x = (uint32_t)start;
        uint64_t n = 0;
        if (sc->kind == J2P_PG_DC_FIRST) {
                while (b.pos < end) {
                        int32_t diff;
                        if (j2p_pg_dc_block(&b, &v->tabs[sc->dctab[sc->slot[x]]], &diff) != J2P_ENT_OK) {
                                b.pos = end;        /* a guessed state ran into an invalid code: any fixed exit will do */
                                x = 0;
                                break;
                        }
                        n++;
                        x = x + 1 == sc->bpm ? 0 : x + 1;
                }
        } else {
                const struct j2p_ent_table *t = &v->tabs[sc->actab[0]];
                while (b.pos < end) {
                        if (x) {                    /* the rest of an EOB run starts here */
                                n += x;
                                x = 0;
                                continue;
                        }
                        if (j2p_pg_acf_block(&b, t, (int)sc->ss, (int)sc->se, (int)sc->al, 0, &x) != J2P_ENT_OK) {
                                b.pos = end;
                                x = 0;
                                break;
                        }
                        n++;
                }
        }
        exit_now[j] = j2p_pg_state(b.pos, x);
        v->cnt[j] = n < g->nblocks ? n : g->nblocks;     /* blocks past the segment's are dropped anyway */
        return round > 0;
}

/* the first block of subsequence j in its scan's decode order */
J2P_HD uint64_t j2p_pg_first(const struct j2p_pg_view *v, const struct j2p_ent_seg *g, uint32_t j) {
        return g->block0 + (v->cnt_x[j] - v->cnt_x[g->sub0]);
}

/* DC first, after the exclusive scan of cnt: decode subsequence j from its exact start state, write
 * its DC differences and sum them per scan slot.  AC first subsequences write zero sums. */
J2P_HD int j2p_pg_dcdiff_one(const struct j2p_pg_view *v, uint32_t j) {
        uint32_t i, end;
        const struct j2p_ent_seg *g = j2p_pg_range(v, j, &i, &end);
        const struct j2p_pg_scan *sc = &v->scans[g->scan];
        uint64_t sum[3] = {0, 0, 0};
        uint32_t n = 0;
        int rc = J2P_ENT_OK;
        if (sc->kind == J2P_PG_DC_FIRST) {
                const uint64_t limit = g->block0 + g->nblocks;
                struct j2p_ent_bits b;
                j2p_ent_seek(&b, v->data + g->data_off, g->nbytes, (uint32_t)(v->start_st[j] >> 32));
                for (uint64_t gi = j2p_pg_first(v, g, j); gi < limit && b.pos < end; gi++, n++) {
                        const uint32_t s = sc->slot[gi % sc->bpm];
                        int32_t diff = 0;
                        rc = j2p_pg_dc_block(&b, &v->tabs[sc->dctab[s]], &diff);
                        if (rc != J2P_ENT_OK) break;
                        v->diff[sc->diff_base + gi] = diff;
                        const uint64_t d = (uint64_t)(int64_t)diff;
                        sum[0] += s == 0 ? d : 0;      /* no dynamic index: keeps the sums in registers */
                        sum[1] += s == 1 ? d : 0;
                        sum[2] += s == 2 ? d : 0;
                }
        }
        v->fcnt[j] = n;
        for (int s = 0; s < 3; s++) v->dcs[(size_t)s * v->nsub + j] = sum[s];
        return rc;
}

/* the step's store of subsequence j: DC first writes (int16_t)(pred << Al) to coefficient 0 of its
 * blocks (after the exclusive scan of dcs); AC first decodes its blocks and writes their bands */
J2P_HD int j2p_pg_store_one(const struct j2p_pg_view *v, uint32_t j) {
        uint32_t i, end;
        const struct j2p_ent_seg *g = j2p_pg_range(v, j, &i, &end);
        const struct j2p_pg_scan *sc = &v->scans[g->scan];
        const struct j2p_ent_file *f = &v->files[sc->file];
        const uint64_t gi0 = j2p_pg_first(v, g, j);
        if (sc->kind == J2P_PG_DC_FIRST) {
                const uint64_t *x = v->dcs_x;
                uint64_t p0 = x[j] - x[g->sub0], p1 = x[v->nsub + j] - x[v->nsub + g->sub0];
                uint64_t p2 = x[2 * (size_t)v->nsub + j] - x[2 * (size_t)v->nsub + g->sub0];
                for (uint64_t gi = gi0; gi < gi0 + v->fcnt[j]; gi++) {
                        const uint32_t m = (uint32_t)(gi / sc->bpm), r = (uint32_t)(gi - (uint64_t)m * sc->bpm), s = sc->slot[r], c = sc->comp[s];
                        const uint64_t d = (uint64_t)(int64_t)v->diff[sc->diff_base + gi];
                        p0 += s == 0 ? d : 0;      /* no dynamic index: keeps the predictions in registers */
                        p1 += s == 1 ? d : 0;
                        p2 += s == 2 ? d : 0;
                        const uint64_t pred = s == 0 ? p0 : s == 1 ? p1 : p2;
                        const uint32_t my = m / sc->mcux, mx = m - my * sc->mcux;
                        const uint32_t bx = mx * sc->bw[s] + sc->dx[r], by = my * sc->bh[s] + sc->dy[r];
                        if (bx < f->wb[c] && by < f->hb[c]) f->out[c][((size_t)by * f->wb[c] + bx) * 64] = (int16_t)(uint16_t)((uint32_t)pred << sc->al);
                }
                return J2P_ENT_OK;
        }
        /* AC first: one component, its real block grid, so a block's index in the scan is its index in the plane */
        const uint64_t limit = g->block0 + g->nblocks;
        const struct j2p_ent_table *t = &v->tabs[sc->actab[0]];
        int16_t *plane = f->out[sc->comp[0]];
        struct j2p_ent_bits b;
        j2p_ent_seek(&b, v->data + g->data_off, g->nbytes, (uint32_t)(v->start_st[j] >> 32));
        uint32_t x = (uint32_t)v->start_st[j];
        uint64_t gi = gi0;
        while (gi < limit && b.pos < end) {
                if (x) {
                        const uint64_t k = x < limit - gi ? x : limit - gi;
                        gi += k;
                        x -= (uint32_t)k;
                        continue;
                }
                const int rc = j2p_pg_acf_block(&b, t, (int)sc->ss, (int)sc->se, (int)sc->al, plane + gi * 64, &x);
                if (rc != J2P_ENT_OK) return rc;
                gi++;
        }
        return J2P_ENT_OK;
}

/* ---- DC refine and AC refine ---------------------------------------------------------------- */
/* DC refine, block `first + t` of chunk ch's segment: one bit per block in decode order, padding
 * blocks included */
J2P_HD void j2p_pg_dcref_one(const struct j2p_pg_view *v, const struct j2p_pg_chunk *ch, uint32_t t) {
        const struct j2p_ent_seg *g = &v->segs[ch->item];
        const uint32_t k = ch->first + t;
        if (k >= g->nblocks || (k >> 3) >= g->nbytes) return;
        if (!((v->data[g->data_off + (k >> 3)] >> (7 - (k & 7))) & 1)) return;
        const struct j2p_pg_scan *sc = &v->scans[g->scan];
        const struct j2p_ent_file *f = &v->files[sc->file];
        const uint32_t gi = g->block0 + k, m = gi / sc->bpm, r = gi - m * sc->bpm, s = sc->slot[r], c = sc->comp[s];
        const uint32_t my = m / sc->mcux, mx = m - my * sc->mcux;
        const uint32_t bx = mx * sc->bw[s] + sc->dx[r], by = my * sc->bh[s] + sc->dy[r];
        if (bx < f->wb[c] && by < f->hb[c]) {
                int16_t *o = &f->out[c][((size_t)by * f->wb[c] + bx) * 64];
                *o = (int16_t)(*o | (1 << sc->al));
        }
}

/* AC refine, before the scan: the zig-zag nonzero mask of block `first + t` of chunk ch's scan */
J2P_HD void j2p_pg_mask_one(const struct j2p_pg_view *v, const struct j2p_pg_chunk *ch, uint32_t t) {
        const struct j2p_pg_scan *sc = &v->scans[ch->item];
        const struct j2p_ent_file *f = &v->files[sc->file];
        const uint32_t c = sc->comp[0], k = ch->first + t;
        if (k >= f->wb[c] * f->hb[c]) return;
        const int16_t *blk = f->out[c] + (size_t)k * 64;
        uint64_t nat = 0;
        for (int p = 0; p < 64; p++) nat |= (uint64_t)(blk[p] != 0) << p;
        uint64_t zz = 0;
        for (int p = 0; p < 64; p++) zz |= ((nat >> j2p_ent_zz[p]) & 1) << p;
        v->mask[sc->mask_base + k] = zz;
}

/* AC refine, walker w: every block of its segment in order, from an EOB run of zero */
J2P_HD int j2p_pg_refine_one(const struct j2p_pg_view *v, uint32_t w) {
        const struct j2p_ent_seg *g = &v->segs[v->rsegs[w]];
        const struct j2p_pg_scan *sc = &v->scans[g->scan];
        const struct j2p_ent_table *t = &v->tabs[sc->actab[0]];
        int16_t *plane = v->files[sc->file].out[sc->comp[0]];
        struct j2p_ent_bits b;
        j2p_ent_seek(&b, v->data + g->data_off, g->nbytes, 0);
        uint32_t run = 0;
        for (uint32_t gi = g->block0; gi < g->block0 + g->nblocks; gi++) {
                const int rc = j2p_pg_refine_block(&b, t, (int)sc->ss, (int)sc->se, (int)sc->al, plane + (size_t)gi * 64,
                                                   v->mask[sc->mask_base + gi], &run);
                if (rc != J2P_ENT_OK) return rc;
        }
        return J2P_ENT_OK;
}

#endif
