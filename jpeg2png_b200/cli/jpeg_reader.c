/* jpeg_reader.c — JPEG file -> quantised DCT coefficients (see jpeg_reader.h).
 *
 * A from-scratch ITU T.81 entropy decoder that stops where libjpeg's jpeg_read_coefficients
 * stops: after Huffman or arithmetic decoding, before dequantisation.  Section references are to
 * T.81.  The QM decoder and the sequential arithmetic block step are ../arith/arith_core.h, shared
 * with the device decoder of libj2parith.so; the progressive arithmetic steps are here.
 */
#include "jpeg_reader.h"
#include "../arith/arith_core.h"

#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

/* zigzag position -> natural (row-major) index, T.81 figure A.6 */
static const uint8_t ZZ[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                               41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                               30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct huff {
        int present;
        uint8_t bits[17];
        uint8_t vals[256];
        int mincode[17], maxcode[18], valptr[17];     /* T.81 F.2.2.3 */
};

struct comp {
        int id, h, v, tq;
        unsigned wb, hb;          /* real block grid (jpeg.c:52-53) */
        unsigned pwb, phb;        /* MCU-padded block grid used while decoding */
        int16_t *blk;             /* [phb][pwb][64], natural order */
        int dc_pred;
        int dc_ctx;               /* arithmetic coding: the DC conditioning category (F.1.4.4.1.2) */
        int td, ta;               /* tables of the current scan */
};

struct dec {
        const uint8_t *p, *end;
        uint32_t acc;
        int nbits;
        int hit_marker;           /* a marker was met inside entropy data (stop feeding bits, give zeros) */
        uint16_t qt[4][64];       /* natural order */
        int qt_present[4];
        struct huff dc[4], ac[4];
        struct comp c[4];
        int ncomp, progressive;
        int adobe_transform;           /* the last Adobe APP14 segment's transform before the first SOS, -1 without one */
        int seen_sos;
        int arith;                     /* SOF9/SOF10: arithmetic coding */
        uint8_t dac_L[16], dac_U[16], dac_K[16];   /* DAC conditioning, T.81's defaults until a DAC sets them */
        uint8_t dc_st[4][J2P_ARITH_DC_BINS], ac_st[4][J2P_ARITH_AC_BINS];   /* the statistics of the current segment */
        uint8_t fixed_st;              /* the fixed-probability bin */
        struct j2p_qm qm;
        uint8_t *abuf;                 /* the current segment's unstuffed bytes */
        size_t abuf_cap;
        unsigned flags;                /* J2P_READ_* */
        unsigned W, H, maxh, maxv, mcux, mcuy;
        unsigned restart_interval;
        char *err;
        size_t errlen;
        int failed;
        struct j2p_jpeg_layout *lay;   /* the layout pass (j2p_read_jpeg_layout), NULL for a full read */
        struct j2p_jpeg_layout4 *lay4; /* the four-plane layout pass (j2p_read_jpeg_layout4) */
        unsigned scans_of[4];          /* layout pass: scans that name each component */
        struct j2p_jpeg_prog_layout *play;   /* the progressive layout pass (j2p_read_jpeg_prog_layout) */
        struct j2p_jpeg_arith_layout *alay;  /* the arithmetic layout pass (j2p_read_jpeg_arith_layout) */
        int headers_only;              /* j2p_jpeg_keep_settings: stop at the first SOS */
        size_t data_cap, seg_cap, scan_cap;
};

static int fail(struct dec *d, const char *fmt, ...) {
        if (!d->failed && d->err && d->errlen) {
                va_list ap;
                va_start(ap, fmt);
                vsnprintf(d->err, d->errlen, fmt, ap);
                va_end(ap);
        }
        d->failed = 1;
        return -1;
}

/* ---- bit reader over entropy-coded data with byte stuffing (B.1.1.5) ----------------------- */
static void fill(struct dec *d) {
        while (d->nbits <= 24) {
                unsigned byte = 0;
                if (!d->hit_marker && d->p < d->end) {
                        byte = *d->p;
                        if (byte == 0xFF) {
                                if (d->p + 1 < d->end && d->p[1] == 0x00) {
                                        d->p += 2;
                                } else {
                                        d->hit_marker = 1;   /* leave the marker in place */
                                        byte = 0;
                                }
                        } else {
                                d->p++;
                        }
                }
                d->acc |= (uint32_t)byte << (24 - d->nbits);
                d->nbits += 8;
        }
}
static inline int getbits(struct dec *d, int n) {
        if (n <= 0) return 0;
        if (n > 16) {                                    /* only a corrupt Huffman table can ask for more (F.1.2.1.1: at most 15/16) */
                fail(d, "corrupt jpeg: bad magnitude category");
                return 0;
        }
        if (d->nbits < n) fill(d);
        const int v = (int)(d->acc >> (32 - n));
        d->acc <<= n;
        d->nbits -= n;
        return v;
}
static inline int getbit(struct dec *d) { return getbits(d, 1); }

static int build_huff(struct dec *d, struct huff *h) {
        int code = 0, k = 0;
        for (int l = 1; l <= 16; l++) {
                h->valptr[l] = k;
                h->mincode[l] = code;
                code += h->bits[l];
                k += h->bits[l];
                h->maxcode[l] = h->bits[l] ? code - 1 : -1;
                if (code > (1 << l)) return fail(d, "corrupt jpeg: bad huffman table");
                code <<= 1;
        }
        h->maxcode[17] = 0x7fffffff;
        h->present = 1;
        return 0;
}
static int decode_huff(struct dec *d, const struct huff *h) {
        int code = 0;
        for (int l = 1; l <= 16; l++) {
                code = (code << 1) | getbit(d);
                if (h->maxcode[l] >= 0 && code <= h->maxcode[l] && code >= h->mincode[l])
                        return h->vals[h->valptr[l] + code - h->mincode[l]];
        }
        fail(d, "corrupt jpeg: bad huffman code");
        return 0;
}
static inline int extend(int v, int s) { return (s < 1 || s > 16) ? 0 : (v < (1 << (s - 1)) ? v - (1 << s) + 1 : v); }   /* F.2.2.1 */

/* ---- block decoders ------------------------------------------------------------------------ */
static void block_sequential(struct dec *d, struct comp *c, int16_t *b) {
        int s = decode_huff(d, &d->dc[c->td]);
        int diff = s ? extend(getbits(d, s), s) : 0;
        c->dc_pred += diff;
        b[0] = (int16_t)c->dc_pred;
        for (int k = 1; k < 64; k++) {
                const int rs = decode_huff(d, &d->ac[c->ta]);
                const int r = rs >> 4;
                s = rs & 15;
                if (s) {
                        k += r;
                        if (k > 63) { fail(d, "corrupt jpeg: coefficient index out of range"); return; }
                        b[ZZ[k]] = (int16_t)extend(getbits(d, s), s);
                } else {
                        if (r != 15) break;     /* EOB */
                        k += 15;
                }
                if (d->failed) return;
        }
}
static void block_dc_first(struct dec *d, struct comp *c, int16_t *b, int al) {
        const int s = decode_huff(d, &d->dc[c->td]);
        const int diff = s ? extend(getbits(d, s), s) : 0;
        c->dc_pred += diff;
        b[0] = (int16_t)(c->dc_pred * (1 << al));
}
static void block_dc_refine(struct dec *d, int16_t *b, int al) {
        if (getbit(d)) b[0] |= (int16_t)(1 << al);
}
static void block_ac_first(struct dec *d, struct comp *c, int16_t *b, int ss, int se, int al, unsigned *eobrun) {
        if (*eobrun > 0) { (*eobrun)--; return; }
        for (int k = ss; k <= se; k++) {
                const int rs = decode_huff(d, &d->ac[c->ta]);
                const int r = rs >> 4, s = rs & 15;
                if (s) {
                        k += r;
                        if (k > 63) { fail(d, "corrupt jpeg: coefficient index out of range"); return; }
                        b[ZZ[k]] = (int16_t)(extend(getbits(d, s), s) * (1 << al));
                } else {
                        if (r == 15) { k += 15; }
                        else {
                                *eobrun = 1u << r;
                                if (r) *eobrun += (unsigned)getbits(d, r);
                                (*eobrun)--;
                                break;
                        }
                }
                if (d->failed) return;
        }
}
static void block_ac_refine(struct dec *d, struct comp *c, int16_t *b, int ss, int se, int al, unsigned *eobrun) {   /* G.1.2.3 */
        const int p1 = 1 << al, m1 = -(1 << al);
        int k = ss;
        if (*eobrun == 0) {
                for (; k <= se; k++) {
                        const int rs = decode_huff(d, &d->ac[c->ta]);
                        int r = rs >> 4, s = rs & 15;
                        if (d->failed) return;
                        if (s) {
                                s = getbit(d) ? p1 : m1;
                        } else if (r != 15) {
                                *eobrun = 1u << r;
                                if (r) *eobrun += (unsigned)getbits(d, r);
                                break;
                        }
                        /* skip over already non-zero coefficients (each takes a correction bit) and r zero ones */
                        do {
                                int16_t *coef = &b[ZZ[k]];
                                if (*coef != 0) {
                                        if (getbit(d) && (*coef & p1) == 0) *coef = (int16_t)(*coef + (*coef >= 0 ? p1 : m1));
                                } else {
                                        if (--r < 0) break;
                                }
                                k++;
                        } while (k <= se);
                        if (s && k <= se) b[ZZ[k]] = (int16_t)s;
                }
        }
        if (*eobrun > 0) {
                for (; k <= se; k++) {
                        int16_t *coef = &b[ZZ[k]];
                        if (*coef != 0 && getbit(d) && (*coef & p1) == 0) *coef = (int16_t)(*coef + (*coef >= 0 ? p1 : m1));
                }
                (*eobrun)--;
        }
}

/* ---- arithmetic-coded blocks (jdarith.c's models: F.1.4.4 and G.1.3) ------------------------- */
static int bad_arith(struct dec *d) { return fail(d, "corrupt jpeg: bad arithmetic code"); }

static void arith_block(struct dec *d, struct comp *c, int16_t *b, int ss, int se, int ah, int al) {
        const int td = c->td, ta = c->ta;
        if (!d->progressive) {
                if (j2p_arith_block_seq(&d->qm, d->dc_st[td], d->ac_st[ta], &c->dc_pred, &c->dc_ctx, d->dac_L[td], d->dac_U[td],
                                        d->dac_K[ta], &d->fixed_st, b) != J2P_ARITH_OK) bad_arith(d);
        } else if (ss == 0 && ah == 0) {                        /* G.1.3.1: DC first */
                int diff;
                if (j2p_arith_dc_diff(&d->qm, d->dc_st[td], &c->dc_ctx, d->dac_L[td], d->dac_U[td], &diff) != J2P_ARITH_OK) { bad_arith(d); return; }
                c->dc_pred += diff;
                b[0] = (int16_t)(int)((unsigned)c->dc_pred << al);
        } else if (ss == 0) {                                   /* DC refine: one bit on the fixed bin */
                if (j2p_qm_decode(&d->qm, &d->fixed_st)) b[0] |= (int16_t)(1 << al);
        } else if (ah == 0) {                                   /* G.1.3.2: AC first */
                if (j2p_arith_ac(&d->qm, d->ac_st[ta], d->dac_K[ta], &d->fixed_st, ss, se, al, b) != J2P_ARITH_OK) bad_arith(d);
        } else {                                                /* G.1.3.3: AC refine */
                const int p1 = 1 << al, m1 = (int)(~0u << al);
                int kex = se;                                   /* the previous stages' EOB */
                for (; kex > 0; kex--)
                        if (b[ZZ[kex]]) break;
                for (int k = ss; k <= se; k++) {
                        uint8_t *st = d->ac_st[ta] + 3 * (k - 1);
                        if (k > kex && j2p_qm_decode(&d->qm, st)) break;      /* EOB */
                        for (;;) {
                                int16_t *coef = &b[ZZ[k]];
                                if (*coef) {                    /* a correction bit */
                                        if (j2p_qm_decode(&d->qm, st + 2)) *coef = (int16_t)(*coef + (*coef < 0 ? m1 : p1));
                                        break;
                                }
                                if (j2p_qm_decode(&d->qm, st + 1)) {          /* newly nonzero */
                                        *coef = (int16_t)(j2p_qm_decode(&d->qm, &d->fixed_st) ? m1 : p1);
                                        break;
                                }
                                st += 3;
                                if (++k > se) { bad_arith(d); return; }
                        }
                }
        }
}

/* the unstuffed bytes the entropy decoders read from *pp: up to the first FF not followed by 00,
 * FF 00 -> FF; writes them to o, returns their count and leaves *pp at the FF */
static size_t unstuff(const uint8_t **pp, const uint8_t *end, uint8_t *o) {
        const uint8_t *p = *pp;
        uint8_t *o0 = o;
        while (p < end) {
                const uint8_t *q = memchr(p, 0xFF, (size_t)(end - p));
                const size_t run = (size_t)((q ? q : end) - p);
                memcpy(o, p, run);
                o += run;
                p += run;
                if (!q) break;
                if (p + 1 < end && p[1] == 0x00) { *o++ = 0xFF; p += 2; }
                else break;
        }
        *pp = p;
        return (size_t)(o - o0);
}

static int grow(void **p, size_t *cap, size_t need, size_t elem) {
        if (need <= *cap) return 0;
        size_t n = *cap ? *cap : 4096 / elem + 1;
        while (n < need) n *= 2;
        void *q = realloc(*p, n * elem);
        if (!q) return -1;
        *p = q;
        *cap = n;
        return 0;
}

/* an arithmetic segment starts (the scan's first, or after RSTn): zeroed statistics and DC
 * contexts, C = A = 0 and CT = -16 over the segment's bytes (F.1.4.4, G.1.3) */
static int arith_segment(struct dec *d, struct comp **sc, int ns) {
        memset(d->dc_st, 0, sizeof d->dc_st);
        memset(d->ac_st, 0, sizeof d->ac_st);
        d->fixed_st = J2P_ARITH_FIXED_STATE;
        for (int i = 0; i < ns; i++) sc[i]->dc_ctx = 0;
        if (grow((void **)&d->abuf, &d->abuf_cap, (size_t)(d->end - d->p) + 1, 1) != 0) return fail(d, "could not allocate memory for coefs");
        const size_t n = unstuff(&d->p, d->end, d->abuf);
        if (n > 0xffffffffu) return fail(d, "unsupported jpeg: an arithmetic segment of %zu bytes", n);
        j2p_qm_start(&d->qm, d->abuf, (uint32_t)n);
        return 0;
}

/* ---- one scan ------------------------------------------------------------------------------ */
static int restart(struct dec *d, struct comp **sc, int ns, unsigned *eobrun, int expect) {
        /* byte-align, then RSTn (E.2.4) */
        d->acc = 0;
        d->nbits = 0;
        d->hit_marker = 0;
        while (d->p + 1 < d->end && !(d->p[0] == 0xFF && d->p[1] >= 0xD0 && d->p[1] <= 0xD7)) {
                if (d->p[0] == 0xFF && d->p[1] != 0x00 && d->p[1] != 0xFF) return fail(d, "corrupt jpeg: missing restart marker");
                d->p++;
        }
        if (d->p + 1 >= d->end) return fail(d, "corrupt jpeg: truncated at restart marker");
        if ((d->p[1] & 7) != (expect & 7)) return fail(d, "corrupt jpeg: restart marker out of sequence");
        d->p += 2;
        for (int i = 0; i < ns; i++) sc[i]->dc_pred = 0;
        *eobrun = 0;
        return 0;
}

/* after a scan's last MCU: leave d->p at the next marker that is not RSTn (extra RSTn and junk are skipped) */
static void skip_to_marker(struct dec *d) {
        while (d->p + 1 < d->end && !(d->p[0] == 0xFF && d->p[1] != 0x00 && !(d->p[1] >= 0xD0 && d->p[1] <= 0xD7) && d->p[1] != 0xFF)) d->p++;
}

static int decode_scan(struct dec *d, struct comp **sc, int ns, int ss, int se, int ah, int al) {
        d->acc = 0;
        d->nbits = 0;
        d->hit_marker = 0;
        for (int i = 0; i < ns; i++) sc[i]->dc_pred = 0;
        if (d->arith && arith_segment(d, sc, ns) != 0) return -1;
        unsigned eobrun = 0, since_restart = 0;
        int rst = 0;
        const int interleaved = ns > 1;
        unsigned nmx, nmy;
        if (interleaved) { nmx = d->mcux; nmy = d->mcuy; }
        else { nmx = sc[0]->wb; nmy = sc[0]->hb; }           /* A.2.3: non-interleaved MCU = one block of the real grid */
        for (unsigned my = 0; my < nmy; my++)
                for (unsigned mx = 0; mx < nmx; mx++) {
                        if (d->restart_interval && since_restart == d->restart_interval) {
                                if (restart(d, sc, ns, &eobrun, rst++) != 0) return -1;
                                if (d->arith && arith_segment(d, sc, ns) != 0) return -1;
                                since_restart = 0;
                        }
                        for (int i = 0; i < ns; i++) {
                                struct comp *c = sc[i];
                                const int bh = interleaved ? c->h : 1, bv = interleaved ? c->v : 1;
                                for (int y = 0; y < bv; y++)
                                        for (int x = 0; x < bh; x++) {
                                                const unsigned bx = interleaved ? mx * c->h + x : mx;
                                                const unsigned by = interleaved ? my * c->v + y : my;
                                                int16_t *b = c->blk + ((size_t)by * c->pwb + bx) * 64;
                                                if (d->arith) arith_block(d, c, b, ss, se, ah, al);
                                                else if (!d->progressive) block_sequential(d, c, b);
                                                else if (ss == 0) { if (ah == 0) block_dc_first(d, c, b, al); else block_dc_refine(d, b, al); }
                                                else if (ah == 0) block_ac_first(d, c, b, ss, se, al, &eobrun);
                                                else block_ac_refine(d, c, b, ss, se, al, &eobrun);
                                                if (d->failed) return -1;
                                        }
                        }
                        since_restart++;
                }
        skip_to_marker(d);
        return 0;
}

/* ---- layout pass: one sequential scan cut into segments ------------------------------------ */
/* S: the scan's descriptor; the segments are appended to *seg (seg_n) and their bytes to *data
 * (data_len), which both layout passes own */
static int layout_scan(struct dec *d, struct comp **sc, int ns, struct j2p_jpeg_scan4 *S, struct j2p_jpeg_segment **seg, unsigned *seg_n,
                       uint8_t **data, size_t *data_len) {
        const int interleaved = ns > 1;
        S->ncomp = (unsigned)ns;
        for (int i = 0; i < ns; i++) {
                S->comp[i] = (unsigned)(sc[i] - d->c);
                S->bw[i] = interleaved ? (unsigned)sc[i]->h : 1;
                S->bh[i] = interleaved ? (unsigned)sc[i]->v : 1;
                memcpy(S->dc[i].bits, d->dc[sc[i]->td].bits, 17);
                memcpy(S->dc[i].vals, d->dc[sc[i]->td].vals, 256);
                memcpy(S->ac[i].bits, d->ac[sc[i]->ta].bits, 17);
                memcpy(S->ac[i].vals, d->ac[sc[i]->ta].vals, 256);
        }
        if (interleaved) { S->mcux = d->mcux; S->mcuy = d->mcuy; }
        else { S->mcux = sc[0]->wb; S->mcuy = sc[0]->hb; }
        S->restart_interval = d->restart_interval;
        const size_t total = (size_t)S->mcux * S->mcuy;
        const size_t nseg = d->restart_interval ? (total + d->restart_interval - 1) / d->restart_interval : 1;
        S->seg0 = *seg_n;
        S->nseg = (unsigned)nseg;
        unsigned eobrun = 0;
        for (size_t k = 0; k < nseg; k++) {
                if (k > 0 && restart(d, sc, ns, &eobrun, (int)(k - 1)) != 0) return -1;
                if (grow((void **)seg, &d->seg_cap, (size_t)*seg_n + 1, sizeof **seg) != 0) return fail(d, "could not allocate memory for coefs");
                /* the bytes fill() would feed: up to the first FF not followed by 00, FF 00 -> FF */
                if (grow((void **)data, &d->data_cap, *data_len + (size_t)(d->end - d->p), 1) != 0) return fail(d, "could not allocate memory for coefs");
                struct j2p_jpeg_segment *g = &(*seg)[(*seg_n)++];
                g->off = *data_len;
                g->len = unstuff(&d->p, d->end, *data + *data_len);
                *data_len += g->len;
                g->mcus = (unsigned)(d->restart_interval && k + 1 < nseg ? d->restart_interval : total - k * (d->restart_interval ? d->restart_interval : 0));
        }
        skip_to_marker(d);
        return 0;
}

/* a scan of at most three components as the three-component layouts store it */
static void narrow_scan(const struct j2p_jpeg_scan4 *S4, struct j2p_jpeg_scan *S) {
        S->ncomp = S4->ncomp;
        for (int i = 0; i < 3; i++) {
                S->comp[i] = S4->comp[i];
                S->bw[i] = S4->bw[i];
                S->bh[i] = S4->bh[i];
                S->dc[i] = S4->dc[i];
                S->ac[i] = S4->ac[i];
        }
        S->mcux = S4->mcux;
        S->mcuy = S4->mcuy;
        S->restart_interval = S4->restart_interval;
        S->seg0 = S4->seg0;
        S->nseg = S4->nseg;
}

/* ---- marker segments ----------------------------------------------------------------------- */
static unsigned be16(const uint8_t *p) { return ((unsigned)p[0] << 8) | p[1]; }

static int parse_dqt(struct dec *d, const uint8_t *s, unsigned len) {
        while (len > 0) {
                const int pq = s[0] >> 4, tq = s[0] & 15;
                if (tq > 3 || pq > 1) return fail(d, "corrupt jpeg: bad DQT");
                const unsigned need = 1 + 64 * (pq + 1);
                if (len < need) return fail(d, "corrupt jpeg: short DQT");
                for (int k = 0; k < 64; k++) d->qt[tq][ZZ[k]] = pq ? (uint16_t)be16(s + 1 + 2 * k) : s[1 + k];
                d->qt_present[tq] = 1;
                s += need;
                len -= need;
        }
        return 0;
}
static int parse_dht(struct dec *d, const uint8_t *s, unsigned len) {
        while (len > 0) {
                if (len < 17) return fail(d, "corrupt jpeg: short DHT");
                const int tc = s[0] >> 4, th = s[0] & 15;
                if (tc > 1 || th > 3) return fail(d, "corrupt jpeg: bad DHT");
                struct huff *h = tc ? &d->ac[th] : &d->dc[th];
                unsigned n = 0;
                h->bits[0] = 0;
                for (int l = 1; l <= 16; l++) { h->bits[l] = s[l]; n += s[l]; }
                if (n > 256 || len < 17 + n) return fail(d, "corrupt jpeg: bad DHT");
                memcpy(h->vals, s + 17, n);
                if (build_huff(d, h) != 0) return -1;
                s += 17 + n;
                len -= 17 + n;
        }
        return 0;
}
static int parse_dac(struct dec *d, const uint8_t *s, unsigned len) {     /* B.2.4.3, as libjpeg's get_dac */
        if (len & 1) return fail(d, "corrupt jpeg: bad DAC length");
        for (; len >= 2; s += 2, len -= 2) {
                const unsigned index = s[0], val = s[1];
                if (index >= 32) return fail(d, "corrupt jpeg: bad DAC table index %u", index);
                if (index >= 16) { d->dac_K[index - 16] = (uint8_t)val; continue; }
                if ((val & 15) > (val >> 4)) return fail(d, "corrupt jpeg: bad DAC value 0x%02x (L > U)", val);
                d->dac_L[index] = (uint8_t)(val & 15);
                d->dac_U[index] = (uint8_t)(val >> 4);
        }
        return 0;
}
static int parse_sof(struct dec *d, const uint8_t *s, unsigned len) {
        if (len < 6) return fail(d, "corrupt jpeg: short SOF");
        if (s[0] != 8) return fail(d, "unsupported jpeg: %d-bit samples", s[0]);
        d->H = be16(s + 1);
        d->W = be16(s + 3);
        d->ncomp = s[5];
        if (d->flags & J2P_READ_CMYK) {
                if (d->ncomp != 1 && d->ncomp != 3 && d->ncomp != 4) return fail(d, "only 1, 3 and 4 component jpegs are supported");
        } else if (d->flags & J2P_READ_GRAY) {
                if (d->ncomp != 1 && d->ncomp != 3) return fail(d, "only 1 and 3 component jpegs are supported");
        } else if (d->ncomp != 3) return fail(d, "only 3 component jpegs are supported");    /* jpeg.c:34 */
        if (d->W == 0 || d->H == 0) return fail(d, "unsupported jpeg: empty image or DNL-defined height");
        if (len < 6 + 3u * d->ncomp) return fail(d, "corrupt jpeg: short SOF");
        d->maxh = d->maxv = 1;
        for (int i = 0; i < d->ncomp; i++) {
                struct comp *c = &d->c[i];
                c->id = s[6 + 3 * i];
                c->h = s[7 + 3 * i] >> 4;
                c->v = s[7 + 3 * i] & 15;
                c->tq = s[8 + 3 * i];
                if (c->h < 1 || c->h > 4 || c->v < 1 || c->v > 4 || c->tq > 3) return fail(d, "corrupt jpeg: bad component spec");
                if ((unsigned)c->h > d->maxh) d->maxh = c->h;
                if ((unsigned)c->v > d->maxv) d->maxv = c->v;
        }
        d->mcux = (d->W + 8 * d->maxh - 1) / (8 * d->maxh);
        d->mcuy = (d->H + 8 * d->maxv - 1) / (8 * d->maxv);
        for (int i = 0; i < d->ncomp; i++) {
                struct comp *c = &d->c[i];
                const unsigned cw = (d->W * c->h + d->maxh - 1) / d->maxh, ch = (d->H * c->v + d->maxv - 1) / d->maxv;   /* A.1.1 */
                c->wb = (cw + 7) / 8;
                c->hb = (ch + 7) / 8;
                c->pwb = d->mcux * c->h;
                c->phb = d->mcuy * c->v;
                if (d->lay || d->lay4 || d->play || d->headers_only) continue;                                     /* the layout passes store no blocks */
                c->blk = calloc((size_t)c->pwb * c->phb * 64, sizeof(int16_t));
                if (!c->blk) return fail(d, "could not allocate memory for coefs");                /* jpeg.c:69 */
        }
        return 0;
}

/* T.81's DAC defaults (L = 0, U = 1, Kx = 5), in force from SOI */
static void dac_defaults(struct dec *d) {
        for (int t = 0; t < 16; t++) {
                d->dac_L[t] = 0;
                d->dac_U[t] = 1;
                d->dac_K[t] = 5;
        }
}

/* The marker loop shared by j2p_read_jpeg_mem and j2p_read_jpeg_layout: reads the headers and
 * decodes every scan (full read) or cuts it into segments (layout pass).  Returns 1 when the layout
 * pass stopped early on a file that is not device-decodable. */
static int read_markers(struct dec *d, const uint8_t *buf, size_t len) {
        int have_sof = 0, done = 0;
        if (len < 4 || buf[0] != 0xFF || buf[1] != 0xD8) { fail(d, "not a jpeg file (no SOI marker)"); return 0; }
        d->p += 2;
        dac_defaults(d);
        d->adobe_transform = -1;
        while (!done && !d->failed) {
                /* find next marker */
                while (d->p < d->end && *d->p != 0xFF) d->p++;
                while (d->p < d->end && *d->p == 0xFF) d->p++;
                if (d->p >= d->end) { fail(d, "corrupt jpeg: premature end of file"); break; }
                const unsigned m = *d->p++;
                if (m == 0xD9) { done = 1; break; }                       /* EOI */
                if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;      /* TEM, stray RSTn */
                if (d->p + 2 > d->end) { fail(d, "corrupt jpeg: truncated marker"); break; }
                const unsigned seglen = be16(d->p);
                if (seglen < 2 || d->p + seglen > d->end) { fail(d, "corrupt jpeg: bad segment length"); break; }
                const uint8_t *s = d->p + 2;
                const unsigned sl = seglen - 2;
                d->p += seglen;
                if (m == 0xDB) parse_dqt(d, s, sl);
                else if (m == 0xC4) parse_dht(d, s, sl);
                else if (m == 0xCC) parse_dac(d, s, sl);
                else if (m == 0xC0 || m == 0xC1 || m == 0xC2 || m == 0xC9 || m == 0xCA) {
                        if (have_sof) { fail(d, "unsupported jpeg: multiple frames"); break; }
                        d->progressive = m == 0xC2 || m == 0xCA;
                        d->arith = m == 0xC9 || m == 0xCA;
                        if ((d->lay || d->lay4) && (d->progressive || d->arith)) return 1;
                        if (d->play && (!d->progressive || d->arith)) return 1;
                        if (d->alay && (d->progressive || !d->arith)) return 1;
                        if ((d->lay || d->play || d->alay) && (d->flags & J2P_READ_CMYK) && sl >= 6 && s[5] == 4) return 1;   /* four components: host reader */
                        if (parse_sof(d, s, sl) == 0) have_sof = 1;
                } else if (m == 0xC3 || (m >= 0xC5 && m <= 0xC7) || m == 0xCB || (m >= 0xCD && m <= 0xCF)) {
                        fail(d, "unsupported jpeg: SOF%u (arithmetic, lossless or hierarchical coding)", m - 0xC0);
                } else if (m == 0xEE) {
                        /* Adobe APP14 (libjpeg's examine_app14): 12 data bytes or more, "Adobe", transform at byte 11 */
                        if (!d->seen_sos && sl >= 12 && memcmp(s, "Adobe", 5) == 0) d->adobe_transform = s[11];
                } else if (m == 0xDD) {
                        if (sl < 2) fail(d, "corrupt jpeg: short DRI"); else d->restart_interval = be16(s);
                } else if (m == 0xDA) {
                        if (!have_sof) { fail(d, "corrupt jpeg: scan before frame header"); break; }
                        if (d->headers_only) break;
                        d->seen_sos = 1;
                        if (sl < 1) { fail(d, "corrupt jpeg: short SOS"); break; }
                        const int ns = s[0];
                        if (ns < 1 || ns > (d->ncomp == 4 ? 4 : 3) || sl < 1 + 2u * ns + 3) { fail(d, "corrupt jpeg: bad SOS"); break; }
                        struct comp *sc[4];
                        for (int i = 0; i < ns; i++) {
                                sc[i] = NULL;
                                for (int k = 0; k < d->ncomp; k++) if (d->c[k].id == s[1 + 2 * i]) sc[i] = &d->c[k];
                                if (!sc[i]) { fail(d, "corrupt jpeg: scan names an unknown component"); break; }
                                sc[i]->td = s[2 + 2 * i] >> 4;
                                sc[i]->ta = s[2 + 2 * i] & 15;
                                if (sc[i]->td > 3 || sc[i]->ta > 3) fail(d, "corrupt jpeg: bad table selector");
                        }
                        if (d->failed) break;
                        if (d->ncomp == 4 && ns > 1) {          /* libjpeg's D_MAX_BLOCKS_IN_MCU, for the files this reader took from it */
                                int bpm = 0;
                                for (int i = 0; i < ns; i++) bpm += sc[i]->h * sc[i]->v;
                                if (bpm > 10) { fail(d, "unsupported jpeg: %d blocks per MCU (at most 10)", bpm); break; }
                        }
                        int ss = s[1 + 2 * ns], se = s[2 + 2 * ns], ah = s[3 + 2 * ns] >> 4, al = s[3 + 2 * ns] & 15;
                        if (!d->progressive) { ss = 0; se = 63; ah = al = 0; }
                        else if (ss > se || se > 63 || (ss == 0 && se != 0) || (ss > 0 && ns != 1) || al > 13) { fail(d, "corrupt jpeg: bad progressive scan parameters"); break; }
                        for (int i = 0; i < ns && !d->arith; i++) {
                                if ((ss == 0 && !(d->progressive && ah) && !d->dc[sc[i]->td].present) ||
                                    ((!d->progressive || ss > 0) && !d->ac[sc[i]->ta].present)) { fail(d, "corrupt jpeg: scan uses an undefined huffman table"); break; }
                        }
                        if (d->failed) break;
                        struct j2p_jpeg_scan4 S4;
                        memset(&S4, 0, sizeof S4);
                        if (d->lay) {
                                for (int i = 0; i < ns; i++)
                                        if (d->scans_of[sc[i] - d->c]++) return 1;      /* a component scanned twice */
                                struct j2p_jpeg_layout *l = d->lay;
                                layout_scan(d, sc, ns, &S4, &l->seg, &l->nseg, &l->data, &l->data_len);
                                narrow_scan(&S4, &l->scan[l->nscan++]);
                        } else if (d->lay4) {
                                for (int i = 0; i < ns; i++)
                                        if (d->scans_of[sc[i] - d->c]++) return 1;      /* a component scanned twice */
                                struct j2p_jpeg_layout4 *l = d->lay4;
                                layout_scan(d, sc, ns, &l->scan[l->nscan++], &l->seg, &l->nseg, &l->data, &l->data_len);
                        } else if (d->play) {
                                struct j2p_jpeg_prog_layout *l = d->play;
                                if (grow((void **)&l->scan, &d->scan_cap, (size_t)l->nscan + 1, sizeof *l->scan) != 0) {
                                        fail(d, "could not allocate memory for coefs");
                                        break;
                                }
                                struct j2p_jpeg_prog_scan *S = &l->scan[l->nscan++];
                                memset(S, 0, sizeof *S);
                                S->ss = (unsigned)ss;
                                S->se = (unsigned)se;
                                S->ah = (unsigned)ah;
                                S->al = (unsigned)al;
                                layout_scan(d, sc, ns, &S4, &l->seg, &l->nseg, &l->data, &l->data_len);
                                narrow_scan(&S4, &S->s);
                        } else if (d->alay) {
                                for (int i = 0; i < ns; i++)
                                        if (d->scans_of[sc[i] - d->c]++) return 1;      /* a component scanned twice */
                                struct j2p_jpeg_arith_layout *l = d->alay;
                                struct j2p_jpeg_scan S;
                                layout_scan(d, sc, ns, &S4, &l->seg, &l->nseg, &l->data, &l->data_len);
                                narrow_scan(&S4, &S);
                                struct j2p_jpeg_arith_scan *A = &l->scan[l->nscan++];
                                A->ncomp = S.ncomp;
                                for (int i = 0; i < 3; i++) {
                                        A->comp[i] = S.comp[i];
                                        A->bw[i] = S.bw[i];
                                        A->bh[i] = S.bh[i];
                                        A->dc_tbl[i] = A->ac_tbl[i] = A->dc_L[i] = A->dc_U[i] = A->ac_K[i] = 0;
                                }
                                for (int i = 0; i < ns; i++) {
                                        A->dc_tbl[i] = (unsigned)sc[i]->td;
                                        A->ac_tbl[i] = (unsigned)sc[i]->ta;
                                        A->dc_L[i] = d->dac_L[sc[i]->td];
                                        A->dc_U[i] = d->dac_U[sc[i]->td];
                                        A->ac_K[i] = d->dac_K[sc[i]->ta];
                                }
                                A->mcux = S.mcux;
                                A->mcuy = S.mcuy;
                                A->restart_interval = S.restart_interval;
                                A->seg0 = S.seg0;
                                A->nseg = S.nseg;
                        } else {
                                decode_scan(d, sc, ns, ss, se, ah, al);
                        }
                }
                /* everything else (APPn, COM, DNL, ...) is skipped */
        }
        if (!d->failed && !have_sof) fail(d, "corrupt jpeg: no frame header");
        return 0;
}

/* the reference's checks of the frame (jpeg.c:40-64) and the planes' geometry and tables */
static void check_planes(struct dec *d, struct coef *coefs) {
        for (int i = 0; i < d->ncomp && !d->failed; i++) {
                struct comp *c = &d->c[i];
                struct coef *o = &coefs[i];
                if (!d->qt_present[c->tq]) { fail(d, "weird jpeg: no quant table pointer"); break; }          /* jpeg.c:40 */
                for (int j = 0; j < 64; j++) {
                        if (d->qt[c->tq][j] == 0) { fail(d, "invalid quantization table"); break; }            /* jpeg.c:43 */
                        o->quant_table[j] = d->qt[c->tq][j];
                }
                if (d->failed) break;
                o->w = c->wb * 8;
                o->h = c->hb * 8;
                o->w_samp = d->maxh / c->h;                                                                    /* jpeg.c:57-58 */
                o->h_samp = d->maxv / c->v;
                if (o->h / 8 != (d->H / o->h_samp + 7) / 8) { fail(d, "jpeg invalid coef h size"); break; }    /* jpeg.c:59-61 */
                if (o->w / 8 != (d->W / o->w_samp + 7) / 8) { fail(d, "jpeg invalid coef w size"); break; }    /* jpeg.c:62-64 */
        }
}

/* Writes only the fields before ncomp (always 3 here), so callers that mirror the struct as it was
 * before ncomp was appended (ctypes users of this entry point) stay within their buffer. */
int j2p_read_jpeg_mem(const uint8_t *buf, size_t len, struct j2p_jpeg *out, char *err, size_t errlen) {
        struct j2p_jpeg j;
        const int rc = j2p_read_jpeg_mem_ex(buf, len, 0, &j, err, errlen);
        memcpy(out, &j, offsetof(struct j2p_jpeg, ncomp));
        return rc;
}

/* the full read behind j2p_read_jpeg_mem_ex and j2p_read_jpeg4_mem: coefs has room for ncomp_max
 * planes (3, or 4 with J2P_READ_CMYK); *ncomp is the frame's count once its header is read (also on
 * failure), *colour the J2P_JPEG_* kind of a four-component frame */
static int read_full(const uint8_t *buf, size_t len, unsigned flags, unsigned *w, unsigned *h, struct coef *coefs, unsigned *ncomp,
                     unsigned *colour, char *err, size_t errlen) {
        struct dec *d = calloc(1, sizeof *d);
        if (!d) return -1;
        d->p = buf; d->end = buf + len; d->err = err; d->errlen = errlen; d->flags = flags;
        if (err && errlen) err[0] = 0;
        read_markers(d, buf, len);
        *ncomp = (unsigned)d->ncomp;
        const int planes_failed = d->failed;        /* before the planes: ncomp may be any count, nothing is allocated */
        if (!d->failed) check_planes(d, coefs);
        if (!d->failed) {
                *w = d->W;
                *h = d->H;
                if (colour && d->ncomp == 4) *colour = d->adobe_transform <= 0 ? J2P_JPEG_CMYK : J2P_JPEG_YCCK;   /* libjpeg's default_decompress_parms */
                for (int i = 0; i < d->ncomp; i++) {
                        struct comp *c = &d->c[i];
                        struct coef *o = &coefs[i];
                        o->data = malloc((size_t)o->w * o->h * sizeof(int16_t));
                        if (!o->data) { fail(d, "could not allocate memory for coefs"); break; }
                        for (unsigned by = 0; by < c->hb; by++)
                                memcpy(o->data + (size_t)by * c->wb * 64, c->blk + (size_t)by * c->pwb * 64, (size_t)c->wb * 64 * sizeof(int16_t));
                }
        }
        for (int i = 0; i < 4; i++) free(d->c[i].blk);
        free(d->abuf);
        const int rc = d->failed ? -1 : 0;
        if (rc != 0 && !planes_failed) for (int i = 0; i < d->ncomp; i++) { free(coefs[i].data); coefs[i].data = NULL; }
        free(d);
        return rc;
}

int j2p_read_jpeg_mem_ex(const uint8_t *buf, size_t len, unsigned flags, struct j2p_jpeg *out, char *err, size_t errlen) {
        memset(out, 0, sizeof *out);
        unsigned ncomp;
        const int rc = read_full(buf, len, flags & ~(unsigned)J2P_READ_CMYK, &out->w, &out->h, out->coefs, &ncomp, NULL, err, errlen);
        if (rc == 0) out->ncomp = ncomp;
        return rc;
}

int j2p_read_jpeg4_mem(const uint8_t *buf, size_t len, unsigned flags, struct j2p_jpeg4 *out, char *err, size_t errlen) {
        memset(out, 0, sizeof *out);
        return read_full(buf, len, flags | J2P_READ_CMYK, &out->w, &out->h, out->coefs, &out->ncomp, &out->colour, err, errlen);
}

int j2p_read_jpeg_layout(const uint8_t *buf, size_t len, struct j2p_jpeg_layout *out, char *err, size_t errlen) {
        return j2p_read_jpeg_layout_ex(buf, len, 0, out, err, errlen);
}

int j2p_read_jpeg_layout_ex(const uint8_t *buf, size_t len, unsigned flags, struct j2p_jpeg_layout *out, char *err, size_t errlen) {
        struct dec *d = calloc(1, sizeof *d);
        if (!d) return -1;
        d->p = buf; d->end = buf + len; d->err = err; d->errlen = errlen; d->flags = flags;
        if (err && errlen) err[0] = 0;
        memset(out, 0, sizeof *out);
        d->lay = out;
        const int stopped = read_markers(d, buf, len);
        int decodable = !stopped && !d->failed;
        for (int i = 0; i < d->ncomp && decodable; i++) decodable = d->scans_of[i] == 1;
        if (decodable) {
                check_planes(d, out->coefs);
                out->w = d->W;
                out->h = d->H;
                out->ncomp = (unsigned)d->ncomp;
                for (int i = 0; i < d->ncomp; i++) { out->comp_h[i] = (unsigned)d->c[i].h; out->comp_v[i] = (unsigned)d->c[i].v; }
        }
        const int rc = d->failed ? -1 : 0;
        out->device_decodable = rc == 0 && decodable;
        if (!out->device_decodable) {
                j2p_free_jpeg_layout(out);
                out->nscan = 0;
        }
        free(d);
        return rc;
}

int j2p_read_jpeg_prog_layout(const uint8_t *buf, size_t len, struct j2p_jpeg_prog_layout *out, char *err, size_t errlen) {
        return j2p_read_jpeg_prog_layout_ex(buf, len, 0, out, err, errlen);
}

int j2p_read_jpeg_prog_layout_ex(const uint8_t *buf, size_t len, unsigned flags, struct j2p_jpeg_prog_layout *out, char *err,
                                 size_t errlen) {
        struct dec *d = calloc(1, sizeof *d);
        if (!d) return -1;
        d->p = buf; d->end = buf + len; d->err = err; d->errlen = errlen; d->flags = flags;
        if (err && errlen) err[0] = 0;
        memset(out, 0, sizeof *out);
        d->play = out;
        const int stopped = read_markers(d, buf, len);
        const int decodable = !stopped && !d->failed;
        if (decodable) {
                check_planes(d, out->coefs);
                out->w = d->W;
                out->h = d->H;
                out->ncomp = (unsigned)d->ncomp;
                for (int i = 0; i < d->ncomp; i++) { out->comp_h[i] = (unsigned)d->c[i].h; out->comp_v[i] = (unsigned)d->c[i].v; }
        }
        const int rc = d->failed ? -1 : 0;
        out->progressive_decodable = rc == 0 && decodable;
        if (!out->progressive_decodable) j2p_free_jpeg_prog_layout(out);
        free(d);
        return rc;
}

void j2p_free_jpeg_prog_layout(struct j2p_jpeg_prog_layout *l) {
        free(l->scan);
        free(l->seg);
        free(l->data);
        l->scan = NULL;
        l->seg = NULL;
        l->data = NULL;
        l->nscan = 0;
        l->nseg = 0;
        l->data_len = 0;
}

int j2p_read_jpeg_arith_layout(const uint8_t *buf, size_t len, struct j2p_jpeg_arith_layout *out, char *err, size_t errlen) {
        return j2p_read_jpeg_arith_layout_ex(buf, len, 0, out, err, errlen);
}

int j2p_read_jpeg_arith_layout_ex(const uint8_t *buf, size_t len, unsigned flags, struct j2p_jpeg_arith_layout *out, char *err,
                                  size_t errlen) {
        struct dec *d = calloc(1, sizeof *d);
        if (!d) return -1;
        d->p = buf; d->end = buf + len; d->err = err; d->errlen = errlen; d->flags = flags;
        if (err && errlen) err[0] = 0;
        memset(out, 0, sizeof *out);
        d->alay = out;
        const int stopped = read_markers(d, buf, len);
        int decodable = !stopped && !d->failed;
        for (int i = 0; i < d->ncomp && decodable; i++) decodable = d->scans_of[i] == 1;
        if (decodable) {
                check_planes(d, out->coefs);
                out->w = d->W;
                out->h = d->H;
                out->ncomp = (unsigned)d->ncomp;
                for (int i = 0; i < d->ncomp; i++) { out->comp_h[i] = (unsigned)d->c[i].h; out->comp_v[i] = (unsigned)d->c[i].v; }
        }
        const int rc = d->failed ? -1 : 0;
        out->arith_decodable = rc == 0 && decodable;
        if (!out->arith_decodable) {
                j2p_free_jpeg_arith_layout(out);
                out->nscan = 0;
        }
        free(d);
        return rc;
}

void j2p_free_jpeg_arith_layout(struct j2p_jpeg_arith_layout *l) {
        free(l->seg);
        free(l->data);
        l->seg = NULL;
        l->data = NULL;
        l->nseg = 0;
        l->data_len = 0;
}

int j2p_read_jpeg_layout4(const uint8_t *buf, size_t len, unsigned flags, struct j2p_jpeg_layout4 *out, char *err, size_t errlen) {
        struct dec *d = calloc(1, sizeof *d);
        if (!d) return -1;
        d->p = buf; d->end = buf + len; d->err = err; d->errlen = errlen; d->flags = flags | J2P_READ_CMYK;
        if (err && errlen) err[0] = 0;
        memset(out, 0, sizeof *out);
        d->lay4 = out;
        const int stopped = read_markers(d, buf, len);
        int decodable = !stopped && !d->failed;
        for (int i = 0; i < d->ncomp && decodable; i++) decodable = d->scans_of[i] == 1;
        if (decodable) {
                check_planes(d, out->coefs);
                out->w = d->W;
                out->h = d->H;
                out->ncomp = (unsigned)d->ncomp;
                if (d->ncomp == 4) out->colour = d->adobe_transform <= 0 ? J2P_JPEG_CMYK : J2P_JPEG_YCCK;
                for (int i = 0; i < d->ncomp; i++) { out->comp_h[i] = (unsigned)d->c[i].h; out->comp_v[i] = (unsigned)d->c[i].v; }
        }
        const int rc = d->failed ? -1 : 0;
        out->device_decodable = rc == 0 && decodable;
        if (!out->device_decodable) {
                j2p_free_jpeg_layout4(out);
                out->nscan = 0;
        }
        free(d);
        return rc;
}

void j2p_free_jpeg_layout4(struct j2p_jpeg_layout4 *l) {
        free(l->seg);
        free(l->data);
        l->seg = NULL;
        l->data = NULL;
        l->nseg = 0;
        l->data_len = 0;
}

void j2p_free_jpeg_layout(struct j2p_jpeg_layout *l) {
        free(l->seg);
        free(l->data);
        l->seg = NULL;
        l->data = NULL;
        l->nseg = 0;
        l->data_len = 0;
}

/* ---- EXIF orientation (tag 0x0112 of IFD0 in the first APP1 "Exif\0\0" segment before SOS) ---- */

static unsigned tiff16(const uint8_t *p, int be) { return be ? ((unsigned)p[0] << 8) | p[1] : ((unsigned)p[1] << 8) | p[0]; }
static uint32_t tiff32(const uint8_t *p, int be) {
        return be ? ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]
                  : ((uint32_t)p[3] << 24) | ((uint32_t)p[2] << 16) | ((uint32_t)p[1] << 8) | p[0];
}

/* t: the TIFF structure after "Exif\0\0", n bytes of it */
static int tiff_orientation(const uint8_t *t, size_t n) {
        if (n < 8) return 1;
        int be;
        if (t[0] == 'I' && t[1] == 'I') be = 0;
        else if (t[0] == 'M' && t[1] == 'M') be = 1;
        else return 1;
        if (tiff16(t + 2, be) != 42) return 1;
        const uint32_t ifd = tiff32(t + 4, be);
        if (ifd > n || n - ifd < 2) return 1;
        const unsigned count = tiff16(t + ifd, be);
        if ((n - ifd - 2) / 12 < count) return 1;                     /* the entries run past the segment */
        for (unsigned i = 0; i < count; i++) {
                const uint8_t *e = t + ifd + 2 + 12u * i;
                if (tiff16(e, be) != 0x0112) continue;
                const unsigned type = tiff16(e + 2, be);
                if (tiff32(e + 4, be) != 1 || (type != 3 && type != 4)) return 1;   /* SHORT or LONG, count 1 */
                const uint32_t v = type == 3 ? tiff16(e + 8, be) : tiff32(e + 8, be);
                return v >= 1 && v <= 8 ? (int)v : 1;
        }
        return 1;
}

int j2p_jpeg_exif_orientation(const void *data, size_t len) {
        const uint8_t *p = data, *end = p + len;
        if (!data || len < 4 || p[0] != 0xFF || p[1] != 0xD8) return 1;
        p += 2;
        for (;;) {
                while (p < end && *p != 0xFF) p++;
                while (p < end && *p == 0xFF) p++;
                if (p >= end) return 1;
                const unsigned m = *p++;
                if (m == 0xD9 || m == 0xDA) return 1;                    /* EOI, SOS: no Exif before the image data */
                if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;      /* TEM, RSTn: no length */
                if (end - p < 2) return 1;
                const unsigned seglen = be16(p);
                if (seglen < 2 || (size_t)(end - p) < seglen) return 1;
                const uint8_t *s = p + 2;
                const size_t sl = seglen - 2;
                p += seglen;
                if (m == 0xE1 && sl >= 6 && memcmp(s, "Exif\0\0", 6) == 0) return tiff_orientation(s + 6, sl - 6);
        }
}

/* ---- the settings of Pillow's quality='keep' ---- */
int j2p_jpeg_keep_settings(const void *data, size_t len, struct j2p_jpeg_keep *out, char *err, size_t errlen) {
        struct dec *d = calloc(1, sizeof *d);
        if (!d) return -1;
        d->p = data; d->end = d->p + len; d->err = err; d->errlen = errlen; d->flags = J2P_READ_GRAY | J2P_READ_CMYK; d->headers_only = 1;
        if (err && errlen) err[0] = 0;
        memset(out, 0, sizeof *out);
        read_markers(d, data, len);
        struct coef coefs[4];                   /* J2P_READ_CMYK: up to four planes */
        memset(coefs, 0, sizeof coefs);
        if (!d->failed) check_planes(d, coefs);
        if (!d->failed) {
                for (int t = 0; t < 4; t++) {
                        if (!d->qt_present[t]) continue;
                        out->present |= 1u << t;
                        memcpy(out->qt[t], d->qt[t], sizeof out->qt[t]);
                }
                out->ncomp = (unsigned)d->ncomp;
                for (int i = 0; i < d->ncomp; i++) { out->comp_h[i] = (unsigned)d->c[i].h; out->comp_v[i] = (unsigned)d->c[i].v; }
        }
        const int rc = d->failed ? -1 : 0;
        free(d);
        return rc;
}
