// jpegenc_plan.h — the host side shared by libj2pjpegenc.so, libj2pjpegopt.so and libj2pjpegprog.so: the quantisation
// tables and their reciprocals, the Annex K Huffman tables and the header templates, the plan of a
// call (the layout of its work area), the steps that both the kernels and the host driver call per
// block, and the serial host driver.  The first two libraries differ only in where an image's
// Huffman tables and header come from: the call's Annex K ones, or the image's own optimized ones
// (jpegopt_core.h), and in the work-area bound of a block that follows.  The progressive encoder
// (../jpegprog) takes the plan's checks, the tables and the blocks step, and lays out its own scans.
#ifndef J2P_JPEGENC_PLAN_H
#define J2P_JPEGENC_PLAN_H

#include <string.h>

#include <vector>

#include "../common/codec_host.h"
#include "jpegenc_core.h"

// ---- tables ------------------------------------------------------------------------------------
static const uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ITU-T T.81 Annex K.1, natural order
static const uint8_t kBaseQuant[2][64] = {
    {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,  14, 13, 16, 24, 40,  57,  69,  56,
     14, 17, 22, 29, 51,  87,  80,  62,  18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99}};

// ITU-T T.81 Annex K.3: code counts per length 1..16, then the symbols; DC0, AC0, DC1, AC1
static const uint8_t kDcBits[2][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}};
static const uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
static const uint8_t kAcBits[2][16] = {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d}, {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
static const uint8_t kAcVals[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
     0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
     0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
     0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
     0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
     0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
     0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
     0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
     0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
     0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
     0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
     0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
     0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
     0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
     0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};

// The call's one set without given tables: the two Annex K tables with IJG quality scaling
// (jpeg_quality_scaling, jpeg_add_quant_table with force_baseline)
static void quality_set(int quality, struct j2p_jpegenc_qtables *q) {
    memset(q, 0, sizeof *q);
    q->ntables = 2;
    const long s = quality < 50 ? 5000 / quality : 200 - 2 * quality;
    for (int tbl = 0; tbl < 2; tbl++)
        for (int i = 0; i < 64; i++) {
            const long v = (kBaseQuant[tbl][i] * s + 50) / 100;
            q->table[tbl][i] = (uint16_t)(v < 1 ? 1 : v > 255 ? 255 : v);
        }
}

// the call's kind: whether it is gray (one-component files) or CMYK, and its components
static bool is_gray(const struct j2p_jpegenc_params *p) { return p->components == 1; }
static bool is_cmyk(const struct j2p_jpegenc_params *p) { return p->cmyk == 1; }
static uint32_t nc_of(const struct j2p_jpegenc_params *p) { return is_cmyk(p) ? 4u : is_gray(p) ? 1u : 3u; }

// the sets of quantisation tables of a call, and set k of them.  A CMYK file's quality tables are
// table 0 alone: libjpeg gives all four components table 0, so table 1 is neither written nor used.
static uint32_t nsets_of(const struct j2p_jpegenc_params *p) { return p->qtables ? p->nqtables : 1u; }

static void set_of(const struct j2p_jpegenc_params *p, uint32_t k, struct j2p_jpegenc_qtables *q) {
    if (p->qtables) *q = p->qtables[k];
    else quality_set(p->quality, q);
    if (!p->qtables && is_cmyk(p)) q->ntables = 1;
}

// the table component c of a file of nc components quantises with, as Pillow maps n tables onto
// them: colour (0 Y, 1 Cb, 2 Cr), one for all, two Y 0 and Cb, Cr 1, three or four Y 0, Cb 1, Cr 2;
// CMYK, min(c, n - 1)
static uint32_t table_of(uint32_t nc, uint32_t n, uint32_t c) {
    if (nc == 4) return c < n - 1 ? c : n - 1;
    return n == 1 || c == 0 ? 0u : n == 2 ? 1u : c;
}

// the tables a file of nc components writes (a DQT each, in this order): 0 .. dqts - 1
static uint32_t dqts_of(const struct j2p_jpegenc_qtables *q, uint32_t nc) {
    return nc == 1 ? 1u : nc == 4 ? q->ntables : q->ntables < 3 ? q->ntables : 3u;
}

// whether table tb needs a 16-bit DQT
static bool wide_table(const struct j2p_jpegenc_qtables *q, uint32_t tb) {
    for (int i = 0; i < 64; i++)
        if (q->table[tb][i] > 255) return true;
    return false;
}

// libjpeg-turbo's reciprocal of a divisor d >= 2 (compute_reciprocal, 16-bit DCT elements):
// (|x| + corr) * recip >> shift is x / d rounded half away from zero for every |x| < 2^15
static void reciprocal(uint32_t d, uint16_t *recip, uint16_t *corr, uint8_t *shift) {
    int b = 31 - __builtin_clz(d);
    int r = 16 + b;
    uint64_t fq = (1ull << r) / d, fr = (1ull << r) % d;
    uint32_t c = d / 2;
    if (fr == 0) {
        fq >>= 1;
        r--;
    } else if (fr <= d / 2) {
        c++;
    } else {
        fq++;
    }
    *recip = (uint16_t)fq;
    *corr = (uint16_t)c;
    *shift = (uint8_t)r;
}

// jpeg_make_c_derived_tbl: canonical codes from the counts per length (Annex C)
J2P_HD void j2p_je_derive(const uint8_t *bits, const uint8_t *vals, uint16_t *code, uint8_t *size) {
    uint32_t c = 0, p = 0;
    for (int len = 1; len <= 16; len++) {
        for (int k = 0; k < bits[len - 1]; k++, p++) {
            code[vals[p]] = (uint16_t)c++;
            size[vals[p]] = (uint8_t)len;
        }
        c <<= 1;
    }
}

static uint8_t *put16(uint8_t *o, uint32_t v) {
    o[0] = (uint8_t)(v >> 8);
    o[1] = (uint8_t)v;
    return o + 2;
}

static uint8_t *put_dht(uint8_t *o, int index, const uint8_t *bits, const uint8_t *vals) {
    uint32_t n = 0;
    for (int k = 0; k < 16; k++) n += bits[k];
    o = put16(o, 0xffc4);
    o = put16(o, 2 + 1 + 16 + n);
    *o++ = (uint8_t)index;
    memcpy(o, bits, 16);
    memcpy(o + 16, vals, n);
    return o + 16 + n;
}

// the luma sampling factors the SOF declares
static uint32_t sof_hs(const struct j2p_jpegenc_params *p) { return p->sampling == J2P_JPEGENC_444 ? 1 : 2; }
static uint32_t sof_vs(const struct j2p_jpegenc_params *p) { return p->sampling == J2P_JPEGENC_420 ? 2 : 1; }

// the length of set k's header template: SOI, APP0 (CMYK: APP14), its DQTs, SOF, DHTs, SOS
static uint32_t head_len_of(const struct j2p_jpegenc_params *p, uint32_t k) {
    struct j2p_jpegenc_qtables q;
    set_of(p, k, &q);
    const uint32_t nc = nc_of(p);
    uint32_t n = 2 + (nc == 4 ? 16 : 18) + (10 + 3 * nc) + (nc == 3 ? 2 * 33 + 2 * 183 : 33 + 183) + (8 + 2 * nc);
    for (uint32_t tb = 0; tb < dqts_of(&q, nc); tb++) n += wide_table(&q, tb) ? 133 : 69;
    return n;
}

// set k of the call: each component's reciprocals, the call's codes and geometry, the header template
static void make_tables(const struct j2p_jpegenc_params *p, uint32_t set, struct j2p_je_tables *t) {
    memset(t, 0, sizeof *t);
    const bool gray = is_gray(p);
    t->hs = gray ? 1 : sof_hs(p);       // a gray component is sampled 1 x 1 whatever the SOF says
    t->vs = gray ? 1 : sof_vs(p);
    t->nc = nc_of(p);
    struct j2p_jpegenc_qtables q;
    set_of(p, set, &q);
    for (uint32_t c = 0; c < t->nc; c++) {
        const uint16_t *tb = q.table[table_of(t->nc, q.ntables, c)];
        for (int i = 0; i < 64; i++) reciprocal((uint32_t)tb[i] << 3, &t->recip[c][i], &t->corr[c][i], &t->shift[c][i]);
    }
    for (int k = 0; k < 64; k++) t->zz[kNatural[k]] = (uint8_t)k;
    j2p_je_derive(kDcBits[0], kDcVals, t->huff.code[0], t->huff.size[0]);
    j2p_je_derive(kAcBits[0], kAcVals[0], t->huff.code[1], t->huff.size[1]);
    j2p_je_derive(kDcBits[1], kDcVals, t->huff.code[2], t->huff.size[2]);
    j2p_je_derive(kAcBits[1], kAcVals[1], t->huff.code[3], t->huff.size[3]);

    uint8_t *o = t->head;
    o = put16(o, 0xffd8);
    static const uint8_t app0[18] = {0xff, 0xe0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
    static const uint8_t app14[16] = {0xff, 0xee, 0, 14, 'A', 'd', 'o', 'b', 'e', 0, 100, 0, 0, 0, 0, 0};   // transform 0: CMYK
    const bool cmyk = t->nc == 4;
    memcpy(o, cmyk ? app14 : app0, cmyk ? 16 : 18);
    o += cmyk ? 16 : 18;
    bool sof1 = false;                  // libjpeg's frame is not baseline with a 16-bit table
    for (uint32_t tbl = 0; tbl < dqts_of(&q, t->nc); tbl++) {
        const bool wide = wide_table(&q, tbl);
        sof1 |= wide;
        o = put16(o, 0xffdb);
        o = put16(o, wide ? 131 : 67);
        *o++ = (uint8_t)(wide << 4 | tbl);
        for (int k = 0; k < 64; k++) {
            const uint16_t v = q.table[tbl][kNatural[k]];
            if (wide) o = put16(o, v);
            else *o++ = (uint8_t)v;
        }
    }
    t->sof_at = (uint32_t)(o - t->head);
    o = put16(o, sof1 ? 0xffc1 : 0xffc0);   // the size is patched per image (j2p_je_head_byte)
    o = put16(o, 8 + 3 * t->nc);
    *o++ = 8;
    o = put16(o, 0);
    o = put16(o, 0);
    *o++ = (uint8_t)t->nc;
    for (uint32_t c = 0; c < t->nc; c++) {
        *o++ = (uint8_t)j2p_je_comp_id(t, c);
        *o++ = (uint8_t)(c ? 0x11 : sof_hs(p) << 4 | sof_vs(p));
        *o++ = (uint8_t)table_of(t->nc, q.ntables, c);
    }
    o = put_dht(o, 0x00, kDcBits[0], kDcVals);
    o = put_dht(o, 0x10, kAcBits[0], kAcVals[0]);
    if (t->nc == 3) {
        o = put_dht(o, 0x01, kDcBits[1], kDcVals);
        o = put_dht(o, 0x11, kAcBits[1], kAcVals[1]);
    }
    static const uint8_t sos[14] = {0xff, 0xda, 0, 12, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0};
    static const uint8_t sos_gray[10] = {0xff, 0xda, 0, 8, 1, 1, 0x00, 0, 63, 0};
    static const uint8_t sos_cmyk[16] = {0xff, 0xda, 0, 14, 4, 'C', 0x00, 'M', 0x00, 'Y', 0x00, 'K', 0x00, 0, 63, 0};
    memcpy(o, gray ? sos_gray : cmyk ? sos_cmyk : sos, j2p_je_sos_len(t));
    t->head_len = (uint32_t)(o - t->head) + j2p_je_sos_len(t);
}

// ---- restart intervals -------------------------------------------------------------------------
// libjpeg's rule: restart_marker_blocks = b gives every scan an interval of b MCUs; restart_marker_rows
// = r (which overrides b, as libjpeg's restart_in_rows overrides restart_interval) gives a scan
// min(r x its MCUs per row, 65535): mcux for an interleaved scan, the component's own block-grid
// width for a non-interleaved one.  0: no restarts.
static uint32_t restart_interval(const struct j2p_jpegenc_params *p, uint32_t per_row) {
    if (p->restart_marker_rows) {
        const uint64_t v = (uint64_t)p->restart_marker_rows * per_row;
        return v < 65535 ? (uint32_t)v : 65535u;
    }
    return (uint32_t)p->restart_marker_blocks;
}

#define J2P_JE_DRI 6u                   // DRI: FF DD 00 04 Ri
#define J2P_JE_RST 2u                   // RSTm: FF D0+m, not stuffed

// byte k of DRI for the interval ri
J2P_HD uint8_t j2p_je_dri_byte(uint32_t ri, uint32_t k) {
    return (uint8_t)(k == 0 ? 0xff : k == 1 ? 0xdd : k == 2 ? 0 : k == 3 ? 4 : k == 4 ? ri >> 8 : ri);
}

// byte k of a header that is hl bytes without DRI and ends in an SOS of sos bytes, head(k), with DRI
// for dri (0: no DRI) inserted before the SOS, as libjpeg's write_scan_header places it
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <class Head>
J2P_HD uint8_t j2p_je_dri_head(uint32_t dri, uint32_t hl, uint32_t sos, uint32_t k, Head head) {
    const uint32_t at = hl - sos;
    if (!dri || k < at) return head(k);
    return k < at + J2P_JE_DRI ? j2p_je_dri_byte(dri, k - at) : head(k - J2P_JE_DRI);
}

// byte k of the RST before interval `part` > 0 of a scan
J2P_HD uint8_t j2p_je_rst_byte(uint32_t part, uint32_t k) { return (uint8_t)(k ? 0xd0 + ((part - 1) & 7) : 0xff); }

// Byte k of a stream's header: the scan header head(k) before its first interval, RST0 + (part - 1)
// mod 8 before interval `part` > 0 (the marker number counts the scan's boundaries from 0).
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <class Head>
J2P_HD uint8_t j2p_je_stream_byte(const struct j2p_je_img *st, uint32_t k, Head head) {
    return st->part ? j2p_je_rst_byte(st->part, k) : head(k);
}

// the length of a baseline stream's header with its image's template t
J2P_HD uint32_t j2p_je_fixed_head_len(const struct j2p_je_tables *t, const struct j2p_je_img *st) {
    return st->part ? J2P_JE_RST : t->head_len + (st->ri ? J2P_JE_DRI : 0);
}

// byte k of a baseline scan header with its image's template t: SOI .. SOS with the image's size
// and its DRI
J2P_HD uint8_t j2p_je_scan_head_byte(const struct j2p_je_tables *t, const struct j2p_je_img *st, uint32_t k) {
    return j2p_je_dri_head(st->ri, t->head_len, j2p_je_sos_len(t), k, [&](uint32_t k1) { return j2p_je_head_byte(t, st, k1); });
}

// byte k of a baseline stream's header: the scan header, or the stream's RST
J2P_HD uint8_t j2p_je_fixed_head_byte(const struct j2p_je_tables *t, const struct j2p_je_img *st, uint32_t k) {
    return j2p_je_stream_byte(st, k, [&](uint32_t k1) { return j2p_je_scan_head_byte(t, st, k1); });
}

// whether stream s ends its image's file (EOI follows it)
J2P_HD bool j2p_je_ends_file(const struct j2p_je_img *strs, uint32_t ns, uint32_t s) { return s + 1 == ns || strs[s + 1].img != strs[s].img; }

// ---- plan --------------------------------------------------------------------------------------
// work: [images][sets of tables][streams] [tile sums][tile offsets][block offsets in the tile][coefficients]
//       [0xFF counts per chunk][their exclusive scan][offsets]
//       (own codes only: [derived tables][headers][header lengths][symbol counts])
//       [entropy words][files]
// A stream is an image's scan, or one restart interval of it.  Without restarts each image is one
// stream and the streams are the images ([streams] is empty); with them, stream p of an image holds
// its MCUs p Ri .. (p + 1) Ri - 1.  The symbol counts sit just before the entropy words, so that one
// memset clears both.
struct Layout {
    uint32_t n, ns, ntiles, nchunks;
    bool plain;                         // no restart intervals: the streams are the images
    uint64_t nblk, words;
    size_t off_imgs, off_tab, off_strs, off_tsum, off_toff, off_intra, off_coef, off_ffc, off_ffpre, off_offs, off_raw, off_out, total;
    size_t off_huff, off_head, off_hlen, off_hist;      // per image; empty without own codes
};

#define J2P_JE_SYMBOLS 256u             // symbol counts per table and image (4 tables)
#define J2P_JE_HEAD_ROOM (J2P_JE_HEAD_MAX + J2P_JE_DRI)        // the longest header of a baseline file

// the checks of a call's arguments
static int check_call(const struct j2p_jpegenc_image *im, unsigned n, const struct j2p_jpegenc_params *p) {
    if (!im) return fail("null argument: images");
    if (!p) return fail("null argument: params");
    if (n == 0) return fail("no images");
    if (p->quality < 1 || p->quality > 100) return fail("quality must be 1 .. 100 (got %d)", p->quality);
    if (p->sampling != J2P_JPEGENC_444 && p->sampling != J2P_JPEGENC_422 && p->sampling != J2P_JPEGENC_420)
        return fail("unknown sampling %d (0: 4:4:4, 1: 4:2:2, 2: 4:2:0)", p->sampling);
    if (p->restart_marker_blocks < 0 || p->restart_marker_blocks > 65535)
        return fail("restart_marker_blocks must be 0 .. 65535 (got %d)", p->restart_marker_blocks);
    if (p->restart_marker_rows < 0 || p->restart_marker_rows > 65535)
        return fail("restart_marker_rows must be 0 .. 65535 (got %d)", p->restart_marker_rows);
    if (p->components != 0 && p->components != 1 && p->components != 3)
        return fail("components must be 0 or 3 (colour) or 1 (gray) (got %d)", p->components);
    if (p->cmyk != 0 && p->cmyk != 1) return fail("cmyk must be 0 or 1 (got %d)", p->cmyk);
    if (p->cmyk && p->components != 0) return fail("cmyk = 1 needs components 0 (got %d)", p->components);
    if (p->qtables && p->nqtables == 0) return fail("qtables given with nqtables 0");
    for (unsigned k = 0; p->qtables && k < p->nqtables; k++) {
        const struct j2p_jpegenc_qtables *q = &p->qtables[k];
        if (q->ntables < 1 || q->ntables > 4) return fail("set %u: ntables must be 1 .. 4 (got %u)", k, q->ntables);
        for (uint32_t tb = 0; tb < q->ntables; tb++)
            for (int i = 0; i < 64; i++)
                if (q->table[tb][i] < 1 || q->table[tb][i] > 8191)
                    return fail("set %u: table %u entry %d is %u; entries must be 1 .. 8191 (8q must fit libjpeg's 16-bit divisor)", k, tb, i,
                                q->table[tb][i]);
    }
    for (unsigned i = 0; i < n; i++) {
        const struct j2p_jpegenc_image *x = &im[i];
        if (!x->data) return fail("image %u: null data pointer", i);
        if (x->width == 0 || x->height == 0 || x->width > 65535 || x->height > 65535)
            return fail("image %u: width and height must be 1 .. 65535 (got %u x %u)", i, x->width, x->height);
        if (p->qtables && x->qtables >= p->nqtables) return fail("image %u: set %u of qtables, which has %u", i, x->qtables, p->nqtables);
    }
    return 0;
}

// image i's descriptor, its blocks from blk0: what the blocks step reads (the stream fields are 0).
// A gray image's MCU is one block, so its MCU grid is its block grid.
static void image_desc(const struct j2p_jpegenc_image *x, uint32_t i, const struct j2p_jpegenc_params *p, uint64_t blk0, struct j2p_je_img *g) {
    const bool gray = is_gray(p);
    const uint32_t hs = gray ? 1 : sof_hs(p), vs = gray ? 1 : sof_vs(p), bpm = gray ? 1 : hs * vs + nc_of(p) - 1;
    memset(g, 0, sizeof *g);
    g->src = (const uint8_t *)x->data;
    g->s_row = x->row_stride;
    g->s_col = x->col_stride;
    g->s_chan = gray ? 0 : x->chan_stride;
    g->w = x->width;
    g->h = x->height;
    g->mcux = (x->width + 8 * hs - 1) / (8 * hs);
    g->mcuy = (x->height + 8 * vs - 1) / (8 * vs);
    g->blk0 = blk0;
    g->nblk = (uint64_t)g->mcux * g->mcuy * bpm;
    g->img = i;
    g->set = p->qtables ? x->qtables : 0;
}

// The running totals of a plan's streams.  add() appends a stream of nb blocks from blk0 (in the
// call's block order of the stream's kind), with wpb words a block of room, a header of at most
// `head` bytes and `tail` bytes after it (EOI), and writes its descriptor into g when g is given.
struct StreamPlan {
    uint64_t ns = 0, tiles = 0, chunks = 0, words = 0, out = 0;
    void add(const struct j2p_je_img &im, uint64_t blk0, uint64_t nb, uint32_t wpb, uint32_t head, uint32_t tail, uint32_t scan, uint32_t part,
             uint32_t ri, struct j2p_je_img *g) {
        const uint64_t nt = (nb + J2P_JE_TILE - 1) / J2P_JE_TILE, raw_bytes = nb * (wpb * 4);
        const uint64_t nc = (raw_bytes + J2P_JE_CHUNK - 1) / J2P_JE_CHUNK;
        if (g) {
            *g = im;
            g->blk0 = blk0;
            g->nblk = nb;
            g->tile0 = (uint32_t)tiles;
            g->ntiles = (uint32_t)nt;
            g->chunk0 = (uint32_t)chunks;
            g->nchunks = (uint32_t)nc;
            g->raw_off = words;
            g->scan = (uint8_t)scan;
            g->part = part;
            g->ri = (uint16_t)ri;
        }
        ns++;
        tiles += nt;
        chunks += nc;
        words += (nb * wpb + 3) / 4 * 4 + 4;   // raw_off stays a multiple of 4 words: chunk_bytes reads uint4
        out += head + 2 * raw_bytes + tail;
    }
    int check(uint64_t nblk) const {
        if (ns >= 0x7fffffffu || tiles >= 0x7fffffffu || chunks >= 0x7fffffffu)
            return fail("too many blocks or restart intervals for one call (%llu blocks, %llu streams)", (unsigned long long)nblk,
                        (unsigned long long)ns);
        return 0;
    }
};

// The plan of a call: wpb entropy words per block of the worst case; own: room for per-image tables
// and headers.  With w, also the plan region (images, streams) at w.
static int make_plan(const struct j2p_jpegenc_image *im, unsigned n, const struct j2p_jpegenc_params *p, uint32_t wpb, bool own, Layout *L,
                     uint8_t *w) {
    if (check_call(im, n, p) != 0) return -1;
    const bool restarts = p->restart_marker_blocks || p->restart_marker_rows;
    uint64_t ns = 0, nblk = 0;
    for (unsigned i = 0; i < n; i++) {          // the streams, to place the arrays
        struct j2p_je_img g;
        image_desc(&im[i], i, p, 0, &g);
        const uint64_t ri = restart_interval(p, g.mcux), mcus = (uint64_t)g.mcux * g.mcuy;
        ns += ri ? (mcus + ri - 1) / ri : 1;
    }
    if (ns >= 0x7fffffffu) return fail("too many restart intervals for one call (%llu)", (unsigned long long)ns);
    size_t o = 0;
    L->off_imgs = o;  o = align16(o + n * sizeof(struct j2p_je_img));
    L->off_tab = o;   o = align16(o + nsets_of(p) * sizeof(struct j2p_je_tables));
    o = (o + 127) & ~(size_t)127;       // each descriptor on one 128-byte line
    L->plain = !restarts;
    L->off_strs = restarts ? o : L->off_imgs;
    if (restarts) o = align16(o + ns * sizeof(struct j2p_je_img));
    struct j2p_je_img *imgs = w ? (struct j2p_je_img *)(w + L->off_imgs) : nullptr, *strs = w ? (struct j2p_je_img *)(w + L->off_strs) : nullptr;
    StreamPlan sp;
    std::vector<uint32_t> head(nsets_of(p));
    for (uint32_t k = 0; k < nsets_of(p); k++) head[k] = head_len_of(p, k);
    for (unsigned i = 0; i < n; i++) {
        struct j2p_je_img g;
        image_desc(&im[i], i, p, nblk, &g);
        const uint32_t bpm = (uint32_t)(g.nblk / ((uint64_t)g.mcux * g.mcuy)), ri = restart_interval(p, g.mcux);
        const uint64_t mcus = (uint64_t)g.mcux * g.mcuy, parts = ri ? (mcus + ri - 1) / ri : 1;
        g.ri = (uint16_t)ri;
        if (imgs && restarts) imgs[i] = g;
        for (uint64_t q = 0; q < parts; q++) {
            const uint64_t m0 = q * ri, m1 = ri && m0 + ri < mcus ? m0 + ri : mcus;
            sp.add(g, nblk + m0 * bpm, (m1 - m0) * bpm, wpb, q ? J2P_JE_RST : head[g.set] + (ri ? J2P_JE_DRI : 0), q + 1 == parts ? 2 : 0, 0,
                   (uint32_t)q, ri, strs ? &strs[sp.ns] : nullptr);
        }
        nblk += g.nblk;
    }
    if (sp.check(nblk) != 0) return -1;
    const size_t m = own ? n : 0;
    L->n = n;
    L->ns = (uint32_t)ns;
    L->nblk = nblk;
    L->ntiles = (uint32_t)sp.tiles;
    L->nchunks = (uint32_t)sp.chunks;
    L->words = sp.words;
    L->off_tsum = o;  o = align16(o + sp.tiles * sizeof(uint32_t));
    L->off_toff = o;  o = align16(o + sp.tiles * sizeof(uint64_t));
    L->off_intra = o; o = align16(o + nblk * sizeof(uint32_t));
    L->off_coef = o;  o = align16(o + nblk * 64 * sizeof(int16_t));
    L->off_ffc = o;   o = align16(o + sp.chunks * sizeof(uint32_t));
    L->off_ffpre = o; o = align16(o + (sp.chunks + 1) * sizeof(uint64_t));
    L->off_offs = o;  o = align16(o + (n + 1) * sizeof(uint64_t));
    L->off_huff = o;  o = align16(o + m * sizeof(struct j2p_je_huff));
    L->off_head = o;  o = align16(o + m * J2P_JE_HEAD_ROOM);
    L->off_hlen = o;  o = align16(o + m * sizeof(uint32_t));
    L->off_hist = o;  o = align16(o + m * 4 * J2P_JE_SYMBOLS * sizeof(uint64_t));
    L->off_raw = o;   o = align16(o + sp.words * sizeof(uint32_t));
    L->off_out = o;   o = align16(o + sp.out);
    L->total = o;
    return 0;
}

// the call's sets of tables at t
static void make_sets(const struct j2p_jpegenc_params *p, struct j2p_je_tables *t) {
    for (uint32_t k = 0; k < nsets_of(p); k++) make_tables(p, k, t + k);
}

// the plan region (images, sets, streams) in host memory
static int fill_plan(const struct j2p_jpegenc_image *im, unsigned n, const struct j2p_jpegenc_params *p, uint32_t wpb, bool own, const Layout &,
                     uint8_t *w) {
    Layout tmp;
    if (make_plan(im, n, p, wpb, own, &tmp, w) != 0) return -1;
    make_sets(p, (struct j2p_je_tables *)(w + tmp.off_tab));
    return 0;
}

// ---- steps shared by the kernels and the host driver ----------------------------------------------
// Geometry and codes are the same in every set: these read the call's set 0.
J2P_HD uint32_t comp_of(const struct j2p_je_tables *t, uint64_t b) {
    const uint32_t k = (uint32_t)(b % j2p_je_bpm(t)), nl = t->hs * t->vs;
    return k < nl ? 0 : 1 + (k - nl);
}

// the Huffman tables block b codes with (j2p_je_htab)
J2P_HD uint32_t htab_of(const struct j2p_je_tables *t, uint64_t b) { return j2p_je_htab(t, comp_of(t, b)); }

// column x of a block whose rows are through pass 1 (rows[y * stride + x]): pass 2, quantise with
// the tables of t (the image's set), and store in zig-zag order; a dummy keeps only its DC
J2P_HD void finish_column(const struct j2p_je_tables *t, const struct j2p_je_where *w, const int *rows, int stride, int x, int16_t *coef) {
    int d[8];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int y = 0; y < 8; y++) d[y] = rows[y * stride + x];
    j2p_je_fdct_1d<2>(d);
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int y = 0; y < 8; y++) {
        const int i = y * 8 + x;
        const int v = w->dummy && i ? 0 : j2p_je_quant(t, (int)w->comp, i, d[y]);
        coef[t->zz[i]] = (int16_t)v;
    }
}

J2P_HD int pred_of(const struct j2p_je_tables *t, const int16_t *coef, uint64_t blk0, uint64_t b) {
    const uint64_t pb = j2p_je_prev(t, b);
    return pb == ~(uint64_t)0 ? 0 : coef[(blk0 + pb) * 64];
}

J2P_HD uint64_t raw_bytes(const struct j2p_je_img *im) { return (im->bits + 7) / 8; }

// ---- host driver -------------------------------------------------------------------------------
// the blocks step of the kernels on one image with its set t, serially: its coefficients at coef +
// im->blk0 * 64
static void host_blocks(const struct j2p_je_img *im, const struct j2p_je_tables *t, int16_t *coef) {
    for (uint64_t b = 0; b < im->nblk; b++) {
        const struct j2p_je_where wh = j2p_je_locate(im, t, b);
        int rows[64];
        for (int y = 0; y < 8; y++) j2p_je_block_row(im, t, &wh, y, rows + 8 * y);
        for (int x = 0; x < 8; x++) finish_column(t, &wh, rows, 8, x, coef + (im->blk0 + b) * 64);
    }
}

// encode_jpeg's default codes: the call's Annex K tables for every image, and the header template of
// its set (t: the sets)
struct FixedCodes {
    const struct j2p_je_tables *t;
    const struct j2p_je_huff *huff(uint32_t) const { return &t->huff; }
    uint32_t head_len(const struct j2p_je_img *st) const { return j2p_je_fixed_head_len(t + st->set, st); }
    uint8_t head_byte(const struct j2p_je_img *st, uint32_t k) const { return j2p_je_fixed_head_byte(t + st->set, st, k); }
};

// The steps of the kernels run serially on host memory.  codes(L, w, imgs, strs, t, coef) (t: the
// sets) runs
// between the blocks and the sizes and returns where each image's Huffman tables and each stream's
// header come from: an object with huff(image), head_len(stream) and head_byte(stream, k), such as
// FixedCodes.
template <class Codes>
static int encode_host_steps(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, uint32_t wpb, bool own,
                             void *work, size_t work_bytes, uint64_t *offsets, Codes codes) {
    Layout L;
    if (make_plan(images, n, params, wpb, own, &L, nullptr) != 0) return -1;
    if (!work || !offsets) return fail("null argument");
    if (work_bytes < L.total) return fail("work area of %zu bytes is smaller than the plan's %zu", work_bytes, L.total);
    uint8_t *w = (uint8_t *)work;
    if (fill_plan(images, n, params, wpb, own, L, w) != 0) return -1;
    const struct j2p_je_img *imgs = (const struct j2p_je_img *)(w + L.off_imgs);
    struct j2p_je_img *strs = (struct j2p_je_img *)(w + L.off_strs);
    const struct j2p_je_tables *t = (const struct j2p_je_tables *)(w + L.off_tab);
    uint32_t *tsum = (uint32_t *)(w + L.off_tsum), *intra = (uint32_t *)(w + L.off_intra), *ffc = (uint32_t *)(w + L.off_ffc);
    uint64_t *toff = (uint64_t *)(w + L.off_toff), *ffpre = (uint64_t *)(w + L.off_ffpre);
    int16_t *coef = (int16_t *)(w + L.off_coef);
    uint32_t *raw = (uint32_t *)(w + L.off_raw);
    uint8_t *out = w + L.off_out;
    memset(w + L.off_hist, 0, L.off_raw - L.off_hist + L.words * sizeof(uint32_t));
    for (unsigned i = 0; i < n; i++) host_blocks(&imgs[i], t + imgs[i].set, coef);      // blocks
    const auto c = codes(L, w, imgs, (const struct j2p_je_img *)strs, t, (const int16_t *)coef);
    for (uint32_t s = 0; s < L.ns; s++) {                               // sizes and scans
        struct j2p_je_img *im = &strs[s];
        uint64_t bits = 0;
        for (uint32_t k = 0; k < im->ntiles; k++) {
            uint32_t sum = 0;
            for (uint64_t b = (uint64_t)k * J2P_JE_TILE; b < im->nblk && b < (uint64_t)(k + 1) * J2P_JE_TILE; b++) {
                intra[im->blk0 + b] = sum;
                sum += j2p_je_block_bits(coef + (im->blk0 + b) * 64, pred_of(t, coef, im->blk0, b), c.huff(im->img), htab_of(t, b));
            }
            tsum[im->tile0 + k] = sum;
            toff[im->tile0 + k] = bits;
            bits += sum;
        }
        im->bits = bits;
        uint64_t pw;
        const uint32_t mask = j2p_je_pad(bits, &pw);
        raw[im->raw_off + pw] |= mask;
    }
    for (uint32_t s = 0; s < L.ns; s++) {                               // emit
        const struct j2p_je_img *im = &strs[s];
        for (uint64_t b = 0; b < im->nblk; b++) {
            const uint64_t pos = toff[im->tile0 + b / J2P_JE_TILE] + intra[im->blk0 + b];
            j2p_je_emit(coef + (im->blk0 + b) * 64, pred_of(t, coef, im->blk0, b), c.huff(im->img), htab_of(t, b), pos,
                        [&](uint64_t k, uint32_t v) { raw[im->raw_off + k] |= v; });
        }
    }
    uint64_t ff = 0, off = 0;                                           // 0xFF counts, stream and file offsets
    for (uint32_t s = 0; s < L.ns; s++) {
        struct j2p_je_img *im = &strs[s];
        const uint32_t *rw = raw + im->raw_off;
        const uint64_t nbytes = raw_bytes(im);
        for (uint32_t k = 0; k < im->nchunks; k++) {
            uint32_t cnt = 0;
            for (uint64_t j = (uint64_t)k * J2P_JE_CHUNK; j < nbytes && j < (uint64_t)(k + 1) * J2P_JE_CHUNK; j++) cnt += j2p_je_byte(rw, j) == 0xff;
            ffc[im->chunk0 + k] = cnt;
            ffpre[im->chunk0 + k] = ff;
            ff += cnt;
        }
        const uint64_t ffi = ff - ffpre[im->chunk0];
        im->file_len = c.head_len(im) + nbytes + ffi + (j2p_je_ends_file(strs, L.ns, s) ? 2 : 0);
        im->file_off = off;
        if (s == 0 || strs[s - 1].img != im->img) offsets[im->img] = off;
        off += im->file_len;
    }
    ffpre[L.nchunks] = ff;
    offsets[n] = off;
    for (uint32_t s = 0; s < L.ns; s++) {                               // files
        const struct j2p_je_img *im = &strs[s];
        uint8_t *o = out + im->file_off;
        for (uint32_t k = 0; k < c.head_len(im); k++) *o++ = c.head_byte(im, k);
        const uint32_t *rw = raw + im->raw_off;
        for (uint64_t j = 0; j < raw_bytes(im); j++) {
            const uint8_t v = j2p_je_byte(rw, j);
            *o++ = v;
            if (v == 0xff) *o++ = 0;
        }
        if (j2p_je_ends_file(strs, L.ns, s)) {
            *o++ = 0xff;
            *o++ = 0xd9;
        }
    }
    return 0;
}

#endif  // J2P_JPEGENC_PLAN_H
