// jpegprog.cu — libj2pjpegprog.so: the device encoder of progressive JPEG files and the serial host
// driver of the same steps.  See jpegprog.h; the scans are in jpegprog_core.h, the steps shared with
// the other encoders in ../jpegenc (jpegenc_plan.h, jpegenc_kernels.cuh) and the table builder in
// ../jpegopt/jpegopt_core.h.
#include <vector>

#include "../jpegenc/jpegenc_kernels.cuh"
#include "jpegprog_core.h"

extern "C" const char *j2p_jpegprog_last_error(void) { return g_err; }

// ---- plan --------------------------------------------------------------------------------------
// Every (image, scan, restart interval) is a stream, described by a j2p_je_img (the stuffing steps'
// view of a bit stream): its image, scan and interval, blk0 and nblk its blocks among the call's
// stream blocks, its tiles, chunks, words, bits and place in the output.  Without restarts a scan is
// one stream.  The streams of one scan are consecutive, and so are their stream blocks, and each
// (image, scan) has a j2p_jp_scanplan: its first stream and the DRI its header carries.
// work: [images][sets of tables][streams][scans] [tile sums][tile offsets][block offsets in the tile][run states]
//       [summaries][coefficients][0xFF counts per chunk][their exclusive scan][offsets]
//       [derived tables][scan headers][their lengths][symbol counts][entropy words][files]
// The symbol counts sit just before the entropy words, so that one memset clears both.
struct PLayout {
    uint32_t n, ns, ntiles, nchunks;
    bool plain;                         // no restart intervals: one stream per (image, scan)
    uint64_t nblk, nsblk, words;
    size_t off_imgs, off_tab, off_str, off_scan, off_tsum, off_toff, off_intra, off_state, off_summ, off_coef, off_ffc, off_ffpre, off_offs,
        off_huff, off_head, off_hlen, off_hist, off_raw, off_out, total;
};

struct j2p_jp_scanplan {
    uint32_t s0;                        // the scan's first stream
    uint32_t dri;                       // the interval its DRI writes, 0 for no DRI (unchanged since the last one)
};

// The streams of a call's images: each stream's descriptor into strs and each scan's plan into scs
// when they are given; returns the totals.
static StreamPlan prog_streams(const struct j2p_je_img *imgs, unsigned n, const struct j2p_jpegenc_params *p, const struct j2p_je_tables *t,
                               struct j2p_je_img *strs, struct j2p_jp_scanplan *scs, uint64_t *nsblk) {
    StreamPlan sp;
    uint64_t sblk = 0;
    const uint32_t nc = t->nc, per = j2p_jp_nscans(nc);
    for (unsigned i = 0; i < n; i++) {
        const struct j2p_je_img *im = &imgs[i];
        uint32_t last_ri = 0;                                   // the interval of the last DRI written
        for (uint32_t k = 0; k < per; k++) {
            const bool ac = j2p_jp_is_ac(nc, k);
            const uint32_t comp = j2p_jp_scan_of(nc, k).comp, wpb = j2p_jp_bound_words(nc, k);
            // an MCU of an AC scan is one block of the component's own grid; of a DC scan, an MCU of the image
            const uint32_t per_row = ac ? j2p_jp_grid_w(im, t, comp) : im->mcux, upm = ac ? 1 : j2p_je_bpm(t);
            const uint64_t mcus = ac ? (uint64_t)per_row * j2p_jp_grid_h(im, t, comp) : (uint64_t)im->mcux * im->mcuy;
            const uint32_t ri = restart_interval(p, per_row);
            const uint64_t parts = ri ? (mcus + ri - 1) / ri : 1;
            if (scs) scs[(size_t)i * per + k] = {(uint32_t)sp.ns, ri != last_ri ? ri : 0u};
            last_ri = ri;
            for (uint64_t q = 0; q < parts; q++) {
                const uint64_t m0 = q * ri, m1 = ri && m0 + ri < mcus ? m0 + ri : mcus;
                sp.add(*im, sblk + m0 * upm, (m1 - m0) * upm, wpb, q ? J2P_JE_RST : J2P_JP_HEAD, k + 1 == per && q + 1 == parts ? 2 : 0, k,
                       (uint32_t)q, ri, strs ? &strs[sp.ns] : nullptr);
            }
            sblk += mcus * upm;
        }
    }
    *nsblk = sblk;
    return sp;
}

// The plan of a call; with w, also its plan region (images, tables, streams, scans) at w.
static int prog_plan(const struct j2p_jpegenc_image *im, unsigned n, const struct j2p_jpegenc_params *p, PLayout *P, uint8_t *w) {
    if (check_call(im, n, p) != 0) return -1;
    std::vector<struct j2p_je_img> imgs(n);
    uint64_t nblk = 0;
    for (unsigned i = 0; i < n; i++) {
        image_desc(&im[i], i, p, nblk, &imgs[i]);
        nblk += imgs[i].nblk;
    }
    struct j2p_je_tables t;             // set 0: the geometry, the same in every set
    make_tables(p, 0, &t);
    uint64_t sblk;
    const StreamPlan sp = prog_streams(imgs.data(), n, p, &t, nullptr, nullptr, &sblk);
    if (sp.check(nblk) != 0) return -1;
    const size_t nsc = (size_t)n * j2p_jp_nscans(t.nc), ntab = (size_t)n * j2p_jp_ntables(t.nc);
    size_t o = 0;
    P->off_imgs = o;  o = align16(o + n * sizeof(struct j2p_je_img));
    P->off_tab = o;   o = align16(o + nsets_of(p) * sizeof(struct j2p_je_tables));
    o = (o + 127) & ~(size_t)127;       // each descriptor on one 128-byte line
    P->off_str = o;   o = align16(o + sp.ns * sizeof(struct j2p_je_img));
    P->off_scan = o;  o = align16(o + nsc * sizeof(struct j2p_jp_scanplan));
    if (w) {
        memcpy(w + P->off_imgs, imgs.data(), n * sizeof(struct j2p_je_img));
        make_sets(p, (struct j2p_je_tables *)(w + P->off_tab));
        prog_streams(imgs.data(), n, p, &t, (struct j2p_je_img *)(w + P->off_str), (struct j2p_jp_scanplan *)(w + P->off_scan), &sblk);
    }
    P->n = n;
    P->ns = (uint32_t)sp.ns;
    P->plain = !p->restart_marker_blocks && !p->restart_marker_rows;
    P->nblk = nblk;
    P->nsblk = sblk;
    P->ntiles = (uint32_t)sp.tiles;
    P->nchunks = (uint32_t)sp.chunks;
    P->words = sp.words;
    P->off_tsum = o;  o = align16(o + sp.tiles * sizeof(uint32_t));
    P->off_toff = o;  o = align16(o + sp.tiles * sizeof(uint64_t));
    P->off_intra = o; o = align16(o + sblk * sizeof(uint32_t));
    P->off_state = o; o = align16(o + sblk * sizeof(uint32_t));
    P->off_summ = o;  o = align16(o + sblk);
    P->off_coef = o;  o = align16(o + nblk * 64 * sizeof(int16_t));
    P->off_ffc = o;   o = align16(o + sp.chunks * sizeof(uint32_t));
    P->off_ffpre = o; o = align16(o + (sp.chunks + 1) * sizeof(uint64_t));
    P->off_offs = o;  o = align16(o + (n + 1) * sizeof(uint64_t));
    P->off_huff = o;  o = align16(o + ntab * sizeof(struct j2p_jp_huff));
    P->off_head = o;  o = align16(o + nsc * J2P_JP_HEAD);
    P->off_hlen = o;  o = align16(o + nsc * sizeof(uint32_t));
    P->off_hist = o;  o = align16(o + ntab * 256 * sizeof(uint64_t));
    P->off_raw = o;   o = align16(o + sp.words * sizeof(uint32_t));
    P->off_out = o;   o = align16(o + sp.out);
    P->total = o;
    return 0;
}

extern "C" int j2p_jpegprog_plan(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, size_t *work_bytes,
                                 size_t *out_offset) {
    PLayout P;
    if (prog_plan(images, n, params, &P, nullptr) != 0) return -1;
    if (work_bytes) *work_bytes = P.total;
    if (out_offset) *out_offset = P.off_out;
    return 0;
}

// ---- steps shared by the kernels and the host driver ----------------------------------------------
// what a block's coding reads
struct Ctx {
    const struct j2p_je_img *imgs, *strs;
    const struct j2p_je_tables *t;
    const int16_t *coef;
    const uint8_t *summ;
    const uint32_t *state;
    bool plain;                         // no restart intervals: stream s is scan s % 10 of image s / 10 (6 gray, 18 CMYK)
    uint32_t nc;                        // the call's kind: 3 colour, 1 gray (the six-scan script), 4 CMYK (18 scans)
};

// the scan and the image of stream s: arithmetic without restart intervals, the descriptor with them
J2P_HD uint32_t scan_of(const Ctx &x, uint32_t s) { return x.plain ? s % j2p_jp_nscans(x.nc) : x.strs[s].scan; }
J2P_HD uint32_t image_of(const Ctx &x, uint32_t s) { return x.plain ? s / j2p_jp_nscans(x.nc) : x.strs[s].img; }

// the first of image i's Huffman table slots (tables and symbol counts), j2p_jp_ntables a image
J2P_HD size_t slot0(const Ctx &x, uint32_t i) { return (size_t)i * j2p_jp_ntables(x.nc); }

// the first block of stream s in its scan's order (the MCU grid's stored order for a DC scan, the
// component's raster order for an AC scan): a multiple of an MCU, so a DC prediction restarts there
J2P_HD uint64_t stream_first(const Ctx &x, uint32_t s) {
    if (x.plain) return 0;
    const struct j2p_je_img *st = &x.strs[s];
    return (uint64_t)st->part * st->ri * (j2p_jp_is_ac(x.nc, st->scan) ? 1u : j2p_je_bpm(x.t));
}

// the coefficients of block j of an AC scan over component comp of image im
J2P_HD const int16_t *ac_coef(const Ctx &x, const struct j2p_je_img *im, uint32_t comp, uint64_t j) {
    return x.coef + (im->blk0 + j2p_jp_stored(im, x.t, comp, j2p_jp_grid_w(im, x.t, comp), (uint32_t)j)) * 64;
}

// block j of stream s into o; the stream's last block flushes the EOB run, as a restart does
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <class Out>
J2P_HD void code_block(const Ctx &x, uint32_t s, uint64_t j, Out &o) {
    const uint32_t k = scan_of(x, s);
    const struct j2p_je_img *st = &x.strs[s], *im = &x.imgs[image_of(x, s)];
    const struct j2p_jp_scan sc = j2p_jp_scan_of(x.nc, k);
    const uint64_t f = stream_first(x, s);
    const bool last = j + 1 == st->nblk;
    if (j2p_jp_is_ac(x.nc, k))
        j2p_jp_code(sc, ac_coef(x, im, sc.comp, f + j), 0, sc.comp, x.state[st->blk0 + j], j, last, o);
    else
        j2p_jp_code(sc, x.coef + (im->blk0 + f + j) * 64, pred_of(x.t, x.coef, im->blk0 + f, j), htab_of(x.t, j), 0, j, last, o);
}

// the summary of block j of AC stream s
J2P_HD uint32_t summary_of(const Ctx &x, uint32_t s, uint64_t j) {
    const struct j2p_jp_scan sc = j2p_jp_scan_of(x.nc, scan_of(x, s));
    return j2p_jp_summary(sc, ac_coef(x, &x.imgs[image_of(x, s)], sc.comp, stream_first(x, s) + j));
}

// Outs of j2p_jp_code: symbol counts, bit counts, and the bits themselves
template <class Count>
struct CountSymbols {
    Count count;
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
    J2P_HD void sym(int tb, int s) { count(tb, s); }
    J2P_HD void bits(uint32_t, int) {}
    J2P_HD void deferred(uint64_t, uint32_t, uint32_t) {}
};

struct CountBits {
    const struct j2p_jp_huff *h;
    uint32_t n;
    J2P_HD void sym(int tb, int s) { n += h[tb].size[s]; }
    J2P_HD void bits(uint32_t, int k) { n += (uint32_t)k; }
    J2P_HD void deferred(uint64_t, uint32_t, uint32_t be) { n += be; }
};

template <class Or>
struct EmitBits {
    const struct j2p_jp_huff *h;
    j2p_je_writer<Or> w;
    Ctx x;
    uint32_t s;
    J2P_HD void sym(int tb, int v) { w(h[tb].code[v], h[tb].size[v]); }
    J2P_HD void bits(uint32_t v, int k) { w(v, k); }
    // the correction bits of the run's blocks that have any, in order
    J2P_HD void deferred(uint64_t first, uint32_t run, uint32_t) {
        const struct j2p_je_img *st = &x.strs[s], *im = &x.imgs[image_of(x, s)];
        const struct j2p_jp_scan sc = j2p_jp_scan_of(x.nc, scan_of(x, s));
        const uint64_t f = stream_first(x, s);
        for (uint64_t q = first; q < first + run; q++)
            if (x.summ[st->blk0 + q] & 63u) j2p_jp_tail(sc, ac_coef(x, im, sc.comp, f + q), *this);
    }
};

// the header of stream st: its scan's header (in heads, its length in hlens; per scans an image),
// or RST
static uint32_t prog_head_len(const uint32_t *hlens, uint32_t per, const struct j2p_je_img *st) {
    return st->part ? J2P_JE_RST : hlens[(size_t)st->img * per + st->scan];
}

static uint8_t prog_head_byte(const uint8_t *heads, uint32_t per, const struct j2p_je_img *st, uint32_t k) {
    return j2p_je_stream_byte(st, k, [&](uint32_t k1) { return heads[((size_t)st->img * per + st->scan) * J2P_JP_HEAD + k1]; });
}

// ---- host driver -------------------------------------------------------------------------------
extern "C" int j2p_jpegprog_encode_host(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, void *work,
                                        size_t work_bytes, uint64_t *offsets) {
    PLayout P;
    if (prog_plan(images, n, params, &P, nullptr) != 0) return -1;
    if (!work || !offsets) return fail("null argument");
    if (work_bytes < P.total) return fail("work area of %zu bytes is smaller than the plan's %zu", work_bytes, P.total);
    uint8_t *w = (uint8_t *)work;
    if (prog_plan(images, n, params, &P, w) != 0) return -1;
    struct j2p_je_img *imgs = (struct j2p_je_img *)(w + P.off_imgs), *strs = (struct j2p_je_img *)(w + P.off_str);
    const struct j2p_jp_scanplan *scs = (const struct j2p_jp_scanplan *)(w + P.off_scan);
    const struct j2p_je_tables *t = (const struct j2p_je_tables *)(w + P.off_tab);
    int16_t *coef = (int16_t *)(w + P.off_coef);
    uint8_t *summ = w + P.off_summ;
    uint32_t *state = (uint32_t *)(w + P.off_state), *raw = (uint32_t *)(w + P.off_raw), *hlens = (uint32_t *)(w + P.off_hlen);
    uint64_t *hist = (uint64_t *)(w + P.off_hist);
    struct j2p_jp_huff *huffs = (struct j2p_jp_huff *)(w + P.off_huff);
    uint8_t *heads = w + P.off_head, *out = w + P.off_out;
    memset(w + P.off_hist, 0, P.off_raw - P.off_hist + P.words * sizeof(uint32_t));
    const uint32_t nc = t->nc, per = j2p_jp_nscans(nc);
    const Ctx x = {imgs, strs, t, coef, summ, state, P.plain, nc};
    for (unsigned i = 0; i < n; i++) host_blocks(&imgs[i], t + imgs[i].set, coef);      // blocks
    for (uint32_t s = 0; s < P.ns; s++) {                               // summaries, runs
        const struct j2p_je_img *st = &strs[s];
        if (!j2p_jp_is_ac(nc, st->scan)) continue;
        for (uint64_t j = 0; j < st->nblk; j++) summ[st->blk0 + j] = (uint8_t)summary_of(x, s, j);
        for (uint64_t j = 0; j < st->nblk; j++)
            if (j == 0 || (summ[st->blk0 + j - 1] & J2P_JP_RESET))
                j2p_jp_walk(j, st->nblk, [&](uint64_t q) { return (uint32_t)summ[st->blk0 + q]; },
                            [&](uint64_t q, uint32_t v) { state[st->blk0 + q] = v; });
    }
    for (uint32_t s = 0; s < P.ns; s++) {                               // hist
        uint64_t *h = hist + (slot0(x, strs[s].img) + j2p_jp_slot(nc, strs[s].scan)) * 256;
        const auto count = [h](int tb, int v) { h[tb * 256 + v]++; };
        CountSymbols<decltype(count)> o = {count};
        for (uint64_t j = 0; j < strs[s].nblk; j++) code_block(x, s, j, o);
    }
    for (unsigned i = 0; i < n; i++) {                                  // tables, scan headers
        struct j2p_jo_scratch scr;
        struct j2p_jp_dht d;
        for (uint32_t tb = 0; tb < j2p_jp_ntables(nc); tb++)
            j2p_jp_table(hist + (slot0(x, i) + tb) * 256, &scr, &d, &huffs[slot0(x, i) + tb], tb, j2p_jo_serial());
        const struct j2p_je_tables *ts = t + imgs[i].set;
        for (uint32_t k = 0; k < per; k++) {
            const size_t q = (size_t)i * per + k;
            hlens[q] = j2p_jp_scan_head_len(ts, &d, k, scs[q].dri);
            for (uint32_t b = 0; b < hlens[q]; b++) heads[q * J2P_JP_HEAD + b] = j2p_jp_scan_head_byte(ts, &imgs[i], &d, k, scs[q].dri, b);
        }
    }
    for (uint32_t s = 0; s < P.ns; s++) {                               // sizes, emit, padding
        struct j2p_je_img *st = &strs[s];
        const struct j2p_jp_huff *h = huffs + slot0(x, st->img) + j2p_jp_slot(nc, st->scan);
        uint64_t pos = 0;
        for (uint64_t j = 0; j < st->nblk; j++) {
            CountBits c = {h, 0};
            code_block(x, s, j, c);
            const auto orw = [&](uint64_t k, uint32_t v) { raw[st->raw_off + k] |= v; };
            EmitBits<decltype(orw)> e = {h, {orw, 0, (uint32_t)(pos & 31), pos >> 5}, x, s};
            code_block(x, s, j, e);
            if (e.w.fill) orw(e.w.word, (uint32_t)(e.w.acc >> 32));
            pos += c.n;
        }
        st->bits = pos;
        uint64_t pw;
        const uint32_t mask = j2p_je_pad(pos, &pw);
        raw[st->raw_off + pw] |= mask;
    }
    uint8_t *o = out;                                                   // files
    for (uint32_t s = 0; s < P.ns; s++) {
        const struct j2p_je_img *st = &strs[s];
        if (s == 0 || strs[s - 1].img != st->img) offsets[st->img] = (uint64_t)(o - out);
        for (uint32_t b = 0; b < prog_head_len(hlens, per, st); b++) *o++ = prog_head_byte(heads, per, st, b);
        const uint32_t *rw = raw + st->raw_off;
        for (uint64_t j = 0; j < raw_bytes(st); j++) {
            const uint8_t v = j2p_je_byte(rw, j);
            *o++ = v;
            if (v == 0xff) *o++ = 0;
        }
        if (j2p_je_ends_file(strs, P.ns, s)) {
            *o++ = 0xff;
            *o++ = 0xd9;
        }
    }
    offsets[n] = (uint64_t)(o - out);
    return 0;
}

// ---- device ------------------------------------------------------------------------------------
static const int kTableThreads = 32 * J2P_JP_TABLES;    // one warp per table of a colour image

// the derived tables of stream s (two for a colour scan 0, one for an AC scan or a gray or CMYK
// scan 0, none for the DC refine) into shared memory, by every thread of the CTA
__device__ __forceinline__ const struct j2p_jp_huff *stage(struct j2p_jp_huff *sh, const struct j2p_jp_huff *huffs, const Ctx &x, uint32_t s) {
    const uint32_t k = scan_of(x, s), nt = j2p_jp_ntab(x.nc, k);
    const uint4 *src = (const uint4 *)(huffs + slot0(x, image_of(x, s)) + j2p_jp_slot(x.nc, k));
    uint4 *dst = (uint4 *)sh;
    for (uint32_t q = threadIdx.x; q < nt * sizeof(struct j2p_jp_huff) / 16; q += blockDim.x) dst[q] = src[q];
    __syncthreads();
    return sh;
}

// the stream of this tile, and this thread's block in it
__device__ __forceinline__ uint32_t tile_block(const struct j2p_je_img *strs, uint32_t ns, uint64_t *j) {
    const uint32_t s = find_image(strs, ns, blockIdx.x, 1);
    *j = (uint64_t)(blockIdx.x - strs[s].tile0) * J2P_JE_TILE + threadIdx.x;
    return s;
}

// x with the call's kind as the constant NC.  k_jp_hist branches once on the kind, which is uniform
// over the launch, and runs its body with as_kind<3>, <1> or <4>, so each kind's body is compiled
// for it alone; k_jp_emit does so for colour and runs gray and CMYK calls through one body with the
// kind as a runtime value (a third body would take it past 64 registers); k_jp_blocks does the same
// with its summaries.
template <uint32_t NC>
__device__ __forceinline__ Ctx as_kind(Ctx x) {
    x.nc = NC;
    return x;
}

// each real block's summary in each AC scan of its component (a lane per scan).  A component's AC
// scans are the gray script's in a gray or a CMYK call, the colour script's otherwise: SC, 1 or 3,
// is that script, and nc the call's kind, which places the scan among the image's.
template <uint32_t SC>
__device__ __forceinline__ void summaries(const struct j2p_je_img *__restrict__ imgs, uint32_t n, const struct j2p_je_tables *__restrict__ t,
                                          uint64_t nblk, const int16_t *__restrict__ coef, const struct j2p_je_img *__restrict__ strs,
                                          const struct j2p_jp_scanplan *__restrict__ scs, bool plain, uint8_t *__restrict__ summ, uint32_t nc) {
    const uint64_t g = ((uint64_t)blockIdx.x * kBlockThreads + threadIdx.x) >> 3;
    if (g >= nblk) return;
    const uint32_t i = find_image(imgs, n, g, 0);
    const struct j2p_je_img *im = &imgs[i];
    const struct j2p_je_where wh = j2p_je_locate(im, t, g - im->blk0);
    const uint32_t lane = threadIdx.x & 7;
    const int ks = j2p_jp_comp_scan(SC, SC == 1 ? 0 : wh.comp, lane);          // the scan in script SC
    if (wh.dummy || ks < 0) return;
    const int k = SC == 1 && nc == 4 ? j2p_jp_comp_scan(4, wh.comp, lane) : ks;  // the scan of the image
    const uint64_t j = (uint64_t)wh.row * j2p_jp_grid_w(im, t, wh.comp) + wh.col;
    const size_t q = (size_t)i * j2p_jp_nscans(nc) + k;
    summ[strs[plain ? q : scs[q].s0].blk0 + j] = (uint8_t)j2p_jp_summary(j2p_jp_scan_of(SC, (uint32_t)ks), coef + g * 64);
}

// kBlockThreads threads, 8 per block: the shared blocks body, then the summaries.  Six CTAs per SM
// (40 registers, as with colour summaries alone): the two summary bodies would otherwise take 48.
__global__ void __launch_bounds__(kBlockThreads, 6) k_jp_blocks(const struct j2p_je_img *__restrict__ imgs, uint32_t n,
                                                            const struct j2p_je_tables *__restrict__ t, uint64_t nblk,
                                                            int16_t *__restrict__ coef, const struct j2p_je_img *__restrict__ strs,
                                                            const struct j2p_jp_scanplan *__restrict__ scs, bool plain,
                                                            uint8_t *__restrict__ summ, uint32_t nc) {
    blocks_body(imgs, n, t, nblk, coef);
    __syncthreads();
    if (nc == 3) summaries<3>(imgs, n, t, nblk, coef, strs, scs, plain, summ, nc);
    else summaries<1>(imgs, n, t, nblk, coef, strs, scs, plain, summ, nc);
}

// The stream-arithmetic kernels take the call's kind and run the body with NC = it, and so PER =
// its scans per image, J2P_JP_SCANS, J2P_JP_SCANS_GRAY or J2P_JP_SCANS_CMYK: three instantiations
// in one kernel.
template <uint32_t NC>
__device__ __forceinline__ void runs_body(const struct j2p_je_img *__restrict__ strs, uint32_t ns, bool plain, const uint8_t *__restrict__ summ,
                                          uint32_t *__restrict__ state) {
    const StreamMap<j2p_jp_nscans(NC)> sm = {strs, ns, plain};
    uint64_t j;
    const uint32_t s = tile_block(sm.strs, sm.ns, &j);
    const struct j2p_je_img *st = &sm.strs[s];
    if (!j2p_jp_is_ac(NC, sm.scan(s)) || j >= st->nblk) return;
    const uint8_t *m = summ + st->blk0;
    if (j && !(m[j - 1] & J2P_JP_RESET)) return;
    uint32_t *out = state + st->blk0;
    j2p_jp_walk(j, st->nblk, [&](uint64_t q) { return (uint32_t)m[q]; }, [&](uint64_t q, uint32_t v) { out[q] = v; });
}

// per block of an AC stream that starts a segment: the walk to the segment's end (a RESET block or
// the stream's end, which a restart marker follows)
__global__ void __launch_bounds__(kTileThreads) k_jp_runs(const struct j2p_je_img *__restrict__ strs, uint32_t ns, bool plain, const uint8_t *__restrict__ summ,
                                                         uint32_t *__restrict__ state, uint32_t nc) {
    if (nc == 1) runs_body<1>(strs, ns, plain, summ, state);
    else if (nc == 4) runs_body<4>(strs, ns, plain, summ, state);
    else runs_body<3>(strs, ns, plain, summ, state);
}

// per tile: the symbols of its blocks counted in shared memory, then added to the image's counts
__device__ __forceinline__ void hist_body(const Ctx &x, uint32_t ns, unsigned long long *__restrict__ hist, uint32_t *cnt) {
    uint64_t j;
    const uint32_t s = tile_block(x.strs, ns, &j), k = scan_of(x, s);
    if (!j2p_jp_ntab(x.nc, k)) return;                  // the DC refine has no symbols
    for (uint32_t q = threadIdx.x; q < 2 * 256; q += kTileThreads) cnt[q] = 0;
    __syncthreads();
    if (j < x.strs[s].nblk) {
        const auto count = [&](int tb, int v) { atomicAdd(&cnt[tb * 256 + v], 1u); };
        CountSymbols<decltype(count)> o = {count};
        code_block(x, s, j, o);
    }
    __syncthreads();
    unsigned long long *h = hist + (slot0(x, image_of(x, s)) + j2p_jp_slot(x.nc, k)) * 256;
    for (uint32_t q = threadIdx.x; q < 2 * 256; q += kTileThreads)
        if (cnt[q]) atomicAdd(h + q, (unsigned long long)cnt[q]);
}

__global__ void __launch_bounds__(kTileThreads) k_jp_hist(const Ctx x, uint32_t ns, unsigned long long *__restrict__ hist) {
    __shared__ uint32_t cnt[2 * 256];
    if (x.nc == 1) hist_body(as_kind<1>(x), ns, hist, cnt);
    else if (x.nc == 4) hist_body(as_kind<4>(x), ns, hist, cnt);
    else hist_body(as_kind<3>(x), ns, hist, cnt);
}

// per image, a warp per table: code lengths, symbols and codes; then its scans' headers, from its
// set's template.  A gray image's warps past its five tables have none to build; a CMYK image's
// seventeen take two rounds of the ten warps.
__global__ void __launch_bounds__(kTableThreads) k_jp_tables(const struct j2p_je_img *__restrict__ imgs, const struct j2p_je_tables *__restrict__ t,
                                                            const struct j2p_jp_scanplan *__restrict__ scs, const uint64_t *__restrict__ hist,
                                                            struct j2p_jp_huff *__restrict__ huffs, uint8_t *__restrict__ heads,
                                                            uint32_t *__restrict__ hlens) {
    __shared__ struct j2p_jo_scratch scr[kTableThreads / 32];
    __shared__ struct j2p_jp_dht d;
    const uint32_t i = blockIdx.x, w = threadIdx.x >> 5, nc = t->nc;
    const uint32_t per = j2p_jp_nscans(nc), ntab = j2p_jp_ntables(nc);
    const WarpLanes L = {threadIdx.x & 31, 32};
    for (uint32_t tb = w; tb < ntab; tb += kTableThreads / 32) {
        const size_t tab = (size_t)i * ntab + tb;
        j2p_jp_table(hist + tab * 256, &scr[w], &d, &huffs[tab], tb, L);
    }
    __syncthreads();
    const struct j2p_je_tables *ts = t + imgs[i].set;
    for (uint32_t k = 0; k < per; k++) {
        const size_t q = (size_t)i * per + k;
        const uint32_t dri = scs[q].dri, len = j2p_jp_scan_head_len(ts, &d, k, dri);
        for (uint32_t b = threadIdx.x; b < len; b += kTableThreads) heads[q * J2P_JP_HEAD + b] = j2p_jp_scan_head_byte(ts, &imgs[i], &d, k, dri, b);
        if (threadIdx.x == 0) hlens[q] = len;
    }
}

// per tile: each block's bits, their exclusive scan in the tile, the tile's sum.  One body with the
// kind as a runtime flag: two specialised bodies would take more registers.
__global__ void __launch_bounds__(kTileThreads) k_jp_sizes(const Ctx x, uint32_t ns, const struct j2p_jp_huff *__restrict__ huffs,
                                                          uint32_t *__restrict__ intra, uint32_t *__restrict__ tsum) {
    typedef cub::BlockScan<uint32_t, kTileThreads> Scan;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ __align__(16) struct j2p_jp_huff sh[2];
    uint64_t j;
    const uint32_t s = tile_block(x.strs, ns, &j);
    const struct j2p_je_img *st = &x.strs[s];
    CountBits c = {stage(sh, huffs, x, s), 0};
    if (j < st->nblk) code_block(x, s, j, c);
    uint32_t excl, total;
    Scan(tmp).ExclusiveSum(c.n, excl, total);
    if (j < st->nblk) intra[st->blk0 + j] = excl;
    if (threadIdx.x == 0) tsum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanThreads) k_jp_scan(struct j2p_je_img *__restrict__ strs, const uint32_t *__restrict__ tsum,
                                                         uint64_t *__restrict__ toff, uint32_t *__restrict__ raw) {
    scan_body(strs, tsum, toff, raw);
}

__device__ __forceinline__ void emit_kind_body(const Ctx &x, uint32_t ns, const struct j2p_jp_huff *__restrict__ huffs,
                                               const uint32_t *__restrict__ intra, const uint64_t *__restrict__ toff, uint32_t *__restrict__ raw,
                                               struct j2p_jp_huff *sh) {
    uint64_t j;
    const uint32_t s = tile_block(x.strs, ns, &j);
    const struct j2p_je_img *st = &x.strs[s];
    const struct j2p_jp_huff *h = stage(sh, huffs, x, s);
    if (j >= st->nblk) return;
    uint32_t *rw = raw + st->raw_off;
    const uint64_t pos = toff[blockIdx.x] + intra[st->blk0 + j];
    const auto orw = [rw](uint64_t k, uint32_t v) { atomicOr(rw + k, v); };
    EmitBits<decltype(orw)> e = {h, {orw, 0, (uint32_t)(pos & 31), pos >> 5}, x, s};
    code_block(x, s, j, e);
    if (e.w.fill) orw(e.w.word, (uint32_t)(e.w.acc >> 32));
}

__global__ void __launch_bounds__(kTileThreads) k_jp_emit(const Ctx x, uint32_t ns, const struct j2p_jp_huff *__restrict__ huffs,
                                                         const uint32_t *__restrict__ intra, const uint64_t *__restrict__ toff,
                                                         uint32_t *__restrict__ raw) {
    __shared__ __align__(16) struct j2p_jp_huff sh[2];
    if (x.nc == 3) emit_kind_body(as_kind<3>(x), ns, huffs, intra, toff, raw, sh);
    else emit_kind_body(x, ns, huffs, intra, toff, raw, sh);
}

__global__ void __launch_bounds__(kChunkThreads) k_jp_ffcount(const struct j2p_je_img *__restrict__ strs, uint32_t ns,
                                                             const uint32_t *__restrict__ raw, uint32_t *__restrict__ ffc) {
    ffcount_body(strs, ns, raw, ffc);
}

template <uint32_t PER>
__device__ __forceinline__ void prog_offsets_body(struct j2p_je_img *__restrict__ strs, uint32_t ns, bool plain, uint32_t n,
                                                  const uint32_t *__restrict__ ffc, uint32_t nchunks, const uint32_t *__restrict__ hlens,
                                                  uint64_t *__restrict__ ffpre, uint64_t *__restrict__ offsets) {
    const StreamMap<PER> sm = {strs, ns, plain};
    offsets_body(strs, sm, n, ffc, nchunks, ffpre, offsets, [&](uint32_t s) { return hlens[sm.scan_index(s)]; });
}

__global__ void __launch_bounds__(kScanThreads) k_jp_offsets(struct j2p_je_img *__restrict__ strs, uint32_t ns, bool plain, uint32_t n,
                                                            const uint32_t *__restrict__ ffc, uint32_t nchunks, const uint32_t *__restrict__ hlens,
                                                            uint64_t *__restrict__ ffpre, uint64_t *__restrict__ offsets, uint32_t nc) {
    if (nc == 1) prog_offsets_body<J2P_JP_SCANS_GRAY>(strs, ns, plain, n, ffc, nchunks, hlens, ffpre, offsets);
    else if (nc == 4) prog_offsets_body<J2P_JP_SCANS_CMYK>(strs, ns, plain, n, ffc, nchunks, hlens, ffpre, offsets);
    else prog_offsets_body<J2P_JP_SCANS>(strs, ns, plain, n, ffc, nchunks, hlens, ffpre, offsets);
}

template <uint32_t PER>
__device__ __forceinline__ void prog_stuff_body(const struct j2p_je_img *__restrict__ strs, uint32_t ns, bool plain, const uint8_t *__restrict__ heads,
                                                const uint32_t *__restrict__ hlens, const uint32_t *__restrict__ raw,
                                                const uint64_t *__restrict__ ffpre, uint8_t *__restrict__ out) {
    const StreamMap<PER> sm = {strs, ns, plain};
    stuff_body(sm, raw, ffpre, out, [&](uint32_t s) { return hlens[sm.scan_index(s)]; },
               [&](uint32_t s, uint32_t k) { return heads[(size_t)sm.scan_index(s) * J2P_JP_HEAD + k]; });
}

__global__ void __launch_bounds__(kChunkThreads) k_jp_stuff(const struct j2p_je_img *__restrict__ strs, uint32_t ns, bool plain, const uint8_t *__restrict__ heads,
                                                           const uint32_t *__restrict__ hlens, const uint32_t *__restrict__ raw,
                                                           const uint64_t *__restrict__ ffpre, uint8_t *__restrict__ out, uint32_t nc) {
    if (nc == 1) prog_stuff_body<J2P_JP_SCANS_GRAY>(strs, ns, plain, heads, hlens, raw, ffpre, out);
    else if (nc == 4) prog_stuff_body<J2P_JP_SCANS_CMYK>(strs, ns, plain, heads, hlens, raw, ffpre, out);
    else prog_stuff_body<J2P_JP_SCANS>(strs, ns, plain, heads, hlens, raw, ffpre, out);
}

extern "C" int j2p_jpegprog_encode(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, void *work,
                                   size_t work_bytes, void *stream, uint64_t *offsets, void *dst, size_t dst_cap, struct j2p_jpegenc_stats *stats) {
    PLayout P;
    if (prog_plan(images, n, params, &P, nullptr) != 0) return -1;
    const auto fill = [&](uint8_t *plan) { return prog_plan(images, n, params, &P, plan); };
    const auto launch = [&](uint8_t *w, cudaStream_t st, const uint8_t *, auto counted) {
        struct j2p_je_img *imgs = (struct j2p_je_img *)(w + P.off_imgs), *strs = (struct j2p_je_img *)(w + P.off_str);
        const struct j2p_jp_scanplan *scs = (const struct j2p_jp_scanplan *)(w + P.off_scan);
        const struct j2p_je_tables *t = (const struct j2p_je_tables *)(w + P.off_tab);
        uint32_t *tsum = (uint32_t *)(w + P.off_tsum), *intra = (uint32_t *)(w + P.off_intra), *ffc = (uint32_t *)(w + P.off_ffc);
        uint32_t *state = (uint32_t *)(w + P.off_state), *raw = (uint32_t *)(w + P.off_raw), *hlens = (uint32_t *)(w + P.off_hlen);
        uint64_t *toff = (uint64_t *)(w + P.off_toff), *ffpre = (uint64_t *)(w + P.off_ffpre), *offs = (uint64_t *)(w + P.off_offs);
        uint64_t *hist = (uint64_t *)(w + P.off_hist);
        int16_t *coef = (int16_t *)(w + P.off_coef);
        uint8_t *summ = w + P.off_summ, *heads = w + P.off_head;
        struct j2p_jp_huff *huffs = (struct j2p_jp_huff *)(w + P.off_huff);
        const uint32_t nc = nc_of(params);
        const Ctx x = {imgs, strs, t, coef, summ, state, P.plain, nc};
        // the symbol counts and the entropy words, which follow them
        const cudaError_t em = cudaMemsetAsync(hist, 0, P.off_raw - P.off_hist + P.words * sizeof(uint32_t), st);
        if (em != cudaSuccess) return fail("clearing the symbol counts and entropy words: %s", cudaGetErrorString(em));
        const uint64_t bgrid = (P.nblk * 8 + kBlockThreads - 1) / kBlockThreads;
        k_jp_blocks<<<(unsigned)bgrid, kBlockThreads, 0, st>>>(imgs, n, t, P.nblk, coef, strs, scs, P.plain, summ, nc);
        counted();
        k_jp_runs<<<P.ntiles, kTileThreads, 0, st>>>(strs, P.ns, P.plain, summ, state, nc);
        counted();
        k_jp_hist<<<P.ntiles, kTileThreads, 0, st>>>(x, P.ns, (unsigned long long *)hist);
        counted();
        k_jp_tables<<<n, kTableThreads, 0, st>>>(imgs, t, scs, hist, huffs, heads, hlens);
        counted();
        k_jp_sizes<<<P.ntiles, kTileThreads, 0, st>>>(x, P.ns, huffs, intra, tsum);
        counted();
        k_jp_scan<<<P.ns, kScanThreads, 0, st>>>(strs, tsum, toff, raw);
        counted();
        k_jp_emit<<<P.ntiles, kTileThreads, 0, st>>>(x, P.ns, huffs, intra, toff, raw);
        counted();
        k_jp_ffcount<<<P.nchunks, kChunkThreads, 0, st>>>(strs, P.ns, raw, ffc);
        counted();
        k_jp_offsets<<<1, kScanThreads, 0, st>>>(strs, P.ns, P.plain, n, ffc, P.nchunks, hlens, ffpre, offs, nc);
        counted();
        k_jp_stuff<<<P.nchunks, kChunkThreads, 0, st>>>(strs, P.ns, P.plain, heads, hlens, raw, ffpre, w + P.off_out, nc);
        counted();
        return 0;
    };
    if (encode_call(images, n, P, P.off_tsum, work, work_bytes, stream, offsets, dst, dst_cap, stats, fill, launch) != 0) return -1;
    if (stats) stats->blocks = P.nblk;
    return 0;
}
