// jpegprog.cu — libj2pjpegprog.so: the device encoder of progressive JPEG files and the serial host
// driver of the same steps.  See jpegprog.h; the scans are in jpegprog_core.h, the steps shared with
// the other encoders in ../jpegenc (jpegenc_plan.h, jpegenc_kernels.cuh) and the table builder in
// ../jpegopt/jpegopt_core.h.
#include <vector>

#include "../jpegenc/jpegenc_kernels.cuh"
#include "jpegprog_core.h"

extern "C" const char *j2p_jpegprog_last_error(void) { return g_err; }

// ---- plan --------------------------------------------------------------------------------------
// Every (image, scan) pair is a stream, described by a j2p_je_img (the stuffing steps' view of a bit
// stream): blk0 and nblk its blocks among the call's stream blocks, its tiles, chunks, words, bits
// and place in the output.  Stream s is scan s % 10 of image s / 10.
// work: [images][tables][streams] [tile sums][tile offsets][block offsets in the tile][run states]
//       [summaries][coefficients][0xFF counts per chunk][their exclusive scan][offsets]
//       [derived tables][stream headers][their lengths][symbol counts][entropy words][files]
// The symbol counts sit just before the entropy words, so that one memset clears both.
struct PLayout {
    uint32_t n, ns, ntiles, nchunks;
    uint64_t nblk, nsblk, words;
    size_t off_imgs, off_tab, off_str, off_tsum, off_toff, off_intra, off_state, off_summ, off_coef, off_ffc, off_ffpre, off_offs,
        off_huff, off_head, off_hlen, off_hist, off_raw, off_out, total;
};

// The plan of a call; with w, also its plan region (images, tables, streams) at w.
static int prog_plan(const struct j2p_jpegenc_image *im, unsigned n, const struct j2p_jpegenc_params *p, PLayout *P, uint8_t *w) {
    Layout L;
    if (make_plan(im, n, p, 0, false, &L, nullptr) != 0) return -1;      // the argument checks
    const size_t ns = (size_t)n * J2P_JP_SCANS;
    size_t o = 0;
    P->off_imgs = o;  o = align16(o + n * sizeof(struct j2p_je_img));
    P->off_tab = o;   o = align16(o + sizeof(struct j2p_je_tables));
    P->off_str = o;   o = align16(o + ns * sizeof(struct j2p_je_img));
    std::vector<uint8_t> tmp;
    if (!w) {
        tmp.resize(o);
        w = tmp.data();
    }
    struct j2p_je_img *imgs = (struct j2p_je_img *)(w + P->off_imgs), *strs = (struct j2p_je_img *)(w + P->off_str);
    struct j2p_je_tables *t = (struct j2p_je_tables *)(w + P->off_tab);
    make_plan(im, n, p, 0, false, &L, imgs);
    make_tables(p, t);
    uint64_t sblk = 0, words = 0, tiles = 0, chunks = 0, out = 0;
    for (unsigned i = 0; i < n; i++) {
        for (uint32_t k = 0; k < J2P_JP_SCANS; k++) {
            const uint32_t comp = j2p_jp_scan_of(k).comp, wpb = j2p_jp_bound_words(k);
            const uint64_t nb = j2p_jp_is_ac(k) ? (uint64_t)j2p_jp_grid_w(&imgs[i], t, comp) * j2p_jp_grid_h(&imgs[i], t, comp) : imgs[i].nblk;
            const uint64_t nt = (nb + J2P_JE_TILE - 1) / J2P_JE_TILE, raw_bytes = nb * wpb * 4;
            const uint64_t nc = (raw_bytes + J2P_JE_CHUNK - 1) / J2P_JE_CHUNK;
            struct j2p_je_img *g = &strs[(size_t)i * J2P_JP_SCANS + k];
            *g = imgs[i];
            g->blk0 = sblk;
            g->nblk = nb;
            g->tile0 = (uint32_t)tiles;
            g->ntiles = (uint32_t)nt;
            g->chunk0 = (uint32_t)chunks;
            g->nchunks = (uint32_t)nc;
            g->raw_off = words;
            g->out_cap = J2P_JP_HEAD + 2 * raw_bytes + (k + 1 == J2P_JP_SCANS ? 2 : 0);
            sblk += nb;
            tiles += nt;
            chunks += nc;
            words += (nb * wpb + 3) / 4 * 4 + 4;   // raw_off stays a multiple of 4 words: chunk_bytes reads uint4
            out += g->out_cap;
        }
    }
    if (tiles >= 0x7fffffffu || chunks >= 0x7fffffffu) return fail("too many blocks for one call (%llu)", (unsigned long long)L.nblk);
    P->n = n;
    P->ns = (uint32_t)ns;
    P->nblk = L.nblk;
    P->nsblk = sblk;
    P->ntiles = (uint32_t)tiles;
    P->nchunks = (uint32_t)chunks;
    P->words = words;
    P->off_tsum = o;  o = align16(o + tiles * sizeof(uint32_t));
    P->off_toff = o;  o = align16(o + tiles * sizeof(uint64_t));
    P->off_intra = o; o = align16(o + sblk * sizeof(uint32_t));
    P->off_state = o; o = align16(o + sblk * sizeof(uint32_t));
    P->off_summ = o;  o = align16(o + sblk);
    P->off_coef = o;  o = align16(o + L.nblk * 64 * sizeof(int16_t));
    P->off_ffc = o;   o = align16(o + chunks * sizeof(uint32_t));
    P->off_ffpre = o; o = align16(o + (chunks + 1) * sizeof(uint64_t));
    P->off_offs = o;  o = align16(o + (n + 1) * sizeof(uint64_t));
    P->off_huff = o;  o = align16(o + (size_t)n * J2P_JP_TABLES * sizeof(struct j2p_jp_huff));
    P->off_head = o;  o = align16(o + ns * J2P_JP_HEAD);
    P->off_hlen = o;  o = align16(o + ns * sizeof(uint32_t));
    P->off_hist = o;  o = align16(o + (size_t)n * J2P_JP_TABLES * 256 * sizeof(uint64_t));
    P->off_raw = o;   o = align16(o + words * sizeof(uint32_t));
    P->off_out = o;   o = align16(o + out);
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
};

// the coefficients of block j of an AC scan over component comp of image im
J2P_HD const int16_t *ac_coef(const Ctx &x, const struct j2p_je_img *im, uint32_t comp, uint64_t j) {
    return x.coef + (im->blk0 + j2p_jp_stored(im, x.t, comp, j2p_jp_grid_w(im, x.t, comp), (uint32_t)j)) * 64;
}

// block j of stream s into o
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <class Out>
J2P_HD void code_block(const Ctx &x, uint32_t s, uint64_t j, Out &o) {
    const uint32_t k = s % J2P_JP_SCANS;
    const struct j2p_je_img *st = &x.strs[s], *im = &x.imgs[s / J2P_JP_SCANS];
    const struct j2p_jp_scan sc = j2p_jp_scan_of(k);
    const bool last = j + 1 == st->nblk;
    if (j2p_jp_is_ac(k))
        j2p_jp_code(sc, ac_coef(x, im, sc.comp, j), 0, sc.comp, x.state[st->blk0 + j], j, last, o);
    else
        j2p_jp_code(sc, x.coef + (im->blk0 + j) * 64, pred_of(x.t, x.coef, im->blk0, j), comp_of(x.t, j), 0, j, last, o);
}

// the summary of block j of AC stream s
J2P_HD uint32_t summary_of(const Ctx &x, uint32_t s, uint64_t j) {
    const struct j2p_jp_scan sc = j2p_jp_scan_of(s % J2P_JP_SCANS);
    return j2p_jp_summary(sc, ac_coef(x, &x.imgs[s / J2P_JP_SCANS], sc.comp, j));
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
        const struct j2p_jp_scan sc = j2p_jp_scan_of(s % J2P_JP_SCANS);
        const struct j2p_je_img *st = &x.strs[s], *im = &x.imgs[s / J2P_JP_SCANS];
        for (uint64_t q = first; q < first + run; q++)
            if (x.summ[st->blk0 + q] & 63u) j2p_jp_tail(sc, ac_coef(x, im, sc.comp, q), *this);
    }
};

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
    const struct j2p_je_tables *t = (const struct j2p_je_tables *)(w + P.off_tab);
    int16_t *coef = (int16_t *)(w + P.off_coef);
    uint8_t *summ = w + P.off_summ;
    uint32_t *state = (uint32_t *)(w + P.off_state), *raw = (uint32_t *)(w + P.off_raw), *hlens = (uint32_t *)(w + P.off_hlen);
    uint64_t *hist = (uint64_t *)(w + P.off_hist);
    struct j2p_jp_huff *huffs = (struct j2p_jp_huff *)(w + P.off_huff);
    uint8_t *heads = w + P.off_head, *out = w + P.off_out;
    memset(w + P.off_hist, 0, P.off_raw - P.off_hist + P.words * sizeof(uint32_t));
    const Ctx x = {imgs, strs, t, coef, summ, state};
    for (unsigned i = 0; i < n; i++) host_blocks(&imgs[i], t, coef);   // blocks
    for (uint32_t s = 0; s < P.ns; s++) {                               // summaries, runs
        if (!j2p_jp_is_ac(s % J2P_JP_SCANS)) continue;
        const struct j2p_je_img *st = &strs[s];
        for (uint64_t j = 0; j < st->nblk; j++) summ[st->blk0 + j] = (uint8_t)summary_of(x, s, j);
        for (uint64_t j = 0; j < st->nblk; j++)
            if (j == 0 || (summ[st->blk0 + j - 1] & J2P_JP_RESET))
                j2p_jp_walk(j, st->nblk, [&](uint64_t q) { return (uint32_t)summ[st->blk0 + q]; },
                            [&](uint64_t q, uint32_t v) { state[st->blk0 + q] = v; });
    }
    for (uint32_t s = 0; s < P.ns; s++) {                               // hist
        uint64_t *h = hist + ((size_t)(s / J2P_JP_SCANS) * J2P_JP_TABLES + j2p_jp_slot(s % J2P_JP_SCANS)) * 256;
        const auto count = [h](int tb, int v) { h[tb * 256 + v]++; };
        CountSymbols<decltype(count)> o = {count};
        for (uint64_t j = 0; j < strs[s].nblk; j++) code_block(x, s, j, o);
    }
    for (unsigned i = 0; i < n; i++) {                                  // tables, headers
        struct j2p_jo_scratch scr;
        struct j2p_jp_dht d;
        for (uint32_t tb = 0; tb < J2P_JP_TABLES; tb++)
            j2p_jp_table(hist + ((size_t)i * J2P_JP_TABLES + tb) * 256, &scr, &d, &huffs[(size_t)i * J2P_JP_TABLES + tb], tb, j2p_jo_serial());
        for (uint32_t k = 0; k < J2P_JP_SCANS; k++) {
            const size_t s = (size_t)i * J2P_JP_SCANS + k;
            hlens[s] = j2p_jp_head_len(&d, k);
            for (uint32_t b = 0; b < hlens[s]; b++) heads[s * J2P_JP_HEAD + b] = j2p_jp_head_byte(t, &imgs[i], &d, k, b);
        }
    }
    for (uint32_t s = 0; s < P.ns; s++) {                               // sizes, emit, padding
        struct j2p_je_img *st = &strs[s];
        const struct j2p_jp_huff *h = huffs + (size_t)(s / J2P_JP_SCANS) * J2P_JP_TABLES + j2p_jp_slot(s % J2P_JP_SCANS);
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
    for (unsigned i = 0; i < n; i++) {
        offsets[i] = (uint64_t)(o - out);
        for (uint32_t k = 0; k < J2P_JP_SCANS; k++) {
            const size_t s = (size_t)i * J2P_JP_SCANS + k;
            for (uint32_t b = 0; b < hlens[s]; b++) *o++ = heads[s * J2P_JP_HEAD + b];
            const uint32_t *rw = raw + strs[s].raw_off;
            for (uint64_t j = 0; j < raw_bytes(&strs[s]); j++) {
                const uint8_t v = j2p_je_byte(rw, j);
                *o++ = v;
                if (v == 0xff) *o++ = 0;
            }
        }
        *o++ = 0xff;
        *o++ = 0xd9;
    }
    offsets[n] = (uint64_t)(o - out);
    return 0;
}

// ---- device ------------------------------------------------------------------------------------
static const int kTableThreads = 32 * J2P_JP_TABLES;    // one warp per table of an image

// the derived tables of stream s (two for scan 0, one for an AC scan, none for the DC refine) into
// shared memory, by every thread of the CTA
__device__ __forceinline__ const struct j2p_jp_huff *stage(struct j2p_jp_huff *sh, const struct j2p_jp_huff *huffs, uint32_t s) {
    const uint32_t k = s % J2P_JP_SCANS, nt = k == 0 ? 2 : j2p_jp_is_ac(k) ? 1 : 0;
    const uint4 *src = (const uint4 *)(huffs + (size_t)(s / J2P_JP_SCANS) * J2P_JP_TABLES + j2p_jp_slot(k));
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

// kBlockThreads threads, 8 per block: the shared blocks body, then each real block's summary in
// each AC scan of its component (a lane per scan)
__global__ void __launch_bounds__(kBlockThreads) k_jp_blocks(const struct j2p_je_img *__restrict__ imgs, uint32_t n,
                                                            const struct j2p_je_tables *__restrict__ t, uint64_t nblk,
                                                            int16_t *__restrict__ coef, const struct j2p_je_img *__restrict__ strs,
                                                            uint8_t *__restrict__ summ) {
    blocks_body(imgs, n, t, nblk, coef);
    __syncthreads();
    const uint64_t g = ((uint64_t)blockIdx.x * kBlockThreads + threadIdx.x) >> 3;
    if (g >= nblk) return;
    const uint32_t i = find_image(imgs, n, g, 0);
    const struct j2p_je_img *im = &imgs[i];
    const struct j2p_je_where wh = j2p_je_locate(im, t, g - im->blk0);
    const int k = j2p_jp_comp_scan(wh.comp, threadIdx.x & 7);
    if (wh.dummy || k < 0) return;
    const uint64_t j = (uint64_t)wh.row * j2p_jp_grid_w(im, t, wh.comp) + wh.col;
    summ[strs[(size_t)i * J2P_JP_SCANS + k].blk0 + j] = (uint8_t)j2p_jp_summary(j2p_jp_scan_of((uint32_t)k), coef + g * 64);
}

// per block of an AC scan that starts a segment: the walk to the segment's end
__global__ void __launch_bounds__(kTileThreads) k_jp_runs(const struct j2p_je_img *__restrict__ strs, uint32_t ns,
                                                         const uint8_t *__restrict__ summ, uint32_t *__restrict__ state) {
    uint64_t j;
    const uint32_t s = tile_block(strs, ns, &j);
    const struct j2p_je_img *st = &strs[s];
    if (!j2p_jp_is_ac(s % J2P_JP_SCANS) || j >= st->nblk) return;
    const uint8_t *m = summ + st->blk0;
    if (j && !(m[j - 1] & J2P_JP_RESET)) return;
    uint32_t *out = state + st->blk0;
    j2p_jp_walk(j, st->nblk, [&](uint64_t q) { return (uint32_t)m[q]; }, [&](uint64_t q, uint32_t v) { out[q] = v; });
}

// per tile: the symbols of its blocks counted in shared memory, then added to the image's counts
__global__ void __launch_bounds__(kTileThreads) k_jp_hist(const Ctx x, uint32_t ns, unsigned long long *__restrict__ hist) {
    __shared__ uint32_t cnt[2 * 256];
    uint64_t j;
    const uint32_t s = tile_block(x.strs, ns, &j), k = s % J2P_JP_SCANS;
    if (k == 6) return;                                 // the DC refine has no symbols
    for (uint32_t q = threadIdx.x; q < 2 * 256; q += kTileThreads) cnt[q] = 0;
    __syncthreads();
    if (j < x.strs[s].nblk) {
        const auto count = [&](int tb, int v) { atomicAdd(&cnt[tb * 256 + v], 1u); };
        CountSymbols<decltype(count)> o = {count};
        code_block(x, s, j, o);
    }
    __syncthreads();
    unsigned long long *h = hist + ((size_t)(s / J2P_JP_SCANS) * J2P_JP_TABLES + j2p_jp_slot(k)) * 256;
    for (uint32_t q = threadIdx.x; q < 2 * 256; q += kTileThreads)
        if (cnt[q]) atomicAdd(h + q, (unsigned long long)cnt[q]);
}

// per image, a warp per table: code lengths, symbols and codes; then its streams' headers
__global__ void __launch_bounds__(kTableThreads) k_jp_tables(const struct j2p_je_img *__restrict__ imgs, const struct j2p_je_tables *__restrict__ t,
                                                            const uint64_t *__restrict__ hist, struct j2p_jp_huff *__restrict__ huffs,
                                                            uint8_t *__restrict__ heads, uint32_t *__restrict__ hlens) {
    __shared__ struct j2p_jo_scratch scr[J2P_JP_TABLES];
    __shared__ struct j2p_jp_dht d;
    const uint32_t i = blockIdx.x, tb = threadIdx.x >> 5;
    const WarpLanes L = {threadIdx.x & 31, 32};
    const size_t tab = (size_t)i * J2P_JP_TABLES + tb;
    j2p_jp_table(hist + tab * 256, &scr[tb], &d, &huffs[tab], tb, L);
    __syncthreads();
    for (uint32_t k = 0; k < J2P_JP_SCANS; k++) {
        const size_t s = (size_t)i * J2P_JP_SCANS + k;
        const uint32_t len = j2p_jp_head_len(&d, k);
        for (uint32_t b = threadIdx.x; b < len; b += kTableThreads) heads[s * J2P_JP_HEAD + b] = j2p_jp_head_byte(t, &imgs[i], &d, k, b);
        if (threadIdx.x == 0) hlens[s] = len;
    }
}

// per tile: each block's bits, their exclusive scan in the tile, the tile's sum
__global__ void __launch_bounds__(kTileThreads) k_jp_sizes(const Ctx x, uint32_t ns, const struct j2p_jp_huff *__restrict__ huffs,
                                                          uint32_t *__restrict__ intra, uint32_t *__restrict__ tsum) {
    typedef cub::BlockScan<uint32_t, kTileThreads> Scan;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ __align__(16) struct j2p_jp_huff sh[2];
    uint64_t j;
    const uint32_t s = tile_block(x.strs, ns, &j);
    const struct j2p_je_img *st = &x.strs[s];
    CountBits c = {stage(sh, huffs, s), 0};
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

__global__ void __launch_bounds__(kTileThreads) k_jp_emit(const Ctx x, uint32_t ns, const struct j2p_jp_huff *__restrict__ huffs,
                                                         const uint32_t *__restrict__ intra, const uint64_t *__restrict__ toff,
                                                         uint32_t *__restrict__ raw) {
    __shared__ __align__(16) struct j2p_jp_huff sh[2];
    uint64_t j;
    const uint32_t s = tile_block(x.strs, ns, &j);
    const struct j2p_je_img *st = &x.strs[s];
    const struct j2p_jp_huff *h = stage(sh, huffs, s);
    if (j >= st->nblk) return;
    uint32_t *rw = raw + st->raw_off;
    const uint64_t pos = toff[blockIdx.x] + intra[st->blk0 + j];
    const auto orw = [rw](uint64_t k, uint32_t v) { atomicOr(rw + k, v); };
    EmitBits<decltype(orw)> e = {h, {orw, 0, (uint32_t)(pos & 31), pos >> 5}, x, s};
    code_block(x, s, j, e);
    if (e.w.fill) orw(e.w.word, (uint32_t)(e.w.acc >> 32));
}

__global__ void __launch_bounds__(kChunkThreads) k_jp_ffcount(const struct j2p_je_img *__restrict__ strs, uint32_t ns,
                                                             const uint32_t *__restrict__ raw, uint32_t *__restrict__ ffc) {
    ffcount_body(strs, ns, raw, ffc);
}

// one CTA: the scan of the 0xFF counts over the call, then each stream's place in the output (its
// header, its stuffed bytes and, after an image's last scan, EOI) and each file's offset
__global__ void __launch_bounds__(kScanThreads) k_jp_offsets(struct j2p_je_img *__restrict__ strs, uint32_t ns, uint32_t n,
                                                            const uint32_t *__restrict__ ffc, uint32_t nchunks, const uint32_t *__restrict__ hlens,
                                                            uint64_t *__restrict__ ffpre, uint64_t *__restrict__ offsets) {
    __shared__ typename ScanU64::TempStorage tmp;
    const uint64_t ff = scan_segment(nchunks, [&](uint32_t k) { return (uint64_t)ffc[k]; }, [&](uint32_t k, uint64_t v) { ffpre[k] = v; }, tmp);
    if (threadIdx.x == 0) ffpre[nchunks] = ff;
    __syncthreads();
    const uint64_t base = scan_segment(
        ns,
        [&](uint32_t s) {
            const struct j2p_je_img *st = &strs[s];
            return hlens[s] + raw_bytes(st) + (ffpre[st->chunk0 + st->nchunks] - ffpre[st->chunk0]) + (s % J2P_JP_SCANS == J2P_JP_SCANS - 1 ? 2 : 0);
        },
        [&](uint32_t s, uint64_t v) { strs[s].file_off = v; }, tmp);
    __syncthreads();
    for (uint32_t s = threadIdx.x; s < ns; s += kScanThreads) strs[s].file_len = (s + 1 < ns ? strs[s + 1].file_off : base) - strs[s].file_off;
    for (uint32_t i = threadIdx.x; i < n; i += kScanThreads) offsets[i] = strs[(size_t)i * J2P_JP_SCANS].file_off;
    if (threadIdx.x == 0) offsets[n] = base;
}

// per chunk: its bytes into the output with a 0x00 after each 0xFF; a stream's first chunk also
// writes its header, the chunk holding an image's last byte the EOI
__global__ void __launch_bounds__(kChunkThreads) k_jp_stuff(const struct j2p_je_img *__restrict__ strs, uint32_t ns,
                                                           const uint8_t *__restrict__ heads, const uint32_t *__restrict__ hlens,
                                                           const uint32_t *__restrict__ raw, const uint64_t *__restrict__ ffpre,
                                                           uint8_t *__restrict__ out) {
    typedef cub::BlockScan<uint32_t, kChunkThreads> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const uint32_t s = find_image(strs, ns, blockIdx.x, 2);
    const struct j2p_je_img *st = &strs[s];
    const uint32_t c = blockIdx.x - st->chunk0, hl = hlens[s];
    const uint64_t nbytes = raw_bytes(st);
    if ((uint64_t)c * J2P_JE_CHUNK >= nbytes) return;
    uint8_t *o0 = out + st->file_off;
    if (c == 0)
        for (uint32_t b = threadIdx.x; b < hl; b += kChunkThreads) o0[b] = heads[(size_t)s * J2P_JP_HEAD + b];
    if (threadIdx.x == 0 && s % J2P_JP_SCANS == J2P_JP_SCANS - 1 && (uint64_t)(c + 1) * J2P_JE_CHUNK >= nbytes) {
        o0[st->file_len - 2] = 0xff;
        o0[st->file_len - 1] = 0xd9;
    }
    uint64_t j0;
    uint32_t cnt;
    uint4 v;
    const uint32_t m = chunk_bytes(st, raw, c, &j0, &cnt, &v);
    uint32_t before;
    Scan(tmp).ExclusiveSum(cnt, before);
    uint8_t *o = o0 + hl + j0 + (ffpre[blockIdx.x] - ffpre[st->chunk0]) + before;
    const uint32_t wv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int q = 0; q < 16; q++) {
        if ((uint32_t)q >= m) break;
        const uint8_t b = (uint8_t)(wv[q >> 2] >> (24 - 8 * (q & 3)));
        *o++ = b;
        if (b == 0xff) *o++ = 0;
    }
}

extern "C" int j2p_jpegprog_encode(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, void *work,
                                   size_t work_bytes, void *stream, uint64_t *offsets, void *dst, size_t dst_cap, struct j2p_jpegenc_stats *stats) {
    PLayout P;
    if (prog_plan(images, n, params, &P, nullptr) != 0) return -1;
    const auto fill = [&](uint8_t *plan) { return prog_plan(images, n, params, &P, plan); };
    const auto launch = [&](uint8_t *w, cudaStream_t st, const uint8_t *, auto counted) {
        struct j2p_je_img *imgs = (struct j2p_je_img *)(w + P.off_imgs), *strs = (struct j2p_je_img *)(w + P.off_str);
        const struct j2p_je_tables *t = (const struct j2p_je_tables *)(w + P.off_tab);
        uint32_t *tsum = (uint32_t *)(w + P.off_tsum), *intra = (uint32_t *)(w + P.off_intra), *ffc = (uint32_t *)(w + P.off_ffc);
        uint32_t *state = (uint32_t *)(w + P.off_state), *raw = (uint32_t *)(w + P.off_raw), *hlens = (uint32_t *)(w + P.off_hlen);
        uint64_t *toff = (uint64_t *)(w + P.off_toff), *ffpre = (uint64_t *)(w + P.off_ffpre), *offs = (uint64_t *)(w + P.off_offs);
        uint64_t *hist = (uint64_t *)(w + P.off_hist);
        int16_t *coef = (int16_t *)(w + P.off_coef);
        uint8_t *summ = w + P.off_summ, *heads = w + P.off_head;
        struct j2p_jp_huff *huffs = (struct j2p_jp_huff *)(w + P.off_huff);
        const Ctx x = {imgs, strs, t, coef, summ, state};
        // the symbol counts and the entropy words, which follow them
        const cudaError_t em = cudaMemsetAsync(hist, 0, P.off_raw - P.off_hist + P.words * sizeof(uint32_t), st);
        if (em != cudaSuccess) return fail("clearing the symbol counts and entropy words: %s", cudaGetErrorString(em));
        const uint64_t bgrid = (P.nblk * 8 + kBlockThreads - 1) / kBlockThreads;
        k_jp_blocks<<<(unsigned)bgrid, kBlockThreads, 0, st>>>(imgs, n, t, P.nblk, coef, strs, summ);
        counted();
        k_jp_runs<<<P.ntiles, kTileThreads, 0, st>>>(strs, P.ns, summ, state);
        counted();
        k_jp_hist<<<P.ntiles, kTileThreads, 0, st>>>(x, P.ns, (unsigned long long *)hist);
        counted();
        k_jp_tables<<<n, kTableThreads, 0, st>>>(imgs, t, hist, huffs, heads, hlens);
        counted();
        k_jp_sizes<<<P.ntiles, kTileThreads, 0, st>>>(x, P.ns, huffs, intra, tsum);
        counted();
        k_jp_scan<<<P.ns, kScanThreads, 0, st>>>(strs, tsum, toff, raw);
        counted();
        k_jp_emit<<<P.ntiles, kTileThreads, 0, st>>>(x, P.ns, huffs, intra, toff, raw);
        counted();
        k_jp_ffcount<<<P.nchunks, kChunkThreads, 0, st>>>(strs, P.ns, raw, ffc);
        counted();
        k_jp_offsets<<<1, kScanThreads, 0, st>>>(strs, P.ns, n, ffc, P.nchunks, hlens, ffpre, offs);
        counted();
        k_jp_stuff<<<P.nchunks, kChunkThreads, 0, st>>>(strs, P.ns, heads, hlens, raw, ffpre, w + P.off_out);
        counted();
        return 0;
    };
    if (encode_call(images, n, P, P.off_tsum, work, work_bytes, stream, offsets, dst, dst_cap, stats, fill, launch) != 0) return -1;
    if (stats) stats->blocks = P.nblk;
    return 0;
}
