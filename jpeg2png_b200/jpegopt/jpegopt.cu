// jpegopt.cu — libj2pjpegopt.so: the device encoder of optimized JPEG files and the serial host
// driver of the same steps.  See jpegopt.h; the steps it shares with libj2pjpegenc.so are in
// ../jpegenc (jpegenc_plan.h, jpegenc_kernels.cuh, jpegenc_core.h), the table builder in
// jpegopt_core.h.
#include "../jpegenc/jpegenc_kernels.cuh"
#include "jpegopt.h"
#include "jpegopt_core.h"

#define J2P_JO_WORDS_PER_BLOCK 53u      // 32-bit words of J2P_JPEGOPT_BLOCK_BITS, rounded up
static_assert(J2P_JO_WORDS_PER_BLOCK * 32 >= J2P_JPEGOPT_BLOCK_BITS && (J2P_JO_WORDS_PER_BLOCK - 1) * 32 < J2P_JPEGOPT_BLOCK_BITS,
              "J2P_JO_WORDS_PER_BLOCK is J2P_JPEGOPT_BLOCK_BITS in words");

extern "C" const char *j2p_jpegopt_last_error(void) { return g_err; }

extern "C" int j2p_jpegopt_plan(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, size_t *work_bytes,
                                size_t *out_offset) {
    Layout L;
    if (make_plan(images, n, params, J2P_JO_WORDS_PER_BLOCK, true, &L, nullptr) != 0) return -1;
    if (work_bytes) *work_bytes = L.total;
    if (out_offset) *out_offset = L.off_out;
    return 0;
}

extern "C" int j2p_jpegopt_build_table(const uint64_t *counts, uint8_t *bits, uint8_t *vals, unsigned *nvals) {
    if (!counts || !bits || !vals || !nvals) return fail("null argument");
    bool any = false;
    for (int k = 0; k < 256; k++) any |= counts[k] != 0;
    if (!any) return fail("a table needs at least one symbol");
    struct j2p_jo_scratch s;
    *nvals = j2p_jo_build(counts, &s, bits, vals, j2p_jo_serial());
    return 0;
}

// ---- host driver -------------------------------------------------------------------------------
// the length and byte k of stream st's header: its image's own header (with its length in hlens), or RST
J2P_HD uint32_t own_head_len(const uint32_t *hlens, const struct j2p_je_img *st) { return st->part ? J2P_JE_RST : hlens[st->img]; }

J2P_HD uint8_t own_head_byte(const uint8_t *heads, const struct j2p_je_img *st, uint32_t k) {
    return j2p_je_stream_byte(st, k, [&](uint32_t k1) { return heads[(size_t)st->img * J2P_JE_HEAD_ROOM + k1]; });
}

// each image's own tables and header, in the work area
struct OwnCodes {
    const struct j2p_je_huff *huffs;
    const uint8_t *heads;
    const uint32_t *hlens;
    const struct j2p_je_huff *huff(uint32_t i) const { return &huffs[i]; }
    uint32_t head_len(const struct j2p_je_img *st) const { return own_head_len(hlens, st); }
    uint8_t head_byte(const struct j2p_je_img *st, uint32_t k) const { return own_head_byte(heads, st, k); }
};

extern "C" int j2p_jpegopt_encode_host(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, void *work,
                                       size_t work_bytes, uint64_t *offsets) {
    const auto codes = [n](const Layout &L, uint8_t *w, const struct j2p_je_img *imgs, const struct j2p_je_img *strs, const struct j2p_je_tables *t,
                           const int16_t *coef) {
        uint64_t *hist = (uint64_t *)(w + L.off_hist);
        struct j2p_je_huff *huffs = (struct j2p_je_huff *)(w + L.off_huff);
        uint8_t *heads = w + L.off_head;
        uint32_t *hlens = (uint32_t *)(w + L.off_hlen);
        for (uint32_t s = 0; s < L.ns; s++) {                           // hist: the DC predictions restart with each stream
            const struct j2p_je_img *st = &strs[s];
            uint64_t *h = hist + (size_t)st->img * 4 * J2P_JE_SYMBOLS;
            for (uint64_t b = 0; b < st->nblk; b++)
                j2p_je_symbols(coef + (st->blk0 + b) * 64, pred_of(t, coef, st->blk0, b), htab_of(t, b),
                               [&](int tb, int v) { h[tb * J2P_JE_SYMBOLS + v]++; }, [](uint32_t, int) {});
        }
        for (unsigned i = 0; i < n; i++) {                              // tables
            const struct j2p_je_img *im = &imgs[i];
            const uint64_t *h = hist + (size_t)i * 4 * J2P_JE_SYMBOLS;
            struct j2p_jo_scratch s;
            struct j2p_jo_dht d;
            for (int tb = 0; tb < (int)j2p_jo_ntables(t); tb++) j2p_jo_table(h + tb * J2P_JE_SYMBOLS, &s, &d, &huffs[i], tb, j2p_jo_serial());
            const struct j2p_je_tables *ts = t + im->set;
            hlens[i] = j2p_jo_file_head_len(ts, im, &d);
            for (uint32_t k = 0; k < hlens[i]; k++) heads[(size_t)i * J2P_JE_HEAD_ROOM + k] = j2p_jo_file_head_byte(ts, im, &d, k);
        }
        return OwnCodes{huffs, heads, hlens};
    };
    return encode_host_steps(images, n, params, J2P_JO_WORDS_PER_BLOCK, true, work, work_bytes, offsets, codes);
}

// ---- device ------------------------------------------------------------------------------------
static const int kTableThreads = 128;       // one warp per table of an image

// image i's derived tables into shared memory, by every thread of the CTA
__device__ __forceinline__ const struct j2p_je_huff *stage(struct j2p_je_huff *sh, const struct j2p_je_huff *huffs, uint32_t i) {
    const uint4 *src = (const uint4 *)(huffs + i);
    uint4 *dst = (uint4 *)sh;
    for (uint32_t k = threadIdx.x; k < sizeof(struct j2p_je_huff) / 16; k += blockDim.x) dst[k] = src[k];
    __syncthreads();
    return sh;
}

__global__ void __launch_bounds__(kBlockThreads) k_jo_blocks(const struct j2p_je_img *__restrict__ imgs, uint32_t n,
                                                            const struct j2p_je_tables *__restrict__ t, uint64_t nblk,
                                                            int16_t *__restrict__ coef) {
    blocks_body(imgs, n, t, nblk, coef);
}

// per tile: the symbols of its blocks counted in shared memory, then added to the image's counts
__global__ void __launch_bounds__(kTileThreads) k_jo_hist(const struct j2p_je_img *__restrict__ strs, uint32_t ns, bool plain,
                                                         const struct j2p_je_tables *__restrict__ t, const int16_t *__restrict__ coef,
                                                         unsigned long long *__restrict__ hist) {
    const StreamMap<1> sm = {strs, ns, plain};
    __shared__ uint32_t cnt[4 * J2P_JE_SYMBOLS];
    for (uint32_t k = threadIdx.x; k < 4 * J2P_JE_SYMBOLS; k += kTileThreads) cnt[k] = 0;
    __syncthreads();
    const uint32_t tile = blockIdx.x;
    const uint32_t s = find_image(sm.strs, sm.ns, tile, 1), i = sm.img(s);
    const struct j2p_je_img *im = &sm.strs[s];
    const uint64_t b = (uint64_t)(tile - im->tile0) * J2P_JE_TILE + threadIdx.x;
    const uint64_t blk0 = im->blk0;
    if (b < im->nblk)
        j2p_je_symbols(coef + (blk0 + b) * 64, pred_of(t, coef, blk0, b), htab_of(t, b),
                       [&](int tb, int s) { atomicAdd(&cnt[tb * J2P_JE_SYMBOLS + s], 1u); }, [](uint32_t, int) {});
    __syncthreads();
    unsigned long long *h = hist + (size_t)i * 4 * J2P_JE_SYMBOLS;
    for (uint32_t k = threadIdx.x; k < 4 * J2P_JE_SYMBOLS; k += kTileThreads)
        if (cnt[k]) atomicAdd(h + k, (unsigned long long)cnt[k]);
}

// per image, a warp per table: code lengths, symbols and codes; then the image's header (from its
// set's template) and its length.  A gray or CMYK image's warps 2 and 3 have no table (its chroma
// counts are all 0).
__global__ void __launch_bounds__(kTableThreads) k_jo_tables(const struct j2p_je_img *__restrict__ imgs, const struct j2p_je_tables *__restrict__ t,
                                                            const uint64_t *__restrict__ hist, struct j2p_je_huff *__restrict__ huffs,
                                                            uint8_t *__restrict__ heads, uint32_t *__restrict__ hlens) {
    __shared__ struct j2p_jo_scratch scr[kTableThreads / 32];
    __shared__ struct j2p_jo_dht d;
    const uint32_t i = blockIdx.x, tb = threadIdx.x >> 5;
    const WarpLanes L = {threadIdx.x & 31, 32};
    if (tb < j2p_jo_ntables(t)) j2p_jo_table(hist + ((size_t)i * 4 + tb) * J2P_JE_SYMBOLS, &scr[tb], &d, &huffs[i], (int)tb, L);
    __syncthreads();
    const struct j2p_je_tables *ts = t + imgs[i].set;
    const uint32_t len = j2p_jo_file_head_len(ts, &imgs[i], &d);
    for (uint32_t k = threadIdx.x; k < len; k += kTableThreads) heads[(size_t)i * J2P_JE_HEAD_ROOM + k] = j2p_jo_file_head_byte(ts, &imgs[i], &d, k);
    if (threadIdx.x == 0) hlens[i] = len;
}

__global__ void __launch_bounds__(kTileThreads) k_jo_sizes(const struct j2p_je_img *__restrict__ strs, uint32_t ns, bool plain,
                                                          const struct j2p_je_tables *__restrict__ t, const int16_t *__restrict__ coef,
                                                          const struct j2p_je_huff *__restrict__ huffs, uint32_t *__restrict__ intra,
                                                          uint32_t *__restrict__ tsum) {
    const StreamMap<1> sm = {strs, ns, plain};
    __shared__ __align__(16) struct j2p_je_huff sh;
    sizes_body(sm, t, coef, intra, tsum, [&](uint32_t i) { return stage(&sh, huffs, i); });
}

__global__ void __launch_bounds__(kScanThreads) k_jo_scan(struct j2p_je_img *__restrict__ strs, const uint32_t *__restrict__ tsum,
                                                         uint64_t *__restrict__ toff, uint32_t *__restrict__ raw) {
    scan_body(strs, tsum, toff, raw);
}

__global__ void __launch_bounds__(kTileThreads) k_jo_emit(const struct j2p_je_img *__restrict__ strs, uint32_t ns, bool plain,
                                                         const struct j2p_je_tables *__restrict__ t, const int16_t *__restrict__ coef,
                                                         const struct j2p_je_huff *__restrict__ huffs, const uint32_t *__restrict__ intra,
                                                         const uint64_t *__restrict__ toff, uint32_t *__restrict__ raw) {
    const StreamMap<1> sm = {strs, ns, plain};
    __shared__ __align__(16) struct j2p_je_huff sh;
    emit_body(sm.strs, sm.ns, t, coef, intra, toff, raw, stage(&sh, huffs, sm.img(find_image(sm.strs, sm.ns, blockIdx.x, 1))));
}

__global__ void __launch_bounds__(kChunkThreads) k_jo_ffcount(const struct j2p_je_img *__restrict__ strs, uint32_t ns,
                                                             const uint32_t *__restrict__ raw, uint32_t *__restrict__ ffc) {
    ffcount_body(strs, ns, raw, ffc);
}

__global__ void __launch_bounds__(kScanThreads) k_jo_offsets(struct j2p_je_img *__restrict__ strs, uint32_t ns, bool plain, uint32_t n,
                                                            const uint32_t *__restrict__ ffc, uint32_t nchunks, const uint32_t *__restrict__ hlens,
                                                            uint64_t *__restrict__ ffpre, uint64_t *__restrict__ offsets) {
    const StreamMap<1> sm = {strs, ns, plain};
    offsets_body(strs, sm, n, ffc, nchunks, ffpre, offsets, [&](uint32_t s) { return hlens[sm.img(s)]; });
}

__global__ void __launch_bounds__(kChunkThreads) k_jo_stuff(const struct j2p_je_img *__restrict__ strs, uint32_t ns, bool plain,
                                                           const uint8_t *__restrict__ heads, const uint32_t *__restrict__ hlens,
                                                           const uint32_t *__restrict__ raw, const uint64_t *__restrict__ ffpre,
                                                           uint8_t *__restrict__ out) {
    const StreamMap<1> sm = {strs, ns, plain};
    stuff_body(sm, raw, ffpre, out, [&](uint32_t s) { return hlens[sm.img(s)]; },
               [&](uint32_t s, uint32_t k) { return heads[(size_t)sm.img(s) * J2P_JE_HEAD_ROOM + k]; });
}

extern "C" int j2p_jpegopt_encode(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, void *work,
                                  size_t work_bytes, void *stream, uint64_t *offsets, void *dst, size_t dst_cap, struct j2p_jpegenc_stats *stats) {
    Layout L;
    if (make_plan(images, n, params, J2P_JO_WORDS_PER_BLOCK, true, &L, nullptr) != 0) return -1;
    const auto fill = [&](uint8_t *plan) { return fill_plan(images, n, params, J2P_JO_WORDS_PER_BLOCK, true, L, plan); };
    const auto launch = [&](uint8_t *w, cudaStream_t st, const uint8_t *, auto counted) {
        struct j2p_je_img *imgs = (struct j2p_je_img *)(w + L.off_imgs), *strs = (struct j2p_je_img *)(w + L.off_strs);
        const struct j2p_je_tables *t = (const struct j2p_je_tables *)(w + L.off_tab);
        uint32_t *tsum = (uint32_t *)(w + L.off_tsum), *intra = (uint32_t *)(w + L.off_intra), *ffc = (uint32_t *)(w + L.off_ffc);
        uint64_t *toff = (uint64_t *)(w + L.off_toff), *ffpre = (uint64_t *)(w + L.off_ffpre), *offs = (uint64_t *)(w + L.off_offs);
        int16_t *coef = (int16_t *)(w + L.off_coef);
        uint32_t *raw = (uint32_t *)(w + L.off_raw);
        uint64_t *hist = (uint64_t *)(w + L.off_hist);
        struct j2p_je_huff *huffs = (struct j2p_je_huff *)(w + L.off_huff);
        uint8_t *heads = w + L.off_head;
        uint32_t *hlens = (uint32_t *)(w + L.off_hlen);
        // the symbol counts and the entropy words, which follow them
        const cudaError_t em = cudaMemsetAsync(hist, 0, L.off_raw - L.off_hist + L.words * sizeof(uint32_t), st);
        if (em != cudaSuccess) return fail("clearing the symbol counts and entropy words: %s", cudaGetErrorString(em));
        const uint64_t bgrid = (L.nblk * 8 + kBlockThreads - 1) / kBlockThreads;
        k_jo_blocks<<<(unsigned)bgrid, kBlockThreads, 0, st>>>(imgs, n, t, L.nblk, coef);
        counted();
        k_jo_hist<<<L.ntiles, kTileThreads, 0, st>>>(strs, L.ns, L.plain, t, coef, (unsigned long long *)hist);
        counted();
        k_jo_tables<<<n, kTableThreads, 0, st>>>(imgs, t, hist, huffs, heads, hlens);
        counted();
        k_jo_sizes<<<L.ntiles, kTileThreads, 0, st>>>(strs, L.ns, L.plain, t, coef, huffs, intra, tsum);
        counted();
        k_jo_scan<<<L.ns, kScanThreads, 0, st>>>(strs, tsum, toff, raw);
        counted();
        k_jo_emit<<<L.ntiles, kTileThreads, 0, st>>>(strs, L.ns, L.plain, t, coef, huffs, intra, toff, raw);
        counted();
        k_jo_ffcount<<<L.nchunks, kChunkThreads, 0, st>>>(strs, L.ns, raw, ffc);
        counted();
        k_jo_offsets<<<1, kScanThreads, 0, st>>>(strs, L.ns, L.plain, n, ffc, L.nchunks, hlens, ffpre, offs);
        counted();
        k_jo_stuff<<<L.nchunks, kChunkThreads, 0, st>>>(strs, L.ns, L.plain, heads, hlens, raw, ffpre, w + L.off_out);
        counted();
        return 0;
    };
    if (encode_call(images, n, L, L.off_tsum, work, work_bytes, stream, offsets, dst, dst_cap, stats, fill, launch) != 0) return -1;
    if (stats) stats->blocks = L.nblk;
    return 0;
}
