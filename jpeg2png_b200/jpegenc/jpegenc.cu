// jpegenc.cu — libj2pjpegenc.so: the device encoder (blocks, sizes, scans, emit, stuffing) and the
// serial host driver of the same steps, with the Annex K Huffman tables.  The plan, the kernel bodies
// and the host driver are shared with libj2pjpegopt.so: jpegenc_plan.h, jpegenc_kernels.cuh and
// jpegenc_core.h.
#include "jpegenc_kernels.cuh"

extern "C" const char *j2p_jpegenc_last_error(void) { return g_err; }

extern "C" int j2p_jpegenc_plan(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, size_t *work_bytes,
                                size_t *out_offset) {
    Layout L;
    if (make_plan(images, n, params, J2P_JE_WORDS_PER_BLOCK, false, &L, nullptr) != 0) return -1;
    if (work_bytes) *work_bytes = L.total;
    if (out_offset) *out_offset = L.off_out;
    return 0;
}

// ---- host driver -------------------------------------------------------------------------------
extern "C" int j2p_jpegenc_encode_host(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, void *work,
                                       size_t work_bytes, uint64_t *offsets) {
    return encode_host_steps(images, n, params, J2P_JE_WORDS_PER_BLOCK, false, work, work_bytes, offsets,
                             [](const Layout &, uint8_t *, const struct j2p_je_img *, const struct j2p_je_img *, const struct j2p_je_tables *t,
                                const int16_t *) {
                                 return FixedCodes{t};
                             });
}

// ---- device ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlockThreads) k_je_blocks(const struct j2p_je_img *__restrict__ imgs, uint32_t n,
                                                            const struct j2p_je_tables *__restrict__ t, uint64_t nblk,
                                                            int16_t *__restrict__ coef) {
    blocks_body(imgs, n, t, nblk, coef);
}

__global__ void __launch_bounds__(kTileThreads) k_je_sizes(const struct j2p_je_img *__restrict__ strs, uint32_t ns, bool plain, const struct j2p_je_tables *__restrict__ t,
                                                          const int16_t *__restrict__ coef, uint32_t *__restrict__ intra,
                                                          uint32_t *__restrict__ tsum) {
    const StreamMap<1> sm = {strs, ns, plain};
    sizes_body(sm, t, coef, intra, tsum, [&](uint32_t) { return &t->huff; });
}

__global__ void __launch_bounds__(kScanThreads) k_je_scan(struct j2p_je_img *__restrict__ strs, const uint32_t *__restrict__ tsum,
                                                         uint64_t *__restrict__ toff, uint32_t *__restrict__ raw) {
    scan_body(strs, tsum, toff, raw);
}

__global__ void __launch_bounds__(kTileThreads) k_je_emit(const struct j2p_je_img *__restrict__ strs, uint32_t ns,
                                                         const struct j2p_je_tables *__restrict__ t, const int16_t *__restrict__ coef,
                                                         const uint32_t *__restrict__ intra, const uint64_t *__restrict__ toff,
                                                         uint32_t *__restrict__ raw) {
    emit_body(strs, ns, t, coef, intra, toff, raw, &t->huff);
}

__global__ void __launch_bounds__(kChunkThreads) k_je_ffcount(const struct j2p_je_img *__restrict__ strs, uint32_t ns,
                                                             const uint32_t *__restrict__ raw, uint32_t *__restrict__ ffc) {
    ffcount_body(strs, ns, raw, ffc);
}

// the scan header's length: its image's template (t: the call's sets), with DRI when the image has
// restart intervals
__device__ __forceinline__ uint32_t fixed_head_len(const StreamMap<1> &sm, const struct j2p_je_tables *t, uint32_t s) {
    const struct j2p_je_img *st = &sm.strs[s];
    return t[st->set].head_len + (!sm.plain && st->ri ? J2P_JE_DRI : 0);
}

__global__ void __launch_bounds__(kScanThreads) k_je_offsets(struct j2p_je_img *__restrict__ strs, uint32_t ns, bool plain, uint32_t n,
                                                            const uint32_t *__restrict__ ffc, uint32_t nchunks, uint64_t *__restrict__ ffpre,
                                                            uint64_t *__restrict__ offsets, const struct j2p_je_tables *__restrict__ t) {
    const StreamMap<1> sm = {strs, ns, plain};
    offsets_body(strs, sm, n, ffc, nchunks, ffpre, offsets, [&](uint32_t s) { return fixed_head_len(sm, t, s); });
}

__global__ void __launch_bounds__(kChunkThreads) k_je_stuff(const struct j2p_je_img *__restrict__ strs, uint32_t ns, bool plain, const struct j2p_je_tables *__restrict__ t,
                                                           const uint32_t *__restrict__ raw, const uint64_t *__restrict__ ffpre,
                                                           uint8_t *__restrict__ out) {
    const StreamMap<1> sm = {strs, ns, plain};
    stuff_body(sm, raw, ffpre, out, [&](uint32_t s) { return fixed_head_len(sm, t, s); }, [&](uint32_t s, uint32_t k) {
        const struct j2p_je_img *st = &sm.strs[s];
        return sm.plain ? j2p_je_head_byte(t + st->set, st, k) : j2p_je_scan_head_byte(t + st->set, st, k);
    });
}

extern "C" int j2p_jpegenc_encode(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, void *work,
                                  size_t work_bytes, void *stream, uint64_t *offsets, void *dst, size_t dst_cap, struct j2p_jpegenc_stats *stats) {
    Layout L;
    if (make_plan(images, n, params, J2P_JE_WORDS_PER_BLOCK, false, &L, nullptr) != 0) return -1;
    const auto fill = [&](uint8_t *plan) { return fill_plan(images, n, params, J2P_JE_WORDS_PER_BLOCK, false, L, plan); };
    const auto launch = [&](uint8_t *w, cudaStream_t st, const uint8_t *, auto counted) {
        struct j2p_je_img *imgs = (struct j2p_je_img *)(w + L.off_imgs), *strs = (struct j2p_je_img *)(w + L.off_strs);
        const struct j2p_je_tables *t = (const struct j2p_je_tables *)(w + L.off_tab);
        uint32_t *tsum = (uint32_t *)(w + L.off_tsum), *intra = (uint32_t *)(w + L.off_intra), *ffc = (uint32_t *)(w + L.off_ffc);
        uint64_t *toff = (uint64_t *)(w + L.off_toff), *ffpre = (uint64_t *)(w + L.off_ffpre), *offs = (uint64_t *)(w + L.off_offs);
        int16_t *coef = (int16_t *)(w + L.off_coef);
        uint32_t *raw = (uint32_t *)(w + L.off_raw);
        const cudaError_t em = cudaMemsetAsync(raw, 0, L.words * sizeof(uint32_t), st);
        if (em != cudaSuccess) return fail("clearing the entropy words: %s", cudaGetErrorString(em));
        const uint64_t bgrid = (L.nblk * 8 + kBlockThreads - 1) / kBlockThreads;
        k_je_blocks<<<(unsigned)bgrid, kBlockThreads, 0, st>>>(imgs, n, t, L.nblk, coef);
        counted();
        k_je_sizes<<<L.ntiles, kTileThreads, 0, st>>>(strs, L.ns, L.plain, t, coef, intra, tsum);
        counted();
        k_je_scan<<<L.ns, kScanThreads, 0, st>>>(strs, tsum, toff, raw);
        counted();
        k_je_emit<<<L.ntiles, kTileThreads, 0, st>>>(strs, L.ns, t, coef, intra, toff, raw);
        counted();
        k_je_ffcount<<<L.nchunks, kChunkThreads, 0, st>>>(strs, L.ns, raw, ffc);
        counted();
        k_je_offsets<<<1, kScanThreads, 0, st>>>(strs, L.ns, L.plain, n, ffc, L.nchunks, ffpre, offs, t);
        counted();
        k_je_stuff<<<L.nchunks, kChunkThreads, 0, st>>>(strs, L.ns, L.plain, t, raw, ffpre, w + L.off_out);
        counted();
        return 0;
    };
    if (encode_call(images, n, L, L.off_tsum, work, work_bytes, stream, offsets, dst, dst_cap, stats, fill, launch) != 0) return -1;
    if (stats) stats->blocks = L.nblk;
    return 0;
}
