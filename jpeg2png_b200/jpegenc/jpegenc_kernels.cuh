// jpegenc_kernels.cuh — the bodies of the encoder's kernels as __device__ functions, shared by
// libj2pjpegenc.so (whose __global__ kernels are thin wrappers around them), libj2pjpegopt.so and
// libj2pjpegprog.so (which runs the blocks, scan and ffcount bodies on its per-scan streams).
// Where an image's Huffman tables and header come from is a parameter:
//   huff(i)                the derived tables of image i (called by every thread of the CTA, before
//                          any of them returns, so that it may stage them in shared memory); the
//                          emit body takes the tables themselves, staged by its caller;
//   head_len(i)            the header's length;
//   head_byte(i, im, k)    its byte k.
#ifndef J2P_JPEGENC_KERNELS_CUH
#define J2P_JPEGENC_KERNELS_CUH

#include <cuda_runtime.h>
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "jpegenc_plan.h"

static const int kBlockThreads = 256;       // 8 threads per block: a row each, then a column each
static const int kTileThreads = J2P_JE_TILE;
static const int kScanThreads = 512;
static const int kScanItems = 8;            // per thread and round of a scan
static const int kChunkThreads = J2P_JE_CHUNK / 16;     // 16 bytes per thread

__device__ __forceinline__ uint32_t find_image(const struct j2p_je_img *imgs, uint32_t n, uint64_t v, int field) {
    uint32_t lo = 0, hi = n - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) / 2;
        const uint64_t s = field == 0 ? imgs[mid].blk0 : field == 1 ? imgs[mid].tile0 : imgs[mid].chunk0;
        if (s <= v) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// Exclusive scan of count values ld(k) over the CTA, kScanThreads x kScanItems per round:
// st(k, prefix) for each, returns the sum.
typedef cub::BlockScan<uint64_t, kScanThreads> ScanU64;

template <class Ld, class St>
__device__ uint64_t scan_segment(uint32_t count, Ld ld, St st, typename ScanU64::TempStorage &tmp) {
    uint64_t base = 0;
    for (uint32_t k0 = 0; k0 < count; k0 += kScanThreads * kScanItems) {
        const uint32_t k1 = k0 + threadIdx.x * kScanItems;
        uint64_t v[kScanItems], sum = 0;
#pragma unroll
        for (int q = 0; q < kScanItems; q++) {
            v[q] = k1 + q < count ? ld(k1 + q) : 0;
            sum += v[q];
        }
        uint64_t excl, total;
        ScanU64(tmp).ExclusiveSum(sum, excl, total);
        uint64_t run = base + excl;
#pragma unroll
        for (int q = 0; q < kScanItems; q++) {
            if (k1 + q < count) st(k1 + q, run);
            run += v[q];
        }
        base += total;
        __syncthreads();
    }
    return base;
}

// kBlockThreads threads, 8 per block: colour, downsampling, FDCT and quantisation
__device__ __forceinline__ void blocks_body(const struct j2p_je_img *__restrict__ imgs, uint32_t n, const struct j2p_je_tables *__restrict__ t,
                                            uint64_t nblk, int16_t *__restrict__ coef) {
    __shared__ int rows[kBlockThreads / 8][8 * 9];
    const uint32_t grp = threadIdx.x >> 3, lane = threadIdx.x & 7;
    const uint64_t g = ((uint64_t)blockIdx.x * kBlockThreads + threadIdx.x) >> 3;
    const bool on = g < nblk;
    struct j2p_je_where wh;
    if (on) {
        const struct j2p_je_img im = imgs[find_image(imgs, n, g, 0)];
        wh = j2p_je_locate(&im, t, g - im.blk0);
        int d[8];
        j2p_je_block_row(&im, t, &wh, (int)lane, d);
#pragma unroll
        for (int x = 0; x < 8; x++) rows[grp][lane * 9 + x] = d[x];
    }
    __syncthreads();
    if (on) finish_column(t, &wh, rows[grp], 9, (int)lane, coef + g * 64);
}

// per tile: each block's bits, their exclusive scan in the tile, the tile's sum
template <class Huff>
__device__ __forceinline__ void sizes_body(const struct j2p_je_img *__restrict__ imgs, uint32_t n, const struct j2p_je_tables *__restrict__ t,
                                           const int16_t *__restrict__ coef, uint32_t *__restrict__ intra, uint32_t *__restrict__ tsum, Huff huff) {
    typedef cub::BlockScan<uint32_t, kTileThreads> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const uint32_t tile = blockIdx.x;
    const uint32_t i = find_image(imgs, n, tile, 1);
    const struct j2p_je_img *im = &imgs[i];
    const struct j2p_je_huff *h = huff(i);
    const uint64_t b = (uint64_t)(tile - im->tile0) * J2P_JE_TILE + threadIdx.x;
    const uint64_t blk0 = im->blk0;
    uint32_t bits = 0;
    if (b < im->nblk) bits = j2p_je_block_bits(coef + (blk0 + b) * 64, pred_of(t, coef, blk0, b), h, comp_of(t, b));
    uint32_t excl, total;
    Scan(tmp).ExclusiveSum(bits, excl, total);
    if (b < im->nblk) intra[blk0 + b] = excl;
    if (threadIdx.x == 0) tsum[tile] = total;
}

// per image: the tiles' bit offsets, the image's bits, the padding 1-bits
__device__ __forceinline__ void scan_body(struct j2p_je_img *__restrict__ imgs, const uint32_t *__restrict__ tsum, uint64_t *__restrict__ toff,
                                          uint32_t *__restrict__ raw) {
    __shared__ typename ScanU64::TempStorage tmp;
    struct j2p_je_img *im = &imgs[blockIdx.x];
    const uint32_t t0 = im->tile0;
    const uint64_t base = scan_segment(im->ntiles, [&](uint32_t k) { return (uint64_t)tsum[t0 + k]; },
                                       [&](uint32_t k, uint64_t v) { toff[t0 + k] = v; }, tmp);
    if (threadIdx.x == 0) {
        im->bits = base;
        uint64_t pw;
        const uint32_t mask = j2p_je_pad(base, &pw);
        if (mask) atomicOr(raw + im->raw_off + pw, mask);
    }
}

__device__ __forceinline__ void emit_body(const struct j2p_je_img *__restrict__ imgs, uint32_t n, const struct j2p_je_tables *__restrict__ t,
                                          const int16_t *__restrict__ coef, const uint32_t *__restrict__ intra, const uint64_t *__restrict__ toff,
                                          uint32_t *__restrict__ raw, const struct j2p_je_huff *huff) {
    const uint32_t tile = blockIdx.x;
    const struct j2p_je_img *im = &imgs[find_image(imgs, n, tile, 1)];
    const uint64_t b = (uint64_t)(tile - im->tile0) * J2P_JE_TILE + threadIdx.x;
    if (b >= im->nblk) return;
    const uint64_t blk0 = im->blk0;
    uint32_t *rw = raw + im->raw_off;
    j2p_je_emit(coef + (blk0 + b) * 64, pred_of(t, coef, blk0, b), huff, comp_of(t, b), toff[tile] + intra[blk0 + b],
                [&](uint64_t k, uint32_t v) { atomicOr(rw + k, v); });
}

// this thread's 16 entropy bytes of a chunk: the bytes (0 past the end) and how many are 0xFF
__device__ __forceinline__ uint32_t chunk_bytes(const struct j2p_je_img *im, const uint32_t *raw, uint32_t c, uint64_t *j0, uint32_t *cnt,
                                                uint4 *v) {
    const uint64_t nbytes = raw_bytes(im);
    *j0 = (uint64_t)c * J2P_JE_CHUNK + threadIdx.x * 16u;
    *v = make_uint4(0, 0, 0, 0);
    *cnt = 0;
    if (*j0 >= nbytes) return 0;
    *v = *(const uint4 *)(raw + im->raw_off + *j0 / 4);                  // raw_off and j0 / 4 are multiples of 4
    const uint32_t m = nbytes - *j0 < 16 ? (uint32_t)(nbytes - *j0) : 16u;
    const uint32_t wv[4] = {v->x, v->y, v->z, v->w};
    uint32_t k = 0;
#pragma unroll
    for (int q = 0; q < 16; q++) k += (uint32_t)q < m && ((wv[q >> 2] >> (24 - 8 * (q & 3))) & 0xff) == 0xff;
    *cnt = k;
    return m;
}

__device__ __forceinline__ void ffcount_body(const struct j2p_je_img *__restrict__ imgs, uint32_t n, const uint32_t *__restrict__ raw,
                                             uint32_t *__restrict__ ffc) {
    typedef cub::BlockReduce<uint32_t, kChunkThreads> Red;
    __shared__ typename Red::TempStorage tmp;
    const struct j2p_je_img *im = &imgs[find_image(imgs, n, blockIdx.x, 2)];
    const uint32_t c = blockIdx.x - im->chunk0;
    if ((uint64_t)c * J2P_JE_CHUNK >= raw_bytes(im)) {
        if (threadIdx.x == 0) ffc[blockIdx.x] = 0;
        return;
    }
    uint64_t j0;
    uint32_t cnt;
    uint4 v;
    chunk_bytes(im, raw, c, &j0, &cnt, &v);
    const uint32_t s = Red(tmp).Sum(cnt);
    if (threadIdx.x == 0) ffc[blockIdx.x] = s;
}

// one CTA: the scan of the 0xFF counts over the call, each file's length and offset
template <class HeadLen>
__device__ __forceinline__ void offsets_body(struct j2p_je_img *__restrict__ imgs, uint32_t n, const uint32_t *__restrict__ ffc, uint32_t nchunks,
                                             uint64_t *__restrict__ ffpre, uint64_t *__restrict__ offsets, HeadLen head_len) {
    __shared__ typename ScanU64::TempStorage tmp;
    const uint64_t ff = scan_segment(nchunks, [&](uint32_t k) { return (uint64_t)ffc[k]; }, [&](uint32_t k, uint64_t v) { ffpre[k] = v; }, tmp);
    if (threadIdx.x == 0) ffpre[nchunks] = ff;
    __syncthreads();
    const uint64_t base = scan_segment(
        n,
        [&](uint32_t i) {
            const struct j2p_je_img *im = &imgs[i];
            return head_len(i) + raw_bytes(im) + (ffpre[im->chunk0 + im->nchunks] - ffpre[im->chunk0]) + 2;
        },
        [&](uint32_t i, uint64_t v) { imgs[i].file_off = v; offsets[i] = v; }, tmp);
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += kScanThreads) imgs[i].file_len = (i + 1 < n ? imgs[i + 1].file_off : base) - imgs[i].file_off;
    if (threadIdx.x == 0) offsets[n] = base;
}

// per chunk: its bytes into the file with a 0x00 after each 0xFF; the first chunk also writes the
// header, the one holding the last byte the EOI
template <class HeadLen, class HeadByte>
__device__ __forceinline__ void stuff_body(const struct j2p_je_img *__restrict__ imgs, uint32_t n, const uint32_t *__restrict__ raw,
                                           const uint64_t *__restrict__ ffpre, uint8_t *__restrict__ out, HeadLen head_len, HeadByte head_byte) {
    typedef cub::BlockScan<uint32_t, kChunkThreads> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const uint32_t i = find_image(imgs, n, blockIdx.x, 2);
    const struct j2p_je_img *im = &imgs[i];
    const uint32_t c = blockIdx.x - im->chunk0;
    const uint64_t nbytes = raw_bytes(im);
    if ((uint64_t)c * J2P_JE_CHUNK >= nbytes) return;
    uint8_t *file = out + im->file_off;
    if (c == 0)
        for (uint32_t k = threadIdx.x; k < head_len(i); k += kChunkThreads) file[k] = head_byte(i, im, k);
    if (threadIdx.x == 0 && (uint64_t)(c + 1) * J2P_JE_CHUNK >= nbytes) {
        file[im->file_len - 2] = 0xff;
        file[im->file_len - 1] = 0xd9;
    }
    uint64_t j0;
    uint32_t cnt;
    uint4 v;
    const uint32_t m = chunk_bytes(im, raw, c, &j0, &cnt, &v);
    uint32_t before;
    Scan(tmp).ExclusiveSum(cnt, before);
    uint8_t *o = file + head_len(i) + j0 + (ffpre[blockIdx.x] - ffpre[im->chunk0]) + before;
    const uint32_t wv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int q = 0; q < 16; q++) {
        if ((uint32_t)q >= m) break;
        const uint8_t b = (uint8_t)(wv[q >> 2] >> (24 - 8 * (q & 3)));
        *o++ = b;
        if (b == 0xff) *o++ = 0;
    }
}

#endif  // J2P_JPEGENC_KERNELS_CUH
