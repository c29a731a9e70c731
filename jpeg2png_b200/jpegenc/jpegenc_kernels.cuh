// jpegenc_kernels.cuh — the bodies of the encoder's kernels as __device__ functions, shared by
// libj2pjpegenc.so (whose __global__ kernels are thin wrappers around them), libj2pjpegopt.so and
// libj2pjpegprog.so.  The blocks body runs on images; the others run on bit streams (an image's
// scan, or one restart interval of it; jpegenc_plan.h), each described by a j2p_je_img that names
// its image.  Where an image's Huffman tables and a stream's header come from is a parameter:
//   huff(i)                the derived tables of image i (called by every thread of the CTA, before
//                          any of them returns, so that it may stage them in shared memory); the
//                          emit body takes the tables themselves, staged by its caller;
//   head_len(s)            the length of the scan header that stream s starts with when it is its
//                          scan's first interval (the others start with RST);
//   head_byte(s, k)        its byte k.
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

// kBlockThreads threads, 8 per block: colour, downsampling, FDCT and quantisation with the tables
// of the image's set (t: the call's sets)
__device__ __forceinline__ void blocks_body(const struct j2p_je_img *__restrict__ imgs, uint32_t n, const struct j2p_je_tables *__restrict__ t,
                                            uint64_t nblk, int16_t *__restrict__ coef) {
    __shared__ int rows[kBlockThreads / 8][8 * 9];
    __shared__ uint32_t sets[kBlockThreads / 8];   // each block's set, with its rows: no register holds it across the barrier
    const uint32_t grp = threadIdx.x >> 3, lane = threadIdx.x & 7;
    const uint64_t g = ((uint64_t)blockIdx.x * kBlockThreads + threadIdx.x) >> 3;
    const bool on = g < nblk;
    struct j2p_je_where wh;
    if (on) {                           // the geometry is the same in every set: set 0's
        const struct j2p_je_img im = imgs[find_image(imgs, n, g, 0)];
        if (lane == 0) sets[grp] = im.set;
        wh = j2p_je_locate(&im, t, g - im.blk0);
        int d[8];
        if (t->nc == 4) j2p_je_block_row<4>(&im, t, &wh, (int)lane, d);
        else j2p_je_block_row<3>(&im, t, &wh, (int)lane, d);
#pragma unroll
        for (int x = 0; x < 8; x++) rows[grp][lane * 9 + x] = d[x];
    }
    __syncthreads();
    if (on) finish_column(t + sets[grp], &wh, rows[grp], 9, (int)lane, coef + g * 64);
}

// Where the kernels find a stream's image, scan and interval.  Without restart intervals (plain)
// every image has PER streams (1, or a progressive file's ten scans), so stream s is scan s % PER of
// image s / PER and the only interval of its scan: the kernels use that arithmetic, as they did
// before restarts existed, and read none of the descriptor's stream fields for it.  With restart
// intervals they read the descriptor.
template <uint32_t PER>
struct StreamMap {
    const struct j2p_je_img *strs;
    uint32_t ns;
    bool plain;
    __device__ __forceinline__ uint32_t img(uint32_t s) const { return plain ? s / PER : strs[s].img; }
    __device__ __forceinline__ uint32_t scan(uint32_t s) const { return plain ? s % PER : strs[s].scan; }
    // the (image, scan) of stream s as one index, img x PER + scan
    __device__ __forceinline__ uint32_t scan_index(uint32_t s) const { return plain ? s : strs[s].img * PER + strs[s].scan; }
    // whether stream s starts with RST rather than its scan's header
    __device__ __forceinline__ bool rst(uint32_t s) const { return !plain && strs[s].part; }
    __device__ __forceinline__ bool first_of_file(uint32_t s) const { return plain ? s % PER == 0 : s == 0 || strs[s - 1].img != strs[s].img; }
    __device__ __forceinline__ bool ends_file(uint32_t s) const { return plain ? s % PER == PER - 1 : j2p_je_ends_file(strs, ns, s); }
};

// per tile: each block's bits, their exclusive scan in the tile, the tile's sum
template <uint32_t PER, class Huff>
__device__ __forceinline__ void sizes_body(const StreamMap<PER> &sm, const struct j2p_je_tables *__restrict__ t, const int16_t *__restrict__ coef,
                                           uint32_t *__restrict__ intra, uint32_t *__restrict__ tsum, Huff huff) {
    typedef cub::BlockScan<uint32_t, kTileThreads> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const uint32_t tile = blockIdx.x, s = find_image(sm.strs, sm.ns, tile, 1);
    const struct j2p_je_img *im = &sm.strs[s];
    const struct j2p_je_huff *h = huff(sm.img(s));
    const uint64_t b = (uint64_t)(tile - im->tile0) * J2P_JE_TILE + threadIdx.x;
    const uint64_t blk0 = im->blk0;
    uint32_t bits = 0;
    if (b < im->nblk) bits = j2p_je_block_bits(coef + (blk0 + b) * 64, pred_of(t, coef, blk0, b), h, htab_of(t, b));
    uint32_t excl, total;
    Scan(tmp).ExclusiveSum(bits, excl, total);
    if (b < im->nblk) intra[blk0 + b] = excl;
    if (threadIdx.x == 0) tsum[tile] = total;
}

// per stream: the tiles' bit offsets, the stream's bits, the padding 1-bits
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

__device__ __forceinline__ void emit_body(const struct j2p_je_img *__restrict__ strs, uint32_t ns, const struct j2p_je_tables *__restrict__ t,
                                          const int16_t *__restrict__ coef, const uint32_t *__restrict__ intra, const uint64_t *__restrict__ toff,
                                          uint32_t *__restrict__ raw, const struct j2p_je_huff *huff) {
    const uint32_t tile = blockIdx.x;
    const struct j2p_je_img *im = &strs[find_image(strs, ns, tile, 1)];
    const uint64_t b = (uint64_t)(tile - im->tile0) * J2P_JE_TILE + threadIdx.x;
    if (b >= im->nblk) return;
    const uint64_t blk0 = im->blk0;
    uint32_t *rw = raw + im->raw_off;
    j2p_je_emit(coef + (blk0 + b) * 64, pred_of(t, coef, blk0, b), huff, htab_of(t, b), toff[tile] + intra[blk0 + b],
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

__device__ __forceinline__ void ffcount_body(const struct j2p_je_img *__restrict__ strs, uint32_t ns, const uint32_t *__restrict__ raw,
                                             uint32_t *__restrict__ ffc) {
    typedef cub::BlockReduce<uint32_t, kChunkThreads> Red;
    __shared__ typename Red::TempStorage tmp;
    const struct j2p_je_img *im = &strs[find_image(strs, ns, blockIdx.x, 2)];
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

// one CTA: the scan of the 0xFF counts over the call, each stream's place in the output (its header:
// its scan's, of head_len(s) bytes, or RST; its stuffed bytes; after an image's last stream, EOI) and
// each file's offset
template <uint32_t PER, class HeadLen>
__device__ __forceinline__ void offsets_body(struct j2p_je_img *__restrict__ strs, const StreamMap<PER> &sm, uint32_t n,
                                             const uint32_t *__restrict__ ffc, uint32_t nchunks, uint64_t *__restrict__ ffpre,
                                             uint64_t *__restrict__ offsets, HeadLen head_len) {
    __shared__ typename ScanU64::TempStorage tmp;
    const uint32_t ns = sm.ns;
    const uint64_t ff = scan_segment(nchunks, [&](uint32_t k) { return (uint64_t)ffc[k]; }, [&](uint32_t k, uint64_t v) { ffpre[k] = v; }, tmp);
    if (threadIdx.x == 0) ffpre[nchunks] = ff;
    __syncthreads();
    const uint64_t base = scan_segment(
        ns,
        [&](uint32_t s) {
            const struct j2p_je_img *st = &strs[s];
            return (sm.rst(s) ? J2P_JE_RST : head_len(s)) + raw_bytes(st) + (ffpre[st->chunk0 + st->nchunks] - ffpre[st->chunk0]) +
                   (sm.ends_file(s) ? 2 : 0);
        },
        [&](uint32_t s, uint64_t v) {
            strs[s].file_off = v;
            if (sm.first_of_file(s)) offsets[sm.img(s)] = v;
        },
        tmp);
    __syncthreads();
    for (uint32_t s = threadIdx.x; s < ns; s += kScanThreads) strs[s].file_len = (s + 1 < ns ? strs[s + 1].file_off : base) - strs[s].file_off;
    if (threadIdx.x == 0) offsets[n] = base;
}

// per chunk: its bytes into the output with a 0x00 after each 0xFF; a stream's first chunk also
// writes its header (its scan's, head_len(s) bytes head_byte(s, k), or RST), the chunk holding an
// image's last byte the EOI
template <uint32_t PER, class HeadLen, class HeadByte>
__device__ __forceinline__ void stuff_body(const StreamMap<PER> &sm, const uint32_t *__restrict__ raw, const uint64_t *__restrict__ ffpre,
                                           uint8_t *__restrict__ out, HeadLen head_len, HeadByte head_byte) {
    typedef cub::BlockScan<uint32_t, kChunkThreads> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const uint32_t s = find_image(sm.strs, sm.ns, blockIdx.x, 2);
    const struct j2p_je_img *st = &sm.strs[s];
    const bool rst = sm.rst(s);
    const uint32_t c = blockIdx.x - st->chunk0, hl = rst ? J2P_JE_RST : head_len(s);
    const uint64_t nbytes = raw_bytes(st);
    if ((uint64_t)c * J2P_JE_CHUNK >= nbytes) return;
    uint8_t *file = out + st->file_off;
    if (c == 0) {
        if (rst) {
            if (threadIdx.x < J2P_JE_RST) file[threadIdx.x] = j2p_je_rst_byte(st->part, threadIdx.x);
        } else {
            for (uint32_t k = threadIdx.x; k < hl; k += kChunkThreads) file[k] = head_byte(s, k);
        }
    }
    if (threadIdx.x == 0 && (uint64_t)(c + 1) * J2P_JE_CHUNK >= nbytes && sm.ends_file(s)) {
        file[st->file_len - 2] = 0xff;
        file[st->file_len - 1] = 0xd9;
    }
    uint64_t j0;
    uint32_t cnt;
    uint4 v;
    const uint32_t m = chunk_bytes(st, raw, c, &j0, &cnt, &v);
    uint32_t before;
    Scan(tmp).ExclusiveSum(cnt, before);
    uint8_t *o = file + hl + j0 + (ffpre[blockIdx.x] - ffpre[st->chunk0]) + before;
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
