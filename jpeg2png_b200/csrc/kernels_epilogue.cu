// kernels_epilogue.cu — what the reference does to the solver's result before libpng sees it,
// as one device pass over the three planes of a frame (or of a batch of frames):
//   luma += 128                                   (jpeg2png.c:156-159)
//   YCbCr -> RGB in double, narrowed to float, clamp to [0, 255]
//                                                 (png.c:39-47, clamp: utils.h CLAMP via png.c:15-17)
// and then, per output mode (EpilogueArgs, kernels.cuh):
//   EP_SCANLINES  scale by (1 << bits) / 256, TRUNCATE, 8-bit or 16-bit big-endian samples (png.c:51-62),
//                 every row prefixed with filter type 0: the image as PNG scanlines, so the host only
//                 has to deflate it (3 or 6 bytes per pixel cross PCIe instead of 12)
//   EP_HWC/EP_CHW interleaved or planar samples for a tensor: 8 bit = the 8-bit PNG sample,
//                 16 bit = the 16-bit PNG sample in native byte order, 32 bit = the clamped float
// With a.nc == 1 (gray export) only the luma is read and written: clamp(float(double(Y + 128))),
// which is the RGB expression with zero chroma (1.402 * 0 and the other products are exact zeros,
// and adding +0 to a double that is not -0 leaves it unchanged).  The branch is uniform per launch.
// With a.oriented (HWC / CHW) the same samples are written flipped or rotated per frame by its EXIF
// orientation (DESIGN §7l): a CTA converts a 32 x 32 tile and writes it where the orientation puts it.
// With a.four (HWC / CHW) the frame is a four-component JPEG's four planes (four_samples, DESIGN §7q):
// four inverted CMYK samples per pixel, or three from Pillow's CMYK -> RGB of them.
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.cuh"
#include "numerics.cuh"

namespace j2p {

constexpr int EP_NT = 256;
constexpr int EP_TILE = 32;                                 // oriented mode: tiles of EP_TILE x EP_TILE pixels
constexpr int EP_TILE_ROW = EP_TILE * 16 + 4;               // largest staged output row (HWC float, four channels), + a pad word
constexpr int EP_STAGE = 4 * EP_TILE * (EP_TILE * 4 + 4);   // largest staged tile (CHW float, four channels), rows padded by a word
static_assert(EP_STAGE >= EP_TILE * EP_TILE_ROW && EP_STAGE >= EP_NT * 16, "the staging buffer holds every mode");

// png.c:15-17 + :44-46: the double expression is narrowed to float by the call to clamp() and
// compared with the double bounds 0. and 255.
__device__ __forceinline__ float clamp_sample(double v) {
    const float x = __double2float_rn(v);
    return (double)x > 255. ? 255.f : ((double)x < 0. ? 0.f : x);
}

// nbytes staged bytes -> global memory, consecutive threads (nt of them: the CTA or a warp) on
// consecutive 4-byte words; dst has any alignment (a scanline starts after its filter byte, a CHW row
// segment at any pixel)
__device__ __forceinline__ void store_bytes(uint8_t *dst, const uint8_t *src, int nbytes, int tid, int nt = EP_NT) {
    const int head = min(nbytes, (int)((4u - ((unsigned)(uintptr_t)dst & 3u)) & 3u));
    if (tid < head) dst[tid] = src[tid];
    const int words = (nbytes - head) >> 2;
    const uint8_t *s = src + head;
    const unsigned o = (unsigned)(uintptr_t)s & 3u;
    const uint32_t *s4 = reinterpret_cast<const uint32_t *>(s - o);
    uint32_t *d4 = reinterpret_cast<uint32_t *>(dst + head);
    for (int i = tid; i < words; i += nt) d4[i] = __byte_perm(s4[i], s4[i + 1], 0x3210u + 0x1111u * o);
    const int done = head + 4 * words;
    if (tid < nbytes - done) dst[done + tid] = src[done + tid];
}

// the samples of pixel (px, row) of a frame: the unsigned value of each of the nc samples (the float's
// bits at 32 bits), before any byte swap
__device__ __forceinline__ void pixel_samples(const EpilogueArgs &a, int frame, int row, int px, bool gray, uint32_t s[3]) {
    float v[3];
    const float *Y = a.plane[0] + (size_t)frame * a.frame_stride[0] + (size_t)row * a.ld[0];
    const float yi = __fadd_rn(Y[px], 128.f);                                                     // jpeg2png.c:158
    const double dy = (double)yi;
    if (gray) {
        v[0] = v[1] = v[2] = clamp_sample(dy);                                                       // png.c:44-46, zero chroma
    } else {
        const float *Cb = a.plane[1] + (size_t)frame * a.frame_stride[1] + (size_t)row * a.ld[1];
        const float *Cr = a.plane[2] + (size_t)frame * a.frame_stride[2] + (size_t)row * a.ld[2];
        const double dcb = (double)Cb[px], dcr = (double)Cr[px];
        v[0] = clamp_sample(__dadd_rn(dy, __dmul_rn(1.402, dcr)));                                       // png.c:44
        v[1] = clamp_sample(__dsub_rn(__dsub_rn(dy, __dmul_rn(0.34414, dcb)), __dmul_rn(0.71414, dcr))); // png.c:45
        v[2] = clamp_sample(__dadd_rn(dy, __dmul_rn(1.772, dcb)));                                       // png.c:46
    }
    const float bitfactor = a.sample == 8 ? 1.0f : 256.0f;                                               // (1 << bits) / 256.
#pragma unroll
    for (int k = 0; k < 3; k++)
        s[k] = a.sample == 32 ? __float_as_uint(v[k]) : __float2uint_rz(__fmul_rn(v[k], bitfactor));    // png.c:44-46 truncation
}

// The samples of pixel (px, row) of a four-plane frame (a.four, DESIGN §7q).  A plane's gray sample
// g is what the gray export writes for it; its inversion is 255 - g (8 bit), 65535 - g (16 bit) or
// 255.f - g (float), Pillow's "CMYK;I" reading of Adobe files.  CMYK: every channel inverted.
// YCCK: channels 0-2 the RGB samples of planes 0-2, channel 3 plane 3 inverted.  With a.nc == 3
// (8 bit) the four 8-bit samples go through Pillow's CMYK -> RGB: nk = 255 - K, t = x * nk + 128,
// each channel clip(nk - ((t + (t >> 8)) >> 8), 0, 255).
__device__ __forceinline__ void four_samples(const EpilogueArgs &a, int frame, int row, int px, uint32_t s[4]) {
    const int c0 = a.four == EP_FOUR_YCCK ? 3 : 0;
    if (c0 == 3) pixel_samples(a, frame, row, px, false, s);
#pragma unroll 1
    for (int c = c0; c < 4; c++) {
        const float *P = a.plane[c] + (size_t)frame * a.frame_stride[c] + (size_t)row * a.ld[c];
        const float g = clamp_sample((double)__fadd_rn(P[px], 128.f));                                // the gray sample
        s[c] = a.sample == 32 ? __float_as_uint(__fsub_rn(255.f, g))
             : (a.sample == 8 ? 255u : 65535u) - __float2uint_rz(__fmul_rn(g, a.sample == 8 ? 1.0f : 256.0f));
    }
    if (a.nc == 3) {
        const int nk = 255 - (int)s[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const int t = (int)s[k] * nk + 128;
            s[k] = (uint32_t)min(max(nk - ((t + (t >> 8)) >> 8), 0), 255);
        }
    }
}

__device__ __forceinline__ void stage_sample(uint8_t *p, uint32_t s, int es) {
    if (es == 1) *p = (uint8_t)s;
    else if (es == 2) *reinterpret_cast<uint16_t *>(p) = (uint16_t)s;
    else *reinterpret_cast<uint32_t *>(p) = s;
}

// Oriented mode: one CTA = the tile (blockIdx.x, blockIdx.y) of frame blockIdx.z.  Each warp reads
// whole tile rows of the planes; the samples are staged in output order for the frame's orientation
// k (EXIF, as Pillow's ImageOps.exif_transpose applies it: k >= 5 transposes, then (k - 1) & 3 =
// 1, 2, 3 flips the columns, both, the rows of the result), and each warp writes staged output rows
// as contiguous segments.  A staged row is padded by one word so the transposed staging stores of a
// warp fall in different banks.
__device__ __forceinline__ void oriented_tile(const EpilogueArgs &a, uint8_t *sm) {
    const int frame = blockIdx.z, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tx0 = blockIdx.x * EP_TILE, ty0 = blockIdx.y * EP_TILE;
    const int tw = min(EP_TILE, a.w - tx0), th = min(EP_TILE, a.h - ty0);
    const int es = a.sample >> 3;
    const bool gray = a.nc == 1, chw = a.mode == EP_CHW;
    const int nc = a.nc;
    int k = a.orient ? a.orient[frame] : 1;
    if (k < 1 || k > 8) k = 1;
    const bool tr = k >= 5;
    const int fl = (k - 1) & 3;
    const bool fx = fl == 1 || fl == 2, fy = fl >= 2;
    const int ow = tr ? th : tw, oh = tr ? tw : th;                         // the tile as written
    const int px_bytes = chw ? es : nc * es;                                // a staged pixel
    const int row_bytes = EP_TILE * px_bytes + 4;                           // a staged output row
    const int plane_stage = EP_TILE * row_bytes;                            // CHW: one channel's staged tile
    if (lane < tw) {
        for (int ly = warp; ly < th; ly += EP_NT / 32) {
            uint32_t s[4];
            if (a.four) four_samples(a, frame, ty0 + ly, tx0 + lane, s);
            else pixel_samples(a, frame, ty0 + ly, tx0 + lane, gray, s);
            const int sx = tr ? ly : lane, sy = tr ? lane : ly;
            const int ox = fx ? ow - 1 - sx : sx, oy = fy ? oh - 1 - sy : sy;
            uint8_t *e = sm + oy * row_bytes + ox * px_bytes;
#pragma unroll
            for (int c = 0; c < 4; c++) {
                if (c >= nc) break;
                stage_sample(chw ? e + c * plane_stage : e + c * es, s[c], es);
            }
        }
    }
    __syncthreads();
    // the output image is SW x SH (transposed for k >= 5); the tile starts at (X0, Y0) there
    const int SW = tr ? a.h : a.w, SH = tr ? a.w : a.h;
    const int sx0 = tr ? ty0 : tx0, sy0 = tr ? tx0 : ty0;
    const int X0 = fx ? SW - sx0 - ow : sx0, Y0 = fy ? SH - sy0 - oh : sy0;
    uint8_t *base = a.out + (size_t)frame * a.frame_bytes;
    const size_t plane_bytes = (size_t)a.w * a.h * es;
    // g lanes per output row segment, so that a warp writes several short segments (CHW) at once
    const int segs = chw ? nc * oh : oh, words = (ow * px_bytes + 3) >> 2;
    const int g = words <= 8 ? 8 : (words <= 16 ? 16 : 32);
    for (int r = warp * (32 / g) + lane / g; r < segs; r += EP_NT / g) {
        const int c = chw ? r / oh : 0, oy = r - c * oh;
        uint8_t *dst = base + c * plane_bytes + ((size_t)(Y0 + oy) * SW + X0) * px_bytes;
        store_bytes(dst, sm + c * plane_stage + oy * row_bytes, ow * px_bytes, lane % g, g);
    }
}

// one CTA = EP_NT consecutive pixels of one row (a.row0 + blockIdx.y) of one frame (blockIdx.z); samples
// are staged in shared memory in output order and written out with coalesced word stores.  With
// a.oriented: one 32 x 32 tile per CTA (oriented_tile).
__global__ void __launch_bounds__(EP_NT) k_scanlines(const EpilogueArgs a) {
    __shared__ __align__(16) uint8_t sm[EP_STAGE + 16];                // + one word read past the end by store_bytes
    if (a.oriented) {
        oriented_tile(a, sm);
        return;
    }
    const int row = a.row0 + (int)blockIdx.y, frame = blockIdx.z, x0 = blockIdx.x * EP_NT, tid = threadIdx.x;
    const int es = a.sample >> 3, npx = min(EP_NT, a.w - x0);           // bytes per sample, pixels of this CTA
    const bool gray = a.nc == 1;
    const int nc = a.nc;                                                // samples per pixel
    if (tid < npx) {
        uint32_t v[4];
        if (a.four) four_samples(a, frame, row, x0 + tid, v);
        else pixel_samples(a, frame, row, x0 + tid, gray, v);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (k >= nc) break;
            uint32_t s = v[k];
            if (a.mode == EP_SCANLINES && es == 2) s = ((s >> 8) & 0xffu) | ((s & 0xffu) << 8);                // png.c:58-60 big-endian
            const int e = a.mode == EP_CHW ? k * EP_NT + tid : tid * nc + k;                                  // staged element
            stage_sample(sm + e * es, s, es);
        }
    }
    __syncthreads();
    uint8_t *base = a.out + (size_t)frame * a.frame_bytes;
    if (a.mode == EP_CHW) {
        const size_t plane_bytes = (size_t)a.w * a.h * es, at = ((size_t)row * a.w + x0) * es;
        for (int k = 0; k < nc; k++) store_bytes(base + k * plane_bytes + at, sm + k * EP_NT * es, npx * es, tid);
        return;
    }
    const int filter = a.mode == EP_SCANLINES;                                                               // one filter byte per scanline
    uint8_t *dst = base + (size_t)row * ((size_t)a.w * nc * es + filter);
    if (filter && x0 == 0 && tid == 0) dst[0] = 0;                                                           // PNG filter type 0 (None)
    store_bytes(dst + filter + (size_t)x0 * nc * es, sm, npx * nc * es, tid);
}

// rows in launches of at most kMaxGridRows (kernels.cuh); the oriented mode in one launch of tiles
// (its caller keeps the tile rows within kMaxGridRows); *nlaunch: launches made
cudaError_t launch_scanlines(const EpilogueArgs &a, int nframes, cudaStream_t s, int *nlaunch) {
    if (a.oriented) {
        k_scanlines<<<dim3((a.w + EP_TILE - 1) / EP_TILE, (a.h + EP_TILE - 1) / EP_TILE, nframes), EP_NT, 0, s>>>(a);
        *nlaunch += 1;
        return cudaGetLastError();
    }
    EpilogueArgs b = a;
    for (b.row0 = 0; b.row0 < a.h; b.row0 += kMaxGridRows) {
        const int rows = a.h - b.row0 < kMaxGridRows ? a.h - b.row0 : kMaxGridRows;
        k_scanlines<<<dim3((a.w + EP_NT - 1) / EP_NT, rows, nframes), EP_NT, 0, s>>>(b);
        *nlaunch += 1;
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace j2p
