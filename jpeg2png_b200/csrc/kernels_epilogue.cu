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
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.cuh"
#include "numerics.cuh"

namespace j2p {

constexpr int EP_NT = 256;

// png.c:15-17 + :44-46: the double expression is narrowed to float by the call to clamp() and
// compared with the double bounds 0. and 255.
__device__ __forceinline__ float clamp_sample(double v) {
    const float x = __double2float_rn(v);
    return (double)x > 255. ? 255.f : ((double)x < 0. ? 0.f : x);
}

// nbytes staged bytes -> global memory, consecutive threads on consecutive 4-byte words; dst has
// any alignment (a scanline starts after its filter byte, a CHW row segment at any pixel)
__device__ __forceinline__ void store_bytes(uint8_t *dst, const uint8_t *src, int nbytes, int tid) {
    const int head = min(nbytes, (int)((4u - ((unsigned)(uintptr_t)dst & 3u)) & 3u));
    if (tid < head) dst[tid] = src[tid];
    const int words = (nbytes - head) >> 2;
    const uint8_t *s = src + head;
    const unsigned o = (unsigned)(uintptr_t)s & 3u;
    const uint32_t *s4 = reinterpret_cast<const uint32_t *>(s - o);
    uint32_t *d4 = reinterpret_cast<uint32_t *>(dst + head);
    for (int i = tid; i < words; i += EP_NT) d4[i] = __byte_perm(s4[i], s4[i + 1], 0x3210u + 0x1111u * o);
    const int done = head + 4 * words;
    if (tid < nbytes - done) dst[done + tid] = src[done + tid];
}

// one CTA = EP_NT consecutive pixels of one row (a.row0 + blockIdx.y) of one frame (blockIdx.z); samples
// are staged in shared memory in output order and written out with coalesced word stores
__global__ void __launch_bounds__(EP_NT) k_scanlines(const EpilogueArgs a) {
    __shared__ __align__(16) uint8_t sm[EP_NT * 12 + 16];               // + one word read past the end by store_bytes
    const int row = a.row0 + (int)blockIdx.y, frame = blockIdx.z, x0 = blockIdx.x * EP_NT, tid = threadIdx.x;
    const int es = a.sample >> 3, npx = min(EP_NT, a.w - x0);           // bytes per sample, pixels of this CTA
    const bool gray = a.nc == 1;
    const int nc = gray ? 1 : 3;                                        // samples per pixel
    if (tid < npx) {
        const int px = x0 + tid;
        float v[3];
        {
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
        }
        const float bitfactor = a.sample == 8 ? 1.0f : 256.0f;                                               // (1 << bits) / 256.
#pragma unroll
        for (int k = 0; k < 3; k++) {
            if (k >= nc) break;
            uint32_t s = a.sample == 32 ? __float_as_uint(v[k]) : __float2uint_rz(__fmul_rn(v[k], bitfactor));   // png.c:44-46 truncation
            if (a.mode == EP_SCANLINES && es == 2) s = ((s >> 8) & 0xffu) | ((s & 0xffu) << 8);                // png.c:58-60 big-endian
            const int e = a.mode == EP_CHW ? k * EP_NT + tid : tid * nc + k;                                  // staged element
            if (es == 1) sm[e] = (uint8_t)s;
            else if (es == 2) reinterpret_cast<uint16_t *>(sm)[e] = (uint16_t)s;
            else reinterpret_cast<uint32_t *>(sm)[e] = s;
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

// rows in launches of at most kMaxGridRows (kernels.cuh); *nlaunch: launches made
cudaError_t launch_scanlines(const EpilogueArgs &a, int nframes, cudaStream_t s, int *nlaunch) {
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
