// project_tile_body.cuh — the bodies of the tiled projection of 1x1 planes and of the step of the pixels
// no block covers (kernels_project_tile.cu), shared by the single-frame and batch kernels of
// libjpeg2png_b200.so and the grouped kernels of libj2pmixed.so (mixed/mixed.cu).
// `geo` (geometry.cuh) supplies the CTA's block index and its frame's grid: the launch grid itself
// (GridGeo), or the CTA's entry in the table of a grouped launch (GroupGeo).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "geometry.cuh"
#include "kernels.cuh"
#include "numerics.cuh"
#include "pdl.cuh"
#include "project_common.cuh"
#include "record.cuh"
#include "strip_sync.cuh"

namespace j2p {

#ifndef J2P_TILE_BLOCKS
#define J2P_TILE_BLOCKS 16            // coefficient blocks per CTA tile (16 or 32: the tables and the norm take 96 threads).  16-block tiles
                                      // run as eight 4-warp CTAs per SM where 32-block tiles run as four 8-warp CTAs: the same resident warps,
                                      // half as many warps behind each of the two CTA barriers
#endif
constexpr int PT_NB = J2P_TILE_BLOCKS;
constexpr int PT_NT = PT_NB * 8;      // 8 threads per block
constexpr int PT_C4 = PT_NB * 2;      // float4 columns per tile row
constexpr int PT_SH = PT_NB == 32 ? 6 : (PT_NB == 16 ? 5 : 7);   // log2(PT_C4)
static_assert(PT_C4 == 1 << PT_SH, "tile width");

#ifndef J2P_TILE_MIN_CTAS
#define J2P_TILE_MIN_CTAS (256 / J2P_TILE_BLOCKS / 2)      // 32 warps per SM either way (64 registers)
#endif

template <bool BATCH, class G>
__device__ __forceinline__ void step_uncovered_body(const FrameDev &F, const int c, const float factor, const G &geo) {
    const PlaneDev &P = F.pl[c];
    const int W = F.W, H = F.H;
    const int frame = BATCH ? (int)geo.bz() : 0;
    const size_t fo = BATCH ? (size_t)frame * F.frame_stride : 0;
    const float *const xk = P.x + fo, *const gk = P.g + fo;
    float *const xm = P.xp + fo;
    Stepper stepper;
    stepper.factor = factor;
    stepper.step = F.step;
    stepper.norm = F.norms[16 * frame + c];
    stepper.rn = 0.f;
    stepper.stepping = stepper.norm != 0.f;
    const unsigned bottom = (unsigned)(H - P.ch) * (unsigned)W, right_w = (unsigned)(W - P.cw);
    const unsigned n = bottom + (unsigned)P.ch * right_w;
    for (unsigned i = geo.bx() * blockDim.x + threadIdx.x; i < n; i += geo.nx() * blockDim.x) {
        unsigned px, py;
        if (i < bottom) {
            py = (unsigned)P.ch + i / (unsigned)W;
            px = i % (unsigned)W;
        } else {
            const unsigned k = i - bottom;
            py = k / right_w;
            px = (unsigned)P.cw + k % right_w;
        }
        const size_t gi = (size_t)py * W + px;
        xm[gi] = stepper(xk[gi], xm[gi], gk[gi]);
    }
}

}  // namespace j2p
