// gradient_packed_body.cuh — the body of the packed sub-gradient kernel (kernels_gradient_packed.cu),
// shared by the single-frame and batch kernels of libjpeg2png_b200.so and the grouped kernel of
// libj2pmixed.so (mixed/mixed.cu), which runs frames of different sizes in one grid.
// `geo` (geometry.cuh) supplies the CTA's block index and its frame's grid: the launch grid itself
// (GridGeo), or the CTA's entry in the table of a grouped launch (GroupGeo).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gradient_common.cuh"
#include "geometry.cuh"
#include "kernels.cuh"
#include "numerics.cuh"
#include "pdl.cuh"
#include "project_common.cuh"
#include "record.cuh"
#include "strip_sync.cuh"

namespace j2p {

// what one row step hands to the next; f2 = the lane's two adjacent columns
template <int NC>
struct RowCarry {
    f2 y[NC];            // FISTA point of the newest row
    f2 gx[NC], gy[NC];   // forward differences of the newest source row
    f2 og[NC];           // gradient of the newest target row after its first nine addends
    f2 tvb[NC];          // its TV "below" quotients   (addend 1 of the next target row)
    f2 ud[NC], dg[NC];   // its TGV "above/below" and diagonal quotients (addends 4, 5 of the next target row)
    bool ok1, ok2;       // row guard (numerics.cuh) of the newest and the second newest row
};

__device__ __forceinline__ f2 shl_from_left(f2 v, float from_left) { return pk(from_left, lo(v)); }    // (left neighbour's hi, own lo)
__device__ __forceinline__ f2 shr_from_right(f2 v, float from_right) { return pk(hi(v), from_right); } // (own hi, right neighbour's lo)

// GPM: how the DCT-distance term is addressed.  1 = every plane is full resolution and covers the
// whole frame (4:4:4): gp has the frame's geometry, one 8-byte load per plane at the pixel offset.
// 0 = generic (any sampling factors, grids smaller than the frame).
#ifdef J2P_GRAD_MAXNREG      // A/B aid: an explicit register budget instead of the resident-CTA bound
#define J2P_GRAD_BOUNDS __maxnreg__(J2P_GRAD_MAXNREG)
#else
#define J2P_GRAD_BOUNDS __launch_bounds__(GM_NT, J2P_GRAD_MIN_CTAS)
#endif

}  // namespace j2p
