// geometry.cuh — where a CTA of an iteration kernel works, as the shared kernel bodies ask for it
// (gradient_packed_body.cuh, project_tile_body.cuh, project_tile22_body.cuh).
//
// A body reads its block index and its frame's grid through `geo` wherever the kernel used to read
// blockIdx and gridDim.  GridGeo is the launch grid itself: the single-frame and batch kernels of
// libjpeg2png_b200.so.  GroupGeo is one entry of a grouped launch's CTA table (libj2pmixed.so): the grid
// is flat, one CTA per entry, and the entry holds the index that CTA has in the batch-kernel grid of
// its own session, so every frame of a group is cut into exactly the CTAs its own session launches.
#pragma once
#include <cuda_runtime.h>

#include "kernels.cuh"

namespace j2p {

#ifdef __CUDACC__
struct GridGeo {
    __device__ __forceinline__ unsigned bx() const { return blockIdx.x; }
    __device__ __forceinline__ unsigned by() const { return blockIdx.y; }
    __device__ __forceinline__ unsigned bz() const { return blockIdx.z; }
    __device__ __forceinline__ unsigned nx() const { return gridDim.x; }
    __device__ __forceinline__ unsigned ny() const { return gridDim.y; }
};
#endif

// One CTA of a grouped launch: its session's descriptor, the plane (uncovered-pixel kernels), and its
// block index (bx, by, bz = frame of the session) in a grid of nx x ny CTAs per frame and plane group.
struct GroupCta {
    unsigned d, c, bx, by, bz, nx, ny, pad;
};

// One session of a group: its frame geometry and buffers with the iterate buffers of one parity, and the
// band geometry its own k_gradient_packed launch has.  F.tables always points at device tables.
struct GroupFrame {
    FrameDev F;
    int band_rows, pad[3];
};

#ifdef __CUDACC__
struct GroupGeo {
    unsigned x, y, z, w, h;
    __device__ __forceinline__ explicit GroupGeo(const GroupCta &e) : x(e.bx), y(e.by), z(e.bz), w(e.nx), h(e.ny) {}
    __device__ __forceinline__ unsigned bx() const { return x; }
    __device__ __forceinline__ unsigned by() const { return y; }
    __device__ __forceinline__ unsigned bz() const { return z; }
    __device__ __forceinline__ unsigned nx() const { return w; }
    __device__ __forceinline__ unsigned ny() const { return h; }
};
#endif

// The grouped kernels of one iteration (libj2pmixed.so, j2p_mixed_iterate): kernel kind, variant and the
// slice of the CTA table each one launches.  A slice with count 0 is not launched.
enum GroupKernel {
    GK_GRAD = 0,        // k_gradient_packed_grouped<NC, TGV, GPM>: variant = GPM (0, 1, 2)
    GK_TILE = 3,        // k_project_tile_grouped<RES>: variant = RES (0, 1)
    GK_TILE22 = 5,      // k_project_tile22_grouped
    GK_UNCOVERED = 6,   // k_step_uncovered_grouped
    GK_UNCOVERED22 = 7, // k_step_uncovered22_grouped
    GK_COUNT = 8
};
struct GroupLaunch {
    unsigned first[GK_COUNT], count[GK_COUNT];   // CTA table slice per GroupKernel slot
};

}  // namespace j2p
