// kernels_project_tile22.cu — step + projection of a 2x2-subsampled plane (4:2:0 chroma) with the
// coalesced, swizzled staging of kernels_project_tile.cu.
//
// Default for 2x2 planes (validated bit for bit on the whole GPU suite against k_project<2,2>,
// whose threads fetch their own 64-byte row pieces, and faster than it at 1080p and 8K).
//
// A coefficient block of a 2x2 plane covers 16 x 16 frame pixels.  Thread j of a block owns
// coefficient row j = frame rows 2j and 2j+1 of that footprint (2 x 16 stepped values in
// registers, compute.c:348-370), exactly like k_project<2,2>.  A CTA owns 16 blocks in a row:
// 256 x 16 frame pixels; its 128 threads copy the three 16 KB arrays with cp.async, consecutive
// lanes on consecutive 16-byte pieces, into shared memory whose 16-byte columns are XOR-swizzled by
// (row >> 1) — the eight threads of a block read rows 2j (+sy), so that is the index that must
// spread them over the banks.  x_{k+1} goes back the same way; gp (coefficient resolution, 8 rows
// of 128 floats per tile) through its own small staging array.
#include <cuda_runtime.h>
#include <stdint.h>

#include "project_tile22_body.cuh"

namespace j2p {

// BATCH: a batch session (FrameDev::nframes); blockIdx.z = frame, blockIdx.x = k * (CTA columns) +
// column for planes c0 + k (a single frame: blockIdx.z = k), as in k_project_tile.
template <bool BATCH>
__global__ void __launch_bounds__(P22_NT, 3) k_project_tile22(const __grid_constant__ FrameDev F, const int c0, const float factor) {
    project_tile22_body<BATCH>(F, c0, factor, GridGeo{});
}

// frame pixels of a 2x2 plane beyond its coefficient grid (W > 2 cw or H > 2 ch): step only.
// BATCH: the frame is blockIdx.z.
template <bool BATCH>
__global__ void k_step_uncovered22(const __grid_constant__ FrameDev F, const int c, const float factor) {
    step_uncovered22_body<BATCH>(F, c, factor, GridGeo{});
}

cudaError_t configure_project_tile22() {
    const cudaError_t e = cudaFuncSetAttribute(k_project_tile22<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P22_SMEM);
    return e != cudaSuccess ? e : cudaFuncSetAttribute(k_project_tile22<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P22_SMEM);
}

// F: already restricted to the rows the session owns (launch_project).  Projects planes
// c .. c+count-1, which must all be 2x2 planes with the same coefficient grid.
// uncovered_only: the tiles have been projected elsewhere (the recording kernels of
// libj2pobjective.so); only the stepped-only pixels remain
cudaError_t launch_project_tile22(const FrameDev &F, int c, int count, float factor, cudaStream_t s, int *nlaunch, bool uncovered_only) {
    const PlaneDev &P = F.pl[c];
    const int bw = P.cw >> 3, bh = P.ch >> 3, gx = (bw + P22_NB - 1) / P22_NB;
    const bool batch = F.nframes > 1;
    cudaError_t e = cudaSuccess;
    for (int y0 = 0; y0 < bh && !uncovered_only && e == cudaSuccess; y0 += kMaxGridRows) {   // one launch unless bh > 65535
        const int rows = bh - y0 < kMaxGridRows ? bh - y0 : kMaxGridRows;
        const FrameDev V = y0 == 0 && rows == bh ? F : rows_view(F, c, count, y0, 16, y0 + rows == bh);
        e = batch ? launch_chain(k_project_tile22<true>, dim3(gx * count, rows, F.nframes), dim3(P22_NT), P22_SMEM, s, V, c, factor)
                  : launch_chain(k_project_tile22<false>, dim3(gx, rows, count), dim3(P22_NT), P22_SMEM, s, V, c, factor);
        *nlaunch += 1;
    }
    for (int k = c; k < c + count && e == cudaSuccess; k++) {
        const PlaneDev &Q = F.pl[k];
        if (2 * Q.cw < F.W || 2 * Q.ch < F.H) {
            const size_t n = (size_t)(F.H - 2 * Q.ch) * F.W + (size_t)2 * Q.ch * (F.W - 2 * Q.cw);
            int blocks = (int)((n + 255) / 256);
            if (batch) {                                             // one launch for the plane in every frame
                const int cap = (132 * 8 + F.nframes - 1) / F.nframes;
                k_step_uncovered22<true><<<dim3(blocks < cap ? blocks : cap, 1, F.nframes), 256, 0, s>>>(F, k, factor);
            } else {
                if (blocks > 132 * 8) blocks = 132 * 8;
                k_step_uncovered22<false><<<blocks, 256, 0, s>>>(F, k, factor);
            }
            e = cudaGetLastError();
            *nlaunch += 1;
        }
    }
    return e;
}

}  // namespace j2p
