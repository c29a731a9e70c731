// kernels_project_tile.cu — step + projection of a full-resolution (1x1) plane with fully
// coalesced, swizzled staging through shared memory.
//
// The arithmetic organisation is the 8-threads-per-block one (thread j owns row j of its block;
// the three 2-D transforms alternate register butterflies with 8x8 shared-memory transposes).
// What this kernel changes is how the pixels travel.  When every thread fetches its own row, a
// warp-level 16-byte access touches 32 sectors and uses half of each: knock-out experiments showed
// that kernel spending more time on memory instructions alone (the L1 sector rate) than the fp64
// conversions need.  Here a CTA owns a
// tile of 16 blocks x 1 block (128 x 8 pixels); its 128 threads copy each 4 KB array with
// consecutive lanes on consecutive 16-byte pieces (cp.async, 512 contiguous bytes per warp
// instruction, every sector used once), into a layout whose 16-byte columns are XOR-swizzled by
// the row so that the per-row reads of the compute mapping are bank-conflict free.  Results go
// back the same way: rows into shared memory, then cooperative coalesced stores.
#include <cuda_runtime.h>
#include <stdint.h>

#include "project_tile_body.cuh"

namespace j2p {

// RES: the plane's coefficient grid is smaller than the frame (compute.c:338), e.g. 1080p luma.
// BATCH: a batch session (FrameDev::nframes); blockIdx.z = frame, blockIdx.x = k * (CTA columns) +
// column for planes c0 + k (a single frame: blockIdx.z = k).  A batch keeps gridDim.z for the frames,
// which may number 65535.
template <bool RES, bool BATCH>
__global__ void __launch_bounds__(PT_NT, J2P_TILE_MIN_CTAS) k_project_tile(const __grid_constant__ FrameDev F, const int c0, const float factor) {
    const GridGeo geo{};
    constexpr bool REC = false;          // the recording variant is k_project_tile_rec (libj2pobjective.so)
    const RecDev R{};
#include "project_tile_body.inc"
}

// Frame pixels of a 1x1 plane that no coefficient block covers (1080p: luma rows 1080..1087) are
// only stepped: compute_projection never visits them (compute.c:349-350).  The region is the
// bottom band (rows >= ch, full width) plus the right band (rows < ch, columns >= cw).
// BATCH: the frame is blockIdx.z.
template <bool BATCH>
__global__ void k_step_uncovered(const __grid_constant__ FrameDev F, const int c, const float factor) {
    step_uncovered_body<BATCH>(F, c, factor, GridGeo{});
}

static cudaError_t launch_step_uncovered(const FrameDev &F, int c, float factor, cudaStream_t s) {
    const PlaneDev &P = F.pl[c];
    const size_t n = (size_t)(F.H - P.ch) * F.W + (size_t)P.ch * (F.W - P.cw);
    int blocks = (int)((n + 255) / 256);
    if (F.nframes > 1) {                                         // one launch for the plane in every frame
        const int cap = (132 * 8 + F.nframes - 1) / F.nframes;
        k_step_uncovered<true><<<dim3(blocks < cap ? blocks : cap, 1, F.nframes), 256, 0, s>>>(F, c, factor);
        return cudaGetLastError();
    }
    if (blocks > 132 * 8) blocks = 132 * 8;
    k_step_uncovered<false><<<blocks, 256, 0, s>>>(F, c, factor);
    return cudaGetLastError();
}

// CTAs of plane P per block row: what calls strip_border_done per side and iteration (session.cu counts them)
int project_tile_border_units(const PlaneDev &P) { return ((P.cw >> 3) + PT_NB - 1) / PT_NB; }

// F: already restricted to the rows the session owns (launch_project).  Projects planes
// c .. c+count-1, which must all be 1x1 planes with the same coefficient grid.
// uncovered_only: the tiles have been projected by the TMA kernel; only the stepped-only pixels remain
cudaError_t launch_project_tile(const FrameDev &F, int c, int count, float factor, cudaStream_t s, int *nlaunch, bool uncovered_only) {
    const PlaneDev &P = F.pl[c];
    const int bw = P.cw >> 3, bh = P.ch >> 3, gx = (bw + PT_NB - 1) / PT_NB;
    const bool batch = F.nframes > 1;
    cudaError_t e = cudaSuccess;
    for (int y0 = 0; y0 < bh && !uncovered_only && e == cudaSuccess; y0 += kMaxGridRows) {   // one launch unless bh > 65535
        const int rows = bh - y0 < kMaxGridRows ? bh - y0 : kMaxGridRows;
        const FrameDev V = y0 == 0 && rows == bh ? F : rows_view(F, c, count, y0, 8, y0 + rows == bh);
        const dim3 grid = batch ? dim3(gx * count, rows, F.nframes) : dim3(gx, rows, count);
        if (batch)
            e = P.resample ? launch_chain(k_project_tile<true, true>, grid, dim3(PT_NT), 0, s, V, c, factor) : launch_chain(k_project_tile<false, true>, grid, dim3(PT_NT), 0, s, V, c, factor);
        else
            e = P.resample ? launch_chain(k_project_tile<true, false>, grid, dim3(PT_NT), 0, s, V, c, factor) : launch_chain(k_project_tile<false, false>, grid, dim3(PT_NT), 0, s, V, c, factor);
        *nlaunch += 1;
    }
    for (int k = c; k < c + count && e == cudaSuccess; k++)
        if (F.pl[k].cw < F.W || F.pl[k].ch < F.H) {
            e = launch_step_uncovered(F, k, factor, s);
            *nlaunch += 1;
        }
    return e;
}

}  // namespace j2p
