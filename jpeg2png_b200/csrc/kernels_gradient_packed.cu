// kernels_gradient_packed.cu — the production sub-gradient kernel: k_gradient on pixel pairs.
//
// Same algorithm, same order of IEEE operations and therefore the same bits as the scalar
// k_gradient of kernels_gradient.cu (which stays as the objective-logging build): FISTA point
// (compute.c:431-440), TV (compute.c:73-113) and second-order TGV (compute.c:128-186) sub-gradient
// as an ordered per-pixel gather (SURVEY.md §8a), the DCT-distance term from `gp`, per-CTA fp64
// sums of g^2 and the last-CTA fold into the norms of compute.c:200-206.
//
// What changed is how the work is organised.  A lane owns two adjacent columns and runs the
// identical sequence on both; the two columns live in one 64-bit register pair (`f2`,
// numerics.cuh), each pair operation being two explicitly rounded scalar fp32 instructions on
// sm_90.  On top of that:
//   * the row-to-row state is ping-ponged between two register sets by unrolling two row steps
//     with swapped roles, which removes the ~45 register copies per row of the scalar kernel;
//   * the DCT-distance term enters as fma(gp, mask, 0) — one instruction that is both the
//     "0 + gp" of compute.c:62 and the validity select;
//   * dead sources are made harmless before the square root (norm^2 := 1, reciprocal := 0) instead
//     of after it, which halves the selects per pixel;
//   * rows travel through a per-warp ring in shared memory, GM_DEPTH rows ahead, filled with cp.async
//     (every lane copies its own 8 bytes and later reads them back itself: no barrier, only
//     cp.async.wait_group).  With the loads held in registers one row ahead, 12 warps x 2.3 KB were
//     all an SM had in flight, and by Little's law that caps the kernel's bandwidth whatever the
//     instruction count;
//   * for strip sessions the two exchanges of an iteration are part of the kernel (strip_sync.cuh).
#include <cuda_runtime.h>
#include <stdint.h>

#include "gradient_packed_body.cuh"

namespace j2p {

// BATCH: a batch session (kernels.cuh, FrameDev::nframes); the frame is blockIdx.z and every frame
// has the grid a single-frame session of its geometry gets.  Its base is formed once, in 64 bits;
// the offsets inside a frame stay 32-bit.  !BATCH compiles to the single-frame kernel unchanged.
template <int NC, bool TGV, int GPM, bool BATCH>
__global__ void J2P_GRAD_BOUNDS k_gradient_packed(const __grid_constant__ FrameDev F, const float factor, const int band_rows) {
    const GridGeo geo{};
    constexpr bool REC = false;          // the recording variant is k_gradient_packed_rec (libj2pobjective.so)
    const RecDev R{};
#include "gradient_packed_body.inc"
}

// ------------------------------------------------------------------------------------------
// host-side launcher (geometry shared with the scalar kernel: grad_geometry in kernels_gradient.cu)
// ------------------------------------------------------------------------------------------
void grad_geometry(int W, int H, int slots, int *ctas_x, int *bands, int *band_rows);

// CTAs of one kernel instantiation resident on the current device at once.  Per instantiation, not
// per kernel family: the one-channel builds (separate mode, -s) need 72..86 registers and fit five
// CTAs per SM where the three-channel joint build fits two — a band geometry sized for the wrong one
// leaves most of the machine idle.
static int sm_count() {
    static int sms[64];
    int dev = 0;
    cudaGetDevice(&dev);
    int &n = sms[dev & 63];
    if (n == 0 && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
        cudaGetLastError();
        n = 132;
    }
    return n;
}
// A batch launches the batched instantiation with every frame on the grid a single-frame session of
// that geometry gets: the band geometry comes from the SINGLE-FRAME instantiation's occupancy, so each
// frame's sums of g^2 are folded in the same order as in its own session (DESIGN.md §7b).
template <int NC, bool TGV, int GPM>
static int instance_per_sm() {
    static const int per_sm = [] {
        int n = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_gradient_packed<NC, TGV, GPM, false>, GM_NT, 0) != cudaSuccess) {
            cudaGetLastError();
            n = 0;
        }
        return n > 0 ? n : 1;
    }();
    return per_sm;
}
template <int NC, bool TGV, int GPM>
static cudaError_t launch_instance(const FrameDev &F, float factor, cudaStream_t s) {
    int cx, bands, rows;
    grad_geometry(F.W, F.t1 - F.t0, sm_count() * instance_per_sm<NC, TGV, GPM>(), &cx, &bands, &rows);
    if (F.nframes > 1) return launch_chain(k_gradient_packed<NC, TGV, GPM, true>, dim3(cx, bands, F.nframes), dim3(GM_NT), 0, s, F, factor, rows);
    return launch_chain(k_gradient_packed<NC, TGV, GPM, false>, dim3(cx, bands), dim3(GM_NT), 0, s, F, factor, rows);
}
template <bool TGV, int GPM>
static cudaError_t launch_packed_nc(const FrameDev &F, float factor, cudaStream_t s) {
    switch (F.nc) {
        case 1: return launch_instance<1, TGV, GPM>(F, factor, s);
        case 2: return launch_instance<2, TGV, GPM>(F, factor, s);
        default: return launch_instance<3, TGV, GPM>(F, factor, s);
    }
}
template <bool TGV, int GPM>
static int per_sm_nc(int nc) {
    switch (nc) {
        case 1: return instance_per_sm<1, TGV, GPM>();
        case 2: return instance_per_sm<2, TGV, GPM>();
        default: return instance_per_sm<3, TGV, GPM>();
    }
}

int packed_gradient_occupancy() {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_gradient_packed<3, true, 1, false>, GM_NT, 0) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return per_sm;
}

// How the DCT-distance term of F is addressed: the kernel's GPM
int packed_gradient_gpm(const FrameDev &F) {
    const int owned = F.t1 - F.t0;
    bool full = true;      // every plane at full resolution over the whole (local) frame: gp has the frame's geometry
    for (int c = 0; c < F.nc; c++) full = full && F.pl[c].sw == 1 && F.pl[c].sh == 1 && F.pl[c].cw == F.W && F.pl[c].ch >= owned;
    // 4:2:0 with aligned grids: luma full width (its last rows may be missing: 1080p), both chroma planes exactly half
    bool c420 = F.nc == 3 && F.pl[0].sw == 1 && F.pl[0].sh == 1 && F.pl[0].cw == F.W;
    for (int c = 1; c < 3 && c420; c++) c420 = F.pl[c].sw == 2 && F.pl[c].sh == 2 && 2 * F.pl[c].cw == F.W && F.pl[c].ch == F.pl[1].ch;
    return full ? 1 : (c420 ? 2 : 0);
}

// The grid launch_instance gives a frame of F's geometry: CTA columns, bands, rows per band.  A group
// (j2p_session_iterate_group) gives every frame this grid, so its sums of g^2 fold in the same order.
void packed_gradient_geometry(const FrameDev &F, int *cx, int *bands, int *rows) {
    const int gpm = packed_gradient_gpm(F);
    int per_sm;
    if (gpm == 2) per_sm = F.use_tgv ? instance_per_sm<3, true, 2>() : instance_per_sm<3, false, 2>();
    else if (gpm == 1) per_sm = F.use_tgv ? per_sm_nc<true, 1>(F.nc) : per_sm_nc<false, 1>(F.nc);
    else per_sm = F.use_tgv ? per_sm_nc<true, 0>(F.nc) : per_sm_nc<false, 0>(F.nc);
    grad_geometry(F.W, F.t1 - F.t0, sm_count() * per_sm, cx, bands, rows);
}

cudaError_t launch_gradient_packed(const FrameDev &F, float factor, cudaStream_t s) {
    const int gpm = packed_gradient_gpm(F);
    if (gpm == 1) return F.use_tgv ? launch_packed_nc<true, 1>(F, factor, s) : launch_packed_nc<false, 1>(F, factor, s);
    if (gpm == 2) return F.use_tgv ? launch_instance<3, true, 2>(F, factor, s) : launch_instance<3, false, 2>(F, factor, s);
    return F.use_tgv ? launch_packed_nc<true, 0>(F, factor, s) : launch_packed_nc<false, 0>(F, factor, s);
}

}  // namespace j2p
