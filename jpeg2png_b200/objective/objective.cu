// objective.cu — libj2pobjective.so: the recording variants of the iteration kernels behind
// j2p_session_record_objective.
//
// A recording session (single frame or batch) iterates with these kernels instead of the solver's: the
// same bodies (gradient_packed_body.inc, project_tile_body.inc, project_tile22_body.cuh,
// project_generic_body.inc) compiled with REC, which adds the objective sums of the reference's -c log
// (record.cuh) and changes nothing else.  Every kernel runs with batch addressing, a single frame as a
// batch of one, so a frame's record does not depend on how many frames share its session.  Each frame
// keeps the CTAs, bands and tiles of its unrecorded batch launch (session.cu passes the sub-gradient's
// geometry), so its sums of g^2, and with them its iterates, are the unrecorded ones bit for bit.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../csrc/gradient_packed_body.cuh"
#include "../csrc/project_generic_body.cuh"
#include "../csrc/project_tile22_body.cuh"
#include "../csrc/project_tile_body.cuh"

namespace j2p {

template <int NC_, bool TGV_, int GPM_>
__global__ void J2P_GRAD_BOUNDS k_gradient_packed_rec(const __grid_constant__ FrameDev F, const float factor, const int band_rows,
                                                      const __grid_constant__ RecDev R) {
    constexpr int NC = NC_, GPM = GPM_;
    constexpr bool TGV = TGV_, BATCH = true, REC = true;
    const GridGeo geo{};
#include "../csrc/gradient_packed_body.inc"
}

template <bool RES_>
__global__ void __launch_bounds__(PT_NT, J2P_TILE_MIN_CTAS) k_project_tile_rec(const __grid_constant__ FrameDev F, const int c0, const float factor,
                                                                             const __grid_constant__ RecDev R) {
    constexpr bool RES = RES_, BATCH = true, REC = true;
    const GridGeo geo{};
#include "../csrc/project_tile_body.inc"
}

__global__ void __launch_bounds__(P22_NT, 3) k_project_tile22_rec(const __grid_constant__ FrameDev F, const int c0, const float factor,
                                                                 const __grid_constant__ RecDev R) {
    project_tile22_body<true, GridGeo, true>(F, c0, factor, GridGeo{}, &R);
}

// one frame per launch (the frame's view, kernels.cuh frame_view); R.pp is that frame's
template <int SW, int SH>
__global__ void __launch_bounds__(P_NT, (SW * SH <= 1) ? J2P_PROJ_MIN_CTAS : 2) k_project_rec(const __grid_constant__ FrameDev F, const ProjPlane G, const float factor,
                                                                                           const __grid_constant__ RecDev R) {
    constexpr bool REC = true;
#include "../csrc/project_generic_body.inc"
}

template <bool TGV, int GPM>
static void *grad_kernel(int nc) {
    switch (nc) {
        case 1: return (void *)k_gradient_packed_rec<1, TGV, GPM>;
        case 2: return (void *)k_gradient_packed_rec<2, TGV, GPM>;
        default: return (void *)k_gradient_packed_rec<3, TGV, GPM>;
    }
}

static cudaError_t launch(void *kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t s, bool chain, void **args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    // the chain of the unrecorded path (pdl.cuh): the gradient and the tile projections are programmatic
    // dependents of the kernel before them; the generic projection is a plain launch
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = chain && pdl_enabled() ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelExC(&cfg, kernel, args);
    if (e != cudaSuccess) cudaGetLastError();
    return e;
}

}  // namespace j2p

using namespace j2p;

// Once per device (the current one): the dynamic shared memory of the 2x2 tile kernel.
extern "C" int j2p_objective_configure(void) {
    const cudaError_t e = cudaFuncSetAttribute(k_project_tile22_rec, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P22_SMEM);
    if (e != cudaSuccess) cudaGetLastError();
    return (int)e;
}

// The recording sub-gradient of every frame of F on the grid (cx, bands) x frames with `rows` rows per
// band: the geometry of the unrecorded launch (session.cu, packed_gradient_geometry).  Returns a cudaError_t.
extern "C" int j2p_objective_gradient(const FrameDev *F, float factor, int cx, int bands, int rows, int gpm, const RecDev *R, void *stream) {
    void *k;
    if (gpm == 2) k = F->use_tgv ? (void *)k_gradient_packed_rec<3, true, 2> : (void *)k_gradient_packed_rec<3, false, 2>;
    else if (gpm == 1) k = F->use_tgv ? grad_kernel<true, 1>(F->nc) : grad_kernel<false, 1>(F->nc);
    else k = F->use_tgv ? grad_kernel<true, 0>(F->nc) : grad_kernel<false, 0>(F->nc);
    void *args[] = {(void *)F, (void *)&factor, (void *)&rows, (void *)R};
    return (int)launch(k, dim3(cx, bands, F->nframes), dim3(GM_NT), 0, (cudaStream_t)stream, true, args);
}

// The recording projection of planes c .. c+count-1 of every frame of F (planes of one geometry; the
// generic kernel takes one plane).  Only the blocks: the pixels no block covers are stepped by the
// solver's own kernels (session.cu).  *nlaunch: kernels launched.  Returns a cudaError_t.
extern "C" int j2p_objective_project(const FrameDev *Fp, int c, int count, float factor, const RecDev *Rp, void *stream, int *nlaunch) {
    const FrameDev &F = *Fp;
    const cudaStream_t s = (cudaStream_t)stream;
    const PlaneDev &P = F.pl[c];
    const int bw = P.cw >> 3, bh = P.ch >> 3;
    cudaError_t e = cudaSuccess;
    *nlaunch = 0;
    if ((P.sw == 1 && P.sh == 1) || (P.sw == 2 && P.sh == 2)) {
        const bool p11 = P.sw == 1;
        const int gx = (bw + PT_NB - 1) / PT_NB;                    // PT_NB == P22_NB
        for (int y0 = 0; y0 < bh && e == cudaSuccess; y0 += kMaxGridRows) {   // one launch unless bh > 65535
            const int rows = bh - y0 < kMaxGridRows ? bh - y0 : kMaxGridRows;
            FrameDev V = y0 == 0 && rows == bh ? F : rows_view(F, c, count, y0, p11 ? 8 : 16, y0 + rows == bh);
            RecDev R = *Rp;
            R.row0 = (unsigned)y0;
            void *args[] = {(void *)&V, (void *)&c, (void *)&factor, (void *)&R};
            void *k = p11 ? (P.resample ? (void *)k_project_tile_rec<true> : (void *)k_project_tile_rec<false>) : (void *)k_project_tile22_rec;
            e = launch(k, dim3(gx * count, rows, F.nframes), dim3(p11 ? PT_NT : P22_NT), p11 ? 0 : P22_SMEM, s, true, args);
            *nlaunch += 1;
        }
        return (int)e;
    }
    // k_project_rec handles one frame: launched once per frame on that frame's view (kernels_project.cu)
    const int tw = 8 * P_BW * P.sw, th = 8 * P_BH * P.sh;
    ProjPlane G;
    G.c = c;
    G.gx = (F.W + tw - 1) / tw;
    const int gy = (F.H + th - 1) / th;
    void *k = P.sw == 2 && P.sh == 1 ? (void *)k_project_rec<2, 1> : (P.sw == 1 && P.sh == 2 ? (void *)k_project_rec<1, 2> : (void *)k_project_rec<0, 0>);
    for (int f = 0; f < F.nframes && e == cudaSuccess; f++) {
        const FrameDev Vf = F.nframes > 1 ? frame_view(F, f) : F;
        for (int y0 = 0; y0 < gy && e == cudaSuccess; y0 += kMaxGridRows) {
            const int rows = gy - y0 < kMaxGridRows ? gy - y0 : kMaxGridRows;
            FrameDev V = y0 == 0 && rows == gy ? Vf : rows_view(Vf, c, 1, y0 * P_BH, 8 * P.sh, y0 + rows == gy);
            RecDev R = *Rp;
            R.pp += (size_t)f * 3 * R.pp_stride;
            R.row0 = (unsigned)y0;
            void *args[] = {(void *)&V, (void *)&G, (void *)&factor, (void *)&R};
            e = launch(k, dim3(G.gx, rows), dim3(P_NT), 0, s, false, args);
            *nlaunch += 1;
        }
    }
    return (int)e;
}

// Partials the projection of one frame writes for plane c (RecDev::pp_count): one per CTA of the tile
// kernels, one per block slot of the generic kernel.
extern "C" unsigned j2p_objective_partials(const FrameDev *F, int c) {
    const PlaneDev &P = F->pl[c];
    const unsigned bw = (unsigned)P.cw >> 3, bh = (unsigned)P.ch >> 3;
    if ((P.sw == 1 && P.sh == 1) || (P.sw == 2 && P.sh == 2)) return (bw + PT_NB - 1) / PT_NB * bh;
    const unsigned tw = 8 * P_BW * P.sw, th = 8 * P_BH * P.sh;
    return (unsigned)((F->W + tw - 1) / tw) * ((F->H + th - 1) / th) * (P_NT / 8);
}
