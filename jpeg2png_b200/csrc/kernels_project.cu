// kernels_project.cu — step + projection kernel, conventional decode, aux_init.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "kernels.cuh"
#include "project_generic_body.cuh"
#include "numerics.cuh"
#include "project_common.cuh"
#include "strip_sync.cuh"
#include "tma_maps.h"


namespace j2p {

cudaError_t launch_project_tile(const FrameDev &F, int c, int count, float factor, cudaStream_t s, int *nlaunch, bool uncovered_only);
cudaError_t configure_project_tma();
bool project_tma_enabled();
cudaError_t launch_project_tma(const FrameDev &F, const TileMaps &M, int c, int count, int xsel, float factor, cudaStream_t s);
cudaError_t configure_project_tile22();
cudaError_t launch_project_tile22(const FrameDev &F, int c, int count, float factor, cudaStream_t s, int *nlaunch, bool uncovered_only);

// k_project — 8 threads per coefficient block (thread j owns row j), 32 blocks per CTA; constants and
// layout in project_generic_body.cuh, the body in project_generic_body.inc.
template <int SW, int SH>
__global__ void __launch_bounds__(P_NT, (SW * SH <= 1) ? J2P_PROJ_MIN_CTAS : 2) k_project(const __grid_constant__ FrameDev F, const ProjPlane G, const float factor) {
    constexpr bool REC = false;          // the recording variant is k_project_rec (libj2pobjective.so)
    const RecDev R{};
#include "project_generic_body.inc"
}

// ------------------------------------------------------------------------------------------
// set-up kernels
// ------------------------------------------------------------------------------------------
// conventional decode of one plane: dequantise + IDCT + raster (jpeg.c:83-92, jpeg2png.c:131-139)
struct QTable { float q[64]; };                                             // by value: 256 B of kernel parameters, no device copy to manage
__global__ void __launch_bounds__(P_NT) k_decode(const int16_t *data, const __grid_constant__ QTable qt, float *out, int cw, int ch) {
    const float *q = qt.q;
    __shared__ __align__(16) float tiles[P_NT / 8][TILE_STRIDE];
    const int tid = threadIdx.x, b = tid >> 3, j = tid & 7;
    const int nb = (cw >> 3) * (ch >> 3);
    const int blk = blockIdx.x * (P_NT / 8) + b;
    if (blk >= nb) return;
    const int bw = cw >> 3, by = blk / bw, bx = blk - by * bw;
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int d = data[(size_t)blk * 64 + j * 8 + i];
        v[i] = __int2float_rn(d * (int)q[j * 8 + i]);                         // int product, one rounding (jpeg.c:88)
    }
    idct8x8_rows(v, tiles[b], j);
#pragma unroll
    for (int i = 0; i < 8; i++) out[(size_t)(by * 8 + j) * cw + bx * 8 + i] = v[i];
}

// aux_init (compute.c:295-309): nearest-neighbour upsample with edge clamp into x and xp
__global__ void k_init_plane(const float *fdata, float *x, float *xp, int W, int H, int cw, int ch, int sw, int sh) {
    const size_t n = (size_t)W * H;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int py = (int)(i / W), px = (int)(i - (size_t)py * W);
        int cx = px / sw, cy = py / sh;
        cx = cx < cw - 1 ? cx : cw - 1;
        cy = cy < ch - 1 ? cy : ch - 1;
        const float v = fdata[(size_t)cy * cw + cx];
        x[i] = v;
        xp[i] = v;
    }
}

// ------------------------------------------------------------------------------------------
// host-side launchers
// ------------------------------------------------------------------------------------------
// 2x2 planes (4:2:0 chroma) go through kernels_project_tile22.cu (coalesced staging; bit-identical
// on the whole GPU suite).
// J2P_PROJ_TILE22=0 selects the register-footprint kernel k_project<2,2> instead (A/B aid; it is
// also what the objective-logging build uses).
static bool g_tile22 = true;

cudaError_t configure_project_kernels() {
    const char *e = getenv("J2P_PROJ_TILE22");
    g_tile22 = !(e && *e == '0');
    const cudaError_t rc = configure_project_tma();
    return rc != cudaSuccess ? rc : configure_project_tile22();
}

// strip sessions: fold the per-rank sums of g^2 in rank order (deterministic), then the norms of
// compute.c:200-206 and their reciprocals
__global__ void k_fold_sums(const double *sums_by_rank, int nranks, int nc, float *norms) {
    const int c = threadIdx.x;
    if (c >= nc) return;
    double s = 0.;
    for (int r = 0; r < nranks; r++) s = __dadd_rn(s, sums_by_rank[r * 3 + c]);
    const float norm = fsqrt(__double2float_rn(s));
    norms[c] = norm;
    norms[4 + c] = __frcp_rn(norm);
}

cudaError_t launch_fold_sums(const double *sums_by_rank, int nranks, int nc, float *norms, cudaStream_t s) {
    k_fold_sums<<<1, 32, 0, s>>>(sums_by_rank, nranks, nc, norms);
    return cudaGetLastError();
}

// *nlaunch: number of kernels launched (planes of one geometry share a launch)
cudaError_t launch_project(const FrameDev &Fin, float factor, cudaStream_t s, int *nlaunch) {
    *nlaunch = 0;
    // the projection is block-local: it only sees the rows the session owns (no halo rows)
    FrameDev F = Fin;
    if (F.t0 != 0 || F.t1 != F.H) {
        const size_t off = (size_t)F.t0 * F.W;
        for (int c = 0; c < F.nc; c++) {
            F.pl[c].x += off;
            F.pl[c].xp += off;
            F.pl[c].g += off;
        }
        F.H = F.t1 - F.t0;
    }
    for (int c = 0; c < F.nc; c++) {
        const PlaneDev &P = F.pl[c];
        const int tw = 8 * P_BW * P.sw, th = 8 * P_BH * P.sh;
        ProjPlane G;
        G.c = c;
        G.gx = (F.W + tw - 1) / tw;
        const int gy = (F.H + th - 1) / th;
        // k_project's CTA rows in launches of at most kMaxGridRows (one launch unless the plane is that tall)
        auto each_rows = [&](const FrameDev &V, auto launch) {
            for (int y0 = 0; y0 < gy; y0 += kMaxGridRows) {
                const int rows = gy - y0 < kMaxGridRows ? gy - y0 : kMaxGridRows;
                launch(y0 == 0 && rows == gy ? V : rows_view(V, c, 1, y0 * P_BH, 8 * P.sh, y0 + rows == gy), dim3(G.gx, rows));
                *nlaunch += 1;
            }
        };
        if (F.log_on && P.sw == 1 && P.sh == 1) {
            each_rows(F, [&](const FrameDev &V, dim3 grid) { k_project<1, 1><<<grid, P_NT, 0, s>>>(V, G, factor); });   // the variant that also sums the log terms
        } else if (P.sw == 1 && P.sh == 1) {
            int count = 1;      // following planes of identical geometry ride in the same launch (grid.z; a batch: grid.x)
            while (c + count < F.nc && F.pl[c + count].sw == 1 && F.pl[c + count].sh == 1 && F.pl[c + count].cw == P.cw &&
                   F.pl[c + count].ch == P.ch)
                count++;
            // persistent TMA-fed kernel where the session has tensor maps; it takes the unrestricted frame
            const bool tma = Fin.host_maps != nullptr && project_tma_enabled();
            if (tma) {
                const cudaError_t et = launch_project_tma(Fin, *static_cast<const TileMaps *>(Fin.host_maps), c, count, Fin.buf_sel, factor, s);
                if (et != cudaSuccess) return et;
                *nlaunch += 1;
            }
            const cudaError_t eb = launch_project_tile(F, c, count, factor, s, nlaunch, tma);
            if (eb != cudaSuccess) return eb;
            c += count - 1;
        }
        else if (P.sw == 2 && P.sh == 2 && g_tile22 && !F.log_on) {
            int count = 1;      // Cb and Cr share one launch
            while (c + count < F.nc && F.pl[c + count].sw == 2 && F.pl[c + count].sh == 2 && F.pl[c + count].cw == P.cw &&
                   F.pl[c + count].ch == P.ch)
                count++;
            const cudaError_t eb = launch_project_tile22(F, c, count, factor, s, nlaunch, false);
            if (eb != cudaSuccess) return eb;
            c += count - 1;
        }
        else {
            // k_project<> handles one frame: a batch launches it once per frame on that frame's view
            for (int f = 0; f < F.nframes; f++) {
                each_rows(F.nframes > 1 ? frame_view(F, f) : F, [&](const FrameDev &V, dim3 grid) {
                    if (P.sw == 2 && P.sh == 2) k_project<2, 2><<<grid, P_NT, 0, s>>>(V, G, factor);
                    else if (P.sw == 2 && P.sh == 1) k_project<2, 1><<<grid, P_NT, 0, s>>>(V, G, factor);
                    else if (P.sw == 1 && P.sh == 2) k_project<1, 2><<<grid, P_NT, 0, s>>>(V, G, factor);
                    else k_project<0, 0><<<grid, P_NT, 0, s>>>(V, G, factor);
                });
            }
        }
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_decode(const int16_t *data, const float *q_host, float *out, int cw, int ch, cudaStream_t s) {
    const int nb = (cw / 8) * (ch / 8);
    QTable qt;
    for (int i = 0; i < 64; i++) qt.q[i] = q_host[i];
    k_decode<<<(nb + P_NT / 8 - 1) / (P_NT / 8), P_NT, 0, s>>>(data, qt, out, cw, ch);
    return cudaGetLastError();
}

cudaError_t launch_init_plane(const float *fdata, float *x, float *xp, int W, int H, int cw, int ch, int sw, int sh,
                              cudaStream_t s) {
    const size_t n = (size_t)W * H;
    int blocks = (int)((n + 255) / 256);
    if (blocks > 132 * 16) blocks = 132 * 16;
    k_init_plane<<<blocks, 256, 0, s>>>(fdata, x, xp, W, H, cw, ch, sw, sh);
    return cudaGetLastError();
}

}  // namespace j2p
