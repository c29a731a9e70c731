// kernels_project.cu — step + projection kernel, conventional decode, aux_init.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "kernels.cuh"
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
cudaError_t launch_project_tile22(const FrameDev &F, int c, int count, float factor, cudaStream_t s, int *nlaunch);

// ------------------------------------------------------------------------------------------
// k_project — 8 threads per coefficient block (thread j owns row j), 32 blocks per CTA.
// Template <SW, SH>: compile-time sampling factors of the plane (float4 I/O, stepped values of
// the whole footprint kept in registers); SW == 0 selects the run-time generic path.
// ------------------------------------------------------------------------------------------
#ifndef J2P_PBW_LOG2
#define J2P_PBW_LOG2 5     // CTA tile = 2^k blocks wide: 32 x 1 blocks = 1 KB contiguous per plane row (DRAM locality)
#endif
constexpr int P_NT = 256, P_BW = 1 << J2P_PBW_LOG2, P_BH = (P_NT / 8) / P_BW;   // CTA tile in coefficient blocks

struct ProjPlane {
    int c;          // plane index
    int gx;         // CTAs per row
};

#ifndef J2P_PROJ_MIN_CTAS
#define J2P_PROJ_MIN_CTAS 4     // resident CTAs per SM for full-resolution planes (register bound 64)
#endif

template <int SW, int SH>
__global__ void __launch_bounds__(P_NT, (SW * SH <= 1) ? J2P_PROJ_MIN_CTAS : 2) k_project(const __grid_constant__ FrameDev F, const ProjPlane G, const float factor) {
    __shared__ __align__(16) float tiles[2][P_NT / 8][TILE_STRIDE];
    __shared__ __align__(16) float sq[3][64];          // q, q*q, RN(1/(q*q)) of this plane
    __shared__ float snorm[2];                         // norm of g, RN(1/norm)   (from k_gradient)
    const int tid = threadIdx.x;
    const int c = G.c;
    const PlaneDev &P = F.pl[c];
    const int ctax = blockIdx.x, ctay = blockIdx.y;
    const int W = F.W, H = F.H;
    const int b = tid >> 3, j = tid & 7;
    const int bx = ctax * P_BW + (b & (P_BW - 1)), by = ctay * P_BH + (b >> J2P_PBW_LOG2);
    const bool real = bx < (P.cw >> 3) && by < (P.ch >> 3);
    const int sw = SW ? SW : P.sw, sh = SW ? SH : P.sh;
    const int cy = by * 8 + j;

    // Everything that comes from HBM is requested before the first wait: the coefficient row, for
    // full-resolution planes the eight pixels of x_k, x_{k-1} and g, and (one thread) the norm.
    int4 draw = make_int4(0, 0, 0, 0);
    float4 ra[2], rp[2], rg[2];
    if (real) {
        draw = __ldg(reinterpret_cast<const int4 *>(P.data + ((size_t)(by * (P.cw >> 3) + bx) * 64 + j * 8)));
        if constexpr (SW == 1 && SH == 1) {
            const size_t gi = (size_t)cy * W + (size_t)bx * 8;
#pragma unroll
            for (int k = 0; k < 2; k++) {
                ra[k] = reinterpret_cast<const float4 *>(P.x + gi)[k];
                rp[k] = reinterpret_cast<const float4 *>(P.xp + gi)[k];
                rg[k] = reinterpret_cast<const float4 *>(P.g + gi)[k];
            }
        }
    }
    if (tid < 64) {
        sq[0][tid] = F.q[c][tid];
        sq[1][tid] = F.qq[c][tid];
        sq[2][tid] = F.rqq[c][tid];
    } else if (tid < 96) {
        strip_norm(F, c, snorm, tid - 64);                         // whole frame: what k_gradient left; strips: fold of every rank's sums
    }
    __syncthreads();
    Stepper stepper;
    stepper.factor = factor;
    stepper.step = F.step;
    stepper.norm = snorm[0];
    stepper.rn = snorm[1];
    stepper.stepping = stepper.norm != 0.f;                        // compute.c:211
    const bool norm_ok = qdiv_divisor_ok(stepper.norm);
    float *tileA = tiles[0][b], *tileB = tiles[1][b];

    if (!real) {
        // pixels of the frame that no coefficient block covers: step only (compute.c:349-350 never visits them)
        for (int i = 0; i < 8; i++)
            for (int sy = 0; sy < sh; sy++)
                for (int sx = 0; sx < sw; sx++) {
                    const int px = (bx * 8 + i) * sw + sx, py = cy * sh + sy;
                    if (px < W && py < H) {
                        const size_t gi = (size_t)py * W + px;
                        P.xp[gi] = stepper(P.x[gi], P.xp[gi], P.g[gi]);
                    }
                }
        return;   // whole 8-lane groups leave together; the remaining lanes still __syncwarp among themselves
    }

    // ---- stepped point of the footprint, block-row means (compute.c:348-370) ------------------
    constexpr int ZW = SW ? SW * 8 : 1, ZH = SW ? SH : 1;
    float z[ZH][ZW];
    float v[8], mean[8];
    if constexpr (SW > 0) {
        unsigned key = 0xffffffffu;
#pragma unroll
        for (int sy = 0; sy < SH; sy++) {
            const size_t gi = (size_t)(cy * SH + sy) * W + (size_t)bx * 8 * SW;
            const float4 *xr = reinterpret_cast<const float4 *>(P.x + gi);
            const float4 *pr = reinterpret_cast<const float4 *>(P.xp + gi);
            const float4 *gr = reinterpret_cast<const float4 *>(P.g + gi);
#pragma unroll
            for (int k = 0; k < SW * 2; k++) {
                float4 a, p, g;
                if constexpr (SW == 1 && SH == 1) {
                    a = ra[k]; p = rp[k]; g = rg[k];
                } else {
                    a = xr[k]; p = pr[k]; g = gr[k];
                }
                z[sy][k * 4 + 0] = stepper.fast(a.x, p.x, g.x, key);
                z[sy][k * 4 + 1] = stepper.fast(a.y, p.y, g.y, key);
                z[sy][k * 4 + 2] = stepper.fast(a.z, p.z, g.z, key);
                z[sy][k * 4 + 3] = stepper.fast(a.w, p.w, g.w, key);
            }
        }
        if (stepper.stepping && !(norm_ok && key >= QDIV_KEY_MIN)) {   // outside the proven range: IEEE division
#pragma unroll
            for (int sy = 0; sy < SH; sy++) {
                const size_t gi = (size_t)(cy * SH + sy) * W + (size_t)bx * 8 * SW;
#pragma unroll
                for (int k = 0; k < SW * 8; k++) z[sy][k] = stepper(P.x[gi + k], P.xp[gi + k], P.g[gi + k]);
            }
        }
#pragma unroll
        for (int i = 0; i < 8; i++) {
            if (SW * SH > 1 || P.resample) {
                float m = 0.f;                                               // compute.c:351
#pragma unroll
                for (int sy = 0; sy < SH; sy++)
#pragma unroll
                    for (int sx = 0; sx < SW; sx++) m = fadd(m, z[sy][i * SW + sx]);
                constexpr int CNT = SW * SH;
                if constexpr ((CNT & (CNT - 1)) == 0) m = fmul(m, 1.0f / CNT);   // exact: power-of-two divisor
                else m = fdiv(m, (float)CNT);                                // compute.c:359
                mean[i] = m;
                v[i] = m;
            } else {
                mean[i] = 0.f;
                v[i] = z[0][i];
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int cx = bx * 8 + i;
            if (P.resample) {
                float m = 0.f;
                for (int sy = 0; sy < sh; sy++)
                    for (int sx = 0; sx < sw; sx++) {
                        const size_t gi = (size_t)(cy * sh + sy) * W + cx * sw + sx;
                        m = fadd(m, stepper(P.x[gi], P.xp[gi], P.g[gi]));
                    }
                m = fdiv(m, P.cnt);
                mean[i] = m;
                v[i] = m;
            } else {
                const size_t gi = (size_t)cy * W + cx;
                mean[i] = 0.f;
                v[i] = stepper(P.x[gi], P.xp[gi], P.g[gi]);
            }
        }
    }

    fdct8x8_rows(v, tileA, j);

    // ---- clamp to the quantisation interval (compute.c:323-331); DCT-distance residual ---------
    const int dw[4] = {draw.x, draw.y, draw.z, draw.w};
    float qv[8], qqv[8], rqv[8];
    {
        const float4 *t0 = reinterpret_cast<const float4 *>(&sq[0][j * 8]);
        const float4 *t1 = reinterpret_cast<const float4 *>(&sq[1][j * 8]);
        const float4 *t2 = reinterpret_cast<const float4 *>(&sq[2][j * 8]);
#pragma unroll
        for (int k = 0; k < 2; k++) {
            const float4 a = t0[k], bq = t1[k], cq = t2[k];
            qv[k * 4] = a.x; qv[k * 4 + 1] = a.y; qv[k * 4 + 2] = a.z; qv[k * 4 + 3] = a.w;
            qqv[k * 4] = bq.x; qqv[k * 4 + 1] = bq.y; qqv[k * 4 + 2] = bq.z; qqv[k * 4 + 3] = bq.w;
            rqv[k * 4] = cq.x; rqv[k * 4 + 1] = cq.y; rqv[k * 4 + 2] = cq.z; rqv[k * 4 + 3] = cq.w;
        }
    }
    float r[8], num[8];
    unsigned rkey = 0xffffffffu;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int di = (i & 1) ? (dw[i >> 1] >> 16) : (int)(short)(dw[i >> 1] & 0xffff);
        const float d = (float)di;
        const float q = qv[i];
        const float lo = fmul(fsub(d, 0.5f), q), hi = fmul(fadd(d, 0.5f), q);
        float t = v[i];
        t = t > hi ? hi : (t < lo ? lo : t);
        v[i] = t;
        num[i] = fsub(t, fmul(d, q));                                        // compute.c:47
        rkey = min(rkey, qdiv_key(num[i]));
        r[i] = qdiv_core(num[i], qqv[i], rqv[i]);                            // compute.c:49; q*q in [1, 2^32] is always a valid divisor
    }
    if (rkey < QDIV_KEY_MIN) {                                               // a residual below 2^-60: IEEE division
#pragma unroll
        for (int i = 0; i < 8; i++) r[i] = fdiv(num[i], qqv[i]);
    }
    if (F.log_on && P.use_prob) {
        // objective term of the NEXT iteration: sum of (residual/q)^2 (compute_simd_step.c:22-26), fp64
        double loc = 0.;
#pragma unroll
        for (int i = 0; i < 8; i++) loc = __dadd_rn(loc, (double)fsq(fdiv(num[i], qv[i])));
        const unsigned gmask = 0xffu << (tid & 24);
        loc = __dadd_rn(loc, __shfl_xor_sync(gmask, loc, 1));
        loc = __dadd_rn(loc, __shfl_xor_sync(gmask, loc, 2));
        loc = __dadd_rn(loc, __shfl_xor_sync(gmask, loc, 4));
        if (j == 0) atomicAdd(&F.logsums[2 + 3 * F.log_slot + c], loc);
    }

    if (P.use_prob) {
        idct8x8_rows_x2(v, r, tileA, tileB, j);
    } else {
        idct8x8_rows(v, tileA, j);
    }
    if (P.use_prob) {
        float4 *gprow = reinterpret_cast<float4 *>(P.gp + (size_t)cy * P.cw + bx * 8);
        const float pa = P.p_alpha;                                          // compute.c:62 (the product)
        gprow[0] = make_float4(fmul(pa, r[0]), fmul(pa, r[1]), fmul(pa, r[2]), fmul(pa, r[3]));
        gprow[1] = make_float4(fmul(pa, r[4]), fmul(pa, r[5]), fmul(pa, r[6]), fmul(pa, r[7]));
    }

    // ---- write x_{k+1} (compute.c:387-403) -------------------------------------------------------
    if constexpr (SW > 0) {
        if (SW * SH > 1 || P.resample) {
#pragma unroll
            for (int sy = 0; sy < SH; sy++) {
                float4 *o = reinterpret_cast<float4 *>(P.xp + (size_t)(cy * SH + sy) * W + (size_t)bx * 8 * SW);
#pragma unroll
                for (int k = 0; k < SW * 2; k++) {
                    float e[4];
#pragma unroll
                    for (int m = 0; m < 4; m++) {
                        const int col = k * 4 + m, i = col / SW;
                        e[m] = fadd(fsub(z[sy][col], mean[i]), v[i]);
                    }
                    o[k] = make_float4(e[0], e[1], e[2], e[3]);
                }
            }
        } else {
            float4 *o = reinterpret_cast<float4 *>(P.xp + (size_t)cy * W + (size_t)bx * 8);
            o[0] = make_float4(v[0], v[1], v[2], v[3]);
            o[1] = make_float4(v[4], v[5], v[6], v[7]);
        }
    } else {
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int cx = bx * 8 + i;
            if (P.resample) {
                for (int sy = 0; sy < sh; sy++)
                    for (int sx = 0; sx < sw; sx++) {
                        const size_t gi = (size_t)(cy * sh + sy) * W + cx * sw + sx;
                        const float zz = stepper(P.x[gi], P.xp[gi], P.g[gi]);
                        P.xp[gi] = fadd(fsub(zz, mean[i]), v[i]);
                    }
            } else {
                P.xp[(size_t)cy * W + cx] = v[i];
            }
        }
    }
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
            const cudaError_t eb = launch_project_tile22(F, c, count, factor, s, nlaunch);
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
