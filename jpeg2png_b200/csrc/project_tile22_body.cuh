// project_tile22_body.cuh — the bodies of the tiled projection of 2x2 planes and of the step of the
// pixels beyond their coefficient grid (kernels_project_tile22.cu), shared by the single-frame and batch
// kernels of libjpeg2png_b200.so and the grouped kernels of libj2pmixed.so (mixed/mixed.cu).
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

constexpr int P22_NB = 16;                 // coefficient blocks per CTA tile (16 x 1)
constexpr int P22_NT = P22_NB * 8;         // 128 threads
constexpr int P22_C4 = P22_NB * 4;         // float4 columns per frame row of the tile (256 pixels)
constexpr int P22_G4 = P22_NB * 2;         // float4 columns per coefficient row of the tile (128 samples)
constexpr size_t P22_SMEM = (size_t)3 * 16 * P22_C4 * sizeof(float4)      // x_k, x_{k-1}, g
                            + (size_t)8 * P22_G4 * sizeof(float4)          // gp staging
                            + (size_t)P22_NB * TILE_STRIDE * sizeof(float) // transpose tiles
                            + 3 * 64 * sizeof(float) + 4 * sizeof(float);  // tables, norm

// REC (k_project_tile22_rec, objective/objective.cu; false everywhere else) also writes the CTA's sum of
// (residual/q)^2 to R->pp (record.cuh), behind `if constexpr (REC)`.
template <bool BATCH, class G, bool REC = false>
__device__ __forceinline__ void project_tile22_body(const FrameDev &F, const int c0, const float factor, const G &geo, const RecDev *R = nullptr) {
    __shared__ double rsum[REC ? P22_NB : 1];                        // REC: each block's sum of (residual/q)^2
    extern __shared__ __align__(16) unsigned char smem22[];
    float4 *sx = reinterpret_cast<float4 *>(smem22);                 // [16][P22_C4]  x_k  -> later x_{k+1}
    float4 *sp = sx + 16 * P22_C4;                                   // [16][P22_C4]  x_{k-1}
    float4 *sg = sp + 16 * P22_C4;                                   // [16][P22_C4]  g
    float4 *sgp = sg + 16 * P22_C4;                                  // [8][P22_G4]   gp out
    float *tiles = reinterpret_cast<float *>(sgp + 8 * P22_G4);      // [P22_NB][TILE_STRIDE]
    float *sq = tiles + P22_NB * TILE_STRIDE;                        // [3][64]
    float *snorm = sq + 3 * 64;                                      // [2]

    const int tid = threadIdx.x;
    const int frame = BATCH ? (int)geo.bz() : 0;
    const int gx = BATCH ? ((F.pl[c0].cw >> 3) + P22_NB - 1) / P22_NB : 0;   // CTA columns per plane
    const int k = BATCH ? (int)geo.bx() / gx : (int)geo.bz();
    const int c = c0 + k;                                            // planes of equal geometry share one launch
    const PlaneDev &P = F.pl[c];
    const size_t fo = BATCH ? (size_t)frame * F.frame_stride : 0;
    const int W = F.W;
    const int bw = P.cw >> 3;
    const int bx0 = (BATCH ? (int)geo.bx() - k * gx : (int)geo.bx()) * P22_NB;
    const int by = strip_row_order(F.sync, geo.by(), geo.ny());   // the grid covers real blocks only
    const int nbx = min(P22_NB, bw - bx0);
    const int valid_c4 = nbx * 4, valid_g4 = nbx * 2;
    const size_t row0 = (size_t)(by * 16) * W + (size_t)bx0 * 16;    // first frame pixel of the tile

    // ---- coalesced, swizzled copy-in: 16 rows x 64 pieces per array, 8 pieces per thread ----------
    // x_k and x_{k-1} of these planes are not written by the kernels this launch may overlap (the
    // gradient kernel, the luma projection; pdl.cuh): their tiles are requested
    // BEFORE the wait; the g tile follows it at once (kernels_project_tile.cu).
#pragma unroll
    for (int i = 0; i < 16 * P22_C4 / P22_NT; i++) {
        const int e = tid + P22_NT * i, row = e / P22_C4, c4 = e % P22_C4;
        if (c4 < valid_c4) {
            const size_t gi = row0 + (size_t)row * W + (size_t)c4 * 4;
            const int pc = row * P22_C4 + (c4 ^ ((row >> 1) & 7));
            cp_async16(&sx[pc], P.x + fo + gi);
            cp_async16(&sp[pc], P.xp + fo + gi);
        }
    }
    pdl_wait();                                                      // the gradient and its norm are complete and visible
    pdl_launch_dependents();
#pragma unroll
    for (int i = 0; i < 16 * P22_C4 / P22_NT; i++) {
        const int e = tid + P22_NT * i, row = e / P22_C4, c4 = e % P22_C4;
        if (c4 < valid_c4) cp_async16(&sg[row * P22_C4 + (c4 ^ ((row >> 1) & 7))], P.g + fo + row0 + (size_t)row * W + (size_t)c4 * 4);
    }
    cp_async_commit();
    const int b = tid >> 3, j = tid & 7;
    const bool real = b < nbx;
    int4 draw = make_int4(0, 0, 0, 0);
    if (real) draw = __ldg(reinterpret_cast<const int4 *>(P.data + (BATCH ? (size_t)frame * F.data_stride : 0) + ((size_t)(by * bw + bx0 + b) * 64 + j * 8)));
    if (tid < 64) {
        if (BATCH) {                                                 // this frame's tables (device copy)
            const float *t = F.tables + ((size_t)frame * F.nc + c) * 192;
            sq[tid] = t[tid];
            sq[64 + tid] = t[64 + tid];
            sq[128 + tid] = t[128 + tid];
        } else {
            sq[tid] = F.q[c][tid];
            sq[64 + tid] = F.qq[c][tid];
            sq[128 + tid] = F.rqq[c][tid];
        }
    }
    if (BATCH) {
        if (tid == 64) {                                             // what k_gradient left for this frame
            snorm[0] = F.norms[16 * frame + c];
            snorm[1] = F.norms[16 * frame + 4 + c];
        }
    } else if (tid >= 64 && tid < 96) {
        strip_norm(F, c, snorm, tid - 64);                           // whole frame: what k_gradient left; strips: fold of every rank's sums
    }
    cp_async_wait<0>();
    __syncthreads();

    Stepper stepper;
    stepper.factor = factor;
    stepper.step = F.step;
    stepper.norm = snorm[0];
    stepper.rn = snorm[1];
    stepper.stepping = stepper.norm != 0.f;                          // compute.c:211
    const bool norm_ok = qdiv_divisor_ok(stepper.norm);
    const bool use_prob = P.use_prob != 0;
    const unsigned gmask = 0xffu << (tid & 24);
    float *tile = tiles + b * TILE_STRIDE;
    double rloc = 0.;                                                // REC: this block's sum (0 for blocks beyond the plane)

    if (real) {
        // ---- stepped point of the 2 x 16 footprint (compute.c:436, :213) --------------------------
        float z[2][16], v[8], mean[8];
        {
            unsigned key = 0xffffffffu;
#pragma unroll
            for (int sy = 0; sy < 2; sy++) {
                const int rowbase = (2 * j + sy) * P22_C4;
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const int pc = rowbase + ((4 * b + k) ^ j);      // (row >> 1) & 7 == j
                    const float4 a = sx[pc], p = sp[pc], g = sg[pc];
                    z[sy][k * 4 + 0] = stepper.fast(a.x, p.x, g.x, key);
                    z[sy][k * 4 + 1] = stepper.fast(a.y, p.y, g.y, key);
                    z[sy][k * 4 + 2] = stepper.fast(a.z, p.z, g.z, key);
                    z[sy][k * 4 + 3] = stepper.fast(a.w, p.w, g.w, key);
                }
            }
            if (stepper.stepping && !(norm_ok && key >= QDIV_KEY_MIN)) {   // outside the proven range: IEEE division
#pragma unroll
                for (int sy = 0; sy < 2; sy++) {
                    const int rowbase = (2 * j + sy) * P22_C4;
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        const int pc = rowbase + ((4 * b + k) ^ j);
                        const float4 a = sx[pc], p = sp[pc], g = sg[pc];
                        z[sy][k * 4 + 0] = stepper(a.x, p.x, g.x);
                        z[sy][k * 4 + 1] = stepper(a.y, p.y, g.y);
                        z[sy][k * 4 + 2] = stepper(a.z, p.z, g.z);
                        z[sy][k * 4 + 3] = stepper(a.w, p.w, g.w);
                    }
                }
            }
        }
        // block-row means over the 2 x 2 samples, sy outer, sx inner (compute.c:351-360)
#pragma unroll
        for (int i = 0; i < 8; i++) {
            float m = 0.f;
            m = fadd(m, z[0][2 * i]);
            m = fadd(m, z[0][2 * i + 1]);
            m = fadd(m, z[1][2 * i]);
            m = fadd(m, z[1][2 * i + 1]);
            m = fmul(m, 0.25f);                                      // / (float)4: exact, power of two
            mean[i] = m;
            v[i] = m;
        }

        fdct8x8_rows(v, tile, j, gmask);

        // ---- clamp to the quantisation interval (compute.c:323-331); residual (compute.c:47-49) --
        const int dw[4] = {draw.x, draw.y, draw.z, draw.w};
        float r[8], num[8];
        unsigned rkey = 0xffffffffu;
        {
            const float4 *t0 = reinterpret_cast<const float4 *>(&sq[j * 8]);
            const float4 *t1 = reinterpret_cast<const float4 *>(&sq[64 + j * 8]);
            const float4 *t2 = reinterpret_cast<const float4 *>(&sq[128 + j * 8]);
            float qv[8], qqv[8], rqv[8];
#pragma unroll
            for (int k = 0; k < 2; k++) {
                const float4 a = t0[k], bq = t1[k], cq = t2[k];
                qv[k * 4] = a.x; qv[k * 4 + 1] = a.y; qv[k * 4 + 2] = a.z; qv[k * 4 + 3] = a.w;
                qqv[k * 4] = bq.x; qqv[k * 4 + 1] = bq.y; qqv[k * 4 + 2] = bq.z; qqv[k * 4 + 3] = bq.w;
                rqv[k * 4] = cq.x; rqv[k * 4 + 1] = cq.y; rqv[k * 4 + 2] = cq.z; rqv[k * 4 + 3] = cq.w;
            }
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const int di = (i & 1) ? (dw[i >> 1] >> 16) : (int)(short)(dw[i >> 1] & 0xffff);
                const float d = (float)di;
                const float q = qv[i];
                const float lo = fmul(fsub(d, 0.5f), q), hi = fmul(fadd(d, 0.5f), q);
                float t = v[i];
                t = t > hi ? hi : (t < lo ? lo : t);
                v[i] = t;
                num[i] = fsub(t, fmul(d, q));
                rkey = min(rkey, qdiv_key(num[i]));
                r[i] = qdiv_core(num[i], qqv[i], rqv[i]);
            }
            if (rkey < QDIV_KEY_MIN) {                               // a residual below 2^-60: IEEE division
#pragma unroll
                for (int i = 0; i < 8; i++) r[i] = fdiv(num[i], qqv[i]);
            }
            if constexpr (REC) {                                   // the block's sum of (residual/q)^2 (compute_simd_step.c:22-26), fp64
                if (use_prob) {
#pragma unroll
                    for (int i = 0; i < 8; i++) rloc = __dadd_rn(rloc, (double)fsq(fdiv(num[i], qv[i])));
                    rloc = __dadd_rn(rloc, __shfl_xor_sync(gmask, rloc, 1));
                    rloc = __dadd_rn(rloc, __shfl_xor_sync(gmask, rloc, 2));
                    rloc = __dadd_rn(rloc, __shfl_xor_sync(gmask, rloc, 4));
                }
            }
        }

        idct8x8_rows(v, tile, j, gmask);
        if (use_prob) idct8x8_rows(r, tile, j, gmask);

        // ---- x_{k+1} = (z - mean) + projected mean (compute.c:390-403), into this thread's own cells
#pragma unroll
        for (int sy = 0; sy < 2; sy++) {
            const int rowbase = (2 * j + sy) * P22_C4;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                float e[4];
#pragma unroll
                for (int m = 0; m < 4; m++) {
                    const int col = k * 4 + m, i = col >> 1;
                    e[m] = fadd(fsub(z[sy][col], mean[i]), v[i]);
                }
                sx[rowbase + ((4 * b + k) ^ j)] = make_float4(e[0], e[1], e[2], e[3]);
            }
        }
        if (use_prob) {
            const float pa = P.p_alpha;                              // compute.c:62 (the product)
#pragma unroll
            for (int h = 0; h < 2; h++)
                sgp[j * P22_G4 + ((2 * b + h) ^ j)] =
                    make_float4(fmul(pa, r[h * 4 + 0]), fmul(pa, r[h * 4 + 1]), fmul(pa, r[h * 4 + 2]), fmul(pa, r[h * 4 + 3]));
        }
    }
    if constexpr (REC) {
        if (j == 0) rsum[b] = rloc;
    }
    __syncthreads();
    if constexpr (REC) {                                             // the CTA's partial, blocks in order (record.cuh)
        if (tid == 0 && use_prob) {
            double sum = 0.;
            for (int k = 0; k < P22_NB; k++) sum = __dadd_rn(sum, rsum[k]);
            R->pp[((size_t)frame * 3 + c) * R->pp_stride + (size_t)(R->row0 + by) * gx + bx0 / P22_NB] = sum;
        }
    }

    // ---- coalesced copy-out: x_{k+1} over x_{k-1} (compute.c:387), gp for the next iteration ------
#pragma unroll
    for (int i = 0; i < 16 * P22_C4 / P22_NT; i++) {
        const int e = tid + P22_NT * i, row = e / P22_C4, c4 = e % P22_C4;
        if (c4 < valid_c4)
            *reinterpret_cast<float4 *>(P.xp + fo + row0 + (size_t)row * W + (size_t)c4 * 4) = sx[row * P22_C4 + (c4 ^ ((row >> 1) & 7))];
    }
    if (use_prob) {
        float *gp0 = P.gp + fo + (size_t)(by * 8) * P.cw + (size_t)bx0 * 8;
#pragma unroll
        for (int i = 0; i < 8 * P22_G4 / P22_NT; i++) {
            const int e = tid + P22_NT * i, row = e / P22_G4, c4 = e % P22_G4;
            if (c4 < valid_g4) *reinterpret_cast<float4 *>(gp0 + (size_t)row * P.cw + (size_t)c4 * 4) = sgp[row * P22_G4 + (c4 ^ row)];
        }
    }

    // ---- strips over peer memory: border rows into the neighbours' halo rows (kernels_project_tile.cu)
    const StripSync &S = F.sync;
    if (!BATCH && S.nranks > 1 && S.fused_halo) {
        const bool top = by == 0 && S.has_up, bottom = by == (int)geo.ny() - 1 && S.has_down;
        if (top || bottom) {
            for (int e = tid; e < 4 * P22_C4; e += P22_NT) {             // 2 rows x 64 pieces, top then bottom
                const int side = e / (2 * P22_C4), r = (e / P22_C4) & 1, c4 = e % P22_C4;
                if (c4 >= valid_c4 || !(side ? bottom : top)) continue;
                const int row = side ? 14 + r : r;
                float *dst = (side ? S.down_dst[c] : S.up_dst[c]) + (size_t)r * W + (size_t)bx0 * 16 + (size_t)c4 * 4;
                *reinterpret_cast<float4 *>(dst) = sx[row * P22_C4 + (c4 ^ ((row >> 1) & 7))];
            }
            if (top) strip_border_done(S, 0);
            if (bottom) strip_border_done(S, 1);
        }
    }
}

template <bool BATCH, class G>
__device__ __forceinline__ void step_uncovered22_body(const FrameDev &F, const int c, const float factor, const G &geo) {
    const PlaneDev &P = F.pl[c];
    const int W = F.W, H = F.H, cwf = 2 * P.cw, chf = 2 * P.ch;
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
    const unsigned bottom = (unsigned)(H - chf) * (unsigned)W, right_w = (unsigned)(W - cwf);
    const unsigned n = bottom + (unsigned)chf * right_w;
    for (unsigned i = geo.bx() * blockDim.x + threadIdx.x; i < n; i += geo.nx() * blockDim.x) {
        unsigned px, py;
        if (i < bottom) {
            py = (unsigned)chf + i / (unsigned)W;
            px = i % (unsigned)W;
        } else {
            const unsigned k = i - bottom;
            py = k / right_w;
            px = (unsigned)cwf + k % right_w;
        }
        const size_t gi = (size_t)py * W + px;
        xm[gi] = stepper(xk[gi], xm[gi], gk[gi]);
    }
}

}  // namespace j2p
