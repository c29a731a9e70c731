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

#include "kernels.cuh"
#include "numerics.cuh"
#include "pdl.cuh"
#include "project_common.cuh"
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
// RES: the plane's coefficient grid is smaller than the frame (compute.c:338), e.g. 1080p luma.
// BATCH: a batch session (FrameDev::nframes); blockIdx.z = frame, blockIdx.x = k * (CTA columns) +
// column for planes c0 + k (a single frame: blockIdx.z = k).  A batch keeps gridDim.z for the frames,
// which may number 65535.
template <bool RES, bool BATCH>
__global__ void __launch_bounds__(PT_NT, J2P_TILE_MIN_CTAS) k_project_tile(const __grid_constant__ FrameDev F, const int c0, const float factor) {
    __shared__ __align__(16) float4 sx[8][PT_C4];                // x_k          -> later x_{k+1}
    __shared__ __align__(16) float4 sp[8][PT_C4];                // x_{k-1}      -> later gp
    __shared__ __align__(16) float4 sg[8][PT_C4];                // g
    __shared__ __align__(16) float tiles[PT_NT / 8][TILE_STRIDE];
    __shared__ __align__(16) float sq[3][64];
    __shared__ float snorm[2];
    const int tid = threadIdx.x;
    const int frame = BATCH ? (int)blockIdx.z : 0;
    const int gx = BATCH ? ((F.pl[c0].cw >> 3) + PT_NB - 1) / PT_NB : 0;   // CTA columns per plane
    const int k = BATCH ? (int)blockIdx.x / gx : (int)blockIdx.z;
    const int c = c0 + k;                                        // planes of equal geometry share one launch
    const PlaneDev &P = F.pl[c];
    const size_t fo = BATCH ? (size_t)frame * F.frame_stride : 0;
    const int W = F.W;
    const int bw = P.cw >> 3;
    const int bx0 = (BATCH ? (int)blockIdx.x - k * gx : (int)blockIdx.x) * PT_NB;
    const int by = strip_row_order(F.sync, blockIdx.y, gridDim.y);   // the grid covers real blocks only
    const int nbx = min(PT_NB, bw - bx0);                           // blocks of this tile that exist
    const int valid_c4 = nbx * 2;
    const size_t row0 = (size_t)(by * 8) * W + (size_t)bx0 * 8;  // first pixel of the tile

    // ---- coalesced, swizzled copy-in ------------------------------------------------------------
    // x_k and x_{k-1} are not written by the gradient kernel this launch depends on (pdl.cuh): their
    // tiles are requested BEFORE the wait, while that kernel drains.  Everything else follows the wait
    // at once: in all but the first wave of CTAs it returns immediately, and the g tile must not queue
    // behind the table loads (20 waves of short-lived CTAs pay their prologue latency in the open).
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int e = tid + PT_NT * i, row = e >> PT_SH, c4 = e & (PT_C4 - 1);
        if (c4 < valid_c4) {
            const size_t gi = row0 + (size_t)row * W + (size_t)c4 * 4;
            cp_async16(&sx[row][c4 ^ row], P.x + fo + gi);
            cp_async16(&sp[row][c4 ^ row], P.xp + fo + gi);
        }
    }
    pdl_wait();                                                  // the gradient and its norm are complete and visible
    pdl_launch_dependents();
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int e = tid + PT_NT * i, row = e >> PT_SH, c4 = e & (PT_C4 - 1);
        if (c4 < valid_c4) cp_async16(&sg[row][c4 ^ row], P.g + fo + row0 + (size_t)row * W + (size_t)c4 * 4);
    }
    cp_async_commit();
    const int b = tid >> 3, j = tid & 7;
    const bool real = b < nbx;
    int4 draw = make_int4(0, 0, 0, 0);
    if (real) draw = __ldg(reinterpret_cast<const int4 *>(P.data + (BATCH ? (size_t)frame * F.data_stride : 0) + ((size_t)(by * bw + bx0 + b) * 64 + j * 8)));   // 512 B per warp, coalesced
    if (tid < 64) {
        if (BATCH) {                                             // this frame's tables (device copy)
            const float *t = F.tables + ((size_t)frame * F.nc + c) * 192;
            sq[0][tid] = t[tid];
            sq[1][tid] = t[64 + tid];
            sq[2][tid] = t[128 + tid];
        } else {
            sq[0][tid] = F.q[c][tid];
            sq[1][tid] = F.qq[c][tid];
            sq[2][tid] = F.rqq[c][tid];
        }
    }
    if (BATCH) {
        if (tid == 64) {                                         // what k_gradient left for this frame
            snorm[0] = F.norms[16 * frame + c];
            snorm[1] = F.norms[16 * frame + 4 + c];
        }
    } else if (tid >= 64 && tid < 96) {
        strip_norm(F, c, snorm, tid - 64);                       // whole frame: what k_gradient left; strips: fold of every rank's sums
    }
    cp_async_wait<0>();
    __syncthreads();

    Stepper stepper;
    stepper.factor = factor;
    stepper.step = F.step;
    stepper.norm = snorm[0];
    stepper.rn = snorm[1];
    stepper.stepping = stepper.norm != 0.f;                        // compute.c:211
    const bool norm_ok = qdiv_divisor_ok(stepper.norm);
    const bool use_prob = P.use_prob != 0;
    constexpr bool resample = RES;
    const unsigned gmask = 0xffu << (tid & 24);
    float *tile = tiles[b];

    if (real) {
        // ---- stepped point (compute.c:436, :213) from this thread's row of the tile --------------
        float z[8], v[8], mean[8];
        {
            unsigned key = 0xffffffffu;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int pc = (2 * b + h) ^ j;
                const float4 a = sx[j][pc], p = sp[j][pc], g = sg[j][pc];
                z[h * 4 + 0] = stepper.fast(a.x, p.x, g.x, key);
                z[h * 4 + 1] = stepper.fast(a.y, p.y, g.y, key);
                z[h * 4 + 2] = stepper.fast(a.z, p.z, g.z, key);
                z[h * 4 + 3] = stepper.fast(a.w, p.w, g.w, key);
            }
            if (stepper.stepping && !(norm_ok && key >= QDIV_KEY_MIN)) {   // outside the proven range: IEEE division
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int pc = (2 * b + h) ^ j;
                    const float4 a = sx[j][pc], p = sp[j][pc], g = sg[j][pc];
                    z[h * 4 + 0] = stepper(a.x, p.x, g.x);
                    z[h * 4 + 1] = stepper(a.y, p.y, g.y);
                    z[h * 4 + 2] = stepper(a.z, p.z, g.z);
                    z[h * 4 + 3] = stepper(a.w, p.w, g.w);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 8; i++) {
            if (resample) {                                        // sampling 1x1 on a coefficient grid smaller than the frame
                const float m = fadd(0.f, z[i]);                   // compute.c:351-359 with one sample: (0 + z) / 1
                mean[i] = m;
                v[i] = m;
            } else {
                mean[i] = 0.f;
                v[i] = z[i];
            }
        }

        fdct8x8_rows(v, tile, j, gmask);

        // ---- clamp to the quantisation interval (compute.c:323-331); residual (compute.c:47-49) --
        const int dw[4] = {draw.x, draw.y, draw.z, draw.w};
        float r[8], num[8];
        unsigned rkey = 0xffffffffu;
        {
            const float4 *t0 = reinterpret_cast<const float4 *>(&sq[0][j * 8]);
            const float4 *t1 = reinterpret_cast<const float4 *>(&sq[1][j * 8]);
            const float4 *t2 = reinterpret_cast<const float4 *>(&sq[2][j * 8]);
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
            if (rkey < QDIV_KEY_MIN) {                             // a residual below 2^-60: IEEE division
#pragma unroll
                for (int i = 0; i < 8; i++) r[i] = fdiv(num[i], qqv[i]);
            }
        }

        idct8x8_rows(v, tile, j, gmask);
        if (use_prob) idct8x8_rows(r, tile, j, gmask);

        // ---- results into this thread's own cells of the staging tiles ---------------------------
        if (resample) {
#pragma unroll
            for (int i = 0; i < 8; i++) v[i] = fadd(fsub(z[i], mean[i]), v[i]);   // compute.c:390-403
        }
        const float pa = P.p_alpha;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int pc = (2 * b + h) ^ j;
            sx[j][pc] = make_float4(v[h * 4 + 0], v[h * 4 + 1], v[h * 4 + 2], v[h * 4 + 3]);
            if (use_prob)
                sp[j][pc] = make_float4(fmul(pa, r[h * 4 + 0]), fmul(pa, r[h * 4 + 1]), fmul(pa, r[h * 4 + 2]), fmul(pa, r[h * 4 + 3]));   // compute.c:62
        }
    }
    __syncthreads();

    // ---- coalesced copy-out: x_{k+1} over x_{k-1} (compute.c:387), gp for the next iteration ----
    float *gp0 = P.gp + fo + (size_t)(by * 8) * P.cw + (size_t)bx0 * 8;
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int e = tid + PT_NT * i, row = e >> PT_SH, c4 = e & (PT_C4 - 1);
        if (c4 < valid_c4) {
            *reinterpret_cast<float4 *>(P.xp + fo + row0 + (size_t)row * W + (size_t)c4 * 4) = sx[row][c4 ^ row];
            if (use_prob) *reinterpret_cast<float4 *>(gp0 + (size_t)row * P.cw + (size_t)c4 * 4) = sp[row][c4 ^ row];
        }
    }

    // ---- strips over peer memory: the strip's first / last two rows also go straight into the
    // neighbours' halo rows (NVLink stores), and the last border CTA of the iteration raises their flag
    const StripSync &S = F.sync;
    if (!BATCH && S.nranks > 1 && S.fused_halo) {
        const bool top = by == 0 && S.has_up, bottom = by == (int)gridDim.y - 1 && S.has_down;
        if (top || bottom) {
            for (int e = tid; e < 4 * PT_C4; e += PT_NT) {                // 2 rows x 64 pieces, top then bottom
                const int side = e >> (PT_SH + 1), r = (e >> PT_SH) & 1, c4 = e & (PT_C4 - 1);
                if (c4 >= valid_c4 || !(side ? bottom : top)) continue;
                const int row = side ? 6 + r : r;
                float *dst = (side ? S.down_dst[c] : S.up_dst[c]) + (size_t)r * W + (size_t)bx0 * 8 + (size_t)c4 * 4;
                *reinterpret_cast<float4 *>(dst) = sx[row][c4 ^ row];
            }
            if (top) strip_border_done(S, 0);
            if (bottom) strip_border_done(S, 1);
        }
    }
}

// Frame pixels of a 1x1 plane that no coefficient block covers (1080p: luma rows 1080..1087) are
// only stepped: compute_projection never visits them (compute.c:349-350).  The region is the
// bottom band (rows >= ch, full width) plus the right band (rows < ch, columns >= cw).
// BATCH: the frame is blockIdx.z.
template <bool BATCH>
__global__ void k_step_uncovered(const __grid_constant__ FrameDev F, const int c, const float factor) {
    const PlaneDev &P = F.pl[c];
    const int W = F.W, H = F.H;
    const int frame = BATCH ? (int)blockIdx.z : 0;
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
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
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
