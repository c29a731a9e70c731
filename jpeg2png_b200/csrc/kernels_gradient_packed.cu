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

#include "gradient_common.cuh"
#include "kernels.cuh"
#include "numerics.cuh"
#include "pdl.cuh"
#include "project_common.cuh"
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
// BATCH: a batch session (kernels.cuh, FrameDev::nframes); the frame is blockIdx.z and every frame
// has the grid a single-frame session of its geometry gets.  Its base is formed once, in 64 bits;
// the offsets inside a frame stay 32-bit.  !BATCH compiles to the single-frame kernel unchanged.
template <int NC, bool TGV, int GPM, bool BATCH>
__global__ void J2P_GRAD_BOUNDS k_gradient_packed(const __grid_constant__ FrameDev F, const float factor, const int band_rows) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const unsigned frame = BATCH ? blockIdx.z : 0u;
    const size_t fo = BATCH ? (size_t)frame * F.frame_stride : 0;     // elements from frame 0's planes to this frame's
    const int W = F.W, H = F.H;
    const int X0 = (blockIdx.x * GM_WARPS + wid) * GM_USE;   // first target column of this warp
    const int yb = F.t0 + blockIdx.y * band_rows;            // first target row of this CTA (local row index)
    const int ye = min(yb + band_rows, F.t1);
    const int s_first = -F.y0g;                              // local index of the frame's first row
    const int px0 = X0 - 2 + 2 * lane;                       // even; W is even => the pair is in or out together
    const bool pair_in = px0 >= 0 && px0 < W;
    const bool is_target = pair_in && lane >= 1 && lane <= 30;
    const bool has_l0 = px0 > 0, has_r1 = px0 + 1 < W - 1;   // hi always has a left neighbour, lo a right one
    const f2 a1s = splat(F.a1), a1n = splat(-F.a1), a2s = splat(F.a2), a2n = splat(-F.a2), a2m2 = splat(fmul(-2.f, F.a2));
    const f2 fac = splat(factor), half2 = splat(0.5f), zero2 = 0ull;
    const f2 one = splat(F.one);                             // see addm2(): sums with a product go through fma(m, one, b)
    const unsigned zero = (unsigned)band_rows >> 31;         // see settle()

    // Everything the kernel reads was written by the projection before it (x_k, gp, the halo rows):
    // nothing but index arithmetic runs ahead of the wait.  The dependents (the projection of this
    // iteration) may take their seats once this kernel is really running.
    pdl_wait();
    pdl_launch_dependents();
    // strip sessions: the halo rows of x_k arrive from the neighbours' projection (strip_sync.cuh)
    if (!BATCH) strip_wait_halo(F.sync, blockIdx.y == 0, blockIdx.y == gridDim.y - 1);

    double acc[NC];
    RowCarry<NC> A, B;
    f2 gmask[NC];                 // 1 where the pixel has such a term, else 0 (compute.c:58-62 footprint, pweight != 0)
#pragma unroll
    for (int c = 0; c < NC; c++) {
        acc[c] = 0.;
        A.y[c] = A.gx[c] = A.gy[c] = A.og[c] = A.tvb[c] = A.ud[c] = A.dg[c] = zero2;
    }
    A.ok1 = A.ok2 = true;

    // which pixels have a DCT-distance term (compute.c:58-62 footprint, pweight != 0).  GPM 1, 2: every
    // in-frame pixel of a plane with pweight != 0 (values of out-of-frame lanes are never stored), so
    // the mask is warp-uniform; generic: per pixel.
    int gpx[NC][2];
#pragma unroll
    for (int c = 0; c < NC; c++) {
        float m[2];
#pragma unroll
        for (int k = 0; k < 2; k++) {
            const int cx = (px0 + k) / F.pl[c].sw;
            const bool has = F.pl[c].use_prob && (GPM != 0 || (pair_in && cx < F.pl[c].cw));
            gpx[c][k] = has && GPM == 0 ? cx : 0;
            m[k] = has ? 1.f : 0.f;
        }
        gmask[c] = pk(m[0], m[1]);
    }

    // Rows/columns outside the frame are never consumed (their sources are dead), so the loads are
    // made unconditional by clamping the address into the frame: no branches.
    //
    // Addressing (GPM != 0).  The session keeps x[0..2], xp[0..2], g[0..2], gp[0..2] in one slab with
    // the same element stride PS between the planes of an array (session.cu).  The kernel holds ONE
    // 64-bit lane pointer per array (array base + the lane's column, made opaque so that it stays in
    // registers) and forms an address as
    //     lane pointer + 4 * (row * W + c * PS)        row * W + c * PS is warp-uniform, 32 bits
    // With one pointer per buffer in the parameter block the compiler re-read the pointers with LDC every
    // row; those LDCs shared a scoreboard with the loads already in flight, each address waited for the
    // previous loads to land, and the one-row prefetch was lost (long_scoreboard the top stall).
    const int pxc = pair_in ? px0 : 0;
    const unsigned PS = F.plane_stride;
    unsigned long long lp_x = 0, lp_xp = 0, lp_g = 0, lp_gp = 0, lp_gpc = 0;
    if (GPM != 0) {
        asm volatile("mad.wide.s32 %0, %1, 4, %2;" : "=l"(lp_x) : "r"(pxc), "l"(F.pl[0].x + fo));
        asm volatile("mad.wide.s32 %0, %1, 4, %2;" : "=l"(lp_xp) : "r"(pxc), "l"(F.pl[0].xp + fo));
        asm volatile("mad.wide.s32 %0, %1, 4, %2;" : "=l"(lp_g) : "r"(pxc), "l"(F.pl[0].g + fo));
        asm volatile("mad.wide.s32 %0, %1, 4, %2;" : "=l"(lp_gp) : "r"(pxc), "l"(F.pl[0].gp + fo));
        if (GPM == 2) asm volatile("mad.wide.s32 %0, %1, 4, %2;" : "=l"(lp_gpc) : "r"(pxc >> 1), "l"(F.pl[0].gp + fo));   // 2x2 planes: one sample per pixel pair
    }
    auto at = [](unsigned long long base, unsigned elem) {          // base + 4 * elem
        unsigned long long a;
        asm("mad.wide.u32 %0, %1, 4, %2;" : "=l"(a) : "r"(elem), "l"(base));
        return a;
    };
    // ---- the row ring: slot (row mod GM_DEPTH) of this warp holds, per lane, x_k and x_{k-1} of `row`
    // and the DCT-distance term of target row `row - 1` (what the step that forms row `row` consumes)
    constexpr int NSLOT = 3 * NC;
    __shared__ float2 ring[GM_WARPS][GM_DEPTH][NSLOT][32];
    const unsigned ring_lane = (unsigned)__cvta_generic_to_shared(&ring[wid][0][0][lane]);
    constexpr unsigned SLOT_BYTES = NSLOT * 32 * sizeof(float2);
    auto cp8 = [](unsigned dst, unsigned long long src) { asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory"); };
    auto cp4 = [](unsigned dst, unsigned long long src) { asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory"); };
    // everything the step that forms `row` needs, into ring slot `slot`; one commit group per row
    auto issue_row = [&](int row, unsigned slot) {
        const unsigned dst = ring_lane + slot * SLOT_BYTES;
        const unsigned ro = (unsigned)min(max(row, 0), H - 1) * (unsigned)W;   // slabs are below 2^32 elements (checked at session creation)
        const unsigned r = (unsigned)(min(max(row - 1, yb), ye - 1) - F.t0);    // target row of the gp term, as a row of the owned region
#pragma unroll
        for (int c = 0; c < NC; c++) {
            if (GPM != 0) {
                cp8(dst + (2 * c) * 256, at(lp_x, ro + c * PS));
                cp8(dst + (2 * c + 1) * 256, at(lp_xp, ro + c * PS));
            } else {
                cp8(dst + (2 * c) * 256, (unsigned long long)(F.pl[c].x + fo + (ro + (unsigned)pxc)));
                cp8(dst + (2 * c + 1) * 256, (unsigned long long)(F.pl[c].xp + fo + (ro + (unsigned)pxc)));
            }
        }
        if (GPM == 1) {                     // every gp plane has the frame's geometry and every target row has its gp row
#pragma unroll
            for (int c = 0; c < NC; c++) cp8(dst + (2 * NC + c) * 256, at(lp_gp, r * (unsigned)W + c * PS));
        } else if (GPM == 2) {              // 4:2:0 with aligned grids: plane 0 full resolution, planes 1, 2 at half resolution
            cp8(dst + (2 * NC) * 256, at(lp_gp, min(r, (unsigned)F.pl[0].ch - 1u) * (unsigned)W));
            const unsigned rc_ = min(r >> 1, (unsigned)F.pl[1].ch - 1u) * (unsigned)(W >> 1);
#pragma unroll
            for (int c = 1; c < NC; c++) cp4(dst + (2 * NC + c) * 256, at(lp_gpc, rc_ + c * PS));
        } else {
#pragma unroll
            for (int c = 0; c < NC; c++) {
                const PlaneDev &P = F.pl[c];
                const float *gr = P.gp + fo + (size_t)min(r / (unsigned)P.sh, (unsigned)P.ch - 1u) * P.cw;
                cp4(dst + (2 * NC + c) * 256, (unsigned long long)(gr + gpx[c][0]));
                cp4(dst + (2 * NC + c) * 256 + 4, (unsigned long long)(gr + gpx[c][1]));
            }
        }
        cp_async_commit();
    };
    // which planes have a gp row for target row s (warp-uniform)
    auto gp_rows_of = [&](int s) {
        const unsigned r = (unsigned)(s - F.t0);
        if (GPM == 1) return 7u;
        if (GPM == 2) return (r < (unsigned)F.pl[0].ch ? 1u : 0u) | ((r >> 1) < (unsigned)F.pl[1].ch ? 6u : 0u);
        unsigned ok = 0;
#pragma unroll
        for (int c = 0; c < NC; c++)
            if (r / (unsigned)F.pl[c].sh < (unsigned)F.pl[c].ch) ok |= 1u << c;
        return ok;
    };

    // One row step: the FISTA point of row i is formed, source row s = i-1 gets its TV and TGV
    // quotients, target row s-1 its last two addends (and is stored), target row s its first nine.
    // P: the carry of the previous step (read), N: the carry this step leaves (written).
    //
    // The whole step is ONE basic block plus one cold fix-up: the differences and both norms first,
    // then a single vote over every guard of the row (FISTA values, both square-root arguments), then
    // both quotient stages on the fast sequences, unconditionally.  A row the vote rejects recomputes
    // both stages with the IEEE instructions afterwards and overrides the results (tv_slow / tgv_slow,
    // out of line).  The earlier build voted and branched per stage (three votes and two
    // fast/slow diamonds per row, plus a branch around the store): the scheduler could not move the
    // TGV arithmetic under the latency of the TV square root and reciprocal, and "wait" (fixed-latency
    // dependency) was the top stall at three warps per scheduler.
    auto row_step = [&](const int i, const RowCarry<NC> &P, RowCarry<NC> &N) {
        // ---- FISTA point of row i (compute.c:436) from the ring slot filled GM_DEPTH steps ago --------
        cp_async_wait<GM_DEPTH - 1>();                          // this lane's oldest group has landed (it reads only its own bytes)
        const unsigned slot = (unsigned)(i - (yb - 2)) & (GM_DEPTH - 1);
        const float2 *rs = &ring[wid][slot][0][lane];
        unsigned ykey = 0xffffffffu;
#pragma unroll
        for (int c = 0; c < NC; c++) {
            const float2 vx = rs[(2 * c) * 32], vp = rs[(2 * c + 1) * 32];
            const f2 x = pk(vx.x, vx.y), xp = pk(vp.x, vp.y);
            N.y[c] = addm2(mul2(fac, sub2(x, xp)), x, one);
            ykey = min(ykey, min(qdiv_key(lo(N.y[c])), qdiv_key(hi(N.y[c]))));
        }
        // the DCT-distance addend of target row s = i-1: 0 + gp where the pixel has one (compute.c:62), else 0
        const unsigned gp_rows_ok = gp_rows_of(i - 1);
        f2 pterm[NC];
#pragma unroll
        for (int c = 0; c < NC; c++) {
            const float2 vg = rs[(2 * NC + c) * 32];
            const f2 g2 = (GPM == 2 && c > 0) ? pk(vg.x, vg.x) : pk(vg.x, vg.y);   // 2x2 planes: one sample per pixel pair
            pterm[c] = fma2(g2, (gp_rows_ok >> c) & 1u ? gmask[c] : zero2, zero2);
        }
        issue_row(i + GM_DEPTH, slot);                          // the slot has just been read; clamped rows at the end are harmless

        const int s = i - 1;
        const bool src_in = pair_in & (s >= 0) & (s < H);
        // No row below the frame's last row: gy := 0 (compute.c:81).  Nothing to do for it: the row
        // loads are clamped into the buffer, whose last row IS the frame's last row whenever that
        // row is reachable, so row s+1 re-reads row s and gy comes out +0.

        // ---- source row s: first differences and the TV norm (compute.c:79-89) ----------------
        f2 gx0[NC], gy0[NC];
        f2 n1 = zero2;
#pragma unroll
        for (int c = 0; c < NC; c++) {
            float yr1 = __shfl_down_sync(0xffffffffu, lo(P.y[c]), 1);
            yr1 = has_r1 ? yr1 : hi(P.y[c]);                    // no right neighbour: gx := 0 (compute.c:79)
            gx0[c] = sub2(shr_from_right(P.y[c], yr1), P.y[c]);
            gy0[c] = sub2(N.y[c], P.y[c]);
            const f2 sx = mul2(gx0[c], gx0[c]), sy = mul2(gy0[c], gy0[c]);
            n1 = c == 0 ? addm2(sy, sx, one) : addm2(sy, addm2(sx, n1, one), one);   // 0 + gx^2 == gx^2: squares are never -0
            N.gx[c] = gx0[c];
            N.gy[c] = gy0[c];
        }
        const bool tl0 = src_in & (lo(n1) != 0.f), tl1 = src_in & (hi(n1) != 0.f);     // sqrtf(x) != 0  <=>  x != 0   (compute.c:97)
        const f2 ss1 = pk(tl0 ? lo(n1) : 1.f, tl1 ? hi(n1) : 1.f);                   // dead source: norm 1, reciprocal 0 => every quotient exactly 0
        bool bad = (ykey < QDIV_YKEY_MIN) | !root_arg_ok(lo(ss1)) | !root_arg_ok(hi(ss1));   // one guard per VALUE (numerics.cuh, "row guard")

        // ---- source row s: second differences and the TGV norm (compute.c:136-152) ------------
        f2 gxx[NC], gyy[NC], sym[NC];
        f2 ss2 = zero2;
        bool gl0 = false, gl1 = false;
        if (TGV) {
            f2 gyPv[NC];
#pragma unroll
            for (int c = 0; c < NC; c++) gyPv[c] = P.gy[c];
            if (__builtin_expect(s <= s_first, false)) {     // no row above in the frame: gxy, gyy := 0 (compute.c:141-143)
                // gxy needs no help: the clamped loads made "row -1" a copy of row 0, so the gx carried
                // from the previous step already equals gx0.  gy of that copy is 0, not gy0.
#pragma unroll
                for (int c = 0; c < NC; c++) gyPv[c] = gy0[c];
            }
            f2 n2 = zero2;
#pragma unroll
            for (int c = 0; c < NC; c++) {
                float gxl = __shfl_up_sync(0xffffffffu, hi(gx0[c]), 1);
                float gyl = __shfl_up_sync(0xffffffffu, hi(gy0[c]), 1);
                gxl = has_l0 ? gxl : lo(gx0[c]);            // no left neighbour: gxx, gyx := 0 (compute.c:137-139)
                gyl = has_l0 ? gyl : lo(gy0[c]);
                gxx[c] = sub2(gx0[c], shl_from_left(gx0[c], gxl));
                const f2 gyx = sub2(gy0[c], shl_from_left(gy0[c], gyl));
                const f2 gxy = sub2(gx0[c], P.gx[c]);
                gyy[c] = sub2(gy0[c], gyPv[c]);
                const f2 u = add2(gxy, gyx);
                sym[c] = mul2(u, half2);                    // (gxy+gyx)/2., exact either way
                // 2*sym^2 as u*sym: 2*RN((u/2)^2) == RN(u*(u/2)) (power-of-two scalings commute with rounding
                // while nothing underflows; rows where that is not guaranteed are flagged by the row guard
                // and recompute n2 in the reference's form in tgv_slow)
                const f2 t = addm2(mul2(gyy[c], gyy[c]), addm2(mul2(u, sym[c]), mul2(gxx[c], gxx[c]), one), one);
                n2 = c == 0 ? t : add2(n2, t);              // 0 + t == t: t is never -0
            }
            gl0 = src_in & (lo(n2) != 0.f);                  // compute.c:158
            gl1 = src_in & (hi(n2) != 0.f);
            ss2 = pk(gl0 ? lo(n2) : 1.f, gl1 ? hi(n2) : 1.f);
            bad = bad | !root_arg_ok(lo(ss2)) | !root_arg_ok(hi(ss2));
        }

        // ---- the row's one vote; the guard window covers the three rows the differences span ----
        const bool ok0 = !__any_sync(0xffffffffu, bad);
        N.ok1 = ok0;
        N.ok2 = P.ok1;
        const bool fast = ok0 && P.ok1 && P.ok2;

        // ---- TV quotients (compute.c:97-105), fast sequences --------------------------------
        f2 tvs0[NC], tvr0[NC], t2s0[NC], lr0[NC];
        {
            const f2 n = sqrt2_core(ss1), nb = neg2(n);
            const f2 yr = rcp2_core(n, nb);
            const f2 y = pk(tl0 ? lo(yr) : 0.f, tl1 ? hi(yr) : 0.f);
            const f2 yl = rcp2_low(nb, y);                                  // two-term reciprocal: four operations per quotient (numerics.cuh)
#pragma unroll
            for (int c = 0; c < NC; c++) {
                tvs0[c] = qdiv2x(mul2(a1n, add2(gx0[c], gy0[c])), nb, y, yl);   // compute.c:98: (a1 * -(gx+gy)) / n
                tvr0[c] = qdiv2x(mul2(a1s, gx0[c]), nb, y, yl);                  // compute.c:100
                N.tvb[c] = qdiv2x(mul2(a1s, gy0[c]), nb, y, yl);                 // compute.c:103
            }
        }
        // ---- TGV quotients (compute.c:158-183), fast sequences ------------------------------
        if (TGV) {
            const f2 n = sqrt2_core(ss2), nb = neg2(n);
            const f2 yr = rcp2_core(n, nb);
            const f2 y = pk(gl0 ? lo(yr) : 0.f, gl1 ? hi(yr) : 0.f);
            const f2 yl = rcp2_low(nb, y);
#pragma unroll
            for (int c = 0; c < NC; c++) {
                // compute.c:165: a2 * (-(2gxx + 2s + 2gyy) / n) == (-2 a2) * (((s + gxx) + gyy) / n): doubling
                // commutes with every rounding involved (no overflow in this range)
                const f2 sx = addm2(sym[c], gxx[c], one);
                t2s0[c] = mul2(a2m2, qdiv2x(add2(sx, gyy[c]), nb, y, yl));
                lr0[c] = mul2(a2s, qdiv2x(sx, nb, y, yl));                           // compute.c:167,170
                N.ud[c] = mul2(a2s, qdiv2x(addm2(sym[c], gyy[c], one), nb, y, yl));        // compute.c:173,176
                N.dg[c] = mul2(a2n, qdiv2x(sym[c], nb, y, yl));                      // compute.c:179,182: a2 * (-s / n)
            }
        } else {
#pragma unroll
            for (int c = 0; c < NC; c++) t2s0[c] = lr0[c] = N.ud[c] = N.dg[c] = zero2;
        }
        // ---- outside the proven range (once in millions of rows): IEEE square root and division ----
        if (__builtin_expect(!fast, false)) {
            {
                TvSlow<NC> io;
#pragma unroll
                for (int c = 0; c < NC; c++) {
                    io.gx[c][0] = lo(gx0[c]); io.gx[c][1] = hi(gx0[c]);
                    io.gy[c][0] = lo(gy0[c]); io.gy[c][1] = hi(gy0[c]);
                }
                tv_slow<NC>(&io, F.a1, src_in);
#pragma unroll
                for (int c = 0; c < NC; c++) {
                    tvs0[c] = pk(settle(io.q[0][c][0], zero), settle(io.q[0][c][1], zero));
                    tvr0[c] = pk(settle(io.q[1][c][0], zero), settle(io.q[1][c][1], zero));
                    N.tvb[c] = pk(settle(io.q[2][c][0], zero), settle(io.q[2][c][1], zero));
                }
            }
            if (TGV) {
                TgvSlow<NC> io;
#pragma unroll
                for (int c = 0; c < NC; c++) {
                    io.gxx[c][0] = lo(gxx[c]); io.gxx[c][1] = hi(gxx[c]);
                    io.gyy[c][0] = lo(gyy[c]); io.gyy[c][1] = hi(gyy[c]);
                    io.sym[c][0] = lo(sym[c]); io.sym[c][1] = hi(sym[c]);
                }
                tgv_slow<NC>(&io, F.a2, src_in);
#pragma unroll
                for (int c = 0; c < NC; c++) {
                    t2s0[c] = pk(settle(io.q[0][c][0], zero), settle(io.q[0][c][1], zero));
                    lr0[c] = pk(settle(io.q[1][c][0], zero), settle(io.q[1][c][1], zero));
                    N.ud[c] = pk(settle(io.q[2][c][0], zero), settle(io.q[2][c][1], zero));
                    N.dg[c] = pk(settle(io.q[3][c][0], zero), settle(io.q[3][c][1], zero));
                }
            }
        }

        // ---- target row s-1: last two addends (TGV below-left, below), store, sum of squares ----
        // Computed in every step; the rows that are not targets of this band (the two lead-in steps
        // and the idle step of an odd band) only suppress the store and add zeros to the sums.
        {
            const bool st = is_target & (i >= yb + 2) & (i <= ye + 1);
            const unsigned ro = (unsigned)max(s - 1, 0) * (unsigned)W;         // targets are inside the frame: pxc == px0
#pragma unroll
            for (int c = 0; c < NC; c++) {
                f2 o = P.og[c];
                if (TGV) {
                    const float dgl = __shfl_up_sync(0xffffffffu, hi(N.dg[c]), 1);
                    o = addm2(N.ud[c], add2(o, shl_from_left(N.dg[c], dgl)), one);
                }
                float2 *dst = GPM != 0 ? reinterpret_cast<float2 *>(at(lp_g, ro + c * PS)) : reinterpret_cast<float2 *>(F.pl[c].g + fo + (ro + (unsigned)pxc));
                if (st) *dst = make_float2(lo(o), hi(o));
                const f2 sq = mul2(o, o);
                acc[c] = __dadd_rn(acc[c], (double)(st ? lo(sq) : 0.f));      // compute.c:203; + 0.0 leaves the sum as it is
                acc[c] = __dadd_rn(acc[c], (double)(st ? hi(sq) : 0.f));
            }
        }

        // ---- target row s: addends 1..9 (DCT distance; TV above, left, self; TGV above, above-right,
        // left, self, right) ---------------------------------------------------------------------
#pragma unroll
        for (int c = 0; c < NC; c++) {
            const float tvr_l = __shfl_up_sync(0xffffffffu, hi(tvr0[c]), 1);
            f2 o = add2(add2(add2(pterm[c], P.tvb[c]), shl_from_left(tvr0[c], tvr_l)), tvs0[c]);
            if (TGV) {
                const float dg_r = __shfl_down_sync(0xffffffffu, lo(P.dg[c]), 1);
                o = add2(addm2(P.ud[c], o, one), shr_from_right(P.dg[c], dg_r));
                const float lr_l = __shfl_up_sync(0xffffffffu, hi(lr0[c]), 1);
                const float lr_r = __shfl_down_sync(0xffffffffu, lo(lr0[c]), 1);
                o = add2(addm2(t2s0[c], add2(o, shl_from_left(lr0[c], lr_l)), one), shr_from_right(lr0[c], lr_r));
            }
            N.og[c] = o;
        }
    };

    // Warps whose strip starts beyond the frame (only in the last CTA column of odd widths) run the
    // same loop on clamped loads and store nothing: control flow depends on block indices and kernel
    // parameters only, so every shuffle is executed convergently.  Two row steps per trip with the
    // roles of the two carries swapped; an odd row count gets one idle step at the end (its loads
    // are clamped, its store is suppressed by the row test inside the step).
#pragma unroll
    for (int d = 0; d < GM_DEPTH; d++) issue_row(yb - 2 + d, d);
    for (int i = yb - 2; i <= ye + 1; i += 2) {
        row_step(i, A, B);
        row_step(i + 1, B, A);
    }
    cp_async_wait<0>();                 // nothing of this thread is in flight when it leaves

    // CTA reduction (fixed order => run-to-run deterministic), then the last-CTA fold
    __shared__ double red[3][GM_WARPS];
    __shared__ double fin[3];
    __shared__ unsigned ticket;
    const int tid = threadIdx.x;
    // this frame's partials, ticket, sums and norms (a single frame: the session's own)
    double *const partials = F.partials + (BATCH ? (size_t)frame * 5 * F.grad_ctas : 0);
    unsigned *const counter = F.counter + frame;
    double *const sums = F.sums + 4 * frame;
    float *const norms = F.norms + 16 * frame;
#pragma unroll
    for (int c = 0; c < NC; c++) {
        const double sum = warp_sum(acc[c]);
        if (lane == 0) red[c][wid] = sum;
    }
    __syncthreads();
    const unsigned cta = blockIdx.y * gridDim.x + blockIdx.x, ncta = gridDim.x * gridDim.y;
    // One thread publishes the CTA's partial sums and takes the ticket with RELEASE semantics: only
    // these few stores have to be visible to the CTA that folds them.  (A __threadfence() by every
    // thread made each CTA wait for all of its gradient stores to drain before it could retire.)
    if (tid == 0) {
#pragma unroll
        for (int c = 0; c < NC; c++) {
            double sum = 0.;
            for (int k = 0; k < GM_WARPS; k++) sum = __dadd_rn(sum, red[c][k]);
            partials[(size_t)c * F.grad_ctas + cta] = sum;
        }
        unsigned t;
        asm volatile("atom.release.gpu.global.add.u32 %0, [%1], 1;" : "=r"(t) : "l"(counter) : "memory");
        ticket = t;
    }
    __syncthreads();
    if (ticket == ncta - 1) {
        __threadfence();
#pragma unroll
        for (int c = 0; c < NC; c++) {
            double sum = 0.;
            for (unsigned k = tid; k < ncta; k += GM_NT) sum = __dadd_rn(sum, __ldcg(&partials[(size_t)c * F.grad_ctas + k]));
            sum = warp_sum(sum);
            if (lane == 0) red[c][wid] = sum;
        }
        __syncthreads();
        if (tid < 3) {
            double sum = 0.;
            if (tid < NC)
                for (int k = 0; k < GM_WARPS; k++) sum = __dadd_rn(sum, red[tid][k]);
            fin[tid] = sum;
            if (tid < NC) {
                const float norm = fsqrt(__double2float_rn(sum));                               // compute.c:205
                sums[tid] = sum;                                                              // strips driven by the host / NCCL combine these
                norms[tid] = norm;
                norms[4 + tid] = __frcp_rn(norm);                                             // shared reciprocal for k_project
            }
        }
        if (tid == 0) *counter = 0u;
        if (!BATCH && F.sync.nranks > 1) {                                                      // strips over peer memory
            __syncthreads();
            strip_post_sums(F.sync, fin, tid);
        }
    }
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
static cudaError_t launch_instance(const FrameDev &F, float factor, cudaStream_t s) {
    static const int per_sm = [] {
        int n = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_gradient_packed<NC, TGV, GPM, false>, GM_NT, 0) != cudaSuccess) {
            cudaGetLastError();
            n = 0;
        }
        return n > 0 ? n : 1;
    }();
    int cx, bands, rows;
    grad_geometry(F.W, F.t1 - F.t0, sm_count() * per_sm, &cx, &bands, &rows);
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

int packed_gradient_occupancy() {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_gradient_packed<3, true, 1, false>, GM_NT, 0) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return per_sm;
}

cudaError_t launch_gradient_packed(const FrameDev &F, float factor, cudaStream_t s) {
    const int owned = F.t1 - F.t0;
    bool full = true;      // every plane at full resolution over the whole (local) frame: gp has the frame's geometry
    for (int c = 0; c < F.nc; c++) full = full && F.pl[c].sw == 1 && F.pl[c].sh == 1 && F.pl[c].cw == F.W && F.pl[c].ch >= owned;
    // 4:2:0 with aligned grids: luma full width (its last rows may be missing: 1080p), both chroma planes exactly half
    bool c420 = F.nc == 3 && F.pl[0].sw == 1 && F.pl[0].sh == 1 && F.pl[0].cw == F.W;
    for (int c = 1; c < 3 && c420; c++) c420 = F.pl[c].sw == 2 && F.pl[c].sh == 2 && 2 * F.pl[c].cw == F.W && F.pl[c].ch == F.pl[1].ch;
    if (full) return F.use_tgv ? launch_packed_nc<true, 1>(F, factor, s) : launch_packed_nc<false, 1>(F, factor, s);
    if (c420) return F.use_tgv ? launch_instance<3, true, 2>(F, factor, s) : launch_instance<3, false, 2>(F, factor, s);
    return F.use_tgv ? launch_packed_nc<true, 0>(F, factor, s) : launch_packed_nc<false, 0>(F, factor, s);
}

}  // namespace j2p
