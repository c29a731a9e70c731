// probe.cu — libj2pprobe.so: the device arithmetic of the solver and the device-only code paths of
// the codec cores, run on the GPU exactly as the kernels compile them, for tests/test_gpu_device_arith.py.
//
// Test infrastructure only: it includes the real headers and restates none of their code, and no
// product library links it.  It is compiled with the solver's floating-point flags (Makefile;
// tests/test_device_probe_host.py keeps the two in step).
//
// Every entry point takes host arrays, allocates, copies, launches, copies back and frees, and
// returns 0, or -1 with a message in probe_last_error().  A sweep returns a probe_tally: mismatches
// per sequence and the first few (sequence, operands, result, reference) as bit patterns.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../jpeg2png_b200/csrc/numerics.cuh"
#include "../../jpeg2png_b200/csrc/project_common.cuh"
#include "../../jpeg2png_b200/entropy/entropy_core.h"
#include "../../jpeg2png_b200/jpegopt/jpegopt_core.h"
#include "../../jpeg2png_b200/progressive/progressive_core.h"

using namespace j2p;

#define PROBE_SEQS 8
#define PROBE_EX 8

extern "C" {
struct probe_tally {
    unsigned long long checked;             // arguments (or pairs) the kernels ran
    unsigned long long bad[PROBE_SEQS];     // mismatches per sequence
    unsigned nex;                           // mismatches seen (the first PROBE_EX are in ex)
    unsigned ex[PROBE_EX][5];               // sequence, operand 1, operand 2, result, reference
};
}

// g_err, fail() and CK() are codec_host.h's (through entropy_core.h)
static int bad_args(const char *entry) { return fail("%s: bad arguments", entry); }

// a device buffer freed on every return path
struct Buf {
    void *p = nullptr;
    ~Buf() {
        if (p) cudaFree(p);
    }
    template <class T>
    T *as() const { return static_cast<T *>(p); }
};
static int dalloc(Buf &b, size_t bytes) {
    CK(cudaMalloc(&b.p, bytes ? bytes : 4));
    CK(cudaMemset(b.p, 0, bytes ? bytes : 4));
    return 0;
}
static int dput(Buf &b, const void *h, size_t bytes) {
    if (dalloc(b, bytes)) return -1;
    if (bytes) CK(cudaMemcpy(b.p, h, bytes, cudaMemcpyHostToDevice));
    return 0;
}
static int dget(void *h, const Buf &b, size_t bytes) {
    if (bytes) CK(cudaMemcpy(h, b.p, bytes, cudaMemcpyDeviceToHost));
    return 0;
}
static int ran(const char *kernel) {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return e == cudaSuccess ? 0 : fail("%s: %s", kernel, cudaGetErrorString(e));
}
static unsigned blocks(size_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

// equal bit for bit, except that the sign of a zero quotient is not part of the contract (numerics.cuh)
__device__ __forceinline__ bool same(float got, float want, bool zero_sign_free) {
    return __float_as_uint(got) == __float_as_uint(want) || (zero_sign_free && want == 0.f && got == 0.f);
}
// one count per CTA of the arguments its threads check (of n from this launch's first)
__device__ __forceinline__ void count_block(probe_tally *t, size_t n) {
    const size_t first = (size_t)blockIdx.x * blockDim.x;
    if (threadIdx.x == 0 && first < n) atomicAdd(&t->checked, (unsigned long long)(n - first < blockDim.x ? n - first : blockDim.x));
}
__device__ void tally(probe_tally *t, int seq, float a, float b, float got, float want, bool zero_sign_free) {
    if (same(got, want, zero_sign_free)) return;
    atomicAdd(&t->bad[seq], 1ull);
    const unsigned k = atomicAdd(&t->nex, 1u);
    if (k < PROBE_EX) {
        t->ex[k][0] = (unsigned)seq;
        t->ex[k][1] = __float_as_uint(a);
        t->ex[k][2] = __float_as_uint(b);
        t->ex[k][3] = __float_as_uint(got);
        t->ex[k][4] = __float_as_uint(want);
    }
}

// ---- the IEEE instructions themselves, for the host to compare with numpy ---------------------
__global__ void k_ieee(const float *a, const float *b, size_t n, float *q, float *s, float *r) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    q[i] = __fdiv_rn(a[i], b[i]);
    s[i] = __fsqrt_rn(a[i]);
    r[i] = __frcp_rn(a[i]);
}

extern "C" int probe_ieee(const float *a, const float *b, size_t n, float *q, float *s, float *r) {
    if (!a || !b || !q || !s || !r) return bad_args("probe_ieee");
    Buf da, db, dq, ds, dr;
    if (dput(da, a, n * 4) || dput(db, b, n * 4) || dalloc(dq, n * 4) || dalloc(ds, n * 4) || dalloc(dr, n * 4)) return -1;
    if (n) k_ieee<<<blocks(n, 256), 256>>>(da.as<float>(), db.as<float>(), n, dq.as<float>(), ds.as<float>(), dr.as<float>());
    if (ran("k_ieee")) return -1;
    return dget(q, dq, n * 4) || dget(s, ds, n * 4) || dget(r, dr, n * 4) ? -1 : 0;
}

// ---- guards and keys -------------------------------------------------------------------------
// flags bit 0: root_arg_ok(x); bit 1: qdiv_divisor_ok(x); bit 2: qdiv_fast's ok for the numerator x
__global__ void k_guards(const float *x, size_t n, uint32_t *flags, uint32_t *keys) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool ok = true;
    (void)qdiv_fast(x[i], 1.0f, 1.0f, ok);
    flags[i] = (root_arg_ok(x[i]) ? 1u : 0u) | (qdiv_divisor_ok(x[i]) ? 2u : 0u) | (ok ? 4u : 0u);
    keys[i] = qdiv_key(x[i]);
}

extern "C" int probe_guards(const float *x, size_t n, uint32_t *flags, uint32_t *keys) {
    if (!x || !flags || !keys) return bad_args("probe_guards");
    Buf dx, df, dk;
    if (dput(dx, x, n * 4) || dalloc(df, n * 4) || dalloc(dk, n * 4)) return -1;
    if (n) k_guards<<<blocks(n, 256), 256>>>(dx.as<float>(), n, df.as<uint32_t>(), dk.as<uint32_t>());
    if (ran("k_guards")) return -1;
    return dget(flags, df, n * 4) || dget(keys, dk, n * 4) ? -1 : 0;
}

extern "C" void probe_constants(uint32_t *out) {
    out[0] = QDIV_KEY_MIN;
    out[1] = QDIV_YKEY_MIN;
}

// ---- square root and reciprocal over a range of bit patterns ---------------------------------
// Sequences: 0 sqrt_core, 1 rcp_core, 2 rcp_core(sqrt_core(s)), 3/4 sqrt2_core lo/hi, 5/6 rcp2_core
// lo/hi.  The hi half walks the same range in reverse (bit pattern lo_bits + hi_bits - x).
__global__ void k_roots(uint32_t lo_bits, uint32_t hi_bits, uint32_t first, uint32_t count, probe_tally *t) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    count_block(t, count);
    if (i >= count) return;
    const uint32_t xb = first + i;
    const float s = __uint_as_float(xb), p = __uint_as_float(lo_bits + (hi_bits - xb));
    const float ns = __fsqrt_rn(s), np = __fsqrt_rn(p);
    const float rs = __frcp_rn(s), rp = __frcp_rn(p);
    tally(t, 0, s, 0.f, sqrt_core(s), ns, false);
    tally(t, 1, s, 0.f, rcp_core(s), rs, false);
    tally(t, 2, s, 0.f, rcp_core(sqrt_core(s)), __frcp_rn(ns), false);
    const f2 sp = pk(s, p);
    const f2 n2 = sqrt2_core(sp);
    tally(t, 3, s, p, lo(n2), ns, false);
    tally(t, 4, p, s, hi(n2), np, false);
    const f2 r2 = rcp2_core(sp, neg2(sp));
    tally(t, 5, s, p, lo(r2), rs, false);
    tally(t, 6, p, s, hi(r2), rp, false);
}

extern "C" int probe_roots(uint32_t lo_bits, uint32_t hi_bits, probe_tally *out) {
    if (!out || hi_bits < lo_bits) return bad_args("probe_roots");
    Buf dt;
    if (dalloc(dt, sizeof(probe_tally))) return -1;
    const uint64_t total = (uint64_t)hi_bits - lo_bits + 1;
    const uint32_t chunk = 1u << 25;                       // a few milliseconds per launch
    for (uint64_t done = 0; done < total; done += chunk) {
        const uint32_t count = (uint32_t)(total - done < chunk ? total - done : chunk);
        k_roots<<<blocks(count, 256), 256>>>(lo_bits, hi_bits, (uint32_t)(lo_bits + done), count, dt.as<probe_tally>());
        if (ran("k_roots")) return -1;
    }
    return dget(out, dt, sizeof(probe_tally));
}

// ---- division: every sequence against div.rn.f32 ---------------------------------------------
// Pair i runs in the lo half of the packed sequences, with pair n-1-i in the hi half.  Sequences:
// 0 qdiv_fast, 1 qdiv_fast's ok (must hold), 2 qdiv_core, 3/4 qdiv2 lo/hi, 5 qdiv4_core with
// rcp_low, 6/7 qdiv2x with rcp2_low lo/hi.  y = RN(1/b) as the kernels compute it.
__global__ void k_div(const float *A, const float *B, size_t n, probe_tally *t) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    count_block(t, n);
    if (i >= n) return;
    const float a = A[i], b = B[i], a2 = A[n - 1 - i], b2 = B[n - 1 - i];
    const float want = __fdiv_rn(a, b), want2 = __fdiv_rn(a2, b2);
    const float y = __frcp_rn(b), y2 = __frcp_rn(b2);
    bool ok = true;
    tally(t, 0, a, b, qdiv_fast(a, b, y, ok), want, true);
    if (!ok) tally(t, 1, a, b, 0.f, 1.f, false);
    tally(t, 2, a, b, qdiv_core(a, b, y), want, true);
    const f2 av = pk(a, a2), nb = neg2(pk(b, b2)), yv = pk(y, y2);
    const f2 q5 = qdiv2(av, nb, yv);
    tally(t, 3, a, b, lo(q5), want, true);
    tally(t, 4, a2, b2, hi(q5), want2, true);
    tally(t, 5, a, b, qdiv4_core(a, b, y, rcp_low(b, y)), want, true);
    const f2 q4 = qdiv2x(av, nb, yv, rcp2_low(nb, yv));
    tally(t, 6, a, b, lo(q4), want, true);
    tally(t, 7, a2, b2, hi(q4), want2, true);
}

extern "C" int probe_div(const float *a, const float *b, size_t n, probe_tally *out) {
    if (!a || !b || !out) return bad_args("probe_div");
    Buf da, db, dt;
    if (dput(da, a, n * 4) || dput(db, b, n * 4) || dalloc(dt, sizeof(probe_tally))) return -1;
    if (n) k_div<<<blocks(n, 256), 256>>>(da.as<float>(), db.as<float>(), n, dt.as<probe_tally>());
    if (ran("k_div")) return -1;
    return dget(out, dt, sizeof(probe_tally));
}

// ---- the gradient's divisor pipeline (k_gradient's TV / TGV quotients) --------------------------
// n = sqrt2_core(ss), y = rcp2_core(n, -n) or 0 for a dead source, yl = rcp2_low, qdiv2x(a, ...);
// sequences 0/1: lo/hi against RN(a / RN(sqrt(ss))), or 0 for a dead source.
__global__ void k_grad_div(const float *ss, const float *A, const uint8_t *live, size_t n, probe_tally *t) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    count_block(t, n);
    if (i >= n) return;
    const size_t k = n - 1 - i;
    const f2 s2 = pk(ss[i], ss[k]);
    const f2 nn = sqrt2_core(s2), nb = neg2(nn);
    const f2 yr = rcp2_core(nn, nb);
    const f2 y = pk(live[i] ? lo(yr) : 0.f, live[k] ? hi(yr) : 0.f);
    const f2 yl = rcp2_low(nb, y);
    const f2 q = qdiv2x(pk(A[i], A[k]), nb, y, yl);
    const float w0 = live[i] ? __fdiv_rn(A[i], __fsqrt_rn(ss[i])) : 0.f;
    const float w1 = live[k] ? __fdiv_rn(A[k], __fsqrt_rn(ss[k])) : 0.f;
    tally(t, 0, A[i], ss[i], lo(q), w0, true);
    tally(t, 1, A[k], ss[k], hi(q), w1, true);
}

extern "C" int probe_grad_div(const float *ss, const float *a, const uint8_t *live, size_t n, probe_tally *out) {
    if (!ss || !a || !live || !out) return bad_args("probe_grad_div");
    Buf ds, da, dl, dt;
    if (dput(ds, ss, n * 4) || dput(da, a, n * 4) || dput(dl, live, n) || dalloc(dt, sizeof(probe_tally))) return -1;
    if (n) k_grad_div<<<blocks(n, 256), 256>>>(ds.as<float>(), da.as<float>(), dl.as<uint8_t>(), n, dt.as<probe_tally>());
    if (ran("k_grad_div")) return -1;
    return dget(out, dt, sizeof(probe_tally));
}

// ---- the 8x8 transforms in the projection kernels' lane layout ---------------------------------
// Lane j of an 8-lane group holds row j of its block; the four groups of a warp own four blocks whose
// tiles are TILE_STRIDE floats apart.  Warp step s (one per warp) covers blocks 4s .. 4s+3 (kind 0:
// fdct8x8_rows, 1: idct8x8_rows), or 8s .. 8s+7 for kind 2 (idct8x8_rows_x2: group g transforms
// blocks 8s+g and 8s+4+g in lockstep).  With `active`, group g of step s runs only if bit g of
// active[s] is set, with its own 8-lane mask as the tile kernels pass it; idle blocks keep `out`.
__global__ void __launch_bounds__(128) k_dct(int kind, const float *in, uint32_t nsteps, const uint8_t *active, float *out) {
    __shared__ __align__(16) float tiles[4][2][4][TILE_STRIDE];
    const uint32_t w = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 3, j = lane & 7;
    const uint32_t s = blockIdx.x * 4 + w;
    if (s >= nsteps) return;                                   // whole warps only
    float *tile = tiles[w][0][g];
    if (kind == 2) {
        const size_t ba = ((size_t)s * 8 + g) * 64 + j * 8, bb = ba + 4 * 64;
        float a[8], b[8];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            a[i] = in[ba + i];
            b[i] = in[bb + i];
        }
        idct8x8_rows_x2(a, b, tile, tiles[w][1][g], (int)j);
#pragma unroll
        for (int i = 0; i < 8; i++) {
            out[ba + i] = a[i];
            out[bb + i] = b[i];
        }
        return;
    }
    const size_t at = ((size_t)s * 4 + g) * 64 + j * 8;
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = in[at + i];
    if (active) {
        if (!((active[s] >> g) & 1)) return;
        const unsigned gmask = 0xffu << (lane & 24);
        if (kind == 0) fdct8x8_rows(v, tile, (int)j, gmask);
        else idct8x8_rows(v, tile, (int)j, gmask);
    } else {
        if (kind == 0) fdct8x8_rows(v, tile, (int)j);
        else idct8x8_rows(v, tile, (int)j);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) out[at + i] = v[i];
}

extern "C" int probe_dct(int kind, const float *in, uint32_t nblocks, const uint8_t *active, float *out) {
    const uint32_t per = kind == 2 ? 8 : 4;
    if (!in || !out || kind < 0 || kind > 2 || nblocks % per || (kind == 2 && active)) return bad_args("probe_dct");
    const uint32_t nsteps = nblocks / per;
    const size_t bytes = (size_t)nblocks * 64 * 4;
    Buf di, da, dout;
    if (dput(di, in, bytes) || dput(dout, out, bytes)) return -1;
    if (active && dput(da, active, nsteps)) return -1;
    if (nsteps) k_dct<<<blocks(nsteps, 4), 128>>>(kind, di.as<float>(), nsteps, active ? da.as<uint8_t>() : nullptr, dout.as<float>());
    if (ran("k_dct")) return -1;
    return dget(out, dout, bytes);
}

// ---- the steppers of the projection kernels --------------------------------------------------
// One thread per pixel pair (2i, 2i+1): Stepper::operator() and Stepper::fast on each pixel (with its
// own key), Stepper2::fast on the pair (one key).  rn = RN(1/norm) as k_gradient's last CTA writes it.
__global__ void k_stepper(float factor, float step, float norm, bool stepping, float one, const float *x, const float *xp, const float *g,
                          size_t npairs, float *ieee, float *fast, uint32_t *key, float *fast2, uint32_t *key2) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npairs) return;
    const Stepper st = {factor, step, norm, __frcp_rn(norm), stepping};
    Stepper2 s2;
    s2.init(st, one);
    for (int h = 0; h < 2; h++) {
        const size_t k = 2 * i + h;
        unsigned kk = 0xffffffffu;
        ieee[k] = st(x[k], xp[k], g[k]);
        fast[k] = st.fast(x[k], xp[k], g[k], kk);
        key[k] = kk;
    }
    unsigned k2 = 0xffffffffu;
    const f2 y = s2.fast(pk(x[2 * i], x[2 * i + 1]), pk(xp[2 * i], xp[2 * i + 1]), pk(g[2 * i], g[2 * i + 1]), k2);
    fast2[2 * i] = lo(y);
    fast2[2 * i + 1] = hi(y);
    key2[i] = k2;
}

extern "C" int probe_stepper(float factor, float step, float norm, int stepping, const float *x, const float *xp, const float *g, size_t n,
                             float *ieee, float *fast, uint32_t *key, float *fast2, uint32_t *key2) {
    if (!x || !xp || !g || !ieee || !fast || !key || !fast2 || !key2 || n % 2) return bad_args("probe_stepper");
    Buf dx, dp, dg, di, df, dk, df2, dk2;
    if (dput(dx, x, n * 4) || dput(dp, xp, n * 4) || dput(dg, g, n * 4) || dalloc(di, n * 4) || dalloc(df, n * 4) || dalloc(dk, n * 4) ||
        dalloc(df2, n * 4) || dalloc(dk2, n * 2))
        return -1;
    if (n)
        k_stepper<<<blocks(n / 2, 256), 256>>>(factor, step, norm, stepping != 0, 1.0f, dx.as<float>(), dp.as<float>(), dg.as<float>(), n / 2,
                                               di.as<float>(), df.as<float>(), dk.as<uint32_t>(), df2.as<float>(), dk2.as<uint32_t>());
    if (ran("k_stepper")) return -1;
    return dget(ieee, di, n * 4) || dget(fast, df, n * 4) || dget(key, dk, n * 4) || dget(fast2, df2, n * 4) || dget(key2, dk2, n * 2) ? -1 : 0;
}

// ---- the warp table builder of k_jo_tables / k_jp_tables ---------------------------------------
// One warp per table, four per CTA, scratch in shared memory; table t is warp t % 4 of CTA t / 4 and
// fills slot t % 4 of its CTA's DHT and code tables.  top: the longest K.2 length.
__global__ void __launch_bounds__(128) k_jo(const uint64_t *counts, uint32_t n, uint8_t *bits, uint8_t *vals, uint32_t *nvals, uint16_t *code,
                                            uint8_t *size, uint32_t *top) {
    __shared__ struct j2p_jo_scratch scr[4];
    __shared__ struct j2p_jo_dht d;
    __shared__ struct j2p_je_huff h;
    const uint32_t tb = threadIdx.x >> 5, t = blockIdx.x * 4 + tb;
    if (t >= n) return;                                        // whole warps only
    const WarpLanes L = {threadIdx.x & 31, 32};
    j2p_jo_table(counts + (size_t)t * 256, &scr[tb], &d, &h, (int)tb, L);
    __syncwarp();
    for (uint32_t k = L.lane; k < 256; k += 32) {
        if (k < 16) bits[(size_t)t * 16 + k] = d.bits[tb][k];
        vals[(size_t)t * 256 + k] = d.vals[tb][k];
        code[(size_t)t * 256 + k] = h.code[tb][k];
        size[(size_t)t * 256 + k] = h.size[tb][k];
    }
    if (L.lane == 0) {
        nvals[t] = d.nvals[tb];
        top[t] = scr[tb].top;
    }
}

extern "C" int probe_jo_tables(const uint64_t *counts, uint32_t n, uint8_t *bits, uint8_t *vals, uint32_t *nvals, uint16_t *code, uint8_t *size,
                               uint32_t *top) {
    if (!counts || !bits || !vals || !nvals || !code || !size || !top) return bad_args("probe_jo_tables");
    Buf dc, db, dv, dn, dcode, dsize, dtop;
    if (dput(dc, counts, (size_t)n * 256 * 8) || dalloc(db, (size_t)n * 16) || dalloc(dv, (size_t)n * 256) || dalloc(dn, (size_t)n * 4) ||
        dalloc(dcode, (size_t)n * 512) || dalloc(dsize, (size_t)n * 256) || dalloc(dtop, (size_t)n * 4))
        return -1;
    if (n)
        k_jo<<<blocks(n, 4), 128>>>(dc.as<uint64_t>(), n, db.as<uint8_t>(), dv.as<uint8_t>(), dn.as<uint32_t>(), dcode.as<uint16_t>(),
                                    dsize.as<uint8_t>(), dtop.as<uint32_t>());
    if (ran("k_jo")) return -1;
    return dget(bits, db, (size_t)n * 16) || dget(vals, dv, (size_t)n * 256) || dget(nvals, dn, (size_t)n * 4) ||
                   dget(code, dcode, (size_t)n * 512) || dget(size, dsize, (size_t)n * 256) || dget(top, dtop, (size_t)n * 4)
               ? -1
               : 0;
}

// ---- j2p_pg_nth and J2P_PG_CTZ64 --------------------------------------------------------------
// nth[i * 65 + k] = j2p_pg_nth(m[i], k) for k = 0 .. 64; ctz[i] = J2P_PG_CTZ64(m[i]) (m[i] != 0 only)
__global__ void k_pg_nth(const uint64_t *m, size_t n, int32_t *nth, int32_t *ctz) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (int k = 0; k <= 64; k++) nth[i * 65 + k] = j2p_pg_nth(m[i], k);
    ctz[i] = m[i] ? J2P_PG_CTZ64(m[i]) : -1;
}

extern "C" int probe_pg_nth(const uint64_t *m, size_t n, int32_t *nth, int32_t *ctz) {
    if (!m || !nth || !ctz) return bad_args("probe_pg_nth");
    Buf dm, dn, dz;
    if (dput(dm, m, n * 8) || dalloc(dn, n * 65 * 4) || dalloc(dz, n * 4)) return -1;
    if (n) k_pg_nth<<<blocks(n, 128), 128>>>(dm.as<uint64_t>(), n, dn.as<int32_t>(), dz.as<int32_t>());
    if (ran("k_pg_nth")) return -1;
    return dget(nth, dn, n * 65 * 4) || dget(ctz, dz, n * 4) ? -1 : 0;
}

// the host twin, as the serial host driver compiles it
extern "C" void probe_pg_nth_host(const uint64_t *m, size_t n, int32_t *nth, int32_t *ctz) {
    for (size_t i = 0; i < n; i++) {
        for (int k = 0; k <= 64; k++) nth[i * 65 + k] = j2p_pg_nth(m[i], k);
        ctz[i] = m[i] ? J2P_PG_CTZ64(m[i]) : -1;
    }
}

// ---- j2p_ent_word -----------------------------------------------------------------------------
// A segment of nbytes at byte `off` (a multiple of 4) of buf, which ends where the padded segment
// ends; out[w] = j2p_ent_word(segment, w) for w < nwords.
__global__ void k_ent_word(const uint8_t *base, uint32_t nbytes, uint32_t nwords, uint32_t *out) {
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nwords) return;
    struct j2p_ent_bits b = {};
    b.base = base;
    b.nbytes = nbytes;
    out[w] = j2p_ent_word(&b, w);
}

extern "C" int probe_ent_word(const uint8_t *buf, uint32_t len, uint32_t off, uint32_t nbytes, uint32_t nwords, uint32_t *out) {
    if (!buf || !out || off % 4 || len % 4 || off + ((nbytes + 3) & ~3u) != len) return bad_args("probe_ent_word");
    Buf db, dout;
    if (dput(db, buf, len) || dalloc(dout, (size_t)nwords * 4)) return -1;
    if (nwords) k_ent_word<<<blocks(nwords, 64), 64>>>(db.as<uint8_t>() + off, nbytes, nwords, dout.as<uint32_t>());
    if (ran("k_ent_word")) return -1;
    return dget(out, dout, (size_t)nwords * 4);
}

extern "C" int probe_ent_word_host(const uint8_t *buf, uint32_t len, uint32_t off, uint32_t nbytes, uint32_t nwords, uint32_t *out) {
    if (!buf || !out || off % 4 || len % 4 || off + ((nbytes + 3) & ~3u) != len) return bad_args("probe_ent_word_host");
    struct j2p_ent_bits b = {};
    b.base = buf + off;
    b.nbytes = nbytes;
    for (uint32_t w = 0; w < nwords; w++) out[w] = j2p_ent_word(&b, w);
    return 0;
}

extern "C" const char *probe_last_error(void) { return g_err; }
