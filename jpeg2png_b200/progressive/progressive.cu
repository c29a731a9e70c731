// progressive.cu — libj2pprogressive.so: packing of progressive JPEG layouts, the device decoder
// (zeroing, sync rounds, exclusive scans, DC differences, then per step the stores, DC refine, masks
// and refine walkers) and the serial host driver of the same phases.  See progressive.h and
// progressive_core.h.
#include <string.h>

#include <vector>

#include "../cli/jpeg_reader.h"
#include "../common/codec_host.h"
#include "progressive_core.h"

extern "C" const char *j2p_progressive_last_error(void) { return g_err; }

static const uint32_t kMagic = 0x4a325047u;     // "J2PG"

static uint32_t kind_of(const struct j2p_jpeg_prog_scan *s) {
    if (s->ss == 0) return s->ah == 0 ? J2P_PG_DC_FIRST : J2P_PG_DC_REFINE;
    return s->ah == 0 ? J2P_PG_AC_FIRST : J2P_PG_AC_REFINE;
}
static bool self_sync(uint32_t kind) { return kind == J2P_PG_DC_FIRST || kind == J2P_PG_AC_FIRST; }
static uint32_t nsub_of(size_t len, unsigned S) { return len * 8 > S ? (uint32_t)((len * 8 + S - 1) / S) : 1; }
static uint32_t chunks_of(uint64_t blocks) { return (uint32_t)((blocks + J2P_PG_CHUNK - 1) / J2P_PG_CHUNK); }

// ---- plan --------------------------------------------------------------------------------------
struct Counts {
    uint32_t nscan = 0, nseg = 0, ntab = 0, nsub = 0, nsteps = 0, nrseg = 0, nchunk = 0;
    uint64_t nblocks = 0, nmask = 0, data = 0;
};

// The scans of step t: (file, scan) for every file with more than t scans.
static int count(const struct j2p_jpeg_prog_layout *const *L, unsigned n, unsigned S, Counts *c) {
    if (S < 32 || S % 32) return fail("subseq_bits must be a positive multiple of 32 (got %u)", S);
    for (unsigned i = 0; i < n; i++) {
        const struct j2p_jpeg_prog_layout *l = L[i];
        if (!l || !l->progressive_decodable) return fail("layout %u is not a progressive layout", i);
        if (l->nscan > c->nsteps) c->nsteps = l->nscan;
    }
    for (unsigned t = 0; t < c->nsteps; t++) {
        uint64_t mask = 0;
        for (unsigned i = 0; i < n; i++) {
            const struct j2p_jpeg_prog_layout *l = L[i];
            if (t >= l->nscan) continue;
            const struct j2p_jpeg_prog_scan *ps = &l->scan[t];
            const struct j2p_jpeg_scan *sc = &ps->s;
            const uint32_t kind = kind_of(ps);
            unsigned bpm = 0;
            for (unsigned s = 0; s < sc->ncomp; s++) bpm += sc->bw[s] * sc->bh[s];
            const uint64_t blocks = (uint64_t)sc->mcux * sc->mcuy * bpm;
            c->nscan++;
            c->ntab += 2 * sc->ncomp;
            c->nseg += sc->nseg;
            if (kind == J2P_PG_DC_FIRST) c->nblocks += blocks;
            if (kind == J2P_PG_AC_REFINE) {
                mask += blocks;
                c->nrseg += sc->nseg;
                c->nchunk += chunks_of(blocks);
            }
            for (unsigned k = 0; k < sc->nseg; k++) {
                const struct j2p_jpeg_segment *g = &l->seg[sc->seg0 + k];
                if (g->len >= (1u << 28)) return fail("layout %u: a segment of %zu bytes is too long", i, g->len);
                if (self_sync(kind)) c->nsub += nsub_of(g->len, S);
                if (kind == J2P_PG_DC_REFINE) c->nchunk += chunks_of((uint64_t)g->mcus * bpm);
                c->data += (g->len + 3) & ~(size_t)3;
            }
        }
        if (mask > c->nmask) c->nmask = mask;
    }
    if (c->nblocks >= 0xffffffffull || c->nmask >= 0xffffffffull || c->nsub >= 0x7fffffffu) return fail("too many blocks for one call");
    return 0;
}

static void offsets(unsigned n, const Counts &c, struct j2p_pg_header *h) {
    h->magic = kMagic;
    h->nfiles = n;
    h->nscan = c.nscan;
    h->nseg = c.nseg;
    h->ntab = c.ntab;
    h->nsub = c.nsub;
    h->nsteps = c.nsteps;
    h->nrseg = c.nrseg;
    h->nchunk = c.nchunk;
    h->nblocks = c.nblocks;
    h->nmask = c.nmask;
    size_t o = align16(sizeof *h);
    h->off_files = o;  o = align16(o + n * sizeof(j2p_ent_file));
    h->off_scans = o;  o = align16(o + c.nscan * sizeof(j2p_pg_scan));
    h->off_segs = o;   o = align16(o + c.nseg * sizeof(j2p_ent_seg));
    h->off_subs = o;   o = align16(o + c.nsub * sizeof(uint32_t));
    h->off_tabs = o;   o = align16(o + c.ntab * sizeof(j2p_ent_table));
    h->off_steps = o;  o = align16(o + c.nsteps * sizeof(j2p_pg_step));
    h->off_rsegs = o;  o = align16(o + c.nrseg * sizeof(uint32_t));
    h->off_chunks = o; o = align16(o + c.nchunk * sizeof(j2p_pg_chunk));
    h->off_data = o;   o = align16(o + c.data);
    h->total = o;
}

// work area: exit states x2, start states, cnt, cnt_x, fcnt, dcs[3], dcs_x[3], diff, mask, flag
static size_t work_layout(const struct j2p_pg_header *h, uint8_t *w, struct j2p_pg_view *v) {
    const size_t ns = h->nsub;
    size_t o = 0;
    auto take = [&](size_t bytes) { uint8_t *p = w ? w + o : nullptr; o = align16(o + bytes); return p; };
    uint8_t *e0 = take(ns * 8), *e1 = take(ns * 8), *st = take(ns * 8);
    uint8_t *cnt = take(ns * 8), *cnt_x = take(ns * 8), *fcnt = take(ns * 4);
    uint8_t *dcs = take(ns * 24), *dcs_x = take(ns * 24);
    uint8_t *diff = take(h->nblocks * 4), *mask = take(h->nmask * 8), *flag = take(4);
    if (v) {
        v->exit_st[0] = (uint64_t *)e0;
        v->exit_st[1] = (uint64_t *)e1;
        v->start_st = (uint64_t *)st;
        v->cnt = (uint64_t *)cnt;
        v->cnt_x = (uint64_t *)cnt_x;
        v->fcnt = (uint32_t *)fcnt;
        v->dcs = (uint64_t *)dcs;
        v->dcs_x = (uint64_t *)dcs_x;
        v->diff = (int32_t *)diff;
        v->mask = (uint64_t *)mask;
        v->changed = (uint32_t *)flag;
    }
    return o;
}

static int view_of(const void *plan_host, const void *plan, void *work, uint32_t *status, struct j2p_pg_view *v,
                   const struct j2p_pg_header **hp) {
    const struct j2p_pg_header *h = (const struct j2p_pg_header *)plan_host;
    if (!h || !plan || !work || !status) return fail("null argument");
    if (h->magic != kMagic) return fail("not a packed progressive plan");
    const uint8_t *b = (const uint8_t *)plan;
    memset(v, 0, sizeof *v);
    v->files = (const j2p_ent_file *)(b + h->off_files);
    v->scans = (const j2p_pg_scan *)(b + h->off_scans);
    v->segs = (const j2p_ent_seg *)(b + h->off_segs);
    v->sub_seg = (const uint32_t *)(b + h->off_subs);
    v->tabs = (const j2p_ent_table *)(b + h->off_tabs);
    v->rsegs = (const uint32_t *)(b + h->off_rsegs);
    v->chunks = (const j2p_pg_chunk *)(b + h->off_chunks);
    v->data = b + h->off_data;
    v->nsub = h->nsub;
    v->subseq_bits = h->subseq_bits;
    v->status = status;
    work_layout(h, (uint8_t *)work, v);
    *hp = h;
    return 0;
}

static const j2p_pg_step *steps_of(const struct j2p_pg_header *h) {
    return (const j2p_pg_step *)((const uint8_t *)h + h->off_steps);
}

extern "C" int j2p_progressive_plan_size(const struct j2p_jpeg_prog_layout *const *layouts, unsigned n, unsigned subseq_bits,
                                         size_t *plan_bytes, size_t *work_bytes) {
    Counts c;
    if (count(layouts, n, subseq_bits, &c) != 0) return -1;
    struct j2p_pg_header h;
    memset(&h, 0, sizeof h);
    offsets(n, c, &h);
    if (plan_bytes) *plan_bytes = h.total;
    if (work_bytes) *work_bytes = work_layout(&h, nullptr, nullptr);
    return 0;
}

extern "C" int j2p_progressive_pack(const struct j2p_jpeg_prog_layout *const *L, unsigned n, unsigned S, int16_t *const *out, void *dst,
                                    size_t plan_bytes) {
    Counts c;
    if (count(L, n, S, &c) != 0) return -1;
    if (!dst || (!out && n)) return fail("null argument");
    uint8_t *b = (uint8_t *)dst;
    struct j2p_pg_header *h = (struct j2p_pg_header *)b;
    memset(h, 0, sizeof *h);
    offsets(n, c, h);
    h->subseq_bits = S;
    if (plan_bytes < h->total) return fail("plan buffer of %zu bytes is smaller than the plan (%llu)", plan_bytes, (unsigned long long)h->total);
    j2p_ent_file *files = (j2p_ent_file *)(b + h->off_files);
    j2p_pg_scan *scans = (j2p_pg_scan *)(b + h->off_scans);
    j2p_ent_seg *segs = (j2p_ent_seg *)(b + h->off_segs);
    uint32_t *subs = (uint32_t *)(b + h->off_subs);
    j2p_ent_table *tabs = (j2p_ent_table *)(b + h->off_tabs);
    j2p_pg_step *steps = (j2p_pg_step *)(b + h->off_steps);
    uint32_t *rsegs = (uint32_t *)(b + h->off_rsegs);
    j2p_pg_chunk *chunks = (j2p_pg_chunk *)(b + h->off_chunks);
    uint8_t *data = b + h->off_data;
    for (unsigned i = 0; i < n; i++) {
        for (int p = 0; p < 3; p++) {
            files[i].wb[p] = L[i]->coefs[p].w / 8;
            files[i].hb[p] = L[i]->coefs[p].h / 8;
            files[i].out[p] = files[i].wb[p] ? out[3 * i + p] : nullptr;     // a gray file's planes 1 and 2 are empty
        }
    }
    // everything in step order, files in input order within a step
    uint32_t iscan = 0, iseg = 0, isub = 0, itab = 0, irseg = 0, ichunk = 0, diff_base = 0;
    uint64_t doff = 0;
    for (unsigned t = 0; t < c.nsteps; t++) {
        j2p_pg_step *st = &steps[t];
        memset(st, 0, sizeof *st);
        st->sub0 = isub;
        st->rseg0 = irseg;
        uint32_t mask_base = 0;
        std::vector<j2p_pg_chunk> dchunks, mchunks;
        for (unsigned i = 0; i < n; i++) {
            const struct j2p_jpeg_prog_layout *l = L[i];
            if (t >= l->nscan) continue;
            const struct j2p_jpeg_prog_scan *ps = &l->scan[t];
            const struct j2p_jpeg_scan *ls = &ps->s;
            j2p_pg_scan *sc = &scans[iscan];
            memset(sc, 0, sizeof *sc);
            sc->file = i;
            sc->kind = kind_of(ps);
            sc->ss = ps->ss;
            sc->se = ps->se;
            sc->al = ps->al;
            sc->ncomp = ls->ncomp;
            sc->mcux = ls->mcux;
            uint32_t bpm = 0;
            for (unsigned s = 0; s < ls->ncomp; s++) {
                sc->comp[s] = ls->comp[s];
                sc->bw[s] = ls->bw[s];
                sc->bh[s] = ls->bh[s];
                sc->dctab[s] = itab++;
                sc->actab[s] = itab++;
                j2p_ent_build_table(&ls->dc[s], &tabs[sc->dctab[s]]);
                j2p_ent_build_table(&ls->ac[s], &tabs[sc->actab[s]]);
                for (unsigned y = 0; y < ls->bh[s]; y++)
                    for (unsigned x = 0; x < ls->bw[s]; x++, bpm++) {
                        sc->slot[bpm] = (uint8_t)s;
                        sc->dx[bpm] = (uint8_t)x;
                        sc->dy[bpm] = (uint8_t)y;
                    }
            }
            sc->bpm = bpm;
            const uint32_t blocks = ls->mcux * ls->mcuy * bpm;
            if (sc->kind == J2P_PG_DC_FIRST) {
                sc->diff_base = diff_base;
                diff_base += blocks;
            }
            if (sc->kind == J2P_PG_AC_REFINE) {
                sc->mask_base = mask_base;
                mask_base += blocks;
                for (uint32_t k = 0; k < chunks_of(blocks); k++) mchunks.push_back({iscan, k * J2P_PG_CHUNK});
            }
            uint32_t mcu0 = 0;
            for (unsigned q = 0; q < ls->nseg; q++, iseg++) {
                const struct j2p_jpeg_segment *lg = &l->seg[ls->seg0 + q];
                j2p_ent_seg *g = &segs[iseg];
                g->data_off = doff;
                g->nbytes = (uint32_t)lg->len;
                g->scan = iscan;
                g->block0 = mcu0 * bpm;
                g->nblocks = lg->mcus * bpm;
                g->sub0 = isub;
                g->nsub = 0;
                if (self_sync(sc->kind)) {
                    g->nsub = nsub_of(lg->len, S);
                    for (uint32_t k = 0; k < g->nsub; k++) subs[isub++] = iseg;
                }
                if (sc->kind == J2P_PG_AC_REFINE) rsegs[irseg++] = iseg;
                if (sc->kind == J2P_PG_DC_REFINE)
                    for (uint32_t k = 0; k < chunks_of(g->nblocks); k++) dchunks.push_back({iseg, k * J2P_PG_CHUNK});
                memcpy(data + doff, l->data + lg->off, lg->len);
                const size_t padded = (lg->len + 3) & ~(size_t)3;
                memset(data + doff + lg->len, 0, padded - lg->len);
                doff += padded;
                mcu0 += lg->mcus;
            }
            iscan++;
        }
        st->nsub = isub - st->sub0;
        st->nrseg = irseg - st->rseg0;
        st->dchunk0 = ichunk;
        st->ndchunk = (uint32_t)dchunks.size();
        for (const auto &k : dchunks) chunks[ichunk++] = k;
        st->mchunk0 = ichunk;
        st->nmchunk = (uint32_t)mchunks.size();
        for (const auto &k : mchunks) chunks[ichunk++] = k;
    }
    return 0;
}

// ---- host driver -------------------------------------------------------------------------------
static void scan_host(const uint64_t *in, uint64_t *out, size_t n, int ncol) {
    for (int c = 0; c < ncol; c++) {
        uint64_t run = 0;
        for (size_t i = 0; i < n; i++) {
            out[c * n + i] = run;
            run += in[c * n + i];
        }
    }
}

static void fail_file(const struct j2p_pg_view *v, uint32_t *status, uint32_t scan, int rc) {
    const uint32_t file = v->scans[scan].file;
    if (rc != J2P_ENT_OK && status[file] == 0) status[file] = (uint32_t)rc;
}

extern "C" int j2p_progressive_decode_host(const void *plan, void *work, uint32_t *status, struct j2p_progressive_stats *stats) {
    struct j2p_pg_view v;
    const struct j2p_pg_header *h;
    if (view_of(plan, plan, work, status, &v, &h) != 0) return -1;
    memset(status, 0, h->nfiles * sizeof(uint32_t));
    for (uint32_t i = 0; i < h->nfiles; i++)
        for (int c = 0; c < 3; c++)
            if (v.files[i].out[c]) memset(v.files[i].out[c], 0, (size_t)v.files[i].wb[c] * v.files[i].hb[c] * 64 * sizeof(int16_t));
    unsigned rounds = 0;
    if (h->nsub) {
        for (;;) {
            int changed = 0;
            for (uint32_t j = 0; j < h->nsub; j++) changed |= j2p_pg_sync_one(&v, j, rounds);
            rounds++;
            if (rounds >= 2 && !changed) break;
        }
        scan_host(v.cnt, v.cnt_x, h->nsub, 1);
        for (uint32_t j = 0; j < h->nsub; j++) fail_file(&v, status, v.segs[v.sub_seg[j]].scan, j2p_pg_dcdiff_one(&v, j));
        scan_host(v.dcs, v.dcs_x, h->nsub, 3);
    }
    const j2p_pg_step *steps = steps_of(h);
    for (uint32_t t = 0; t < h->nsteps; t++) {
        const j2p_pg_step &st = steps[t];
        for (uint32_t j = st.sub0; j < st.sub0 + st.nsub; j++) fail_file(&v, status, v.segs[v.sub_seg[j]].scan, j2p_pg_store_one(&v, j));
        for (uint32_t k = st.dchunk0; k < st.dchunk0 + st.ndchunk; k++)
            for (uint32_t b = 0; b < J2P_PG_CHUNK; b++) j2p_pg_dcref_one(&v, &v.chunks[k], b);
        for (uint32_t k = st.mchunk0; k < st.mchunk0 + st.nmchunk; k++)
            for (uint32_t b = 0; b < J2P_PG_CHUNK; b++) j2p_pg_mask_one(&v, &v.chunks[k], b);
        for (uint32_t w = st.rseg0; w < st.rseg0 + st.nrseg; w++) fail_file(&v, status, v.segs[v.rsegs[w]].scan, j2p_pg_refine_one(&v, w));
    }
    if (stats) {
        memset(stats, 0, sizeof *stats);
        stats->rounds = rounds;
        stats->steps = h->nsteps;
        stats->subsequences = h->nsub;
        stats->refine_segments = h->nrseg;
    }
    return 0;
}

// ---- device ------------------------------------------------------------------------------------
static const int kThreads = 128;
static const int kScanThreads = 1024, kScanItems = 4;
static const unsigned kRoundsPerCheck = 4;
static const unsigned kZeroSplit = 8;           // CTAs per plane of the zeroing

// one CTA row per (file, plane), kZeroSplit CTAs along it
__global__ void __launch_bounds__(256) k_pg_zero(struct j2p_pg_view v) {
    const uint32_t p = blockIdx.x, c = p % 3;
    const struct j2p_ent_file *f = &v.files[p / 3];
    uint4 *o = (uint4 *)f->out[c];
    const size_t n = (size_t)f->wb[c] * f->hb[c] * 8;      // 8 uint4 per block
    for (size_t i = (size_t)blockIdx.y * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.y * blockDim.x) o[i] = make_uint4(0, 0, 0, 0);
}

__global__ void __launch_bounds__(kThreads) k_pg_sync(struct j2p_pg_view v, uint32_t round) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= v.nsub) return;
    if (j2p_pg_sync_one(&v, j, round)) *v.changed = 1;
}

__device__ __forceinline__ void fail_file_dev(const struct j2p_pg_view &v, uint32_t scan, int rc) {
    if (rc != J2P_ENT_OK) atomicCAS(&v.status[v.scans[scan].file], 0u, (uint32_t)rc);
}

__global__ void __launch_bounds__(kThreads) k_pg_dcdiff(struct j2p_pg_view v) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= v.nsub) return;
    fail_file_dev(v, v.segs[v.sub_seg[j]].scan, j2p_pg_dcdiff_one(&v, j));
}

__global__ void __launch_bounds__(kThreads) k_pg_store(struct j2p_pg_view v, uint32_t sub0, uint32_t nsub) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nsub) return;
    const uint32_t j = sub0 + k;
    fail_file_dev(v, v.segs[v.sub_seg[j]].scan, j2p_pg_store_one(&v, j));
}

__global__ void __launch_bounds__(J2P_PG_CHUNK) k_pg_dcref(struct j2p_pg_view v, uint32_t chunk0) {
    j2p_pg_dcref_one(&v, &v.chunks[chunk0 + blockIdx.x], threadIdx.x);
}

__global__ void __launch_bounds__(J2P_PG_CHUNK) k_pg_mask(struct j2p_pg_view v, uint32_t chunk0) {
    j2p_pg_mask_one(&v, &v.chunks[chunk0 + blockIdx.x], threadIdx.x);
}

__global__ void __launch_bounds__(32) k_pg_refine(struct j2p_pg_view v, uint32_t rseg0, uint32_t nrseg) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nrseg) return;
    const uint32_t w = rseg0 + k;
    fail_file_dev(v, v.segs[v.rsegs[w]].scan, j2p_pg_refine_one(&v, w));
}

// exclusive scan of ncol columns of n uint64 each (column c at in + c * n), one CTA
__global__ void __launch_bounds__(kScanThreads) k_pg_scan(const uint64_t *__restrict__ in, uint64_t *__restrict__ out, uint32_t n, int ncol) {
    __shared__ uint64_t warp_sums[kScanThreads / 32];
    __shared__ uint64_t tile_total;
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    for (int c = 0; c < ncol; c++) {
        const uint64_t *src = in + (size_t)c * n;
        uint64_t *dst = out + (size_t)c * n;
        uint64_t carry = 0;
        for (uint32_t base = 0; base < n; base += kScanThreads * kScanItems) {
            uint64_t x[kScanItems], sum = 0;
            const uint32_t i0 = base + (uint32_t)t * kScanItems;
#pragma unroll
            for (int k = 0; k < kScanItems; k++) {
                x[k] = i0 + k < n ? src[i0 + k] : 0;
                sum += x[k];
            }
            uint64_t incl = sum;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint64_t y = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += y;
            }
            if (lane == 31) warp_sums[wid] = incl;
            __syncthreads();
            if (wid == 0) {
                uint64_t w = warp_sums[lane], wi = w;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const uint64_t y = __shfl_up_sync(0xffffffffu, wi, d);
                    if (lane >= d) wi += y;
                }
                warp_sums[lane] = wi - w;
                if (lane == 31) tile_total = wi;
            }
            __syncthreads();
            uint64_t run = carry + warp_sums[wid] + incl - sum;
#pragma unroll
            for (int k = 0; k < kScanItems; k++) {
                if (i0 + k < n) dst[i0 + k] = run;
                run += x[k];
            }
            carry += tile_total;
            __syncthreads();
        }
    }
}

extern "C" int j2p_progressive_decode(const void *plan_host, const void *plan_dev, void *work_dev, uint32_t *status_dev, void *stream,
                                      struct j2p_progressive_stats *stats) {
    struct j2p_pg_view v;
    const struct j2p_pg_header *h;
    if (view_of(plan_host, plan_dev, work_dev, status_dev, &v, &h) != 0) return -1;
    const cudaStream_t st = (cudaStream_t)stream;
    struct j2p_progressive_stats s;
    memset(&s, 0, sizeof s);
    s.steps = h->nsteps;
    s.subsequences = h->nsub;
    s.refine_segments = h->nrseg;
    CK(cudaMemsetAsync(status_dev, 0, h->nfiles * sizeof(uint32_t), st));
    if (h->nfiles) {
        k_pg_zero<<<dim3(3 * h->nfiles, kZeroSplit), 256, 0, st>>>(v);
        CK(cudaGetLastError());
        s.launches++;
    }
    if (h->nsub) {
        const unsigned grid = (h->nsub + kThreads - 1) / kThreads;
        // a segment of m subsequences is exact after m rounds at most; a round with no change ends it
        uint32_t max_rounds = 2;
        const struct j2p_ent_seg *segs = (const struct j2p_ent_seg *)((const uint8_t *)plan_host + h->off_segs);
        for (uint32_t k = 0; k < h->nseg; k++)
            if (segs[k].nsub + 2 > max_rounds) max_rounds = segs[k].nsub + 2;
        for (;;) {
            for (unsigned k = 0; k < kRoundsPerCheck; k++) {
                if (k + 1 == kRoundsPerCheck) CK(cudaMemsetAsync(v.changed, 0, sizeof(uint32_t), st));
                k_pg_sync<<<grid, kThreads, 0, st>>>(v, s.rounds);
                CK(cudaGetLastError());
                s.rounds++;
                s.launches++;
            }
            uint32_t changed = 0;
            CK(cudaMemcpyAsync(&changed, v.changed, sizeof changed, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            s.round_trips++;
            if (!changed) break;
            if (s.rounds > max_rounds) return fail("sync rounds did not converge (%u rounds)", s.rounds);
        }
        k_pg_scan<<<1, kScanThreads, 0, st>>>(v.cnt, v.cnt_x, h->nsub, 1);
        CK(cudaGetLastError());
        k_pg_dcdiff<<<grid, kThreads, 0, st>>>(v);
        CK(cudaGetLastError());
        k_pg_scan<<<1, kScanThreads, 0, st>>>(v.dcs, v.dcs_x, h->nsub, 3);
        CK(cudaGetLastError());
        s.launches += 3;
    }
    const j2p_pg_step *steps = steps_of(h);
    for (uint32_t t = 0; t < h->nsteps; t++) {
        const j2p_pg_step &p = steps[t];
        if (p.nsub) {
            k_pg_store<<<(p.nsub + kThreads - 1) / kThreads, kThreads, 0, st>>>(v, p.sub0, p.nsub);
            CK(cudaGetLastError());
            s.step_launches++;
        }
        if (p.ndchunk) {
            k_pg_dcref<<<p.ndchunk, J2P_PG_CHUNK, 0, st>>>(v, p.dchunk0);
            CK(cudaGetLastError());
            s.step_launches++;
        }
        if (p.nmchunk) {
            k_pg_mask<<<p.nmchunk, J2P_PG_CHUNK, 0, st>>>(v, p.mchunk0);
            CK(cudaGetLastError());
            s.step_launches++;
        }
        if (p.nrseg) {
            // a walker is serial: few walkers get a CTA each, so no two share a warp's issue slots
            const unsigned per = p.nrseg <= 4096 ? 1 : 32;
            k_pg_refine<<<(p.nrseg + per - 1) / per, per, 0, st>>>(v, p.rseg0, p.nrseg);
            CK(cudaGetLastError());
            s.step_launches++;
        }
    }
    s.launches += s.step_launches;
    if (stats) *stats = s;
    return 0;
}
