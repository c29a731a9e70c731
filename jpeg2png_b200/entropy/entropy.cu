// entropy.cu — libj2pentropy.so: packing of JPEG layouts, the device decoder (sync rounds, exclusive
// scans, final pass, DC pass) and the serial host driver of the same phases.  See entropy.h and
// entropy_core.h.
#include <string.h>

#include "../cli/jpeg_reader.h"
#include "../common/codec_host.h"
#include "entropy_core.h"

extern "C" const char *j2p_entropy_last_error(void) { return g_err; }

static const uint32_t kMagic = 0x4a32454eu;     // "J2EN"

// ---- plan --------------------------------------------------------------------------------------
struct Counts {
    uint32_t nscan = 0, nseg = 0, nsub = 0, nslot = 3;
    uint64_t nblocks = 0, data = 0;
};

// Layout: struct j2p_jpeg_layout (planes of three-component and gray files, out[3 * i + c]) or
// struct j2p_jpeg_layout4 (four-component files, out[4 * i + c]); NP: its planes per file
template <class Layout>
static int count(const Layout *const *L, unsigned n, unsigned S, Counts *c) {
    if (S < 32 || S % 32) return fail("subseq_bits must be a positive multiple of 32 (got %u)", S);
    for (unsigned i = 0; i < n; i++) {
        const Layout *l = L[i];
        if (!l || !l->device_decodable) return fail("layout %u is not device-decodable", i);
        for (unsigned k = 0; k < l->nscan; k++) {
            const auto *sc = &l->scan[k];
            unsigned bpm = 0;
            for (unsigned s = 0; s < sc->ncomp; s++) bpm += sc->bw[s] * sc->bh[s];
            if (bpm > J2P_ENT_MAX_BPM) return fail("layout %u: %u blocks per MCU", i, bpm);
            if (sc->ncomp > 3) c->nslot = 4;
            c->nblocks += (uint64_t)sc->mcux * sc->mcuy * bpm;
        }
        c->nscan += l->nscan;
        c->nseg += l->nseg;
        for (unsigned k = 0; k < l->nseg; k++) {
            const size_t len = l->seg[k].len;
            if (len >= (1u << 28)) return fail("layout %u: a segment of %zu bytes is too long", i, len);
            c->nsub += len * 8 > S ? (uint32_t)((len * 8 + S - 1) / S) : 1;
            c->data += (len + 3) & ~(size_t)3;
        }
    }
    if (c->nblocks >= 0xffffffffull || c->nsub >= 0x7fffffffu) return fail("too many blocks for one call");
    return 0;
}

static void offsets(unsigned n, const Counts &c, struct j2p_ent_header *h) {
    h->magic = kMagic;
    h->nfiles = n;
    h->nscan = c.nscan;
    h->nseg = c.nseg;
    h->ntab = 2 * J2P_ENT_PLANES * c.nscan;
    h->nslot = c.nslot;
    h->nsub = c.nsub;
    h->nblocks = c.nblocks;
    size_t o = align16(sizeof *h);
    h->off_files = o; o = align16(o + n * sizeof(j2p_ent_file));
    h->off_scans = o; o = align16(o + c.nscan * sizeof(j2p_ent_scan));
    h->off_segs = o;  o = align16(o + c.nseg * sizeof(j2p_ent_seg));
    h->off_subs = o;  o = align16(o + c.nsub * sizeof(uint32_t));
    h->off_tabs = o;  o = align16(o + h->ntab * sizeof(j2p_ent_table));
    h->off_data = o;  o = align16(o + c.data);
    h->total = o;
}

// work area: exit states x2, start states, cnt, cnt_x, fcnt, dcs[nslot], dcs_x[nslot], diff, flag
static size_t work_layout(const struct j2p_ent_header *h, uint8_t *w, struct j2p_ent_view *v) {
    const size_t ns = h->nsub;
    size_t o = 0;
    auto take = [&](size_t bytes) { uint8_t *p = w ? w + o : nullptr; o = align16(o + bytes); return p; };
    uint8_t *e0 = take(ns * 8), *e1 = take(ns * 8), *st = take(ns * 8);
    uint8_t *cnt = take(ns * 4), *cnt_x = take(ns * 4), *fcnt = take(ns * 4);
    uint8_t *dcs = take(ns * 4 * h->nslot), *dcs_x = take(ns * 4 * h->nslot);
    uint8_t *diff = take(h->nblocks * 4), *flag = take(4);
    if (v) {
        v->exit_st[0] = (uint64_t *)e0;
        v->exit_st[1] = (uint64_t *)e1;
        v->start_st = (uint64_t *)st;
        v->cnt = (uint32_t *)cnt;
        v->cnt_x = (uint32_t *)cnt_x;
        v->fcnt = (uint32_t *)fcnt;
        v->dcs = (uint32_t *)dcs;
        v->dcs_x = (uint32_t *)dcs_x;
        v->diff = (int32_t *)diff;
        v->changed = (uint32_t *)flag;
    }
    return o;
}

static int view_of(const void *plan_host, const void *plan, void *work, uint32_t *status, struct j2p_ent_view *v,
                   const struct j2p_ent_header **hp) {
    const struct j2p_ent_header *h = (const struct j2p_ent_header *)plan_host;
    if (!h || !plan || !work || !status) return fail("null argument");
    if (h->magic != kMagic) return fail("not a packed entropy plan");
    const uint8_t *b = (const uint8_t *)plan;
    memset(v, 0, sizeof *v);
    v->files = (const j2p_ent_file *)(b + h->off_files);
    v->scans = (const j2p_ent_scan *)(b + h->off_scans);
    v->segs = (const j2p_ent_seg *)(b + h->off_segs);
    v->sub_seg = (const uint32_t *)(b + h->off_subs);
    v->tabs = (const j2p_ent_table *)(b + h->off_tabs);
    v->data = b + h->off_data;
    v->nsub = h->nsub;
    v->subseq_bits = h->subseq_bits;
    v->nslot = h->nslot;
    v->status = status;
    work_layout(h, (uint8_t *)work, v);
    *hp = h;
    return 0;
}

template <class Layout>
static int plan_size(const Layout *const *layouts, unsigned n, unsigned subseq_bits, size_t *plan_bytes, size_t *work_bytes) {
    Counts c;
    if (count(layouts, n, subseq_bits, &c) != 0) return -1;
    struct j2p_ent_header h;
    memset(&h, 0, sizeof h);
    offsets(n, c, &h);
    if (plan_bytes) *plan_bytes = h.total;
    if (work_bytes) *work_bytes = work_layout(&h, nullptr, nullptr);
    return 0;
}

template <class Layout, int NP>
static int pack(const Layout *const *L, unsigned n, unsigned S, int16_t *const *out, void *dst, size_t plan_bytes) {
    Counts c;
    if (count(L, n, S, &c) != 0) return -1;
    if (!dst || (!out && n)) return fail("null argument");
    uint8_t *b = (uint8_t *)dst;
    struct j2p_ent_header *h = (struct j2p_ent_header *)b;
    memset(h, 0, sizeof *h);
    offsets(n, c, h);
    h->subseq_bits = S;
    if (plan_bytes < h->total) return fail("plan buffer of %zu bytes is smaller than the plan (%llu)", plan_bytes, (unsigned long long)h->total);
    j2p_ent_file *files = (j2p_ent_file *)(b + h->off_files);
    j2p_ent_scan *scans = (j2p_ent_scan *)(b + h->off_scans);
    j2p_ent_seg *segs = (j2p_ent_seg *)(b + h->off_segs);
    uint32_t *subs = (uint32_t *)(b + h->off_subs);
    j2p_ent_table *tabs = (j2p_ent_table *)(b + h->off_tabs);
    uint8_t *data = b + h->off_data;
    uint32_t iscan = 0, iseg = 0, isub = 0, diff_base = 0;
    uint64_t doff = 0;
    for (unsigned i = 0; i < n; i++) {
        const Layout *l = L[i];
        j2p_ent_file *f = &files[i];
        memset(f, 0, sizeof *f);
        for (int p = 0; p < NP; p++) {
            f->wb[p] = l->coefs[p].w / 8;
            f->hb[p] = l->coefs[p].h / 8;
            f->out[p] = f->wb[p] ? out[NP * i + p] : nullptr;    // a gray file's planes 1 and 2 are empty
        }
        for (unsigned k = 0; k < l->nscan; k++, iscan++) {
            const auto *ls = &l->scan[k];
            j2p_ent_scan *sc = &scans[iscan];
            memset(sc, 0, sizeof *sc);
            sc->file = i;
            sc->ncomp = ls->ncomp;
            sc->mcux = ls->mcux;
            uint32_t bpm = 0;
            for (unsigned s = 0; s < ls->ncomp; s++) {
                sc->comp[s] = ls->comp[s];
                sc->bw[s] = ls->bw[s];
                sc->bh[s] = ls->bh[s];
                sc->dctab[s] = 2 * J2P_ENT_PLANES * iscan + 2 * s;
                sc->actab[s] = 2 * J2P_ENT_PLANES * iscan + 2 * s + 1;
                j2p_ent_build_table(&ls->dc[s], &tabs[sc->dctab[s]]);
                j2p_ent_build_table(&ls->ac[s], &tabs[sc->actab[s]]);
                for (unsigned y = 0; y < ls->bh[s]; y++)
                    for (unsigned x = 0; x < ls->bw[s]; x++, bpm++) {
                        sc->slot[bpm] = (uint8_t)s;
                        sc->dx[bpm] = (uint8_t)x;
                        sc->dy[bpm] = (uint8_t)y;
                    }
            }
            for (unsigned s = ls->ncomp; s < J2P_ENT_PLANES; s++)
                memset(&tabs[2 * J2P_ENT_PLANES * iscan + 2 * s], 0, 2 * sizeof(j2p_ent_table));   // unused slots
            sc->bpm = bpm;
            sc->diff_base = diff_base;
            diff_base += ls->mcux * ls->mcuy * bpm;
            uint32_t mcu0 = 0;
            for (unsigned q = 0; q < ls->nseg; q++, iseg++) {
                const struct j2p_jpeg_segment *ls_g = &l->seg[ls->seg0 + q];
                j2p_ent_seg *g = &segs[iseg];
                g->data_off = doff;
                g->nbytes = (uint32_t)ls_g->len;
                g->scan = iscan;
                g->block0 = mcu0 * bpm;
                g->nblocks = ls_g->mcus * bpm;
                g->sub0 = isub;
                g->nsub = ls_g->len * 8 > S ? (uint32_t)((ls_g->len * 8 + S - 1) / S) : 1;
                for (uint32_t t = 0; t < g->nsub; t++) subs[isub++] = iseg;
                memcpy(data + doff, l->data + ls_g->off, ls_g->len);
                const size_t padded = (ls_g->len + 3) & ~(size_t)3;
                memset(data + doff + ls_g->len, 0, padded - ls_g->len);
                doff += padded;
                mcu0 += ls_g->mcus;
            }
        }
    }
    return 0;
}

extern "C" int j2p_entropy_plan_size(const struct j2p_jpeg_layout *const *layouts, unsigned n, unsigned subseq_bits,
                                     size_t *plan_bytes, size_t *work_bytes) {
    return plan_size(layouts, n, subseq_bits, plan_bytes, work_bytes);
}

extern "C" int j2p_entropy_pack(const struct j2p_jpeg_layout *const *L, unsigned n, unsigned S, int16_t *const *out, void *dst,
                                size_t plan_bytes) {
    return pack<struct j2p_jpeg_layout, 3>(L, n, S, out, dst, plan_bytes);
}

extern "C" int j2p_entropy_plan_size4(const struct j2p_jpeg_layout4 *const *layouts, unsigned n, unsigned subseq_bits,
                                      size_t *plan_bytes, size_t *work_bytes) {
    return plan_size(layouts, n, subseq_bits, plan_bytes, work_bytes);
}

extern "C" int j2p_entropy_pack4(const struct j2p_jpeg_layout4 *const *L, unsigned n, unsigned S, int16_t *const *out, void *dst,
                                 size_t plan_bytes) {
    return pack<struct j2p_jpeg_layout4, 4>(L, n, S, out, dst, plan_bytes);
}

// ---- host driver -------------------------------------------------------------------------------
static void scan_host(const uint32_t *in, uint32_t *out, size_t n, int ncol) {
    for (int c = 0; c < ncol; c++) {
        uint32_t run = 0;
        for (size_t i = 0; i < n; i++) {
            out[c * n + i] = run;
            run += in[c * n + i];
        }
    }
}

extern "C" int j2p_entropy_decode_host(const void *plan, void *work, uint32_t *status, struct j2p_entropy_stats *stats) {
    struct j2p_ent_view v;
    const struct j2p_ent_header *h;
    if (view_of(plan, plan, work, status, &v, &h) != 0) return -1;
    memset(status, 0, h->nfiles * sizeof(uint32_t));
    unsigned rounds = 0;
    for (;;) {
        int changed = 0;
        for (uint32_t j = 0; j < h->nsub; j++) changed |= j2p_ent_sync_one(&v, j, rounds);
        rounds++;
        if (rounds >= 2 && !changed) break;
    }
    scan_host(v.cnt, v.cnt_x, h->nsub, 1);
    for (uint32_t j = 0; j < h->nsub; j++) {
        const int rc = j2p_ent_final_one(&v, j);
        const uint32_t file = v.scans[v.segs[v.sub_seg[j]].scan].file;
        if (rc != J2P_ENT_OK && status[file] == 0) status[file] = (uint32_t)rc;
    }
    scan_host(v.dcs, v.dcs_x, h->nsub, (int)h->nslot);
    for (uint32_t j = 0; j < h->nsub; j++) j2p_ent_dc_one(&v, j);
    if (stats) {
        stats->rounds = rounds;
        stats->round_trips = 0;
        stats->launches = 0;
        stats->subsequences = h->nsub;
    }
    return 0;
}

// ---- device ------------------------------------------------------------------------------------
static const int kThreads = 128;
static const int kScanThreads = 1024, kScanItems = 8;
static const unsigned kRoundsPerCheck = 4;

__global__ void __launch_bounds__(kThreads) k_ent_sync(struct j2p_ent_view v, uint32_t round) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= v.nsub) return;
    if (j2p_ent_sync_one(&v, j, round)) *v.changed = 1;
}

__global__ void __launch_bounds__(kThreads) k_ent_final(struct j2p_ent_view v) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= v.nsub) return;
    const int rc = j2p_ent_final_one(&v, j);
    if (rc != J2P_ENT_OK) atomicCAS(&v.status[v.scans[v.segs[v.sub_seg[j]].scan].file], 0u, (uint32_t)rc);
}

__global__ void __launch_bounds__(kThreads) k_ent_dc(struct j2p_ent_view v) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= v.nsub) return;
    j2p_ent_dc_one(&v, j);
}

// exclusive scan of ncol columns of n uint32 each (column c at in + c * n), one CTA
__global__ void __launch_bounds__(kScanThreads) k_ent_scan(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, uint32_t n, int ncol) {
    __shared__ uint32_t warp_sums[kScanThreads / 32];
    __shared__ uint32_t tile_total;
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    for (int c = 0; c < ncol; c++) {
        const uint32_t *src = in + (size_t)c * n;
        uint32_t *dst = out + (size_t)c * n;
        uint32_t carry = 0;
        for (uint32_t base = 0; base < n; base += kScanThreads * kScanItems) {
            uint32_t x[kScanItems], sum = 0;
            const uint32_t i0 = base + (uint32_t)t * kScanItems;
#pragma unroll
            for (int k = 0; k < kScanItems; k++) {
                x[k] = i0 + k < n ? src[i0 + k] : 0;
                sum += x[k];
            }
            uint32_t incl = sum;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += y;
            }
            if (lane == 31) warp_sums[wid] = incl;
            __syncthreads();
            if (wid == 0) {
                uint32_t w = warp_sums[lane], wi = w;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const uint32_t y = __shfl_up_sync(0xffffffffu, wi, d);
                    if (lane >= d) wi += y;
                }
                warp_sums[lane] = wi - w;
                if (lane == 31) tile_total = wi;
            }
            __syncthreads();
            uint32_t run = carry + warp_sums[wid] + incl - sum;
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

extern "C" int j2p_entropy_decode(const void *plan_host, const void *plan_dev, void *work_dev, uint32_t *status_dev, void *stream,
                                  struct j2p_entropy_stats *stats) {
    struct j2p_ent_view v;
    const struct j2p_ent_header *h;
    if (view_of(plan_host, plan_dev, work_dev, status_dev, &v, &h) != 0) return -1;
    const cudaStream_t st = (cudaStream_t)stream;
    struct j2p_entropy_stats s = {0, 0, 0, h->nsub};
    CK(cudaMemsetAsync(status_dev, 0, h->nfiles * sizeof(uint32_t), st));
    if (h->nsub) {
        const unsigned grid = (h->nsub + kThreads - 1) / kThreads;
        // a segment of m subsequences is exact after m rounds at most; a round with no change ends it
        uint32_t max_rounds = 2;
        for (uint32_t k = 0; k < h->nseg; k++) {
            const struct j2p_ent_seg *g = (const struct j2p_ent_seg *)((const uint8_t *)plan_host + h->off_segs) + k;
            if (g->nsub + 2 > max_rounds) max_rounds = g->nsub + 2;
        }
        // Rounds go in groups of kRoundsPerCheck; the host reads the flag of a group's last round only.
        // A round whose starts did not change costs a compare per subsequence, a round trip tens of us.
        for (;;) {
            for (unsigned k = 0; k < kRoundsPerCheck; k++) {
                if (k + 1 == kRoundsPerCheck) CK(cudaMemsetAsync(v.changed, 0, sizeof(uint32_t), st));
                k_ent_sync<<<grid, kThreads, 0, st>>>(v, s.rounds);
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
        k_ent_scan<<<1, kScanThreads, 0, st>>>(v.cnt, v.cnt_x, h->nsub, 1);
        CK(cudaGetLastError());
        k_ent_final<<<grid, kThreads, 0, st>>>(v);
        CK(cudaGetLastError());
        k_ent_scan<<<1, kScanThreads, 0, st>>>(v.dcs, v.dcs_x, h->nsub, (int)h->nslot);
        CK(cudaGetLastError());
        k_ent_dc<<<grid, kThreads, 0, st>>>(v);
        CK(cudaGetLastError());
        s.launches += 4;
    }
    if (stats) *stats = s;
    return 0;
}
