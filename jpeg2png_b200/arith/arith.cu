// arith.cu — libj2parith.so: packing of arithmetic layouts, the device decoder (one thread per
// restart segment) and the serial host driver of the same per-segment code.  See arith.h and
// arith_core.h.
#include <string.h>

#include "../cli/jpeg_reader.h"
#include "../common/codec_host.h"
#include "arith.h"
#include "arith_core.h"

extern "C" const char *j2p_arith_last_error(void) { return g_err; }

static const uint32_t kMagic = 0x4a324152u;     // "J2AR"
#define J2P_AR_MAX_BPM 48       // blocks per MCU: three components of up to 4x4 (the reader allows 4)

// ---- plan --------------------------------------------------------------------------------------
struct j2p_ar_file {
    int16_t *out[3];            // int16 [hb][wb][64] per plane, natural order
    uint32_t wb[3], hb[3];      // real block grids
};
struct j2p_ar_scan {
    uint32_t file, ncomp, bpm, mcux;
    uint32_t comp[3], bw[3], bh[3];
    uint32_t dcslot[3], acslot[3];  // the statistics of each component: the first scan slot with its table
    uint32_t L[3], U[3], K[3];      // DAC conditioning
    uint8_t slot[J2P_AR_MAX_BPM], dx[J2P_AR_MAX_BPM], dy[J2P_AR_MAX_BPM];   // block r of an MCU
};
struct j2p_ar_seg {
    uint64_t data_off;
    uint32_t nbytes, scan, mcu0, nmcu;
};
struct j2p_ar_header {
    uint32_t magic, nfiles, nscan, nseg;
    uint64_t off_files, off_scans, off_segs, off_data, total;
};
struct j2p_ar_view {
    const j2p_ar_file *files;
    const j2p_ar_scan *scans;
    const j2p_ar_seg *segs;
    const uint8_t *data;
    uint32_t nseg;
    uint32_t *status;
};

// Per-segment scratch (shared memory on the device): DC statistics of three tables, AC statistics of
// three tables, the fixed bin, then the DC prediction and conditioning category of three components.
enum { kDcOff = 0, kAcOff = 3 * J2P_ARITH_DC_BINS, kFixedOff = kAcOff + 3 * J2P_ARITH_AC_BINS, kPredOff = kFixedOff + 4,
       kCtxOff = kPredOff + 12, kScratch = (kCtxOff + 12 + 15) & ~15 };

static int count(const struct j2p_jpeg_arith_layout *const *L, unsigned n, uint32_t *nscan, uint32_t *nseg, uint64_t *data) {
    *nscan = *nseg = 0;
    *data = 0;
    for (unsigned i = 0; i < n; i++) {
        const struct j2p_jpeg_arith_layout *l = L[i];
        if (!l || !l->arith_decodable) return fail("layout %u is not arithmetic-decodable", i);
        *nscan += l->nscan;
        *nseg += l->nseg;
        for (unsigned k = 0; k < l->nseg; k++) {
            if (l->seg[k].len >= 0xffffffffu) return fail("layout %u: a segment of %zu bytes is too long", i, l->seg[k].len);
            *data += l->seg[k].len;
        }
    }
    return 0;
}

static void offsets(unsigned n, uint32_t nscan, uint32_t nseg, uint64_t data, struct j2p_ar_header *h) {
    h->magic = kMagic;
    h->nfiles = n;
    h->nscan = nscan;
    h->nseg = nseg;
    size_t o = align16(sizeof *h);
    h->off_files = o; o = align16(o + n * sizeof(j2p_ar_file));
    h->off_scans = o; o = align16(o + nscan * sizeof(j2p_ar_scan));
    h->off_segs = o;  o = align16(o + nseg * sizeof(j2p_ar_seg));
    h->off_data = o;  o = align16(o + data);
    h->total = o;
}

static int view_of(const void *plan_host, const void *plan, uint32_t *status, j2p_ar_view *v, const j2p_ar_header **hp) {
    const j2p_ar_header *h = (const j2p_ar_header *)plan_host;
    if (!h || !plan || !status) return fail("null argument");
    if (h->magic != kMagic) return fail("not a packed arithmetic plan");
    const uint8_t *b = (const uint8_t *)plan;
    v->files = (const j2p_ar_file *)(b + h->off_files);
    v->scans = (const j2p_ar_scan *)(b + h->off_scans);
    v->segs = (const j2p_ar_seg *)(b + h->off_segs);
    v->data = b + h->off_data;
    v->nseg = h->nseg;
    v->status = status;
    *hp = h;
    return 0;
}

extern "C" int j2p_arith_plan_size(const struct j2p_jpeg_arith_layout *const *layouts, unsigned n, size_t *plan_bytes, size_t *work_bytes) {
    uint32_t nscan, nseg;
    uint64_t data;
    if (count(layouts, n, &nscan, &nseg, &data) != 0) return -1;
    j2p_ar_header h;
    memset(&h, 0, sizeof h);
    offsets(n, nscan, nseg, data, &h);
    if (plan_bytes) *plan_bytes = h.total;
    if (work_bytes) *work_bytes = 0;
    return 0;
}

extern "C" int j2p_arith_pack(const struct j2p_jpeg_arith_layout *const *L, unsigned n, int16_t *const *out, void *dst, size_t plan_bytes) {
    uint32_t nscan, nseg;
    uint64_t ndata;
    if (count(L, n, &nscan, &nseg, &ndata) != 0) return -1;
    if (!dst || (!out && n)) return fail("null argument");
    uint8_t *b = (uint8_t *)dst;
    j2p_ar_header *h = (j2p_ar_header *)b;
    memset(h, 0, sizeof *h);
    offsets(n, nscan, nseg, ndata, h);
    if (plan_bytes < h->total) return fail("plan buffer of %zu bytes is smaller than the plan (%llu)", plan_bytes, (unsigned long long)h->total);
    j2p_ar_file *files = (j2p_ar_file *)(b + h->off_files);
    j2p_ar_scan *scans = (j2p_ar_scan *)(b + h->off_scans);
    j2p_ar_seg *segs = (j2p_ar_seg *)(b + h->off_segs);
    uint8_t *data = b + h->off_data;
    uint32_t iscan = 0, iseg = 0;
    uint64_t doff = 0;
    for (unsigned i = 0; i < n; i++) {
        const struct j2p_jpeg_arith_layout *l = L[i];
        j2p_ar_file *f = &files[i];
        for (int p = 0; p < 3; p++) {
            f->wb[p] = l->coefs[p].w / 8;
            f->hb[p] = l->coefs[p].h / 8;
            f->out[p] = f->wb[p] ? out[3 * i + p] : nullptr;     // a gray file's planes 1 and 2 are empty
        }
        for (unsigned k = 0; k < l->nscan; k++, iscan++) {
            const struct j2p_jpeg_arith_scan *ls = &l->scan[k];
            j2p_ar_scan *sc = &scans[iscan];
            memset(sc, 0, sizeof *sc);
            sc->file = i;
            sc->ncomp = ls->ncomp;
            sc->mcux = ls->mcux;
            uint32_t bpm = 0;
            for (unsigned s = 0; s < ls->ncomp; s++) {
                sc->comp[s] = ls->comp[s];
                sc->bw[s] = ls->bw[s];
                sc->bh[s] = ls->bh[s];
                sc->dcslot[s] = sc->acslot[s] = s;
                for (unsigned t = 0; t < s; t++) {              // components on one table share its statistics
                    if (ls->dc_tbl[t] == ls->dc_tbl[s] && sc->dcslot[s] == s) sc->dcslot[s] = t;
                    if (ls->ac_tbl[t] == ls->ac_tbl[s] && sc->acslot[s] == s) sc->acslot[s] = t;
                }
                sc->L[s] = ls->dc_L[s];
                sc->U[s] = ls->dc_U[s];
                sc->K[s] = ls->ac_K[s];
                for (unsigned y = 0; y < ls->bh[s]; y++)
                    for (unsigned x = 0; x < ls->bw[s]; x++, bpm++) {
                        sc->slot[bpm] = (uint8_t)s;
                        sc->dx[bpm] = (uint8_t)x;
                        sc->dy[bpm] = (uint8_t)y;
                    }
            }
            sc->bpm = bpm;
            uint32_t mcu0 = 0;
            for (unsigned q = 0; q < ls->nseg; q++, iseg++) {
                const struct j2p_jpeg_segment *lg = &l->seg[ls->seg0 + q];
                j2p_ar_seg *g = &segs[iseg];
                g->data_off = doff;
                g->nbytes = (uint32_t)lg->len;
                g->scan = iscan;
                g->mcu0 = mcu0;
                g->nmcu = lg->mcus;
                memcpy(data + doff, l->data + lg->off, lg->len);
                doff += lg->len;
                mcu0 += lg->mcus;
            }
        }
    }
    return 0;
}

// ---- one segment -------------------------------------------------------------------------------
// Decodes segment j with the scratch area (kScratch bytes, 16-byte aligned): every block of its MCUs
// in order, the blocks inside the plane's real grid written whole (zeros included), MCU padding
// decoded and dropped.  Returns J2P_ARITH_OK or J2P_ARITH_BAD_CODE.
__host__ __device__ static int arith_segment(const j2p_ar_view &v, uint32_t j, uint8_t *scratch) {
    const j2p_ar_seg &g = v.segs[j];
    const j2p_ar_scan &sc = v.scans[g.scan];
    const j2p_ar_file &f = v.files[sc.file];
    uint4 *z = (uint4 *)scratch;
    for (int k = 0; k < kScratch / 16; k++) z[k] = make_uint4(0, 0, 0, 0);
    uint8_t *fixed = scratch + kFixedOff;
    *fixed = J2P_ARITH_FIXED_STATE;
    int *pred = (int *)(scratch + kPredOff), *ctx = (int *)(scratch + kCtxOff);
    struct j2p_qm q;
    j2p_qm_start(&q, v.data + g.data_off, g.nbytes);
    for (uint32_t m = g.mcu0; m < g.mcu0 + g.nmcu; m++) {
        const uint32_t mx = m % sc.mcux, my = m / sc.mcux;
        for (uint32_t r = 0; r < sc.bpm; r++) {
            const uint32_t s = sc.slot[r], c = sc.comp[s];
            const uint32_t bx = mx * sc.bw[s] + sc.dx[r], by = my * sc.bh[s] + sc.dy[r];
            int16_t *b = nullptr;
            if (bx < f.wb[c] && by < f.hb[c]) {
                b = f.out[c] + ((size_t)by * f.wb[c] + bx) * 64;
                uint4 *bz = (uint4 *)b;
                for (int k = 0; k < 8; k++) bz[k] = make_uint4(0, 0, 0, 0);
            }
            if (j2p_arith_block_seq(&q, scratch + kDcOff + J2P_ARITH_DC_BINS * sc.dcslot[s], scratch + kAcOff + J2P_ARITH_AC_BINS * sc.acslot[s],
                                    pred + s, ctx + s, (int)sc.L[s], (int)sc.U[s], (int)sc.K[s], fixed, b) != J2P_ARITH_OK)
                return J2P_ARITH_BAD_CODE;
        }
    }
    return J2P_ARITH_OK;
}

// ---- host driver -------------------------------------------------------------------------------
extern "C" int j2p_arith_decode_host(const void *plan, void *work, uint32_t *status, struct j2p_arith_stats *stats) {
    (void)work;
    j2p_ar_view v = {};
    const j2p_ar_header *h = nullptr;
    if (view_of(plan, plan, status, &v, &h) != 0) return -1;
    memset(status, 0, h->nfiles * sizeof(uint32_t));
    alignas(16) uint8_t scratch[kScratch];
    for (uint32_t j = 0; j < h->nseg; j++) {
        const int rc = arith_segment(v, j, scratch);
        const uint32_t file = v.scans[v.segs[j].scan].file;
        if (rc != J2P_ARITH_OK && status[file] == 0) status[file] = (uint32_t)rc;
    }
    if (stats) {
        stats->launches = 0;
        stats->segments = h->nseg;
    }
    return 0;
}

// ---- device ------------------------------------------------------------------------------------
static const int kThreads = 32;         // 32 x kScratch bytes of statistics per CTA

__global__ void __launch_bounds__(kThreads) k_arith_decode(j2p_ar_view v) {
    __shared__ __align__(16) uint8_t scratch[kThreads * kScratch];
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= v.nseg) return;
    const int rc = arith_segment(v, j, scratch + threadIdx.x * kScratch);
    if (rc != J2P_ARITH_OK) atomicCAS(&v.status[v.scans[v.segs[j].scan].file], 0u, (uint32_t)rc);
}

extern "C" int j2p_arith_decode(const void *plan_host, const void *plan_dev, void *work_dev, uint32_t *status_dev, void *stream,
                                struct j2p_arith_stats *stats) {
    (void)work_dev;
    j2p_ar_view v = {};
    const j2p_ar_header *h = nullptr;
    if (view_of(plan_host, plan_dev, status_dev, &v, &h) != 0) return -1;
    const cudaStream_t st = (cudaStream_t)stream;
    struct j2p_arith_stats s = {0, h->nseg};
    CK(cudaMemsetAsync(status_dev, 0, h->nfiles * sizeof(uint32_t), st));
    if (h->nseg) {
        k_arith_decode<<<(h->nseg + kThreads - 1) / kThreads, kThreads, 0, st>>>(v);
        CK(cudaGetLastError());
        s.launches++;
    }
    if (stats) *stats = s;
    return 0;
}
