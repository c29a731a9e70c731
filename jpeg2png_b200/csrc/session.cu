// session.cu — host side of the solver: HBM residency, the iteration loop, the C ABI.
//
// Implements the `j2p_*` session layer of include/jpeg2png_b200.h.  One session = one frame (or
// one strip of a frame) on one device with its own CUDA stream; sessions share no mutable state,
// so `compute()` built on top of them is re-entrant like the reference (jpeg2png.c:147, :330).
//
// HBM layout per plane c (W x H = working frame, cw x ch = coefficient grid):
//   x, xp   H*W fp32   iterate x_k and x_{k-1}; k_project overwrites xp with x_{k+1}, then the
//                      two pointers swap (reference SWAP at compute.c:438)
//   g       H*W fp32   sub-gradient
//   gp      ch*cw fp32 DCT-distance gradient for the next step, coefficient resolution
//   data    ch*cw i16  quantised coefficients (read-only)
//   fdata0  ch*cw fp32 conventional decode (kept so a session can be re-armed without host I/O)
// plus per session: partials [3][grad_ctas] fp64, norms [3] fp32, one ticket counter.
//
// A batch session (j2p_session_create_batch) holds N frames of one geometry.  Frame f's x, xp, g,
// gp are the slab of one frame repeated at a fixed frame stride; data and fdata0 likewise, each in
// one block; partials [frame][5][grad_ctas], norms [frame][16], sums [frame][4], counters [frame];
// the quantisation tables in device memory as [frame][nc][3][64].  An iteration is the launches of
// a single-frame session, each covering every frame (kernels.cuh, FrameDev::nframes).
#include <cuda_runtime.h>

#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <time.h>

#include <atomic>
#include <algorithm>
#include <map>
#include <string>
#include <mutex>
#include <utility>
#include <vector>

#include "../../include/jpeg2png_b200.h"
#include "copy_pool.h"
#include "geometry.cuh"
#include "kernels.cuh"
#include "record.cuh"
#include "tma_maps.h"

namespace j2p {
int grad_cta_count(int W, int H);
cudaError_t configure_kernels(int *slots);
cudaError_t launch_gradient(const FrameDev &F, float factor, cudaStream_t s);
cudaError_t launch_project(const FrameDev &F, float factor, cudaStream_t s, int *nlaunch);
cudaError_t launch_fold_sums(const double *sums_by_rank, int nranks, int nc, float *norms, cudaStream_t s);
cudaError_t launch_decode(const int16_t *data, const float *q_host, float *out, int cw, int ch, cudaStream_t s);
cudaError_t launch_init_plane(const float *fdata, float *x, float *xp, int W, int H, int cw, int ch, int sw, int sh,
                              cudaStream_t s);
bool project_tma_enabled();
int project_tma_border_units(const PlaneDev &P);
int project_tile_border_units(const PlaneDev &P);
cudaError_t launch_scanlines(const EpilogueArgs &a, int nframes, cudaStream_t s, int *nlaunch);
// kernels_strip.cu: the strip exchanges over peer memory (parameter blocks in kernels.cuh)
cudaError_t launch_halo_exchange(const HaloPeers &P, unsigned seq, unsigned *ticket, int *err, int wait_for_arrival, cudaStream_t s);
// kernels_gradient_packed.cu: the packed gradient's GPM and grid for a frame (what a group gives it)
int packed_gradient_gpm(const FrameDev &F);
void packed_gradient_geometry(const FrameDev &F, int *cx, int *bands, int *rows);
// the stepped-only pixels of 1x1 / 2x2 planes (uncovered_only), next to the recording projection
cudaError_t launch_project_tile(const FrameDev &F, int c, int count, float factor, cudaStream_t s, int *nlaunch, bool uncovered_only);
cudaError_t launch_project_tile22(const FrameDev &F, int c, int count, float factor, cudaStream_t s, int *nlaunch, bool uncovered_only);
}  // namespace j2p

using namespace j2p;

static thread_local char g_err[512] = "";

static int fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
    return code;
}

#define CK(call)                                                                                      \
    do {                                                                                              \
        cudaError_t e_ = (call);                                                                      \
        if (e_ != cudaSuccess) {                                                                      \
            cudaGetLastError();   /* a refused launch also sets the thread's last error: later calls must not see it */ \
            return fail(J2P_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
        }                                                                                             \
    } while (0)

constexpr int kEventRing = 32;
// An event is recorded after every kEventStride-th iteration only: an event record between two kernels
// keeps the second from being launched as a programmatic dependent of the first (pdl.cuh).  Waiting
// for iteration i means waiting for the first recorded iteration >= i (stream order), or for the
// stream when none has been recorded yet.
constexpr unsigned kEventStride = 4;

// ---- device memory: a process-wide cache of device blocks keyed by (device, exact size).  A
// session takes its ~25 blocks from it and gives them back when it is destroyed (its stream is
// idle by then), so a compute() call pays for cudaMalloc only the first time a frame size is seen
// and never for cudaFree's device-wide synchronisation.  (cudaMallocAsync with an unbounded
// release threshold did the same on paper; inside a process that also runs PyTorch its calls
// took milliseconds per session.)
struct DevCache {
    std::mutex mu;
    std::multimap<std::pair<int, size_t>, void *> blocks;
    size_t held[64] = {};                                              // bytes cached per device
    // bytes kept at most PER DEVICE (J2P_DEVCACHE_GB, default 8); beyond that blocks are freed
    static size_t cap() {
        static const size_t c = [] {
            const char *e = getenv("J2P_DEVCACHE_GB");
            const double gb = e && *e ? atof(e) : 8.0;
            return (size_t)((gb < 0 ? 0 : gb) * (double)(1u << 30));
        }();
        return c;
    }
    // best fit: the smallest cached block of at least `bytes` that wastes at most a quarter of
    // itself (a batch of JPEGs of many sizes re-uses blocks instead of piling up exact sizes)
    void *get(int dev, size_t bytes, size_t *got) {
        std::lock_guard<std::mutex> l(mu);
        auto it = blocks.lower_bound({dev, bytes});
        if (it == blocks.end() || it->first.first != dev || it->first.second > bytes + bytes / 4 + 4096) return nullptr;
        void *p = it->second;
        *got = it->first.second;
        held[dev & 63] -= *got;
        blocks.erase(it);
        return p;
    }
    bool put(int dev, void *p, size_t bytes) {
        std::lock_guard<std::mutex> l(mu);
        if (held[dev & 63] + bytes > cap()) return false;
        blocks.insert({{dev, bytes}, p});
        held[dev & 63] += bytes;
        return true;
    }
    // give every idle block of `dev` back to the driver (the current device must be `dev`)
    void trim(int dev) {
        std::lock_guard<std::mutex> l(mu);
        for (auto it = blocks.lower_bound({dev, 0}); it != blocks.end() && it->first.first == dev;) {
            cudaFree(it->second);
            it = blocks.erase(it);
        }
        held[dev & 63] = 0;
    }
};
static DevCache g_dev_cache;

// ---- host <-> device staging for pageable caller memory (the reference's struct coef buffers are
// malloc-family memory): 8 MB pinned chunks, double buffered, the pageable side copied by the
// threads of copy_pool.h.
constexpr size_t kStageChunk = 8u << 20;
constexpr int kStageSlots = 4;
struct PinnedPool {
    std::mutex mu;
    std::vector<void *> free_list;
    void *get() {
        {
            std::lock_guard<std::mutex> l(mu);
            if (!free_list.empty()) {
                void *p = free_list.back();
                free_list.pop_back();
                return p;
            }
        }
        void *p = nullptr;
        if (cudaHostAlloc(&p, kStageChunk, cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            return nullptr;
        }
        return p;
    }
    void put(void *p) {
        std::lock_guard<std::mutex> l(mu);
        free_list.push_back(p);
    }
};
static PinnedPool g_pinned;

static void par_memcpy(void *dst, const void *src, size_t bytes) { CopyPool::instance().copy(dst, src, bytes); }

// Make a freshly allocated host buffer resident before it is needed: ask for huge pages where the
// kernel offers them on request, then first-touch every page with the copy threads.  compute()
// calls this for its result buffers while the device is still iterating.
extern "C" void j2p_host_prefault(void *p, size_t bytes) {
    if (!p || bytes == 0) return;
#ifdef MADV_HUGEPAGE
    const uintptr_t huge = (uintptr_t)2u << 20;
    const uintptr_t a = ((uintptr_t)p + huge - 1) & ~(huge - 1), e = ((uintptr_t)p + bytes) & ~(huge - 1);
    if (e > a) madvise((void *)a, (size_t)(e - a), MADV_HUGEPAGE);      // a hint; failure is harmless
#endif
    CopyPool::instance().touch(p, bytes);
}

struct j2p_session {
    int device = 0;
    cudaStream_t stream = nullptr;
    FrameDev F{};
    j2p_frame_desc desc{};
    TileMaps maps;                    // TMA descriptors of the plane buffers (tma_maps.h)
    float *slab = nullptr;            // x, xp, g, gp of every plane (see create_impl)
    size_t slab_bytes = 0;
    float *x[3] = {}, *xp[3] = {}, *g[3] = {}, *gp[3] = {}, *fdata0[3] = {};   // frame 0's planes
    int16_t *data[3] = {};
    unsigned nframes = 1;             // frames of a batch session (1: an ordinary session)
    size_t fdata_stride = 0;          // elements from one frame's fdata0 planes to the next frame's
    std::vector<float> tables;        // host copy of the tables, [frame][nc][3][64]: q, q*q, RN(1/(q*q))
    float *dev_tables = nullptr;      // batch sessions: the device copy the kernels read
    bool tables_stale = false;        // tables changed since the last device copy
    bool stale = false;               // batch sessions: planes uploaded since the last re-arm
    std::vector<char> uploaded;       // per plane = frame * nchannel + channel
    bool strip = false;       // row strip of a larger frame (multi-GPU tiling)
    bool ipc_exported = false; // peers hold cudaIpc mappings of this session's plane buffers: never recycle them
    float pending_factor = 0.f;
    float t = 1.f;            // FISTA momentum state (compute.c:426)
    unsigned next_iter = 0;
    unsigned long long launches = 0;
    int logging = 0;
    double log_host[8] = {};          // last device copy of logsums
    long long log_host_iter = -1;     // iteration log_host belongs to
    unsigned long long next_log_iter = 0;
    cudaEvent_t ev[kEventRing] = {};
    long long ev_iter[kEventRing];
    std::vector<std::pair<void *, size_t>> dev_blocks;   // everything this session took from the device cache
    void *stage[kStageSlots] = {};            // pinned staging ring (lazily taken from the process-wide pool)
    cudaEvent_t stage_ev[kStageSlots] = {};
    unsigned stage_next = 0;
    cudaEvent_t export_ev = nullptr;          // orders j2p_session_export on a caller stream with the session stream
    cudaEvent_t upload_ev = nullptr;          // orders j2p_session_upload_device after its producer stream
    unsigned long long uid = 0;               // unique over the process (a group's plan names its sessions by it)
    unsigned long long tables_gen = 0;        // bumped whenever a quantisation table is set
    struct GroupPlan *group = nullptr;        // the plan of the last group this session led (j2p_session_iterate_group)
    cudaEvent_t group_ev = nullptr;           // orders a group's launches with this session's stream
    // j2p_session_record_objective: the kernels of libj2pobjective.so and the device record (record.cuh)
    bool recording = false;
    bool rec_armed = false;                   // the record holds every iteration since the last arm
    double *rec_hist = nullptr;               // [desc.iterations][nframes][REC_FIELDS]
    double *rec_pp = nullptr;                 // projection partials [nframes][3][rec_pp_stride]
    unsigned rec_pp_stride = 0, rec_pp_count[3] = {};
};
static void free_group_plan(GroupPlan *g);

// x_k <-> x_{k-1} after an iteration (reference SWAP at compute.c:438); all planes together, which
// keeps pl[c].x == pl[0].x + c * plane_stride
static void swap_iterates(FrameDev &F) {
    for (int c = 0; c < F.nc; c++) {
        PlaneDev &P = F.pl[c];
        float *tp = P.x; P.x = P.xp; P.xp = tp;
    }
    F.buf_sel ^= 1;
}

template <typename T>
static cudaError_t dev_alloc(j2p_session *s, T **p, size_t bytes) {
    bytes = bytes ? (bytes + 255) & ~(size_t)255 : 256;
    size_t got = bytes;
    void *q = g_dev_cache.get(s->device, bytes, &got);
    if (!q) {
        got = bytes;
        cudaError_t e = cudaMalloc(&q, bytes);
        if (e == cudaErrorMemoryAllocation) {          // the cache may be sitting on the memory: release it, try once more
            cudaGetLastError();
            g_dev_cache.trim(s->device);
            e = cudaMalloc(&q, bytes);
        }
        if (e != cudaSuccess) return e;
    }
    s->dev_blocks.push_back({q, got});
    *p = reinterpret_cast<T *>(q);
    return cudaSuccess;
}

static std::once_flag g_cfg_once[64];
static cudaError_t g_cfg_err[64];
static int g_cfg_cc[64];
static int g_cfg_slots[64];

extern "C" const char *j2p_last_error(void) { return g_err; }

extern "C" const char *j2p_version(void) { return "jpeg2png_b200 0.1 (sm_90a)"; }

extern "C" int j2p_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

// per-thread device binding of the drop-in entry (-1 = process default: J2P_DEVICE, else 0)
static thread_local int g_thread_device = -1;

extern "C" int j2p_set_thread_device(int device) {
    if (device < 0) {
        g_thread_device = -1;
        return J2P_OK;
    }
    const int n = j2p_device_count();
    if (device >= n) return fail(J2P_ERR_ARG, "device %d out of range (%d visible)", device, n);
    g_thread_device = device;
    return J2P_OK;
}

extern "C" int j2p_thread_device(void) {
    if (g_thread_device >= 0) return g_thread_device;
    const char *env = getenv("J2P_DEVICE");
    return env && *env ? atoi(env) : 0;
}

extern "C" unsigned j2p_session_width(const j2p_session *s) { return s ? (unsigned)s->F.W : 0; }
extern "C" unsigned j2p_session_height(const j2p_session *s) { return s ? (unsigned)s->F.Hg : 0; }
extern "C" void *j2p_session_stream(j2p_session *s) { return s ? (void *)s->stream : nullptr; }
static float *plane_x(j2p_session *s, unsigned plane);
extern "C" void *j2p_session_plane_ptr(j2p_session *s, unsigned plane) {
    float *x = s ? plane_x(s, plane) : nullptr;
    if (s && !x) fail(J2P_ERR_ARG, "plane %u out of range (%zu planes)", plane, s->uploaded.size());
    return x;
}
extern "C" unsigned long long j2p_session_launches(const j2p_session *s) { return s ? s->launches : 0; }

extern "C" void j2p_session_destroy(j2p_session *s) {
    if (!s) return;
    cudaSetDevice(s->device);
    if (s->stream) cudaStreamSynchronize(s->stream);
    for (auto &blk : s->dev_blocks)                   // the stream is idle: nothing uses the blocks any more
        if (s->ipc_exported || !g_dev_cache.put(s->device, blk.first, blk.second)) cudaFree(blk.first);   // exported blocks go back to the driver, not to another session
    for (int i = 0; i < kEventRing; i++)
        if (s->ev[i]) cudaEventDestroy(s->ev[i]);
    for (int k = 0; k < kStageSlots; k++) {          // the stream is idle: no DMA touches the ring any more
        if (s->stage_ev[k]) cudaEventDestroy(s->stage_ev[k]);
        if (s->stage[k]) g_pinned.put(s->stage[k]);
    }
    if (s->export_ev) cudaEventDestroy(s->export_ev);
    if (s->upload_ev) cudaEventDestroy(s->upload_ev);
    if (s->group_ev) cudaEventDestroy(s->group_ev);
    free_group_plan(s->group);                       // the stream is idle: no group launch reads the plan any more
    if (s->stream) cudaStreamDestroy(s->stream);
    delete s;
}

// row0/rows select a horizontal strip of the frame (frame rows); rows == 0 means the whole frame.
static int create_impl(j2p_session *s, int device, const j2p_frame_desc *d, unsigned row0, unsigned rows, unsigned nframes) {
    const int ndev = j2p_device_count();
    if (ndev <= 0) return fail(J2P_ERR_NODEVICE, "no CUDA device available (the solver has no CPU fallback)");
    if (device < 0 || device >= ndev) return fail(J2P_ERR_ARG, "device %d out of range (0..%d)", device, ndev - 1);
    if (d->nchannel < 1 || d->nchannel > 3) return fail(J2P_ERR_ARG, "nchannel must be 1..3 (compute.c:118)");
    s->device = device;
    s->desc = *d;
    CK(cudaSetDevice(device));
    if (device >= 64) return fail(J2P_ERR_ARG, "device ordinal %d not supported", device);
    std::call_once(g_cfg_once[device], [&] {            // once per device and process: these queries are slow
        int major = 0, minor = 0;
        cudaError_t e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device);
        g_cfg_cc[device] = major * 10 + minor;
        g_cfg_err[device] = e != cudaSuccess ? e : (major * 10 + minor == 90 ? configure_kernels(&g_cfg_slots[device]) : cudaSuccess);
    });
    if (g_cfg_cc[device] != 90)          // sm_90a code loads on compute capability 9.0 only
        return fail(J2P_ERR_NODEVICE, "device %d is sm_%d; this library is built for sm_90a only", device, g_cfg_cc[device]);
    CK(g_cfg_err[device]);

    FrameDev &F = s->F;
    F.nc = (int)d->nchannel;
    unsigned W = 0, H = 0;
    for (unsigned c = 0; c < d->nchannel; c++) {                       // compute.c:410-416
        if (d->plane_w[c] == 0 || d->plane_h[c] == 0 || (d->plane_w[c] & 7) || (d->plane_h[c] & 7))
            return fail(J2P_ERR_ARG, "plane %u size %ux%u is not a positive multiple of 8", c, d->plane_w[c], d->plane_h[c]);
        if (d->w_samp[c] < 1 || d->h_samp[c] < 1) return fail(J2P_ERR_ARG, "plane %u has a zero sampling factor", c);
        if (d->plane_w[c] * d->w_samp[c] > W) W = d->plane_w[c] * d->w_samp[c];
        if (d->plane_h[c] * d->h_samp[c] > H) H = d->plane_h[c] * d->h_samp[c];
    }
    if ((unsigned long long)W * H > 0x7fffffffull) return fail(J2P_ERR_ARG, "frame %ux%u too large", W, H);
    F.W = (int)W;
    F.Hg = (int)H;
    if (rows == 0) {        // whole-frame session: the local buffer is the frame
        row0 = 0;
        rows = H;
    }
    if (row0 + rows > H) return fail(J2P_ERR_ARG, "strip rows %u..%u exceed the frame height %u", row0, row0 + rows, H);
    for (unsigned c = 0; c < d->nchannel; c++) {
        const unsigned mcu = 8 * d->h_samp[c];
        if (row0 % mcu || ((row0 + rows) % mcu && row0 + rows != H))
            return fail(J2P_ERR_ARG, "strip rows %u..%u are not aligned to the %u-row blocks of plane %u", row0, row0 + rows, mcu, c);
        if (d->plane_h[c] * d->h_samp[c] <= row0) return fail(J2P_ERR_ARG, "strip starts below the coefficient rows of plane %u", c);
    }
    // a strip carries two halo rows on every side that has a neighbour (the stencil reach, SURVEY.md §8a)
    const unsigned halo_top = row0 > 0 ? 2 : 0, halo_bot = row0 + rows < H ? 2 : 0;
    s->strip = !(row0 == 0 && rows == H);
    F.H = (int)(rows + halo_top + halo_bot);
    F.y0g = (int)row0 - (int)halo_top;
    F.t0 = (int)halo_top;
    F.t1 = (int)(halo_top + rows);
    const size_t n = (size_t)W * F.H;

    // scalars, evaluated on the host in the reference's own float expressions
    const float radius = sqrtf((float)H * (float)W) / 2;                // compute.c:425 (whole frame)
    F.step = radius / sqrtf((float)(1 + d->iterations));                // compute.c:443
    F.a1 = (float)(1. / (double)sqrtf((float)d->nchannel));             // compute.c:90
    const float tgv_alpha = d->weight / sqrtf((float)(4 / 2));          // compute.c:258
    F.a2 = (float)(((double)tgv_alpha * 1.) / (double)sqrtf((float)d->nchannel));   // compute.c:154
    F.use_tgv = d->weight != 0.f;                                       // compute.c:257
    F.one = 1.0f;

    CK(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
    for (int i = 0; i < kEventRing; i++) {
        CK(cudaEventCreateWithFlags(&s->ev[i], cudaEventDisableTiming));
        s->ev_iter[i] = -1;
    }
    // One slab holds x[0..nc), xp[0..nc), g[0..nc), gp[0..nc), every plane PS elements after the
    // previous one of its array (gp planes are smaller than PS; the rest of their slot is unused).
    // The gradient kernel addresses an array from one lane pointer plus c * PS (FrameDev::
    // plane_stride), and a strip session exports ONE cudaIpc handle.
    const size_t PS = (n + 63) & ~(size_t)63;                            // 256-byte aligned planes
    const size_t slab_elems = PS * 4 * d->nchannel;                      // one frame
    if (slab_elems > 0xffffffffull) return fail(J2P_ERR_ARG, "frame %ux%u too large for 32-bit element offsets", W, H);
    CK(dev_alloc(s, &s->slab, slab_elems * sizeof(float) * nframes));
    s->slab_bytes = slab_elems * sizeof(float) * nframes;
    F.slab = s->slab;
    F.plane_stride = (unsigned)PS;
    s->nframes = nframes;
    F.nframes = (int)nframes;
    F.frame_stride = slab_elems;
    // coefficients and the conventional decode: every plane of every frame in one block each, planes
    // 256-byte aligned
    size_t at_data[3], at_fd[3], data_elems = 0, fd_elems = 0;
    for (unsigned c = 0; c < d->nchannel; c++) {
        const unsigned cy0 = row0 / d->h_samp[c];
        unsigned cy1 = (row0 + rows + d->h_samp[c] - 1) / d->h_samp[c];
        if (cy1 > d->plane_h[c]) cy1 = d->plane_h[c];
        const size_t nc = (size_t)d->plane_w[c] * (cy1 - cy0);
        at_data[c] = data_elems;
        at_fd[c] = fd_elems;
        data_elems += (nc + 127) & ~(size_t)127;
        fd_elems += (nc + 63) & ~(size_t)63;
    }
    F.data_stride = data_elems;
    s->fdata_stride = fd_elems;
    int16_t *data_blk = nullptr;
    float *fd_blk = nullptr;
    CK(dev_alloc(s, &data_blk, data_elems * sizeof(int16_t) * nframes));
    CK(dev_alloc(s, &fd_blk, fd_elems * sizeof(float) * nframes));
    s->tables.assign((size_t)nframes * d->nchannel * 192, 0.f);
    s->uploaded.assign((size_t)nframes * d->nchannel, 0);
    F.tables = nullptr;
    F.host_tables = s->tables.data();
    if (nframes > 1) {
        CK(dev_alloc(s, &s->dev_tables, s->tables.size() * sizeof(float)));
        F.tables = s->dev_tables;
    }
    size_t at_x[3], at_xp[3], at_g[3], at_gp[3];
    for (unsigned c = 0; c < d->nchannel; c++) {
        at_x[c] = PS * (0 * d->nchannel + c);
        at_xp[c] = PS * (1 * d->nchannel + c);
        at_g[c] = PS * (2 * d->nchannel + c);
        at_gp[c] = PS * (3 * d->nchannel + c);
    }
    for (unsigned c = 0; c < d->nchannel; c++) {
        PlaneDev &P = F.pl[c];
        // coefficient rows this session holds: those whose footprint lies in the owned frame rows
        const unsigned cy0 = row0 / d->h_samp[c];
        unsigned cy1 = (row0 + rows + d->h_samp[c] - 1) / d->h_samp[c];
        if (cy1 > d->plane_h[c]) cy1 = d->plane_h[c];
        P.cw = (int)d->plane_w[c]; P.ch = (int)(cy1 - cy0);
        P.sw = (int)d->w_samp[c]; P.sh = (int)d->h_samp[c];
        P.resample = !(d->plane_w[c] == W && d->plane_h[c] == H);       // compute.c:338
        P.use_prob = d->pweight[c] != 0.f;                              // compute.c:244
        P.p_alpha = d->pweight[c] * 2 * 255 * sqrtf(2);                 // compute.c:245
        P.cnt = (float)(d->w_samp[c] * d->h_samp[c]);                   // compute.c:359
        s->x[c] = s->slab + at_x[c];
        s->xp[c] = s->slab + at_xp[c];
        s->g[c] = s->slab + at_g[c];
        s->gp[c] = s->slab + at_gp[c];
        s->fdata0[c] = fd_blk + at_fd[c];
        s->data[c] = data_blk + at_data[c];
        P.x = s->x[c]; P.xp = s->xp[c]; P.g = s->g[c]; P.gp = s->gp[c]; P.data = s->data[c];
    }
    // tensor maps for the TMA-fed projection: the two iterate buffers and the gradient of every plane
    // that has a tiled projection kernel; a driver without the entry point leaves the cp.async kernels
    bool maps_ok = nframes == 1;                                        // a batch always takes the cp.async kernels
    for (unsigned c = 0; c < d->nchannel && maps_ok; c++) {
        const bool p11 = d->w_samp[c] == 1 && d->h_samp[c] == 1, p22 = d->w_samp[c] == 2 && d->h_samp[c] == 2;
        if (!p11 && !p22) continue;
        const int box_rows = p11 ? 8 : 16;
        maps_ok = encode_plane_map(&s->maps.m[c][0], s->x[c], F.W, F.H, box_rows) == 0 &&
                  encode_plane_map(&s->maps.m[c][1], s->xp[c], F.W, F.H, box_rows) == 0 &&
                  encode_plane_map(&s->maps.m[c][2], s->g[c], F.W, F.H, box_rows) == 0;
        if (maps_ok && p11) maps_ok = encode_plane_map(&s->maps.m[c][3], s->gp[c], F.pl[c].cw, F.pl[c].ch, 8) == 0;
    }
    F.host_maps = maps_ok ? &s->maps : nullptr;
    F.buf_sel = 0;
    F.grad_ctas = grad_cta_count(F.W, F.t1 - F.t0);
    F.grad_slots = g_cfg_slots[device];
    CK(dev_alloc(s, &F.partials, sizeof(double) * 5 * (size_t)F.grad_ctas * nframes));
    CK(dev_alloc(s, &F.norms, sizeof(float) * 16 * nframes));     // per frame: [0..2] norms, [4..6] reciprocals, [8..10] strip sequence numbers
    CK(dev_alloc(s, &F.sums, sizeof(double) * 4 * nframes));
    CK(dev_alloc(s, &F.logsums, sizeof(double) * 8));
    CK(cudaMemsetAsync(F.logsums, 0, sizeof(double) * 8, s->stream));
    F.log_on = 0;
    F.log_slot = 0;
    CK(dev_alloc(s, &F.counter, sizeof(unsigned) * nframes));
    CK(cudaMemsetAsync(F.counter, 0, sizeof(unsigned) * nframes, s->stream));
    CK(cudaMemsetAsync(F.norms, 0, sizeof(float) * 16 * nframes, s->stream));
    return J2P_OK;
}

extern "C" int j2p_session_create(j2p_session **out, int device, const struct j2p_frame_desc *d) {
    return j2p_session_create_strip(out, device, d, 0, 0);
}

static int create_session(j2p_session **out, int device, const struct j2p_frame_desc *d, unsigned row0, unsigned rows,
                          unsigned nframes) {
    if (!out || !d) return fail(J2P_ERR_ARG, "null argument");
    *out = nullptr;
    j2p_session *s = new j2p_session();
    static std::atomic<unsigned long long> uid_seq{0};
    s->uid = ++uid_seq;
    const int rc = create_impl(s, device, d, row0, rows, nframes);
    if (rc != J2P_OK) {
        char keep[sizeof g_err];
        memcpy(keep, g_err, sizeof keep);
        j2p_session_destroy(s);
        cudaGetLastError();
        memcpy(g_err, keep, sizeof keep);
        return rc;
    }
    *out = s;
    return J2P_OK;
}

extern "C" int j2p_session_create_strip(j2p_session **out, int device, const struct j2p_frame_desc *d, unsigned row0,
                                        unsigned rows) {
    return create_session(out, device, d, row0, rows, 1);
}

extern "C" int j2p_session_create_batch(j2p_session **out, int device, const struct j2p_frame_desc *d, unsigned nframes) {
    if (out) *out = nullptr;
    if (nframes == 0) return fail(J2P_ERR_ARG, "a batch needs at least one frame");
    if (nframes > 65535) return fail(J2P_ERR_ARG, "a batch holds at most 65535 frames (%u requested)", nframes);
    return create_session(out, device, d, 0, 0, nframes);
}

extern "C" unsigned j2p_session_frames(const j2p_session *s) { return s ? s->nframes : 0; }

// strip entry points: refused on a batch of more than one frame
static int refuse_batch(const j2p_session *s, const char *what) {
    return fail(J2P_ERR_ARG, "%s is not available on a batch session (%u frames)", what, s->nframes);
}

static int reset_impl(j2p_session *s) {
    FrameDev &F = s->F;
    for (size_t k = 0; k < s->uploaded.size(); k++)
        if (!s->uploaded[k]) return fail(J2P_ERR_ARG, "plane %zu (frame %zu, channel %zu) has not been uploaded", k, k / F.nc, k % F.nc);
    F.buf_sel = 0;
    for (int c = 0; c < F.nc; c++) {
        PlaneDev &P = F.pl[c];
        P.x = s->x[c];
        P.xp = s->xp[c];
    }
    for (unsigned f = 0; f < s->nframes; f++) {
        const size_t fo = (size_t)f * F.frame_stride;
        for (int c = 0; c < F.nc; c++) {
            PlaneDev &P = F.pl[c];
            // owned rows only; a strip's halo rows are filled by the driver's first halo exchange
            const size_t off = (size_t)F.t0 * F.W;
            CK(launch_init_plane(s->fdata0[c] + f * s->fdata_stride, P.x + fo + off, P.xp + fo + off, F.W, F.t1 - F.t0, P.cw, P.ch, P.sw,
                                 P.sh, s->stream));
            s->launches++;
            // first step: cos == data*q exactly, so the DCT-distance gradient is exactly 0 (compute.c:283 vs :47)
            CK(cudaMemsetAsync(P.gp + fo, 0, (size_t)P.cw * P.ch * sizeof(float), s->stream));
        }
    }
    if (s->dev_tables && s->tables_stale) {     // pageable source: the copy has read it when the call returns
        CK(cudaMemcpyAsync(s->dev_tables, s->tables.data(), s->tables.size() * sizeof(float), cudaMemcpyHostToDevice, s->stream));
        s->tables_stale = false;
    }
    s->stale = false;
    s->t = 1.f;
    s->next_iter = 0;
    for (int i = 0; i < kEventRing; i++) s->ev_iter[i] = -1;            // events of an earlier solve say nothing about this one
    s->next_log_iter = 0;
    s->log_host_iter = -1;
    CK(cudaMemsetAsync(F.logsums, 0, sizeof(double) * 8, s->stream));    // iteration 0: DCT distance is exactly 0
    if (s->rec_hist) {
        CK(cudaMemsetAsync(s->rec_hist, 0, sizeof(double) * REC_FIELDS * s->desc.iterations * s->nframes, s->stream));
        s->rec_armed = s->recording;
    }
    return J2P_OK;
}

extern "C" int j2p_session_reset(j2p_session *s) {
    if (!s) return fail(J2P_ERR_ARG, "null session");
    CK(cudaSetDevice(s->device));
    return reset_impl(s);
}

// J2P_TRACE=1: where the host time of the transfers goes (stderr; measurement aid)
static bool trace_on() {
    static const bool on = [] { const char *e = getenv("J2P_TRACE"); return e && *e == '1'; }();
    return on;
}
static double now_ms() {
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
}
// ---- staging ring: four pinned 8 MB buffers per session, each with the event of the last DMA that
// used it.  A transfer of any size walks the ring; nothing drains between the arrays of an upload,
// so the host copy of one array overlaps the DMA of the previous one.
// reuse_idle (uploads): take a buffer whose last DMA has already completed before touching another
// one.  Pinning is the expensive part of a short solve — sixteen command-line threads pinning four
// 8 MB buffers each spent half of a batch inside cudaHostAlloc — and
// the three small uploads of a 1080p file never have two DMAs in flight.  Downloads keep the strict
// rotation: there a buffer is free only once the HOST has copied it out, which the events do not say.
static int stage_slot(j2p_session *s, int *slot_out, bool reuse_idle = false) {
    if (reuse_idle) {
        for (int i = 0; i < kStageSlots; i++) {
            const int k = (int)((s->stage_next + i) % kStageSlots);
            if (!s->stage[k]) continue;
            const cudaError_t q = cudaEventQuery(s->stage_ev[k]);
            if (q == cudaSuccess) {
                s->stage_next = (unsigned)k + 1;
                *slot_out = k;
                return J2P_OK;
            }
            if (q != cudaErrorNotReady) return fail(J2P_ERR_CUDA, "%s", cudaGetErrorString(q));
            cudaGetLastError();
        }
    }
    const int k = (int)(s->stage_next++ % kStageSlots);
    if (!s->stage[k]) {
        s->stage[k] = g_pinned.get();
        if (!s->stage[k]) return fail(J2P_ERR_CUDA, "pinned staging allocation failed");
        CK(cudaEventCreateWithFlags(&s->stage_ev[k], cudaEventDisableTiming));
    }
    CK(cudaEventSynchronize(s->stage_ev[k]));         // the buffer's previous DMA is done (no-op if never recorded)
    *slot_out = k;
    return J2P_OK;
}

// pageable host -> device on the session stream.  Returns when `src` has been read completely
// (the caller may free it); the DMA of the last chunks may still be in flight.
static int staged_h2d(j2p_session *s, void *dst, const void *src, size_t bytes) {
    const double t_begin = now_ms();
    double t_wait = 0., t_copy = 0.;
    for (size_t off = 0; off < bytes;) {
        const size_t n = bytes - off < kStageChunk ? bytes - off : kStageChunk;
        int k;
        const double t0 = now_ms();
        const int rc = stage_slot(s, &k, true);
        if (rc != J2P_OK) return rc;
        const double t1 = now_ms();
        par_memcpy(s->stage[k], (const char *)src + off, n);
        t_wait += t1 - t0;
        t_copy += now_ms() - t1;
        CK(cudaMemcpyAsync((char *)dst + off, s->stage[k], n, cudaMemcpyHostToDevice, s->stream));
        CK(cudaEventRecord(s->stage_ev[k], s->stream));
        off += n;
    }
    if (trace_on())
        fprintf(stderr, "j2p trace:   h2d %zu B: %.2f ms (waiting for a buffer %.2f, host copy %.2f)\n", bytes, now_ms() - t_begin, t_wait, t_copy);
    return J2P_OK;
}

// device -> pageable host; returns when `dst` is complete
static int staged_d2h(j2p_session *s, void *dst, const void *src, size_t bytes) {
    const size_t nchunks = (bytes + kStageChunk - 1) / kStageChunk;
    int slot[kStageSlots];
    // every buffer is free on the host side here (earlier downloads have copied theirs out): start the
    // rotation at a buffer that is already pinned instead of pinning the next one
    for (int i = 0; i < kStageSlots; i++)
        if (s->stage[i]) {
            s->stage_next = (unsigned)i;
            break;
        }
    // keep up to kStageSlots - 1 DMAs in flight ahead of the host copy
    size_t issued = 0;
    auto issue = [&]() -> int {
        const size_t off = issued * kStageChunk, n = bytes - off < kStageChunk ? bytes - off : kStageChunk;
        int k;
        const int rc = stage_slot(s, &k);
        if (rc != J2P_OK) return rc;
        CK(cudaMemcpyAsync(s->stage[k], (const char *)src + off, n, cudaMemcpyDeviceToHost, s->stream));
        CK(cudaEventRecord(s->stage_ev[k], s->stream));
        slot[issued % kStageSlots] = k;
        issued++;
        return J2P_OK;
    };
    for (size_t i = 0; i < nchunks; i++) {
        while (issued < nchunks && issued < i + (size_t)(kStageSlots - 1)) {
            const int rc = issue();
            if (rc != J2P_OK) return rc;
        }
        const int k = slot[i % kStageSlots];
        CK(cudaEventSynchronize(s->stage_ev[k]));
        const size_t off = i * kStageChunk, n = bytes - off < kStageChunk ? bytes - off : kStageChunk;
        par_memcpy((char *)dst + off, s->stage[k], n);
    }
    return J2P_OK;
}

// the quantisation tables of `plane` (q, qq, rqq), shared by both uploads
static int set_tables(j2p_session *s, unsigned plane, const uint16_t *quant, float **tab_out) {
    FrameDev &F = s->F;
    const unsigned f = plane / (unsigned)F.nc, c = plane % (unsigned)F.nc;
    float *tab = s->tables.data() + (size_t)plane * 192;                // q, qq, rqq of this frame and plane
    for (int j = 0; j < 64; j++)
        if (quant[j] == 0) return fail(J2P_ERR_ARG, "invalid quantization table (zero entry, jpeg.c:41-45)");
    for (int j = 0; j < 64; j++) {
        tab[j] = (float)quant[j];
        tab[64 + j] = tab[j] * tab[j];                                  // fp32 product (compute.c:49)
        tab[128 + j] = (float)(1.0 / (double)tab[64 + j]);              // RN(1/qq): fp64 quotient narrowed once is correctly rounded
        if (f == 0) {                                                   // what the single-frame kernels read
            F.q[c][j] = tab[j];
            F.qq[c][j] = tab[64 + j];
            F.rqq[c][j] = tab[128 + j];
        }
    }
    s->tables_stale = true;
    s->tables_gen++;
    *tab_out = tab;
    return J2P_OK;
}

// after a plane's upload: re-arm a single-frame session once all its planes are in
static int plane_uploaded(j2p_session *s, unsigned plane) {
    s->uploaded[plane] = 1;
    // A batch is re-armed once, by the first iterate (or reset) after its uploads: re-arming after
    // every plane would cost nframes * nchannel resets per solve.
    if (s->nframes > 1) {
        s->stale = true;
        return J2P_OK;
    }
    bool all = true;
    for (int k = 0; k < s->F.nc; k++) all = all && s->uploaded[k];
    if (all) return reset_impl(s);
    return J2P_OK;
}

// `plane` = frame * nchannel + channel (an ordinary session: the channel)
extern "C" int j2p_session_upload(j2p_session *s, unsigned plane, const int16_t *data, const uint16_t *quant,
                                  const float *fdata) {
    if (!s || !data || !quant) return fail(J2P_ERR_ARG, "null argument");
    if (plane >= s->uploaded.size()) return fail(J2P_ERR_ARG, "plane %u out of range (%zu planes)", plane, s->uploaded.size());
    CK(cudaSetDevice(s->device));
    FrameDev &F = s->F;
    const unsigned f = plane / (unsigned)F.nc, c = plane % (unsigned)F.nc;
    PlaneDev &P = F.pl[c];
    const size_t nc = (size_t)P.cw * P.ch;
    float *tab;
    int rcs = set_tables(s, plane, quant, &tab);
    if (rcs != J2P_OK) return rcs;
    int16_t *ddst = s->data[c] + (size_t)f * F.data_stride;
    float *fdst = s->fdata0[c] + (size_t)f * s->fdata_stride;
    rcs = staged_h2d(s, ddst, data, nc * sizeof(int16_t));
    if (rcs != J2P_OK) return rcs;
    if (fdata) {
        rcs = staged_h2d(s, fdst, fdata, nc * sizeof(float));
        if (rcs != J2P_OK) return rcs;
    } else {
        CK(launch_decode(ddst, tab, fdst, P.cw, P.ch, s->stream));
        s->launches++;
    }
    // The host arrays have been read completely (they sit in the pinned ring or on the device);
    // the stream is NOT drained here, so the next plane's host copy overlaps this plane's DMA.
    return plane_uploaded(s, plane);
}

// coefficients already in device memory: the session stream waits for `stream`, copies them device
// to device and runs the conventional decode, as j2p_session_upload(..., fdata = NULL) does
extern "C" int j2p_session_upload_device(j2p_session *s, unsigned plane, const int16_t *data_dev, const uint16_t *quant,
                                         void *stream) {
    if (!s || !data_dev || !quant) return fail(J2P_ERR_ARG, "null argument");
    if (plane >= s->uploaded.size()) return fail(J2P_ERR_ARG, "plane %u out of range (%zu planes)", plane, s->uploaded.size());
    for (int j = 0; j < 64; j++)
        if (quant[j] == 0) return fail(J2P_ERR_ARG, "invalid quantization table (zero entry, jpeg.c:41-45)");
    CK(cudaSetDevice(s->device));
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, data_dev) != cudaSuccess) {
        cudaGetLastError();
        return fail(J2P_ERR_ARG, "data_dev is not a CUDA pointer");
    }
    if (attr.type != cudaMemoryTypeDevice || attr.device != s->device)
        return fail(J2P_ERR_ARG, "data_dev is not device memory on device %d", s->device);
    FrameDev &F = s->F;
    const unsigned f = plane / (unsigned)F.nc, c = plane % (unsigned)F.nc;
    PlaneDev &P = F.pl[c];
    float *tab;
    const int rc = set_tables(s, plane, quant, &tab);
    if (rc != J2P_OK) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    if (st && st != s->stream) {
        if (!s->upload_ev) CK(cudaEventCreateWithFlags(&s->upload_ev, cudaEventDisableTiming));
        CK(cudaEventRecord(s->upload_ev, st));
        CK(cudaStreamWaitEvent(s->stream, s->upload_ev, 0));
    }
    int16_t *ddst = s->data[c] + (size_t)f * F.data_stride;
    float *fdst = s->fdata0[c] + (size_t)f * s->fdata_stride;
    CK(cudaMemcpyAsync(ddst, data_dev, (size_t)P.cw * P.ch * sizeof(int16_t), cudaMemcpyDeviceToDevice, s->stream));
    CK(launch_decode(ddst, tab, fdst, P.cw, P.ch, s->stream));
    s->launches++;
    return plane_uploaded(s, plane);
}

static int record_gradient(j2p_session *s, unsigned iter, float factor);
static int record_project(j2p_session *s, unsigned iter, float factor, int *nlaunch);

// one solver iteration (number `iter`) on the session stream; optional events around each kernel
static int one_iteration(j2p_session *s, unsigned iter, cudaEvent_t e0, cudaEvent_t e1, cudaEvent_t e2) {
    FrameDev &F = s->F;
    // FISTA momentum (compute.c:431-432, :440), host floats
    const float tnext = (1 + sqrtf(1 + 4 * (s->t * s->t))) / 2;
    const float factor = (s->t - 1) / tnext;
    s->t = tnext;
    if (e0) CK(cudaEventRecord(e0, s->stream));
    if (s->recording) {                                                  // the same iteration with the objective recorded
        int rc = record_gradient(s, iter, factor);
        if (rc != J2P_OK) return rc;
        if (e1) CK(cudaEventRecord(e1, s->stream));
        int nproj = 0;
        rc = record_project(s, iter, factor, &nproj);
        if (rc != J2P_OK) return rc;
        if (e2) CK(cudaEventRecord(e2, s->stream));
        s->launches += 1 + (unsigned)nproj;
        swap_iterates(F);                                                // compute.c:438
        return J2P_OK;
    }
    CK(launch_gradient(F, factor, s->stream));
    if (e1) CK(cudaEventRecord(e1, s->stream));
    if (F.log_on) {
        // k_project accumulates the DCT-distance objective of the NEXT iteration into the other slot
        F.log_slot = (int)((s->next_log_iter + 1) & 1);
        CK(cudaMemsetAsync(F.logsums + 2 + 3 * F.log_slot, 0, 3 * sizeof(double), s->stream));
    }
    int nproj = 0;
    CK(launch_project(F, factor, s->stream, &nproj));
    if (F.log_on) {
        CK(cudaMemcpyAsync(s->log_host, F.logsums, 8 * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
        s->log_host_iter = s->next_log_iter;
        s->next_log_iter++;
    }
    if (e2) CK(cudaEventRecord(e2, s->stream));
    s->launches += 1 + (unsigned)nproj;
    swap_iterates(F);                                                    // compute.c:438
    return J2P_OK;
}

static int check_ready(j2p_session *s, unsigned first) {
    for (size_t k = 0; k < s->uploaded.size(); k++)
        if (!s->uploaded[k]) return fail(J2P_ERR_ARG, "plane %zu has not been uploaded", k);
    if ((first == 0 && s->next_iter != 0) || s->stale) {
        const int rc = reset_impl(s);
        if (rc != J2P_OK) return rc;
    }
    if (first != s->next_iter) return fail(J2P_ERR_ARG, "iterations must be contiguous (expected %u, got %u)", s->next_iter, first);
    return J2P_OK;
}

// ---- strip sessions: one iteration in two halves, the driver combines sums and exchanges halos ----
extern "C" int j2p_session_gradient(j2p_session *s) {
    if (!s) return fail(J2P_ERR_ARG, "null session");
    if (s->nframes > 1) return refuse_batch(s, "j2p_session_gradient");
    CK(cudaSetDevice(s->device));
    for (int c = 0; c < s->F.nc; c++)
        if (!s->uploaded[c]) return fail(J2P_ERR_ARG, "plane %d has not been uploaded", c);
    // FISTA momentum (compute.c:431-432, :440), host floats
    const float tnext = (1 + sqrtf(1 + 4 * (s->t * s->t))) / 2;
    s->pending_factor = (s->t - 1) / tnext;
    s->t = tnext;
    CK(launch_gradient(s->F, s->pending_factor, s->stream));
    s->launches++;
    return J2P_OK;
}

extern "C" void *j2p_session_sums_ptr(j2p_session *s) {
    if (s && s->nframes > 1) {
        refuse_batch(s, "j2p_session_sums_ptr");
        return nullptr;
    }
    return s ? (void *)s->F.sums : nullptr;
}

extern "C" int j2p_session_project(j2p_session *s, const double *sums_by_rank, unsigned nranks) {
    if (!s || !sums_by_rank || nranks == 0) return fail(J2P_ERR_ARG, "bad argument");
    if (s->nframes > 1) return refuse_batch(s, "j2p_session_project");
    CK(cudaSetDevice(s->device));
    FrameDev &F = s->F;
    CK(launch_fold_sums(sums_by_rank, (int)nranks, F.nc, F.norms, s->stream));
    int nproj = 0;
    CK(launch_project(F, s->pending_factor, s->stream, &nproj));
    s->launches += 1 + (unsigned)nproj;                                 // the fold kernel + the projection launches
    swap_iterates(F);                                                    // compute.c:438
    s->next_iter++;
    return J2P_OK;
}

extern "C" int j2p_session_halo(j2p_session *s, unsigned c, int side, void **send, void **recv, size_t *count) {
    if (!s || !send || !recv || !count) return fail(J2P_ERR_ARG, "null argument");
    if (s->nframes > 1) return refuse_batch(s, "j2p_session_halo");
    if (c >= (unsigned)s->F.nc || (side != 0 && side != 1)) return fail(J2P_ERR_ARG, "bad channel or side");
    const FrameDev &F = s->F;
    float *x = F.pl[c].x;
    const size_t W = (size_t)F.W;
    const bool has = side == 0 ? F.t0 > 0 : F.t1 < F.H;
    *count = has ? 2 * W : 0;
    if (side == 0) {
        *send = x + (size_t)F.t0 * W;             // first two owned rows -> upper neighbour's bottom halo
        *recv = x;                                // rows above the strip  <- upper neighbour's last two rows
    } else {
        *send = x + (size_t)(F.t1 - 2) * W;       // last two owned rows  -> lower neighbour's top halo
        *recv = x + (size_t)F.t1 * W;
    }
    return J2P_OK;
}

extern "C" int j2p_session_copy_halo_to_prev(j2p_session *s) {
    if (!s) return fail(J2P_ERR_ARG, "null session");
    if (s->nframes > 1) return refuse_batch(s, "j2p_session_copy_halo_to_prev");
    CK(cudaSetDevice(s->device));
    const FrameDev &F = s->F;
    const size_t W = (size_t)F.W;
    for (int c = 0; c < F.nc; c++) {
        if (F.t0 > 0) CK(cudaMemcpyAsync(F.pl[c].xp, F.pl[c].x, (size_t)F.t0 * W * sizeof(float), cudaMemcpyDeviceToDevice, s->stream));
        if (F.t1 < F.H)
            CK(cudaMemcpyAsync(F.pl[c].xp + (size_t)F.t1 * W, F.pl[c].x + (size_t)F.t1 * W, (size_t)(F.H - F.t1) * W * sizeof(float),
                               cudaMemcpyDeviceToDevice, s->stream));
    }
    return J2P_OK;
}

extern "C" int j2p_session_strip_info(const j2p_session *s, unsigned *local_rows, unsigned *first_owned, unsigned *owned_rows) {
    if (!s) return fail(J2P_ERR_ARG, "null session");
    if (s->nframes > 1) return refuse_batch(s, "j2p_session_strip_info");
    if (local_rows) *local_rows = (unsigned)s->F.H;
    if (first_owned) *first_owned = (unsigned)s->F.t0;
    if (owned_rows) *owned_rows = (unsigned)(s->F.t1 - s->F.t0);
    return J2P_OK;
}

extern "C" int j2p_session_iterate(j2p_session *s, unsigned first, unsigned n) {
    if (!s) return fail(J2P_ERR_ARG, "null session");
    if (s->strip) return fail(J2P_ERR_ARG, "a strip session is driven with j2p_session_gradient / j2p_session_project");
    CK(cudaSetDevice(s->device));
    if (s->recording) {
        if ((unsigned long long)first + n > s->desc.iterations)
            return fail(J2P_ERR_ARG, "the objective record holds %u iterations; iterations %u..%llu asked for", s->desc.iterations, first,
                        (unsigned long long)first + n - 1);
        if (first != 0 && !s->rec_armed && !s->stale)
            return fail(J2P_ERR_ARG, "recording was switched on after iteration 0: iterate from first == 0 to re-arm the record");
    }
    int rc = check_ready(s, first);
    if (rc != J2P_OK) return rc;
    for (unsigned i = first; i < first + n; i++) {
        rc = one_iteration(s, i, nullptr, nullptr, nullptr);
        if (rc != J2P_OK) return rc;
        if (i % kEventStride == kEventStride - 1) {
            const int slot = (int)((i / kEventStride) % kEventRing);
            CK(cudaEventRecord(s->ev[slot], s->stream));
            s->ev_iter[slot] = (long long)i;
        }
    }
    s->next_iter = first + n;
    return J2P_OK;
}

extern "C" int j2p_session_profile(j2p_session *s, unsigned n, float *ms_gradient, float *ms_project) {
    if (!s || !ms_gradient || !ms_project || n == 0) return fail(J2P_ERR_ARG, "bad argument");
    CK(cudaSetDevice(s->device));
    if (s->recording && n > s->desc.iterations)
        return fail(J2P_ERR_ARG, "the objective record holds %u iterations; %u asked for", s->desc.iterations, n);
    int rc = check_ready(s, 0);
    if (rc != J2P_OK) return rc;
    cudaEvent_t e[3];
    for (int k = 0; k < 3; k++) CK(cudaEventCreate(&e[k]));
    double sg = 0., sp = 0.;
    for (unsigned i = 0; i < n; i++) {
        rc = one_iteration(s, i, e[0], e[1], e[2]);
        if (rc != J2P_OK) return rc;
        CK(cudaEventSynchronize(e[2]));
        float a = 0.f, b = 0.f;
        CK(cudaEventElapsedTime(&a, e[0], e[1]));
        CK(cudaEventElapsedTime(&b, e[1], e[2]));
        sg += a;
        sp += b;
    }
    for (int k = 0; k < 3; k++) cudaEventDestroy(e[k]);
    s->next_iter = n;
    *ms_gradient = (float)(sg / n);
    *ms_project = (float)(sp / n);
    return J2P_OK;
}

extern "C" int j2p_session_wait_iteration(j2p_session *s, unsigned iter) {
    if (!s) return fail(J2P_ERR_ARG, "null session");
    CK(cudaSetDevice(s->device));
    if (iter >= s->next_iter) return fail(J2P_ERR_ARG, "iteration %u has not been queued", iter);
    // the first iteration at or after `iter` that carries an event
    const unsigned marked = iter | (kEventStride - 1);
    const int slot = (int)((marked / kEventStride) % kEventRing);
    if (marked < s->next_iter && s->ev_iter[slot] >= (long long)marked) {
        // the slot holds `marked` itself, or (recycled after kEventRing * kEventStride more iterations) a later
        // iteration: events mark where an iteration was QUEUED, and stream order makes the older one complete
        // once the later one is
        CK(cudaEventSynchronize(s->ev[slot]));
    } else {
        CK(cudaStreamSynchronize(s->stream));     // nothing recorded at or after it yet: the tail of a solve
    }
    return J2P_OK;
}

// current iterate of `plane` = frame * nchannel + channel, or null when out of range
static float *plane_x(j2p_session *s, unsigned plane) {
    if (plane >= s->uploaded.size()) return nullptr;
    const unsigned f = plane / (unsigned)s->F.nc, c = plane % (unsigned)s->F.nc;
    return s->F.pl[c].x + (size_t)f * s->F.frame_stride;
}

extern "C" int j2p_session_download(j2p_session *s, unsigned plane, float *out) {
    if (!s || !out) return fail(J2P_ERR_ARG, "null argument");
    float *x = plane_x(s, plane);
    if (!x) return fail(J2P_ERR_ARG, "plane %u out of range (%zu planes)", plane, s->uploaded.size());
    CK(cudaSetDevice(s->device));
    // the rows this session owns (the whole frame, or the strip without its halo rows)
    const size_t n = (size_t)s->F.W * (size_t)(s->F.t1 - s->F.t0);
    return staged_d2h(s, out, x + (size_t)s->F.t0 * s->F.W, n * sizeof(float));
}

// The reference's post-processing of a joint result (jpeg2png.c:156-159 luma += 128; png.c:39-62
// YCbCr -> RGB, clamp, scale, truncate, 8 bit or 16 bit big-endian) on the device, delivered as PNG
// scanlines: h rows of 1 + w*3*bits/8 bytes, each starting with filter type 0.
extern "C" int j2p_session_download_scanlines(j2p_session *s, unsigned w, unsigned h, unsigned bits, unsigned char *out) {
    return j2p_session_download_frame_scanlines(s, 0, w, h, bits, out);
}

extern "C" int j2p_session_download_frame_scanlines(j2p_session *s, unsigned frame, unsigned w, unsigned h, unsigned bits,
                                                    unsigned char *out) {
    if (!s || !out) return fail(J2P_ERR_ARG, "null argument");
    if (frame >= s->nframes) return fail(J2P_ERR_ARG, "frame %u out of range (%u frames)", frame, s->nframes);
    if (s->F.nc != 3 || s->strip) return fail(J2P_ERR_ARG, "scanlines need a whole-frame session with three planes (joint mode)");
    if (bits != 8 && bits != 16) return fail(J2P_ERR_ARG, "bits must be 8 or 16");
    if (w == 0 || h == 0 || w > (unsigned)s->F.W || h > (unsigned)s->F.H) return fail(J2P_ERR_ARG, "image %ux%u does not fit the %dx%d frame", w, h, s->F.W, s->F.H);
    CK(cudaSetDevice(s->device));
    const size_t bytes = (size_t)h * ((size_t)w * 3 * (bits / 8) + 1);
    uint8_t *dev = nullptr;
    CK(dev_alloc(s, &dev, bytes));                   // returns to the device cache with the session
    EpilogueArgs a{};
    a.nc = 3;
    for (int c = 0; c < 3; c++) {
        a.plane[c] = plane_x(s, frame * 3 + (unsigned)c);
        a.frame_stride[c] = s->F.frame_stride;
        a.ld[c] = s->F.W;
    }
    a.w = (int)w;
    a.h = (int)h;
    a.mode = EP_SCANLINES;
    a.sample = (int)bits;
    a.frame_bytes = bytes;
    a.out = dev;
    int nep = 0;
    CK(launch_scanlines(a, 1, s->stream, &nep));
    s->launches += (unsigned)nep;
    return staged_d2h(s, out, dev, bytes);
}

// ---- export into caller device memory: the colour epilogue with a tensor layout, on the caller's
// stream, ordered after the solve that produced the planes and before anything later queued on a
// session stream can overwrite them.  `ss`: one joint session, or the Y, Cb, Cr separate sessions;
// nout: samples per pixel, 3 (RGB) or 1 (gray: plane 0 of the one session ss[0] alone).  oriented:
// the tiled mode of the epilogue, each frame flipped or rotated by orient[frame - frame0] (device
// memory; NULL = every frame 1).
// four (EpilogueFour): the four-plane mode, whose files have q[k] planes in session k (frame0 and
// nframes count files; j2p_session_export_four checked the q[k]).
static int export_impl(j2p_session *const *ss, int nsess, int nout, unsigned frame0, unsigned nframes, const struct j2p_image_out *o,
                       void *dst, void *stream, bool oriented = false, const unsigned char *orient = nullptr, int four = EP_FOUR_NONE,
                       const unsigned *q = nullptr) {
    if (!o || !dst) return fail(J2P_ERR_ARG, "null argument");
    j2p_session *s0 = ss[0];
    const unsigned nfiles = four ? s0->nframes * (unsigned)s0->F.nc / q[0] : s0->nframes;
    if (nframes == 0) return fail(J2P_ERR_ARG, "nframes must be at least 1");
    if (frame0 >= nfiles || nframes > nfiles - frame0)
        return fail(J2P_ERR_ARG, "frames %u..%u out of range (%u frames)", frame0, frame0 + nframes, nfiles);
    if (o->sample != 8 && o->sample != 16 && o->sample != 32) return fail(J2P_ERR_ARG, "sample must be 8, 16 or 32 (got %u)", o->sample);
    if (o->layout != J2P_LAYOUT_HWC && o->layout != J2P_LAYOUT_CHW) return fail(J2P_ERR_ARG, "unknown layout %u", o->layout);
    if (o->w == 0 || o->h == 0) return fail(J2P_ERR_ARG, "image %ux%u is empty", o->w, o->h);
    EpilogueArgs a{};
    a.nc = nout;
    a.four = four;
    for (int c = 0, k = 0, j = 0; c < (four ? 4 : nout); c++) {
        j2p_session *s = ss[four ? k : (nsess == 1 ? 0 : c)];
        const int W = s->F.W, H = s->F.Hg;
        if (o->w > (unsigned)W || o->h > (unsigned)H) return fail(J2P_ERR_ARG, "image %ux%u does not fit the %dx%d frame of plane %d", o->w, o->h, W, H, c);
        if (four) {         // file f's plane c is plane f * q[k] + j of session k
            a.plane[c] = plane_x(s, frame0 * q[k] + (unsigned)j);
            a.frame_stride[c] = (unsigned long long)(q[k] / (unsigned)s->F.nc) * s->F.frame_stride;
            if (++j == (int)q[k]) { k++; j = 0; }
        } else {
            a.plane[c] = plane_x(s, nsess == 1 ? frame0 * (unsigned)s->F.nc + (unsigned)c : frame0);
            a.frame_stride[c] = s->F.frame_stride;
        }
        a.ld[c] = W;
    }
    const size_t image_bytes = (size_t)o->w * o->h * (size_t)nout * (o->sample / 8);
    if (o->frame_bytes < image_bytes) return fail(J2P_ERR_ARG, "frame_bytes %zu is smaller than one image (%zu bytes)", o->frame_bytes, image_bytes);
    a.w = (int)o->w;
    a.h = (int)o->h;
    a.mode = o->layout == J2P_LAYOUT_HWC ? EP_HWC : EP_CHW;
    a.sample = (int)o->sample;
    a.frame_bytes = o->frame_bytes;
    a.out = (uint8_t *)dst;
    a.oriented = oriented;
    a.orient = orient;
    if (oriented && (o->h + 31) / 32 > (unsigned)kMaxGridRows)
        return fail(J2P_ERR_ARG, "an oriented export of %u rows has more than %d rows of 32-pixel tiles", o->h, kMaxGridRows);
    CK(cudaSetDevice(s0->device));
    if (orient) {
        cudaPointerAttributes attr;
        if (cudaPointerGetAttributes(&attr, orient) != cudaSuccess) {
            cudaGetLastError();
            return fail(J2P_ERR_ARG, "orientation is not a CUDA pointer");
        }
        if (attr.type != cudaMemoryTypeDevice || attr.device != s0->device)
            return fail(J2P_ERR_ARG, "orientation is not device memory on device %d", s0->device);
    }
    const cudaStream_t st = stream ? (cudaStream_t)stream : s0->stream;
    // every session stream other than the launch stream: the launch waits for its solve ...
    for (int k = 0; k < nsess; k++) {
        j2p_session *s = ss[k];
        if (s->stream == st) continue;
        if (!s->export_ev) CK(cudaEventCreateWithFlags(&s->export_ev, cudaEventDisableTiming));
        CK(cudaEventRecord(s->export_ev, s->stream));
        CK(cudaStreamWaitEvent(st, s->export_ev, 0));
    }
    int nep = 0;
    CK(launch_scanlines(a, (int)nframes, st, &nep));
    s0->launches += (unsigned)nep;
    // ... and the session stream waits for the export before a later upload / reset / iterate
    for (int k = 0; k < nsess; k++) {
        j2p_session *s = ss[k];
        if (s->stream == st) continue;
        CK(cudaEventRecord(s->export_ev, st));
        CK(cudaStreamWaitEvent(s->stream, s->export_ev, 0));
    }
    return J2P_OK;
}

extern "C" int j2p_session_export(j2p_session *s, unsigned frame0, unsigned nframes, const struct j2p_image_out *o, void *dst,
                                  void *stream) {
    if (!s) return fail(J2P_ERR_ARG, "null session");
    if (s->F.nc != 3 || s->strip) return fail(J2P_ERR_ARG, "j2p_session_export needs a whole-frame session with three planes (joint mode)");
    return export_impl(&s, 1, 3, frame0, nframes, o, dst, stream);
}

extern "C" int j2p_session_export_gray(j2p_session *s, unsigned frame0, unsigned nframes, const struct j2p_image_out *o, void *dst,
                                       void *stream) {
    if (!s) return fail(J2P_ERR_ARG, "null session");
    if ((s->F.nc != 1 && s->F.nc != 3) || s->strip)
        return fail(J2P_ERR_ARG, "j2p_session_export_gray needs a whole-frame session with one or three planes (has %d)", s->F.nc);
    return export_impl(&s, 1, 1, frame0, nframes, o, dst, stream);
}

extern "C" int j2p_session_export_separate(j2p_session *y, j2p_session *cb, j2p_session *cr, unsigned frame0, unsigned nframes,
                                           const struct j2p_image_out *o, void *dst, void *stream) {
    if (!y || !cb || !cr) return fail(J2P_ERR_ARG, "null session");
    j2p_session *ss[3] = {y, cb, cr};
    for (int c = 0; c < 3; c++) {
        if (ss[c]->F.nc != 1 || ss[c]->strip)
            return fail(J2P_ERR_ARG, "j2p_session_export_separate needs three whole-frame sessions with one plane each (plane %d has %d)", c, ss[c]->F.nc);
        if (ss[c]->nframes != y->nframes) return fail(J2P_ERR_ARG, "the separate sessions hold different frame counts (%u, %u)", y->nframes, ss[c]->nframes);
        if (ss[c]->device != y->device) return fail(J2P_ERR_ARG, "the separate sessions live on different devices (%d, %d)", y->device, ss[c]->device);
    }
    return export_impl(ss, 3, 3, frame0, nframes, o, dst, stream);
}

extern "C" int j2p_session_export_oriented(j2p_session *const *sessions, unsigned nsessions, unsigned channels, unsigned frame0,
                                           unsigned nframes, const unsigned char *orientation, const struct j2p_image_out *o,
                                           void *dst, void *stream) {
    if (!sessions) return fail(J2P_ERR_ARG, "null argument");
    if (!((nsessions == 1 && (channels == 1 || channels == 3)) || (nsessions == 3 && channels == 3)))
        return fail(J2P_ERR_ARG, "j2p_session_export_oriented takes one session with 1 or 3 channels or three sessions with 3 (got %u, %u)",
                    nsessions, channels);
    for (unsigned k = 0; k < nsessions; k++)
        if (!sessions[k]) return fail(J2P_ERR_ARG, "null session");
    j2p_session *s = sessions[0];
    if (nsessions == 3) {
        for (int c = 0; c < 3; c++) {
            if (sessions[c]->F.nc != 1 || sessions[c]->strip)
                return fail(J2P_ERR_ARG, "a separate oriented export needs three whole-frame sessions with one plane each (plane %d has %d)", c,
                            sessions[c]->F.nc);
            if (sessions[c]->nframes != s->nframes)
                return fail(J2P_ERR_ARG, "the separate sessions hold different frame counts (%u, %u)", s->nframes, sessions[c]->nframes);
            if (sessions[c]->device != s->device)
                return fail(J2P_ERR_ARG, "the separate sessions live on different devices (%d, %d)", s->device, sessions[c]->device);
        }
    } else if (channels == 3) {
        if (s->F.nc != 3 || s->strip) return fail(J2P_ERR_ARG, "a joint oriented export needs a whole-frame session with three planes");
    } else if ((s->F.nc != 1 && s->F.nc != 3) || s->strip) {
        return fail(J2P_ERR_ARG, "a gray oriented export needs a whole-frame session with one or three planes (has %d)", s->F.nc);
    }
    return export_impl(sessions, (int)nsessions, (int)channels, frame0, nframes, o, dst, stream, true, orientation);
}

extern "C" int j2p_session_export_four(j2p_session *const *sessions, unsigned nsessions, unsigned kind, unsigned channels,
                                       unsigned frame0, unsigned nframes, const unsigned char *orientation,
                                       const struct j2p_image_out *o, void *dst, void *stream) {
    if (!sessions || !o) return fail(J2P_ERR_ARG, "null argument");
    if (kind != J2P_FOUR_CMYK && kind != J2P_FOUR_YCCK) return fail(J2P_ERR_ARG, "unknown four-component kind %u", kind);
    if (channels != 4 && channels != 3) return fail(J2P_ERR_ARG, "a four-component export writes 4 or 3 channels (got %u)", channels);
    if (channels == 3 && o->sample != 8) return fail(J2P_ERR_ARG, "the CMYK -> RGB conversion is defined for 8-bit samples only (got %u)", o->sample);
    if (nsessions < 1 || nsessions > 4) return fail(J2P_ERR_ARG, "a four-component export takes 1 to 4 sessions (got %u)", nsessions);
    unsigned long long planes = 0;
    for (unsigned k = 0; k < nsessions; k++) {
        j2p_session *s = sessions[k];
        if (!s) return fail(J2P_ERR_ARG, "null session");
        if ((s->F.nc != 1 && s->F.nc != 3) || s->strip)
            return fail(J2P_ERR_ARG, "a four-component export needs whole-frame sessions with one or three planes (session %u has %d)", k, s->F.nc);
        if (s->device != sessions[0]->device)
            return fail(J2P_ERR_ARG, "the sessions live on different devices (%d, %d)", sessions[0]->device, s->device);
        planes += (unsigned long long)s->nframes * (unsigned)s->F.nc;
    }
    unsigned q[4] = {0, 0, 0, 0}, sum = 0;
    const unsigned long long nfiles = planes / 4;
    for (unsigned k = 0; k < nsessions; k++) {
        const unsigned long long p = (unsigned long long)sessions[k]->nframes * (unsigned)sessions[k]->F.nc;
        if (planes % 4 || p % nfiles || p / nfiles > 4 || (p / nfiles) % (unsigned)sessions[k]->F.nc)
            return fail(J2P_ERR_ARG, "the sessions do not hold whole planes of %llu files (session %u: %llu planes)", nfiles, k, p);
        q[k] = (unsigned)(p / nfiles);
        sum += q[k];
    }
    if (sum != 4) return fail(J2P_ERR_ARG, "the sessions hold %u planes per file, not 4", sum);
    if (sessions[0]->F.nc == 3 && kind != J2P_FOUR_YCCK)
        return fail(J2P_ERR_ARG, "a three-plane session holds the Y, Cb and Cr of a YCCK file");
    for (unsigned k = 1; k < nsessions; k++)
        if (sessions[k]->F.nc != 1) return fail(J2P_ERR_ARG, "only the first session may hold three planes");
    return export_impl(sessions, (int)nsessions, (int)channels, frame0, nframes, o, dst, stream, orientation != nullptr, orientation,
                       kind == J2P_FOUR_CMYK ? EP_FOUR_CMYK : EP_FOUR_YCCK, q);
}

extern "C" int j2p_session_sync(j2p_session *s) {
    if (!s) return fail(J2P_ERR_ARG, "null session");
    CK(cudaSetDevice(s->device));
    CK(cudaStreamSynchronize(s->stream));
    return J2P_OK;
}

extern "C" int j2p_session_set_logging(j2p_session *s, int enabled) {
    if (!s) return fail(J2P_ERR_ARG, "null session");
    if (enabled && s->strip) return fail(J2P_ERR_ARG, "objective logging is not available on strip sessions");
    if (enabled && s->nframes > 1) return refuse_batch(s, "objective logging");
    if (enabled && s->recording) return fail(J2P_ERR_ARG, "the session records the objective (j2p_session_record_objective); logging is the other way to get it");
    s->logging = enabled != 0;
    s->F.log_on = s->logging;
    return J2P_OK;
}

// Objective terms of the most recently queued iteration, as the reference's SIMD build logs them
// (compute.c:232-272, compute_simd_step.c:61): prob_dist = 0.5 * sum (residual/q)^2 over the
// planes with pweight != 0, tv / tv2 = fp64 sums of alpha*norm, objective = their sum over the
// float total_alpha.  Synchronises the session stream.
// The four logged numbers from the raw sums of one iteration: tv, tv2 and each plane's sum of
// (residual/q)^2.  Shared by j2p_session_objective and j2p_session_objective_history.
static void objective_terms(const j2p_session *s, double tv, double tv2_raw, const double *prob_raw, double out[4]) {
    const FrameDev &F = s->F;
    double prob = 0.;
    float total_alpha = 0.f;
    for (int c = 0; c < F.nc; c++) {
        if (F.pl[c].use_prob) {                                         // compute.c:244-247
            total_alpha += F.pl[c].p_alpha;
            prob += 0.5 * prob_raw[c];
        }
    }
    total_alpha += (float)F.nc;                                         // compute.c:252
    double tv2 = 0.;
    if (F.use_tgv) {                                                    // compute.c:257-260
        const float alpha = s->desc.weight / sqrtf((float)(4 / 2));
        total_alpha += alpha * (float)F.nc;
        tv2 = tv2_raw;
    }
    out[0] = (tv + tv2 + prob) / (double)total_alpha;                   // compute.c:271
    out[1] = prob;
    out[2] = tv;
    out[3] = tv2;
}

extern "C" int j2p_session_objective(j2p_session *s, double out[4]) {
    if (!s || !out) return fail(J2P_ERR_ARG, "null argument");
    if (!s->logging || s->log_host_iter < 0) return fail(J2P_ERR_ARG, "no logged iteration (call j2p_session_set_logging(s, 1) before iterating)");
    CK(cudaSetDevice(s->device));
    CK(cudaStreamSynchronize(s->stream));
    const int slot = (int)(s->log_host_iter & 1);
    objective_terms(s, s->log_host[0], s->log_host[1], s->log_host + 2 + 3 * slot, out);
    return J2P_OK;
}

// ---- the objective recorded on the device (libj2pobjective.so, objective/objective.cu) --------------
// Loaded on first use from next to this library, like libj2pmixed.so.
#include <dlfcn.h>
namespace {
struct ObjectiveApi {
    int (*configure)(void) = nullptr;
    int (*gradient)(const FrameDev *, float, int, int, int, int, const RecDev *, void *) = nullptr;
    int (*project)(const FrameDev *, int, int, float, const RecDev *, void *, int *) = nullptr;
    unsigned (*partials)(const FrameDev *, int) = nullptr;
    char err[400] = "";
};
const ObjectiveApi &objective_api() {
    static const ObjectiveApi api = [] {
        ObjectiveApi a;
        Dl_info info;
        if (!dladdr((void *)&j2p_session_objective, &info) || !info.dli_fname) {
            snprintf(a.err, sizeof a.err, "cannot locate libjpeg2png_b200.so to find libj2pobjective.so");
            return a;
        }
        std::string path(info.dli_fname);
        const size_t slash = path.rfind('/');
        path = (slash == std::string::npos ? std::string(".") : path.substr(0, slash)) + "/../objective/libj2pobjective.so";
        void *h = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
        if (!h) {
            snprintf(a.err, sizeof a.err, "libj2pobjective.so (the recording kernels) cannot be loaded: %s", dlerror());
            return a;
        }
        a.configure = (int (*)(void))dlsym(h, "j2p_objective_configure");
        a.gradient = (decltype(a.gradient))dlsym(h, "j2p_objective_gradient");
        a.project = (decltype(a.project))dlsym(h, "j2p_objective_project");
        a.partials = (decltype(a.partials))dlsym(h, "j2p_objective_partials");
        if (!a.configure || !a.gradient || !a.project || !a.partials) {
            snprintf(a.err, sizeof a.err, "%s does not export the j2p_objective_* entry points", path.c_str());
            a.configure = nullptr;
            a.gradient = nullptr;
        }
        return a;
    }();
    return api;
}
std::once_flag g_objective_once[64];
int g_objective_cfg[64];
}  // namespace

// what the recording kernels see: the session's descriptor with the device tables (a single frame runs
// with batch addressing too), and row `iter` of the record
static FrameDev record_view(const j2p_session *s) {
    FrameDev V = s->F;
    V.tables = s->dev_tables;
    return V;
}
static RecDev record_args(const j2p_session *s, unsigned iter) {
    RecDev R{};
    R.hist = s->rec_hist;
    R.pp = s->rec_pp;
    R.iter = iter;
    R.nframes = s->nframes;
    R.pp_stride = s->rec_pp_stride;
    for (int c = 0; c < 3; c++) R.pp_count[c] = s->rec_pp_count[c];
    return R;
}

static int record_gradient(j2p_session *s, unsigned iter, float factor) {
    const FrameDev V = record_view(s);
    const RecDev R = record_args(s, iter);
    int cx, bands, rows;
    packed_gradient_geometry(V, &cx, &bands, &rows);                    // the unrecorded launch's bands
    CK((cudaError_t)objective_api().gradient(&V, factor, cx, bands, rows, packed_gradient_gpm(V), &R, (void *)s->stream));
    return J2P_OK;
}

// launch_project's planes and launches, each projection kernel replaced by its recording variant
static int record_project(j2p_session *s, unsigned iter, float factor, int *nlaunch) {
    const FrameDev V = record_view(s);
    const RecDev R = record_args(s, iter);
    *nlaunch = 0;
    for (int c = 0; c < V.nc; c++) {
        const PlaneDev &P = V.pl[c];
        const bool p11 = P.sw == 1 && P.sh == 1, p22 = P.sw == 2 && P.sh == 2;
        int count = 1;      // following planes of identical geometry ride in the same launch
        while ((p11 || p22) && c + count < V.nc && V.pl[c + count].sw == P.sw && V.pl[c + count].sh == P.sh && V.pl[c + count].cw == P.cw &&
               V.pl[c + count].ch == P.ch)
            count++;
        int n = 0;
        CK((cudaError_t)objective_api().project(&V, c, count, factor, &R, (void *)s->stream, &n));
        *nlaunch += n;
        n = 0;
        if (p11) CK(launch_project_tile(s->F, c, count, factor, s->stream, &n, true));
        else if (p22) CK(launch_project_tile22(s->F, c, count, factor, s->stream, &n, true));
        *nlaunch += n;
        c += count - 1;
    }
    return J2P_OK;
}

extern "C" int j2p_session_record_objective(j2p_session *s, int enabled) {
    if (!s) return fail(J2P_ERR_ARG, "null session");
    if (!enabled) {
        s->recording = false;
        s->rec_armed = false;
        return J2P_OK;
    }
    if (s->strip) return fail(J2P_ERR_ARG, "the objective cannot be recorded on a strip session");
    if (s->logging) return fail(J2P_ERR_ARG, "the session logs the objective (j2p_session_set_logging); recording is the other way to get it");
    const ObjectiveApi &api = objective_api();
    if (!api.gradient) return fail(J2P_ERR_CUDA, "%s", api.err);
    CK(cudaSetDevice(s->device));
    std::call_once(g_objective_once[s->device & 63], [&] { g_objective_cfg[s->device & 63] = api.configure(); });
    CK((cudaError_t)g_objective_cfg[s->device & 63]);
    if (!s->rec_hist) {
        unsigned stride = 1;
        for (int c = 0; c < s->F.nc; c++) {
            s->rec_pp_count[c] = api.partials(&s->F, c);
            stride = std::max(stride, s->rec_pp_count[c]);
        }
        s->rec_pp_stride = stride;
        CK(dev_alloc(s, &s->rec_hist, sizeof(double) * REC_FIELDS * s->desc.iterations * s->nframes));
        CK(dev_alloc(s, &s->rec_pp, sizeof(double) * 3 * stride * s->nframes));
    }
    if (!s->dev_tables) {                // a single frame: its tables on the device as well (the kernels run with batch addressing)
        CK(dev_alloc(s, &s->dev_tables, s->tables.size() * sizeof(float)));
        s->tables_stale = true;
    }
    if (s->tables_stale) {               // pageable source: the copy has read it when the call returns
        CK(cudaMemcpyAsync(s->dev_tables, s->tables.data(), s->tables.size() * sizeof(float), cudaMemcpyHostToDevice, s->stream));
        s->tables_stale = false;
    }
    if (!s->recording) CK(cudaMemsetAsync(s->rec_hist, 0, sizeof(double) * REC_FIELDS * s->desc.iterations * s->nframes, s->stream));
    s->recording = true;
    s->rec_armed = s->next_iter == 0;
    return J2P_OK;
}

extern "C" int j2p_session_objective_history(j2p_session *s, unsigned first, unsigned count, double *out) {
    if (!s || (!out && count)) return fail(J2P_ERR_ARG, "null argument");
    if (!s->recording) return fail(J2P_ERR_ARG, "the session does not record the objective (call j2p_session_record_objective(s, 1) before iterating)");
    const unsigned done = s->rec_armed && !s->stale ? s->next_iter : 0;
    if ((unsigned long long)first + count > done)
        return fail(J2P_ERR_ARG, "iterations %u..%llu have not been recorded (%u recorded)", first, (unsigned long long)first + count - 1, done);
    if (count == 0) return J2P_OK;
    CK(cudaSetDevice(s->device));
    CK(cudaStreamSynchronize(s->stream));
    const size_t row = (size_t)s->nframes * REC_FIELDS;
    std::vector<double> raw(row * count);
    CK(cudaMemcpy(raw.data(), s->rec_hist + (size_t)first * row, raw.size() * sizeof(double), cudaMemcpyDeviceToHost));
    for (unsigned f = 0; f < s->nframes; f++)
        for (unsigned i = 0; i < count; i++) {
            const double *r = raw.data() + (size_t)i * row + (size_t)f * REC_FIELDS;
            objective_terms(s, r[0], r[1], r + 2, out + ((size_t)f * count + i) * 4);
        }
    return J2P_OK;
}

// ---- native strip loop: NCCL on the session stream --------------------------------------------
// The two exchanges of a strip iteration (all-gather of the three fp64 sums, neighbour exchange of
// the two border rows) are enqueued from here, on the session's own stream, between the kernels:
// no host round trip per iteration, the host only runs ahead of the device.  NCCL is resolved at
// run time (dlopen of libnccl.so.2 — inside a torch process that is the copy torch already loaded),
// so the library has no link-time dependency on it and single-GPU users never touch it.
#include <dlfcn.h>

namespace {
typedef struct ncclComm *nccl_comm_t;
struct nccl_uid { char internal[128]; };                                 // NCCL_UNIQUE_ID_BYTES
enum { kNcclFloat32 = 7, kNcclFloat64 = 8 };                             // ncclDataType_t values (nccl.h)
struct NcclApi {
    int (*GetUniqueId)(nccl_uid *);
    int (*CommInitRank)(nccl_comm_t *, int, nccl_uid, int);
    int (*CommDestroy)(nccl_comm_t);
    int (*Send)(const void *, size_t, int, int, nccl_comm_t, cudaStream_t);
    int (*Recv)(void *, size_t, int, int, nccl_comm_t, cudaStream_t);
    int (*AllGather)(const void *, void *, size_t, int, nccl_comm_t, cudaStream_t);
    int (*GroupStart)();
    int (*GroupEnd)();
    const char *(*GetErrorString)(int);
    bool ok = false;
};
NcclApi g_nccl;
std::once_flag g_nccl_once;

const NcclApi *nccl_api() {
    std::call_once(g_nccl_once, [] {
        void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return;
        NcclApi &a = g_nccl;
#define J2P_SYM(field, name) *(void **)(&a.field) = dlsym(h, name)
        J2P_SYM(GetUniqueId, "ncclGetUniqueId");
        J2P_SYM(CommInitRank, "ncclCommInitRank");
        J2P_SYM(CommDestroy, "ncclCommDestroy");
        J2P_SYM(Send, "ncclSend");
        J2P_SYM(Recv, "ncclRecv");
        J2P_SYM(AllGather, "ncclAllGather");
        J2P_SYM(GroupStart, "ncclGroupStart");
        J2P_SYM(GroupEnd, "ncclGroupEnd");
        J2P_SYM(GetErrorString, "ncclGetErrorString");
#undef J2P_SYM
        a.ok = a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.Send && a.Recv && a.AllGather && a.GroupStart && a.GroupEnd &&
               a.GetErrorString;
    });
    return g_nccl.ok ? &g_nccl : nullptr;
}
}  // namespace

// What a rank publishes so that the others can map its memory (cudaIpc, same node)
struct P2PInfo {
    cudaIpcMemHandle_t mail, flags, slab;
    unsigned long long x_off[3], xp_off[3];      // element offsets of the two iterate buffers of every plane inside the slab
    int t0, t1, H, W, nc, ok;
};

struct j2p_comm {
    nccl_comm_t comm = nullptr;
    int nranks = 0, rank = 0, device = 0;
    double *gathered = nullptr;                                          // [nranks][3] fp64, device
    // ---- peer-memory binding to one session (the default; J2P_STRIP_P2P=0 keeps NCCL in the loop) ----
    j2p_session *bound = nullptr;
    int p2p_state = 0;                                                   // 0 = not tried, 1 = bound, -1 = unavailable (NCCL path)
    double *mail = nullptr;                                              // [2][nranks][4] doubles, written by every rank
    // flag words of a rank: [0, 2*nranks) mailbox flags; then, at 2*nranks + k:
    //   0 "my upper neighbour has delivered its rows", 1 "my lower neighbour has delivered",
    //   2 ticket of the stand-alone halo kernel, 3 error word, 4/5 tickets of the border CTAs (top / bottom)
    unsigned *flags = nullptr;
    std::vector<void *> opened;                                          // cudaIpcOpenMemHandle results to close again
    double *peer_mail[8] = {};                                           // every rank's mailbox / flag block as mapped here (own: local)
    unsigned *peer_flags[8] = {};
    float *up_buf[3][2] = {}, *down_buf[3][2] = {};                      // the neighbours' two plane buffers, mapped here
    unsigned *up_flags = nullptr, *down_flags = nullptr;                 // the neighbours' flag blocks, mapped here
    int up_t1 = 0, down_t0 = 0;                                          // the neighbours' owned-row bounds (their local indices)
    unsigned seq_sums = 0, seq_halo = 0;                                 // sums exchanges / halo deliveries so far (same on every rank)
    int fused_halo = 0;                                                  // the projection kernels deliver the border rows themselves
    unsigned border_ctas[2] = {0, 0};
};

#define NK(call)                                                                                      \
    do {                                                                                              \
        int r_ = (call);                                                                              \
        if (r_ != 0) return fail(J2P_ERR_CUDA, "%s failed: %s (%s:%d)", #call, api->GetErrorString(r_), __FILE__, __LINE__); \
    } while (0)

extern "C" int j2p_comm_unique_id(void *out, size_t bytes) {
    const NcclApi *api = nccl_api();
    if (!api) return fail(J2P_ERR_NODEVICE, "libnccl.so.2 could not be loaded: %s", dlerror());
    if (!out || bytes < sizeof(nccl_uid)) return fail(J2P_ERR_ARG, "the id buffer must hold %zu bytes", sizeof(nccl_uid));
    NK(api->GetUniqueId((nccl_uid *)out));
    return J2P_OK;
}

extern "C" int j2p_comm_create(j2p_comm **out, int device, int nranks, int rank, const void *id, size_t bytes) {
    if (!out || !id || bytes < sizeof(nccl_uid) || nranks < 1 || rank < 0 || rank >= nranks) return fail(J2P_ERR_ARG, "bad argument");
    const NcclApi *api = nccl_api();
    if (!api) return fail(J2P_ERR_NODEVICE, "libnccl.so.2 could not be loaded: %s", dlerror());
    CK(cudaSetDevice(device));
    j2p_comm *c = new j2p_comm;
    c->nranks = nranks;
    c->rank = rank;
    c->device = device;
    nccl_uid uid;
    memcpy(&uid, id, sizeof uid);
    int r = api->CommInitRank(&c->comm, nranks, uid, rank);
    if (r != 0) {
        delete c;
        return fail(J2P_ERR_CUDA, "ncclCommInitRank failed: %s", api->GetErrorString(r));
    }
    if (cudaMalloc(&c->gathered, sizeof(double) * 3 * (size_t)nranks) != cudaSuccess) {
        api->CommDestroy(c->comm);
        delete c;
        return fail(J2P_ERR_CUDA, "cudaMalloc failed: %s", cudaGetErrorString(cudaGetLastError()));
    }
    *out = c;
    return J2P_OK;
}

extern "C" void j2p_comm_destroy(j2p_comm *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    for (void *p : c->opened) cudaIpcCloseMemHandle(p);
    cudaFree(c->mail);
    cudaFree(c->flags);
    const NcclApi *api = nccl_api();
    if (api && c->comm) api->CommDestroy(c->comm);
    cudaFree(c->gathered);
    delete c;
}

// 1 if the loop exchanges through peer memory, 0 if it calls NCCL (decided at the first iterate call)
extern "C" int j2p_comm_protocol(const j2p_comm *c) { return c && c->p2p_state == 1 ? 1 : 0; }

// 0 = fine; non-zero = a peer-memory wait timed out on the device (results are invalid)
extern "C" int j2p_comm_status(j2p_comm *c) {
    if (!c) return fail(J2P_ERR_ARG, "null communicator");
    if (c->p2p_state != 1) return J2P_OK;
    CK(cudaSetDevice(c->device));
    CK(cudaDeviceSynchronize());
    int err = 0;
    CK(cudaMemcpy(&err, c->flags + 2 * c->nranks + 3, sizeof err, cudaMemcpyDeviceToHost));
    if (err) return fail(J2P_ERR_CUDA, "a peer-memory exchange timed out (rank %d)", c->rank);
    return J2P_OK;
}

// ---- peer-memory binding ------------------------------------------------------------------------
// Collective.  Publishes this rank's mailbox, flags and plane buffers as cudaIpc handles (the plane
// buffers are plain cudaMalloc blocks from the device cache), gathers everybody's with NCCL, maps
// every rank's mailbox and the two neighbours' planes.  Every rank ends with the same verdict
// (a second gather), so the loop never mixes the NCCL and the peer-memory protocol.
static int p2p_bind(j2p_comm *c, j2p_session *s, const NcclApi *api) {
    c->bound = s;
    c->p2p_state = -1;
    if (c->nranks > 8) return J2P_OK;
    const int nr = c->nranks;
    const FrameDev &F = s->F;
    P2PInfo mine;
    memset(&mine, 0, sizeof mine);
    mine.t0 = F.t0; mine.t1 = F.t1; mine.H = F.H; mine.W = F.W; mine.nc = F.nc;
    bool ok = cudaMalloc(&c->mail, sizeof(double) * 2 * nr * 4) == cudaSuccess &&
              cudaMalloc(&c->flags, sizeof(unsigned) * (2 * nr + 8)) == cudaSuccess &&
              cudaMemset(c->mail, 0, sizeof(double) * 2 * nr * 4) == cudaSuccess &&
              cudaMemset(c->flags, 0, sizeof(unsigned) * (2 * nr + 8)) == cudaSuccess &&
              cudaIpcGetMemHandle(&mine.mail, c->mail) == cudaSuccess && cudaIpcGetMemHandle(&mine.flags, c->flags) == cudaSuccess;
    ok = ok && cudaIpcGetMemHandle(&mine.slab, s->slab) == cudaSuccess;
    for (int k = 0; k < F.nc; k++) {
        mine.x_off[k] = (unsigned long long)(s->x[k] - s->slab);
        mine.xp_off[k] = (unsigned long long)(s->xp[k] - s->slab);
    }
    mine.ok = ok ? 1 : 0;
    cudaGetLastError();

    // gather the descriptors (in place: my entry sits at its final position)
    std::vector<P2PInfo> all((size_t)nr);
    P2PInfo *d_all = nullptr;
    CK(cudaMalloc(&d_all, sizeof(P2PInfo) * (size_t)nr));
    CK(cudaMemcpy(d_all + c->rank, &mine, sizeof mine, cudaMemcpyHostToDevice));
    NK(api->AllGather(d_all + c->rank, d_all, sizeof(P2PInfo), /*ncclChar*/ 0, c->comm, s->stream));
    CK(cudaStreamSynchronize(s->stream));
    CK(cudaMemcpy(all.data(), d_all, sizeof(P2PInfo) * (size_t)nr, cudaMemcpyDeviceToHost));
    for (int p = 0; p < nr; p++) ok = ok && all[p].ok && all[p].W == F.W && all[p].nc == F.nc;

    auto open = [&](const cudaIpcMemHandle_t &h) -> void * {
        void *q = nullptr;
        if (cudaIpcOpenMemHandle(&q, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = false; return nullptr; }
        c->opened.push_back(q);
        return q;
    };
    if (ok) {
        for (int p = 0; p < nr && ok; p++) {
            if (p == c->rank) { c->peer_mail[p] = c->mail; c->peer_flags[p] = c->flags; continue; }
            c->peer_mail[p] = (double *)open(all[p].mail);
            c->peer_flags[p] = (unsigned *)open(all[p].flags);
            const bool up = p == c->rank - 1, down = p == c->rank + 1;
            if (!up && !down) continue;
            float *peer_slab = (float *)open(all[p].slab);
            for (int k = 0; k < F.nc && ok; k++) {
                float *b0 = peer_slab + all[p].x_off[k], *b1 = peer_slab + all[p].xp_off[k];
                if (up) { c->up_buf[k][0] = b0; c->up_buf[k][1] = b1; }
                else { c->down_buf[k][0] = b0; c->down_buf[k][1] = b1; }
            }
            if (up) { c->up_flags = c->peer_flags[p]; c->up_t1 = all[p].t1; }
            else { c->down_flags = c->peer_flags[p]; c->down_t0 = all[p].t0; }
        }
    }
    // common verdict
    int *d_ok = reinterpret_cast<int *>(d_all);
    const int mine_ok = ok ? 1 : 0;
    CK(cudaMemcpy(d_ok + c->rank, &mine_ok, sizeof(int), cudaMemcpyHostToDevice));
    NK(api->AllGather(d_ok + c->rank, d_ok, sizeof(int), /*ncclChar*/ 0, c->comm, s->stream));
    CK(cudaStreamSynchronize(s->stream));
    std::vector<int> oks((size_t)nr);
    CK(cudaMemcpy(oks.data(), d_ok, sizeof(int) * (size_t)nr, cudaMemcpyDeviceToHost));
    cudaFree(d_all);
    for (int p = 0; p < nr; p++) ok = ok && oks[p] == 1;
    c->p2p_state = ok ? 1 : -1;
    if (ok) {
        s->ipc_exported = true;
        // Can the projection kernels deliver the border rows themselves?  Needs every plane to span
        // the frame width (no stepped-only columns at the strip borders) and to go through one of
        // the two tiled projection kernels (1x1 or 2x2 sampling).  The same on every rank: it only
        // depends on the frame description.
        bool fused = true;
        unsigned ctas = 0;
        for (int k = 0; k < F.nc; k++) {
            const PlaneDev &P = F.pl[k];
            const bool tiled = (P.sw == 1 && P.sh == 1) || (P.sw == 2 && P.sh == 2);
            fused = fused && tiled && P.cw * P.sw == F.W;
            // units of work per block row that deliver border rows: warp tiles of the TMA kernel, CTA tiles of the cp.async kernels
            if (P.sw == 1 && F.host_maps && project_tma_enabled()) ctas += (unsigned)project_tma_border_units(P);
            else if (P.sw == 1) ctas += (unsigned)project_tile_border_units(P);
            else ctas += (unsigned)(((P.cw >> 3) + 15) / 16);                     // kernels_project_tile22.cu: 16 blocks per CTA tile
        }
        const char *e = getenv("J2P_STRIP_FUSED_HALO");
        if (e && *e == '0') fused = false;
        c->fused_halo = fused ? 1 : 0;
        c->border_ctas[0] = c->border_ctas[1] = ctas;
    }
    return J2P_OK;
}

// the two border rows of the current iterate to both neighbours, over peer memory
static int exchange_halos_p2p(j2p_session *s, j2p_comm *c, int wait_for_arrival) {
    const FrameDev &F = s->F;
    const size_t W = (size_t)F.W;
    const int nr = c->nranks;
    HaloPeers hp;
    memset(&hp, 0, sizeof hp);
    hp.has_up = F.t0 > 0 && c->rank > 0;
    hp.has_down = F.t1 < F.H && c->rank + 1 < nr;
    c->seq_halo++;                                                       // counted on every rank, also those without neighbours
    if (!hp.has_up && !hp.has_down) return J2P_OK;
    hp.nc = F.nc;
    hp.n4 = (unsigned)(2 * W / 4);
    for (int k = 0; k < F.nc; k++) {
        const int b = F.pl[k].x == s->x[k] ? 0 : 1;                       // which physical buffer holds the current iterate (same on every rank)
        hp.up_src[k] = F.pl[k].x + (size_t)F.t0 * W;
        hp.down_src[k] = F.pl[k].x + (size_t)(F.t1 - 2) * W;
        if (hp.has_up) hp.up_dst[k] = c->up_buf[k][b] + (size_t)c->up_t1 * W;              // the upper strip's rows below its last owned row
        if (hp.has_down) hp.down_dst[k] = c->down_buf[k][b] + (size_t)(c->down_t0 - 2) * W; // the lower strip's rows above its first owned row
    }
    // flag words of a rank: [2*nr + 0] "my upper neighbour has delivered", [2*nr + 1] "my lower neighbour has delivered"
    if (hp.has_up) hp.up_flag = c->up_flags + 2 * nr + 1;
    if (hp.has_down) hp.down_flag = c->down_flags + 2 * nr + 0;
    hp.from_up = c->flags + 2 * nr + 0;
    hp.from_down = c->flags + 2 * nr + 1;
    CK(launch_halo_exchange(hp, c->seq_halo, c->flags + 2 * nr + 2, reinterpret_cast<int *>(c->flags + 2 * nr + 3), wait_for_arrival, s->stream));
    s->launches++;
    return J2P_OK;
}

// the two border rows of the current iterate, all planes, both neighbours: one NCCL group
static int exchange_halos_nccl(j2p_session *s, j2p_comm *c, const NcclApi *api) {
    const FrameDev &F = s->F;
    const size_t W = (size_t)F.W;
    const bool up = F.t0 > 0 && c->rank > 0, down = F.t1 < F.H && c->rank + 1 < c->nranks;
    if (!up && !down) return J2P_OK;
    NK(api->GroupStart());
    for (int k = 0; k < F.nc; k++) {
        float *x = F.pl[k].x;
        if (up) {
            NK(api->Send(x + (size_t)F.t0 * W, 2 * W, kNcclFloat32, c->rank - 1, c->comm, s->stream));
            NK(api->Recv(x + (size_t)(F.t0 - 2) * W, 2 * W, kNcclFloat32, c->rank - 1, c->comm, s->stream));
        }
        if (down) {
            NK(api->Send(x + (size_t)(F.t1 - 2) * W, 2 * W, kNcclFloat32, c->rank + 1, c->comm, s->stream));
            NK(api->Recv(x + (size_t)F.t1 * W, 2 * W, kNcclFloat32, c->rank + 1, c->comm, s->stream));
        }
    }
    NK(api->GroupEnd());
    return J2P_OK;
}

// The in-kernel exchanges of one iteration (StripSync, kernels.cuh): sequence numbers and the
// destinations of this iteration's border rows.  x_{k+1} is written over xp, so the rows go into
// the neighbours' buffer with the same physical index (the x/xp roles alternate in lockstep on
// every rank).
static void fill_sync(j2p_session *s, j2p_comm *c) {
    FrameDev &F = s->F;
    StripSync &S = F.sync;
    const size_t W = (size_t)F.W;
    const int nr = c->nranks;
    S.nranks = nr;
    S.rank = c->rank;
    S.seq = c->seq_sums + 1;
    S.halo_seq = c->seq_halo;
    S.fused_halo = c->fused_halo;
    S.has_up = F.t0 > 0 && c->rank > 0;
    S.has_down = F.t1 < F.H && c->rank + 1 < nr;
    S.border_ctas[0] = c->border_ctas[0];
    S.border_ctas[1] = c->border_ctas[1];
    for (int p = 0; p < nr; p++) {
        S.mail[p] = c->peer_mail[p];
        S.mail_flag[p] = c->peer_flags[p];
    }
    S.my_mail = c->mail;
    S.my_flag = c->flags;
    for (int k = 0; k < F.nc; k++) {
        const int b = F.pl[k].xp == s->x[k] ? 0 : 1;                      // physical buffer that receives x_{k+1}
        S.up_dst[k] = S.has_up ? c->up_buf[k][b] + (size_t)c->up_t1 * W : nullptr;
        S.down_dst[k] = S.has_down ? c->down_buf[k][b] + (size_t)(c->down_t0 - 2) * W : nullptr;
    }
    S.up_flag = S.has_up ? c->up_flags + 2 * nr + 1 : nullptr;
    S.down_flag = S.has_down ? c->down_flags + 2 * nr + 0 : nullptr;
    S.from_up = c->flags + 2 * nr + 0;
    S.from_down = c->flags + 2 * nr + 1;
    S.border_ticket = c->flags + 2 * nr + 4;
    S.err = reinterpret_cast<int *>(c->flags + 2 * nr + 3);
}

// `n` iterations of this rank's strip; collective over the communicator (every rank calls it with
// the same n).  The first call after (re)arming the session also fills the halo rows of x_0 and
// x_{-1}.  Everything is queued on the session stream; use j2p_session_sync / download to wait.
//
// Peer-memory protocol (the default on one node; DESIGN.md §7): an iteration is exactly the two
// solver kernels, the exchanges happen inside them.  J2P_STRIP_P2P=0, or peers whose memory cannot
// be mapped, fall back to ncclAllGather + ncclSend/ncclRecv between the kernels.
extern "C" int j2p_session_iterate_strip(j2p_session *s, j2p_comm *c, unsigned n) {
    if (s && s->nframes > 1) return refuse_batch(s, "j2p_session_iterate_strip");
    if (!s || !c) return fail(J2P_ERR_ARG, "null argument");
    const NcclApi *api = nccl_api();
    if (!api) return fail(J2P_ERR_NODEVICE, "libnccl.so.2 could not be loaded");
    if (c->device != s->device) return fail(J2P_ERR_ARG, "communicator and session live on different devices");
    CK(cudaSetDevice(s->device));
    for (int k = 0; k < s->F.nc; k++)
        if (!s->uploaded[k]) return fail(J2P_ERR_ARG, "plane %d has not been uploaded", k);
    FrameDev &F = s->F;
    int rc;
    static const bool want_p2p = [] {
        const char *e = getenv("J2P_STRIP_P2P"), *g = getenv("J2P_GRAD_SCALAR");
        return !(e && *e == '0') && !(g && *g == '1');                   // the in-kernel exchanges live in the packed gradient kernel
    }();
    if (want_p2p && c->p2p_state == 0 && (rc = p2p_bind(c, s, api)) != J2P_OK) return rc;
    const bool p2p = want_p2p && c->p2p_state == 1 && c->bound == s;
    if (s->next_iter == 0) {
        if ((rc = p2p ? exchange_halos_p2p(s, c, 1) : exchange_halos_nccl(s, c, api)) != J2P_OK) return rc;
        if ((rc = j2p_session_copy_halo_to_prev(s)) != J2P_OK) return rc;
    }
    for (unsigned i = 0; i < n; i++) {
        const float tnext = (1 + sqrtf(1 + 4 * (s->t * s->t))) / 2;      // compute.c:431-432, :440
        const float factor = (s->t - 1) / tnext;
        s->t = tnext;
        int nproj = 0;
        if (p2p) {
            fill_sync(s, c);
            CK(launch_gradient(F, factor, s->stream));                   // waits for the halo rows, posts the sums
            CK(launch_project(F, factor, s->stream, &nproj));            // waits for the sums, delivers the border rows
            F.sync.nranks = 0;                                           // the session's other entry points see a plain strip
            c->seq_sums++;
            s->launches += 1 + (unsigned)nproj;
        } else {
            CK(launch_gradient(F, factor, s->stream));
            NK(api->AllGather(F.sums, c->gathered, 3, kNcclFloat64, c->comm, s->stream));
            CK(launch_fold_sums(c->gathered, c->nranks, F.nc, F.norms, s->stream));
            CK(launch_project(F, factor, s->stream, &nproj));
            s->launches += 2 + (unsigned)nproj;                          // gradient, fold, projection launches
        }
        swap_iterates(F);                                                // compute.c:438
        s->next_iter++;
        if (p2p) {
            if (c->fused_halo) c->seq_halo++;                            // delivered by the projection kernels
            else if ((rc = exchange_halos_p2p(s, c, 0)) != J2P_OK) return rc;   // stand-alone copy, no wait: the next gradient waits
        } else if ((rc = exchange_halos_nccl(s, c, api)) != J2P_OK) return rc;
    }
    return J2P_OK;
}

// ---- groups: sessions of different frame sizes iterated in one launch chain ----------------------
// The grouped kernels live in libj2pmixed.so (mixed/mixed.cu), next to this library in the package
// tree, loaded on first use.  A group's plan (geometry.cuh): one GroupFrame per session and parity,
// one GroupCta per CTA of every grouped kernel, and device tables for one-frame sessions (their kernels
// read the tables from the parameter block).  It is built once and kept in the first session until
// the group's sessions or their arming change.
namespace {
struct MixedApi {
    int (*configure)(void) = nullptr;
    int (*iterate)(const GroupFrame *, const GroupCta *, const GroupLaunch *, int, int, float, void *, int *) = nullptr;
    char err[400] = "";
};
const MixedApi &mixed_api() {
    static const MixedApi api = [] {
        MixedApi a;
        Dl_info info;
        if (!dladdr((void *)&j2p_session_iterate_group, &info) || !info.dli_fname) {
            snprintf(a.err, sizeof a.err, "cannot locate libjpeg2png_b200.so to find libj2pmixed.so");
            return a;
        }
        std::string path(info.dli_fname);
        const size_t slash = path.rfind('/');
        path = (slash == std::string::npos ? std::string(".") : path.substr(0, slash)) + "/../mixed/libj2pmixed.so";
        void *h = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
        if (!h) {
            snprintf(a.err, sizeof a.err, "libj2pmixed.so (the grouped kernels) cannot be loaded: %s", dlerror());
            return a;
        }
        a.configure = (int (*)(void))dlsym(h, "j2p_mixed_configure");
        a.iterate = (decltype(a.iterate))dlsym(h, "j2p_mixed_iterate");
        if (!a.configure || !a.iterate) {
            snprintf(a.err, sizeof a.err, "%s does not export j2p_mixed_configure / j2p_mixed_iterate", path.c_str());
            a.configure = nullptr;
            a.iterate = nullptr;
        }
        return a;
    }();
    return api;
}
std::once_flag g_mixed_once[64];
int g_mixed_cfg[64];
}  // namespace

struct GroupPlan {
    std::vector<unsigned long long> key;     // the sessions (uid): their geometry and buffers never change
    std::vector<unsigned long long> tables_gen;   // the one-frame sessions' tables the device copy holds
    GroupFrame *frames = nullptr;    // device [2][n]: parity 0, parity 1
    GroupCta *ctas = nullptr;        // device, every grouped kernel's slice (L)
    float *tables = nullptr;         // device tables of the one-frame sessions
    GroupLaunch L{};
    int gpm_nc = 0, tgv = 0;
    std::vector<unsigned> launches;  // per session: what one j2p_session_iterate iteration adds to its count
    std::vector<GroupFrame> h_frames;
    std::vector<GroupCta> h_ctas;
    std::vector<float> h_tables;
};

static void free_group_plan(GroupPlan *g) {
    if (!g) return;
    cudaFree(g->frames);
    cudaFree(g->ctas);
    cudaFree(g->tables);
    delete g;
}

// the launches one iteration of `s` makes on its own (one_iteration: the gradient, then launch_project
// for 1x1 / 2x2 planes, planes of one geometry sharing a launch, a launch per 65535 block rows, and one
// per plane with pixels no block covers)
static unsigned own_launches(const FrameDev &F) {
    unsigned n = 1;
    for (int c = 0; c < F.nc; c++) {
        const PlaneDev &P = F.pl[c];
        int count = 1;
        while (c + count < F.nc && F.pl[c + count].sw == P.sw && F.pl[c + count].sh == P.sh && F.pl[c + count].cw == P.cw &&
               F.pl[c + count].ch == P.ch)
            count++;
        n += (unsigned)(((P.ch >> 3) + kMaxGridRows - 1) / kMaxGridRows);
        for (int k = c; k < c + count; k++)
            n += F.pl[k].sw * F.pl[k].cw < F.W || F.pl[k].sh * F.pl[k].ch < F.H ? 1u : 0u;
        c += count - 1;
    }
    return n;
}

static int build_group_plan(j2p_session *const *ss, unsigned n, GroupPlan *g) {
    std::vector<GroupCta> slot[GK_COUNT];
    size_t ntab = 0;
    for (unsigned d = 0; d < n; d++)
        if (ss[d]->nframes == 1) ntab += ss[d]->tables.size();
    g->h_tables.reserve(ntab);
    g->h_frames.assign(2 * (size_t)n, GroupFrame{});
    g->launches.resize(n);
    if (ntab) CK(cudaMalloc(&g->tables, ntab * sizeof(float)));
    for (unsigned d = 0; d < n; d++) {
        const j2p_session *s = ss[d];
        FrameDev F = s->F;
        for (int c = 0; c < F.nc; c++) {                    // parity 0: x_k in the first iterate buffer
            F.pl[c].x = s->x[c];
            F.pl[c].xp = s->xp[c];
        }
        F.buf_sel = 0;
        if (s->nframes == 1) {
            F.tables = g->tables + g->h_tables.size();
            g->h_tables.insert(g->h_tables.end(), s->tables.begin(), s->tables.end());
        }
        int cx, bands, rows;
        packed_gradient_geometry(F, &cx, &bands, &rows);
        const int gpm = packed_gradient_gpm(F);
        g->launches[d] = own_launches(F);
        GroupFrame &G0 = g->h_frames[d], &G1 = g->h_frames[n + d];
        G0.F = F;
        G0.band_rows = rows;
        G1 = G0;
        for (int c = 0; c < F.nc; c++) std::swap(G1.F.pl[c].x, G1.F.pl[c].xp);
        G1.F.buf_sel = 1;
        for (unsigned f = 0; f < s->nframes; f++) {
            for (int by = 0; by < bands; by++)
                for (int bx = 0; bx < cx; bx++) slot[GK_GRAD + gpm].push_back({d, 0, (unsigned)bx, (unsigned)by, f, (unsigned)cx, (unsigned)bands, 0});
            for (int c = 0; c < F.nc; c++) {
                const PlaneDev &P = F.pl[c];
                const bool p11 = P.sw == 1;                 // the join rules leave 1x1 and 2x2 planes only
                const int bw = P.cw >> 3, bh = P.ch >> 3, gx = (bw + 15) / 16;   // PT_NB == P22_NB == 16 blocks per tile
                std::vector<GroupCta> &tiles = slot[p11 ? GK_TILE + (P.resample ? 1 : 0) : GK_TILE22];
                for (int by = 0; by < bh; by++)
                    for (int bx = 0; bx < gx; bx++) tiles.push_back({d, (unsigned)c, (unsigned)bx, (unsigned)by, f, (unsigned)gx, (unsigned)bh, 0});
                const size_t cwf = (size_t)P.sw * P.cw, chf = (size_t)P.sh * P.ch;
                if (cwf < (size_t)F.W || chf < (size_t)F.H) {
                    // any split of the region is the same per-pixel step; this is the batch path's
                    const size_t px = ((size_t)F.H - chf) * F.W + chf * (F.W - cwf);
                    const size_t cap = s->nframes > 1 ? (132 * 8 + s->nframes - 1) / s->nframes : 132 * 8;
                    const size_t blocks = std::min((px + 255) / 256, cap);
                    for (size_t b = 0; b < blocks; b++)
                        slot[p11 ? GK_UNCOVERED : GK_UNCOVERED22].push_back({d, (unsigned)c, (unsigned)b, 0, f, (unsigned)blocks, 1, 0});
                }
            }
        }
    }
    for (int k = 0; k < GK_COUNT; k++) {
        if (slot[k].size() > 0x7fffffffu) return fail(J2P_ERR_ARG, "the group needs more than 2^31 CTAs in one launch");
        g->L.first[k] = (unsigned)g->h_ctas.size();
        g->L.count[k] = (unsigned)slot[k].size();
        g->h_ctas.insert(g->h_ctas.end(), slot[k].begin(), slot[k].end());
    }
    j2p_session *s0 = ss[0];
    CK(cudaMalloc(&g->frames, g->h_frames.size() * sizeof(GroupFrame)));
    CK(cudaMalloc(&g->ctas, g->h_ctas.size() * sizeof(GroupCta)));
    // host vectors live as long as the plan: the copies may still be in flight when this returns
    CK(cudaMemcpyAsync(g->frames, g->h_frames.data(), g->h_frames.size() * sizeof(GroupFrame), cudaMemcpyHostToDevice, s0->stream));
    CK(cudaMemcpyAsync(g->ctas, g->h_ctas.data(), g->h_ctas.size() * sizeof(GroupCta), cudaMemcpyHostToDevice, s0->stream));
    if (ntab) CK(cudaMemcpyAsync(g->tables, g->h_tables.data(), ntab * sizeof(float), cudaMemcpyHostToDevice, s0->stream));
    g->gpm_nc = s0->F.nc;
    g->tgv = s0->F.use_tgv;
    for (unsigned d = 0; d < n; d++) {
        g->key.push_back(ss[d]->uid);
        g->tables_gen.push_back(ss[d]->tables_gen);
    }
    return J2P_OK;
}

// After uploads: the one-frame sessions' tables into the plan's device copy again (the CTA table and the
// descriptors depend on geometry and buffers only).  Ordered on the launch stream after earlier groups.
static int refresh_group_tables(j2p_session *const *ss, unsigned n, GroupPlan *g) {
    bool stale = false;
    for (unsigned d = 0; d < n; d++) stale = stale || (ss[d]->nframes == 1 && g->tables_gen[d] != ss[d]->tables_gen);
    if (!stale) return J2P_OK;
    size_t at = 0;
    for (unsigned d = 0; d < n; d++) {
        if (ss[d]->nframes != 1) continue;
        std::copy(ss[d]->tables.begin(), ss[d]->tables.end(), g->h_tables.begin() + at);
        at += ss[d]->tables.size();
        g->tables_gen[d] = ss[d]->tables_gen;
    }
    // pageable source: the copy has read h_tables when the call returns
    CK(cudaMemcpyAsync(g->tables, g->h_tables.data(), g->h_tables.size() * sizeof(float), cudaMemcpyHostToDevice, ss[0]->stream));
    return J2P_OK;
}

// the first reason `s` (index k) cannot join a group led by s0, or nullptr
static int refuse_join(const j2p_session *s0, const j2p_session *s, unsigned k) {
    const j2p_frame_desc &a = s0->desc, &b = s->desc;
    if (s->device != s0->device) return fail(J2P_ERR_ARG, "group session %u is on device %d, session 0 on %d", k, s->device, s0->device);
    if (s->strip) return fail(J2P_ERR_ARG, "group session %u is a strip session", k);
    if (s->logging) return fail(J2P_ERR_ARG, "group session %u logs the objective", k);
    if (s->recording) return fail(J2P_ERR_ARG, "group session %u records the objective", k);
    if (b.nchannel != a.nchannel) return fail(J2P_ERR_ARG, "group session %u has %u planes, session 0 %u", k, b.nchannel, a.nchannel);
    for (unsigned c = 0; c < b.nchannel; c++) {
        if (!((b.w_samp[c] == 1 && b.h_samp[c] == 1) || (b.w_samp[c] == 2 && b.h_samp[c] == 2)))
            return fail(J2P_ERR_ARG, "group session %u plane %u is sampled %ux%u; a group takes 1x1 and 2x2 planes only", k, c, b.w_samp[c], b.h_samp[c]);
        if (b.w_samp[c] != a.w_samp[c] || b.h_samp[c] != a.h_samp[c])
            return fail(J2P_ERR_ARG, "group session %u plane %u is sampled %ux%u, session 0 %ux%u", k, c, b.w_samp[c], b.h_samp[c], a.w_samp[c], a.h_samp[c]);
        if (memcmp(&b.pweight[c], &a.pweight[c], sizeof(float)))
            return fail(J2P_ERR_ARG, "group session %u plane %u has pweight %g, session 0 %g", k, c, b.pweight[c], a.pweight[c]);
    }
    if (memcmp(&b.weight, &a.weight, sizeof(float))) return fail(J2P_ERR_ARG, "group session %u has weight %g, session 0 %g", k, b.weight, a.weight);
    if (b.iterations != a.iterations) return fail(J2P_ERR_ARG, "group session %u has %u iterations, session 0 %u", k, b.iterations, a.iterations);
    return J2P_OK;
}

extern "C" int j2p_session_iterate_group(j2p_session *const *sessions, unsigned n, unsigned first, unsigned count) {
    if (!sessions || n == 0) return fail(J2P_ERR_ARG, "a group needs at least one session");
    for (unsigned k = 0; k < n; k++)
        if (!sessions[k]) return fail(J2P_ERR_ARG, "group session %u is null", k);
    j2p_session *s0 = sessions[0];
    unsigned long long frames = 0;
    for (unsigned k = 0; k < n; k++) {
        const int rc = refuse_join(s0, sessions[k], k);
        if (rc != J2P_OK) return rc;
        for (unsigned j = 0; j < k; j++)
            if (sessions[j] == sessions[k]) return fail(J2P_ERR_ARG, "group session %u is session %u again", k, j);
        frames += sessions[k]->nframes;
        if (frames > 65535) return fail(J2P_ERR_ARG, "group session %u takes the group past 65535 frames", k);
    }
    CK(cudaSetDevice(s0->device));
    // every session is checked before any is re-armed: a refused call changes nothing
    for (unsigned k = 0; k < n; k++) {
        const j2p_session *s = sessions[k];
        for (size_t p = 0; p < s->uploaded.size(); p++)
            if (!s->uploaded[p]) return fail(J2P_ERR_ARG, "group session %u: plane %zu has not been uploaded", k, p);
        const unsigned next = s->stale ? 0u : s->next_iter;      // a re-arm (check_ready) starts at 0
        if (first != 0 && first != next)
            return fail(J2P_ERR_ARG, "group session %u: iterations must be contiguous (expected %u, got %u)", k, next, first);
    }
    for (unsigned k = 0; k < n; k++) {
        const int rc = check_ready(sessions[k], first);
        if (rc != J2P_OK) {
            char why[sizeof g_err];
            memcpy(why, g_err, sizeof why);
            return fail(rc, "group session %u: %s", k, why);
        }
    }
    if (count == 0) return J2P_OK;
    const MixedApi &api = mixed_api();
    if (!api.iterate) return fail(J2P_ERR_CUDA, "%s", api.err);
    std::call_once(g_mixed_once[s0->device & 63], [&] { g_mixed_cfg[s0->device & 63] = api.configure(); });
    CK((cudaError_t)g_mixed_cfg[s0->device & 63]);

    GroupPlan *g = s0->group;
    bool same = g && g->key.size() == n;
    for (unsigned k = 0; same && k < n; k++) same = g->key[k] == sessions[k]->uid;
    if (!same) {
        if (g) {
            CK(cudaStreamSynchronize(s0->stream));      // the old plan may still be read by queued launches
            free_group_plan(g);
            s0->group = nullptr;
        }
        g = new GroupPlan();
        const int rc = build_group_plan(sessions, n, g);
        if (rc != J2P_OK) {
            cudaStreamSynchronize(s0->stream);
            free_group_plan(g);
            return rc;
        }
        s0->group = g;
    } else {
        const int rc = refresh_group_tables(sessions, n, g);
        if (rc != J2P_OK) return rc;
    }
    // the launch stream waits for what every other session's stream has queued (uploads, re-arm)
    for (unsigned k = 1; k < n; k++) {
        j2p_session *s = sessions[k];
        if (s->stream == s0->stream) continue;
        if (!s->group_ev) CK(cudaEventCreateWithFlags(&s->group_ev, cudaEventDisableTiming));
        CK(cudaEventRecord(s->group_ev, s->stream));
        CK(cudaStreamWaitEvent(s0->stream, s->group_ev, 0));
    }
    for (unsigned i = first; i < first + count; i++) {
        // FISTA momentum (compute.c:431-432, :440): every session is at iteration i, so at the same t
        const float tnext = (1 + sqrtf(1 + 4 * (s0->t * s0->t))) / 2;
        const float factor = (s0->t - 1) / tnext;
        int nl = 0;
        const cudaError_t e = (cudaError_t)api.iterate(g->frames + (size_t)s0->F.buf_sel * n, g->ctas, &g->L, g->gpm_nc, g->tgv, factor, s0->stream, &nl);
        CK(e);
        for (unsigned k = 0; k < n; k++) {
            j2p_session *s = sessions[k];
            s->t = tnext;
            s->launches += g->launches[k];
            swap_iterates(s->F);                                             // compute.c:438
        }
    }
    // ... and every other session's stream waits for the group's last launch
    for (unsigned k = 0; k < n; k++) {
        j2p_session *s = sessions[k];
        if (k > 0 && s->stream != s0->stream) {
            CK(cudaEventRecord(s->group_ev, s0->stream));
            CK(cudaStreamWaitEvent(s->stream, s->group_ev, 0));
        }
        // the iterations j2p_session_wait_iteration may ask for: marked where the whole group is complete
        for (unsigned i = first; i < first + count; i++)
            if (i % kEventStride == kEventStride - 1) {
                const int slot = (int)((i / kEventStride) % kEventRing);
                CK(cudaEventRecord(s->ev[slot], s->stream));
                s->ev_iter[slot] = (long long)i;
            }
        s->next_iter = first + count;
    }
    return J2P_OK;
}
