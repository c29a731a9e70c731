// kernels.cuh — device-side parameter blocks shared by the kernels and session.cu.
#pragma once
#include <stdint.h>

namespace j2p {

// One colour plane as the kernels see it.  For a strip session (multi-GPU row tiling) the
// frame-sized buffers hold the strip's rows plus the halo rows, the coefficient-sized ones only
// the strip's own coefficient rows.
struct PlaneDev {
    float *x;             // current iterate x_k, H x W raster              (reference aux.fdata)
    float *xp;            // previous iterate x_{k-1}; receives x_{k+1}     (reference aux.fista)
    float *g;             // objective sub-gradient, H x W raster           (reference aux.obj_gradient)
    float *gp;            // DCT-distance gradient for the NEXT step at coefficient resolution,
                          // ch x cw raster: p_alpha * idct((cos - data*q)/q^2)   (compute.c:38-70)
    const int16_t *data;  // quantised coefficients, [blocks][64] natural order
    int cw, ch;           // coefficient grid in samples (ch: rows held by this session)
    int sw, sh;           // upsampling factors
    int resample;         // !(cw == W && ch == H) for the WHOLE frame      (compute.c:338)
    int use_prob;         // pweight != 0                                   (compute.c:244)
    float p_alpha;        // pweight*2*255*sqrtf(2)                         (compute.c:245)
    float cnt;            // (float)(sw*sh), the divisor of the block mean     (compute.c:359)
};

// Strip sessions over peer memory (multi-GPU row tiling, DESIGN.md §7): the two exchanges of an
// iteration happen INSIDE the two kernels.  k_gradient's last CTA stores this rank's three sums of
// g^2 into every rank's mailbox (NVLink stores through cudaIpc mappings) and raises a flag there;
// every CTA of the projection waits for all flags of the iteration and folds the sums in rank
// order; the projection CTAs that produce the strip's first / last two rows also store them into
// the neighbours' halo rows, and the last of them raises the neighbours' halo flag, which the
// first / last row band of the neighbours' next k_gradient waits for.  nranks <= 1: no in-kernel
// exchange (whole-frame session, or a strip driven through NCCL / the host).
struct StripSync {
    int nranks, rank;
    unsigned seq;                   // 1-based index of this iteration's sums exchange (same on every rank)
    unsigned halo_seq;              // the halo flags must have reached this before k_gradient reads the halo rows
    int fused_halo;                 // the projection kernels deliver the border rows themselves
    int has_up, has_down;
    unsigned border_ctas[2];        // projection CTAs per iteration that hold the top / bottom border rows
    double *mail[8];                // rank p's mailbox as mapped here: [2 slots][nranks][4] doubles
    unsigned *mail_flag[8];         // rank p's mailbox flags: [2 slots][nranks]
    const double *my_mail;          // this rank's own mailbox / flags (local addresses)
    const unsigned *my_flag;
    float *up_dst[3], *down_dst[3]; // where rows [t0, t0+2) / [t1-2, t1) of x_{k+1} go in the neighbours, per plane
    unsigned *up_flag, *down_flag;  // the neighbours' words "my lower / upper neighbour has delivered"
    const unsigned *from_up, *from_down;   // this rank's own words
    unsigned *border_ticket;        // [2] local counters of finished border CTAs (top, bottom)
    int *err;                       // set when a wait timed out (results invalid; never hangs a box)
};

struct FrameDev {
    int W, H, nc;         // H: rows held locally (strip + halo rows); whole frame: H == Hg
    int Hg;               // height of the whole frame
    int y0g;              // frame row of local row 0
    int t0, t1;           // local rows [t0, t1) this session owns (targets); the rest is halo
    PlaneDev pl[3];
    float *slab;          // the allocation that holds x, xp, g, gp of every plane
    const void *host_maps;// host pointer to the session's TileMaps (tma_maps.h), or null: no TMA path for this session
    int buf_sel;          // 0: pl[c].x is the session's first iterate buffer, 1: the second (which tensor map is x_k)
    unsigned plane_stride;// elements between consecutive planes of one array: pl[c].x == pl[0].x + c * plane_stride, same for xp, g, gp
    float q[3][64];       // quantisation tables as float
    float qq[3][64];      // q*q (fp32 product, compute.c:49)
    float rqq[3][64];     // RN(1/(q*q)), the shared reciprocal of the residual division
    float a1;             // (float)(1./sqrtf(nc))                          (compute.c:90)
    float a2;             // (float)(alpha*1./sqrtf(nc)), alpha = weight/sqrtf(2)   (compute.c:154,258)
    int use_tgv;          // weight != 0                                    (compute.c:257)
    float step;           // radius / sqrtf(1 + iterations)                 (compute.c:425,443)
    float one;            // 1.0f, opaque to the compiler: addm2() in numerics.cuh
    double *partials;     // [5][grad_ctas] per-CTA sums of g^2 (and, when logging, of the TV / TGV norms)
    double *sums;         // [3] this session's sum of g^2 (strip mode: combined across ranks by the driver)
    float *norms;         // [0..2] sqrtf((float)sum g^2) (compute.c:200-206); [4..6] RN(1/norm)
    unsigned *counter;    // CTAs-done ticket for the last-CTA reduction
    int grad_ctas;
    int grad_slots;       // CTAs of k_gradient resident on this device at once (band geometry)
    StripSync sync;
    // objective logging (compute.c:271-272), only when the caller asked for a CSV log
    int log_on;
    int log_slot;         // which of the two prob_dist slots k_project accumulates into
    double *logsums;      // [0]=tv, [1]=tv2, [2+3*slot+c] = sum over plane c of (residual/q)^2
    // Batch sessions (nframes > 1, several frames of one geometry; session.cu): the pointers above
    // are frame 0's.  Frame f's x, xp, g, gp sit f * frame_stride elements after them, its
    // coefficients f * data_stride elements after pl[c].data, its tables (q, qq, rqq) at
    // tables[f][c][3][64] instead of q/qq/rqq, and its reduction state at partials + f * 5 * grad_ctas,
    // sums + 4 f, norms + 16 f, counter + f.  The batched kernels take the frame from blockIdx.z.
    int nframes;
    unsigned long long frame_stride, data_stride;
    const float *tables;  // device [nframes][nc][3][64]; null for single-frame sessions
    const float *host_tables;  // the host copy of it (per-frame launches of the generic projection)
};

// Frame f's view of a batch for a kernel that handles one frame (a per-frame launch).
inline FrameDev frame_view(const FrameDev &F, int f) {
    FrameDev V = F;
    V.nframes = 1;
    V.tables = nullptr;
    const unsigned long long fo = (unsigned long long)f * F.frame_stride;
    for (int c = 0; c < F.nc; c++) {
        V.pl[c].x += fo;
        V.pl[c].xp += fo;
        V.pl[c].g += fo;
        V.pl[c].gp += fo;
        V.pl[c].data += (unsigned long long)f * F.data_stride;
        for (int k = 0; k < 64; k++) {
            const float *t = F.host_tables + ((size_t)f * F.nc + c) * 192;
            V.q[c][k] = t[k];
            V.qq[c][k] = t[64 + k];
            V.rqq[c][k] = t[128 + k];
        }
    }
    V.partials += (size_t)f * 5 * F.grad_ctas;
    V.sums += 4 * (size_t)f;
    V.norms += 16 * (size_t)f;
    V.counter += f;
    return V;
}

// CUDA caps gridDim.y and gridDim.z at 65535.  The projection and epilogue grids have one CTA row
// per block row (or pixel row) of a plane, so a taller plane is covered by several launches of at
// most kMaxGridRows CTA rows each, every one on a view that starts further down the frame.
constexpr int kMaxGridRows = 65535;

// Planes [c0, c0 + count) seen from coefficient block row `brow` on; a block row spans `frame_rows`
// frame rows (8 * the vertical sampling factor).  Strip borders: only the view that holds a border
// row delivers it to the neighbour.  The kernels address every array relative to the plane
// pointers, so the offsets here are the only 64-bit products the split needs.
inline FrameDev rows_view(const FrameDev &F, int c0, int count, int brow, int frame_rows, bool last) {
    FrameDev V = F;
    const size_t px = (size_t)brow * frame_rows * (size_t)F.W;
    for (int c = c0; c < c0 + count; c++) {
        PlaneDev &P = V.pl[c];
        P.x += px;
        P.xp += px;
        P.g += px;
        P.gp += (size_t)brow * 8 * P.cw;
        P.data += (size_t)brow * (P.cw >> 3) * 64;
        P.ch = P.ch > 8 * brow ? P.ch - 8 * brow : 0;
    }
    V.H = F.H - brow * frame_rows;
    if (brow > 0) V.sync.has_up = 0;
    if (!last) V.sync.has_down = 0;
    return V;
}

// ---- the colour epilogue (kernels_epilogue.cu, k_scanlines): YCbCr planes of `nframes` frames ->
// RGB in one of three output forms.  Each plane has its own base, row stride and frame stride, so
// the three planes may come from one joint session or from three separate-mode sessions whose
// frames differ in size.  With nc == 1 only the luma plane is read and each pixel is one sample:
// the R (= G = B) sample of that luma with zero chroma.
// With `oriented` set (HWC / CHW only) a CTA covers a tile of the image instead of a row segment,
// and each frame is written flipped or rotated by its EXIF orientation (orient[frame], 1..8).
// With `four` set (HWC / CHW only) the frame has four planes (a four-component JPEG, DESIGN §7q):
// EP_FOUR_CMYK, each plane's gray sample inverted; EP_FOUR_YCCK, planes 0-2 as RGB and plane 3's gray
// sample inverted.  nc == 4 writes those samples, nc == 3 (8-bit only) Pillow's CMYK -> RGB of them.
enum EpilogueMode { EP_SCANLINES = 0, EP_HWC = 1, EP_CHW = 2 };
enum EpilogueFour { EP_FOUR_NONE = 0, EP_FOUR_CMYK = 1, EP_FOUR_YCCK = 2 };
struct EpilogueArgs {
    const float *plane[4];               // frame 0's Y, Cb, Cr (current iterates); Y alone when nc == 1; four planes with `four`
    int nc;                              // samples per pixel: 3 (RGB) or 1 (gray); 4 or 3 with `four`
    unsigned long long frame_stride[4];  // elements from one frame's plane to the next frame's
    int ld[4];                           // row stride of each plane, elements
    int four;                            // EpilogueFour
    int w, h;                            // visible image, at most every plane's frame
    int row0;                            // first image row of this launch (launch_scanlines)
    int mode;                            // EpilogueMode
    int sample;                          // bits per sample: 8 or 16 (scanlines), 8, 16 or 32 (HWC / CHW)
    unsigned long long frame_bytes;      // output bytes from one frame to the next
    uint8_t *out;
    int oriented;                        // tiled mapping with per-frame orientation (HWC / CHW)
    const uint8_t *orient;               // device, one value per launched frame; NULL: every frame 1
};

// ---- the stand-alone halo kernel (kernels_strip.cu); pointers into OTHER ranks' memory are cudaIpc
// mappings made by session.cu
struct HaloPeers {
    float *up_dst[3];         // where this strip's first two rows go: the upper neighbour's bottom halo rows, per plane
    float *down_dst[3];       // where the last two rows go: the lower neighbour's top halo rows
    const float *up_src[3];   // this strip's first two owned rows
    const float *down_src[3]; // this strip's last two owned rows
    unsigned *up_flag, *down_flag;         // the neighbours' words for "my lower / upper neighbour has delivered"
    const unsigned *from_up, *from_down;   // this rank's own words
    int has_up, has_down, nc;
    unsigned n4;              // float4s per plane and side: 2 rows * W / 4
};

}  // namespace j2p
