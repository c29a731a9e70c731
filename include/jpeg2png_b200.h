/* jpeg2png_b200.h — C ABI of the B200-native jpeg2png solver (libjpeg2png_b200.so).
 *
 * Plain C, plain pointers and sizes.  Two layers:
 *
 *   1. The DROP-IN layer: `compute()` with exactly the signature, ownership rules and side
 *      effects of the reference solver entry (reference compute.h:8, compute.c:407-465) and the
 *      data contract `struct coef` (reference jpeg2png.h:7-20).  A reference build links this
 *      library instead of its own compute.o/box.o/ooura/dct.o and nothing else changes
 *      (see INTEGRATION.md).
 *
 *   2. The SESSION layer (`j2p_*`): the same solver with the device residency made explicit,
 *      so that a caller (bench, batch driver, multi-GPU strip driver) can keep coefficient
 *      planes resident in HBM, time the iteration loop without the host<->device copies, and
 *      run several frames on several streams/devices.  `compute()` is implemented on top of it.
 *
 * There is NO CPU fallback anywhere behind this header: if no CUDA device is usable every entry
 * point fails (drop-in layer: die() -> exit(EXIT_FAILURE) like the reference, utils.c:20-28;
 * session layer: negative return code + j2p_last_error()).
 */
#ifndef JPEG2PNG_B200_H
#define JPEG2PNG_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------------
 * Data contract — layout-identical to the reference's `struct coef` (jpeg2png.h:7-20).
 *   h, w            plane size in samples (multiples of 8; jpeg.c:52-53)
 *   h_samp, w_samp  upsampling factors of this plane w.r.t. the frame (jpeg.c:57-58)
 *   data            quantised DCT coefficients, int16, [blocks][64] natural order, blocks in
 *                   raster order (jpeg.c:68-77); read-only for the solver, owned by the caller
 *   fdata           in : conventional decode, raster h x w, 0-centred (jpeg2png.c:127-139)
 *                   out: solver result, raster H x W of the working frame (compute.c:455-461)
 *   quant_table     natural order, all entries non-zero (jpeg.c:41-46)
 * ------------------------------------------------------------------------------------- */
struct coef {
        unsigned h;
        unsigned w;
        unsigned h_samp;
        unsigned w_samp;
        int16_t *data;
        float *fdata;
        uint16_t quant_table[64];
};

/* Reference logger.h:6-11 and progressbar.h:4-7: the solver writes log->iteration every
 * iteration (compute.c:428), calls logger_log once per iteration (compute.c:271-272) and
 * progressbar_inc once per iteration when pb != NULL (compute.c:449-452). */
struct logger;
struct progressbar;

/* ---------------------------------------------------------------------------------------
 * 1. Drop-in entry.  Replaces reference compute.c:407-465.
 *
 *   - consumes coefs[c].fdata (it must come from aligned_alloc/malloc, utils.h:89-106) and sets
 *     it to a 16-byte-aligned malloc-family buffer of H*W floats owned by the caller — the
 *     consumed buffer itself when the plane already has frame size, a new one (and the old one
 *     freed, compute.c:304-305, :458) otherwise;
 *   - overwrites coefs[c].w/h with the frame size W,H (compute.c:460-461);
 *   - re-entrant: may be called concurrently from several host threads (jpeg2png.c:147, :330);
 *     each call has its own CUDA stream and device buffers.  What the calls share is internally
 *     locked and holds no solver state: a cache of idle device blocks, pinned staging buffers and
 *     the host copy threads;
 *   - errors: message on stderr prefixed "jpeg2png: " and exit(EXIT_FAILURE) (utils.c:11-28).
 *
 * The callbacks are resolved at link time exactly like in the reference: the host program
 * provides logger_log() and progressbar_inc() (reference logger.c:20-27, progressbar.c:52-54).
 * When the library is loaded stand-alone (tests, bench) weak no-op defaults are used.
 * ------------------------------------------------------------------------------------- */
void compute(unsigned nchannel, struct coef *coefs, struct logger *log, struct progressbar *pb,
             float weight, float *pweight, unsigned iterations);

/* ---------------------------------------------------------------------------------------
 * 2. Session layer.
 * ------------------------------------------------------------------------------------- */
typedef struct j2p_session j2p_session;

enum {
        J2P_OK = 0,
        J2P_ERR_ARG = -1,      /* bad argument (sizes not multiples of 8, nchannel > 3, ...) */
        J2P_ERR_CUDA = -2,     /* a CUDA runtime call failed; see j2p_last_error()           */
        J2P_ERR_NODEVICE = -3  /* no usable sm_100 device                                    */
};

/* Thread-local text of the last failure on this host thread ("" if none). */
const char *j2p_last_error(void);

/* Number of CUDA devices visible to this process (0 if none / no driver). */
int j2p_device_count(void);

/* Which device the drop-in compute() uses when called from THIS host thread (the reference's
 * compute() has no device argument, compute.h:8).  -1 (the initial state of every thread) = the
 * process default: environment J2P_DEVICE, else device 0.  The reference calls compute() from
 * OpenMP threads for the three planes (jpeg2png.c:147-152) and for files (jpeg2png.c:330); a host
 * that binds each of those threads to its own device spreads them over the GPUs of the box. */
int j2p_set_thread_device(int device);
int j2p_thread_device(void);

/* Describes one frame to solve: the planes that are optimised TOGETHER (reference joint mode:
 * nchannel = 3, jpeg2png.c:144; separate mode: three sessions with nchannel = 1, :147-152).
 * A horizontal strip of the frame (multi-GPU spatial tiling) is selected at creation time with
 * j2p_session_create_strip(). */
struct j2p_frame_desc {
        unsigned nchannel;       /* 1..3 */
        unsigned plane_w[3];     /* coef->w  */
        unsigned plane_h[3];     /* coef->h  */
        unsigned w_samp[3];      /* coef->w_samp */
        unsigned h_samp[3];      /* coef->h_samp */
        float weight;            /* TGV weight (-w), compute.c:257-260 */
        float pweight[3];        /* DCT-distance weights (-p), compute.c:244-245 */
        unsigned iterations;     /* total iteration count (fixes the step size, compute.c:443) */
};

/* Create a session on `device` (cudaSetDevice ordinal).  Allocates all HBM working buffers. */
int j2p_session_create(j2p_session **out, int device, const struct j2p_frame_desc *desc);
void j2p_session_destroy(j2p_session *s);

/* ---- batch sessions: many frames of one geometry, one launch chain per iteration ----------------
 * `nframes` frames that all have the geometry and solver parameters of `desc` (plane sizes,
 * sampling factors, weight, pweight, iterations); quantisation tables and coefficients are per
 * frame.  Every iteration solves all frames with the launches one frame would take (4:4:4 and
 * 4:2:0; other sampling factors launch the projection of those planes once per frame), and every
 * frame's result is bit-identical to solving it alone in j2p_session_create's session on the same
 * device.  A batch of one behaves exactly like j2p_session_create.
 *
 * The per-plane calls (j2p_session_upload, j2p_session_download, j2p_session_plane_ptr) address
 * plane = frame * nchannel + channel; the whole-session calls (reset, iterate, profile,
 * wait_iteration, sync, stream, launches) act on the whole batch.  A batch is re-armed once, by the
 * first j2p_session_iterate(s, 0, n) or j2p_session_reset after its planes were uploaded, so new
 * frames can be uploaded into a batch and solved again.  Objective logging and the strip calls are
 * refused on a batch of more than one frame (J2P_ERR_ARG); so are nframes == 0 and out-of-range
 * planes or frames.  j2p_session_record_objective records the objective of every frame of a batch. */
int j2p_session_create_batch(j2p_session **out, int device, const struct j2p_frame_desc *desc,
                             unsigned nframes);
/* Frames of the session (1 for every session not made by j2p_session_create_batch). */
unsigned j2p_session_frames(const j2p_session *s);

/* ---- row strips of one frame across several GPUs (SURVEY.md §8e, BASELINE config 4) ------------
 * A strip session holds frame rows [row0, row0+rows) of the frame described by `desc` (which
 * always describes the WHOLE frame) plus two halo rows on every side that has a neighbour.
 * row0 and row0+rows must be multiples of 8*h_samp of every plane (row0+rows may also be the
 * frame height).  Uploads then carry only the coefficient rows of the strip.  One iteration is
 *     j2p_session_gradient(s);                       k_gradient on the owned rows
 *     <all-gather the 3 doubles at j2p_session_sums_ptr(s) over the ranks>
 *     j2p_session_project(s, gathered, nranks);      fold in rank order -> norms, step + projection
 *     <exchange halos: j2p_session_halo(s, c, side, &send, &recv, &count)>
 * The driver (jpeg2png_b200/strips.py) does the two communication steps with torch.distributed
 * (NCCL over NVLink on GPUs).  After (re)arming a strip session the driver exchanges the halos of
 * the initial iterate once and calls j2p_session_copy_halo_to_prev(). */
int j2p_session_create_strip(j2p_session **out, int device, const struct j2p_frame_desc *desc,
                             unsigned row0, unsigned rows);
int j2p_session_strip_info(const j2p_session *s, unsigned *local_rows, unsigned *first_owned,
                           unsigned *owned_rows);
int j2p_session_gradient(j2p_session *s);
void *j2p_session_sums_ptr(j2p_session *s);
int j2p_session_project(j2p_session *s, const double *sums_by_rank, unsigned nranks);
/* side 0 = top, 1 = bottom.  send: first/last two owned rows of the current iterate; recv: the
 * halo rows beyond them; count: floats to move (0 if there is no neighbour on that side). */
int j2p_session_halo(j2p_session *s, unsigned channel, int side, void **send, void **recv,
                     size_t *count);
int j2p_session_copy_halo_to_prev(j2p_session *s);

/* Native strip loop.  One process per GPU: rank 0 obtains an id with j2p_comm_unique_id(), hands
 * its 128 bytes to the other ranks by any means (the Python driver broadcasts it with
 * torch.distributed), every rank calls j2p_comm_create().  Ranks are the strips in top-to-bottom
 * order.  j2p_session_iterate_strip() is collective; its first call after (re)arming a session also
 * exchanges the halos of the initial iterate; the host never waits inside the loop.
 *
 * On one node (up to 8 ranks) the first call maps the peers' memory (cudaIpc over NVLink) and from
 * then on an iteration is exactly the two solver kernels: the gradient kernel's last CTA stores
 * this rank's sums of g^2 into every rank's mailbox, the projection kernels wait for all of them,
 * fold them in rank order and store the strip's border rows straight into the neighbours' halo
 * rows, the next gradient kernel's border bands wait for those (sequence-numbered flags,
 * st.release.sys / ld.acquire.sys).  When peer memory cannot be mapped, or with J2P_STRIP_P2P=0, the
 * exchanges are ncclAllGather + ncclSend/ncclRecv queued between the kernels.  NCCL is resolved at
 * run time with dlopen("libnccl.so.2"): no link-time dependency.  Same results either way.
 * Destroy the communicator before the session it was used with. */
typedef struct j2p_comm j2p_comm;
#define J2P_COMM_ID_BYTES 128
int j2p_comm_unique_id(void *out, size_t bytes);
int j2p_comm_create(j2p_comm **out, int device, int nranks, int rank, const void *id, size_t bytes);
void j2p_comm_destroy(j2p_comm *c);
int j2p_session_iterate_strip(j2p_session *s, j2p_comm *c, unsigned n);
/* 0, or an error if an in-kernel wait of the peer-memory protocol timed out on the device (a peer
 * died; results are invalid; every wait gives up after about two seconds of GPU clock instead of
 * hanging the device).  Synchronises the device. */
int j2p_comm_status(j2p_comm *c);
/* 1 if j2p_session_iterate_strip exchanges through peer memory, 0 if through NCCL. */
int j2p_comm_protocol(const j2p_comm *c);

/* Working-frame size W x H = max over planes of (plane_w*w_samp, plane_h*h_samp) (compute.c:410-416). */
unsigned j2p_session_width(const j2p_session *s);
unsigned j2p_session_height(const j2p_session *s);

/* Host -> HBM.  `data`: int16 [blocks][64]; `quant`: uint16[64]; `fdata`: raster plane_h x plane_w
 * conventional decode.  Performs the reference aux_init (compute.c:278-310) on the device:
 * cos = data*quant, nearest-neighbour upsample with edge clamp, fista = fdata.  Returns as soon
 * as the host arrays have been read (into the session's pinned staging ring): the caller may free
 * them; the DMA of the last chunks and the set-up kernels are still queued on the session stream. */
int j2p_session_upload(j2p_session *s, unsigned channel, const int16_t *data,
                       const uint16_t *quant, const float *fdata);

/* j2p_session_upload(s, plane, ..., fdata = NULL) for coefficients that are already in device memory
 * (for instance decoded there by libj2pentropy.so).  `data_dev`: int16 [blocks][64] on the session's
 * device; `quant`: host uint16[64].  The session stream waits for the work queued on `stream` so far
 * (a cudaStream_t; NULL: no wait, the data is ready for the session stream), then copies `data_dev`
 * device to device and runs the conventional decode; the same re-arming rules as
 * j2p_session_upload apply.  Returns once the work is queued: `data_dev` must stay valid until the
 * session stream has copied it.  J2P_ERR_ARG: null pointers, plane out of range, a zero table entry,
 * and memory that is not device memory on the session's device. */
int j2p_session_upload_device(j2p_session *s, unsigned plane, const int16_t *data_dev,
                              const uint16_t *quant, void *stream);

/* Re-arm the iteration state from the already-resident coefficient planes and the resident copy
 * of the conventional decode (no host traffic) — lets a benchmark time the loop repeatedly. */
int j2p_session_reset(j2p_session *s);

/* Run `n` solver iterations starting at iteration index `first` (0-based) on the session stream.
 * Asynchronous.  The FISTA momentum sequence (compute.c:431-432) restarts when first == 0. */
int j2p_session_iterate(j2p_session *s, unsigned first, unsigned n);

/* Measurement aid: runs `n` iterations from a freshly re-armed state with CUDA events recorded
 * on the session stream around each kernel, and returns the mean device time per launch of the
 * gradient kernel and of the step+projection kernel (milliseconds). */
int j2p_session_profile(j2p_session *s, unsigned n, float *ms_gradient, float *ms_project);

/* Block the host until iteration `iter` (0-based, already queued by j2p_session_iterate) has
 * finished on the device.  This is what lets `compute()` advance the reference's progress bar
 * (compute.c:449-452) at the pace of the device without draining the stream. */
int j2p_session_wait_iteration(j2p_session *s, unsigned iter);

/* HBM -> host: the current iterate of `channel`, H x W floats raster (batch sessions:
 * plane = frame * nchannel + channel). */
int j2p_session_download(j2p_session *s, unsigned channel, float *out);

/* HBM -> host, joint (3-plane) whole-frame sessions: the image as the reference hands it to libpng,
 * computed on the device — luma += 128 (jpeg2png.c:156-159), YCbCr -> RGB in double, clamp,
 * scale by (1 << bits)/256, truncate (png.c:39-47), 8-bit or 16-bit big-endian samples
 * (png.c:51-62) — laid out as PNG scanlines: h rows of 1 + w*3*bits/8 bytes, every row starting
 * with filter type 0.  w x h is the visible image (jpeg->w, jpeg->h), at most the frame size.
 * 3 or 6 bytes per pixel cross PCIe instead of 12. */
int j2p_session_download_scanlines(j2p_session *s, unsigned w, unsigned h, unsigned bits,
                                   unsigned char *out);
/* The same for frame `frame` of a batch session (j2p_session_download_scanlines is frame 0). */
int j2p_session_download_frame_scanlines(j2p_session *s, unsigned frame, unsigned w, unsigned h,
                                         unsigned bits, unsigned char *out);

/* ---- export of the RGB image into caller-owned device memory (tensors) -------------------------
 * The colour conversion of j2p_session_download_scanlines, written into `dst` on the device for
 * frames [frame0, frame0 + nframes) of a session, nothing staged through the host.  Per sample,
 * x = the YCbCr -> RGB expression in double on (luma + 128 in fp32), narrowed to float and clamped
 * to [0, 255] (jpeg2png.c:156-159, png.c:39-47); then
 *   sample 8:  uint8  trunc(x)          = the 8-bit PNG sample
 *   sample 16: uint16 trunc(x * 256)    = the 16-bit PNG sample (-1), in native byte order
 *   sample 32: float  x
 * HWC: h rows of w pixels of 3 samples (R, G, B); CHW: the R plane, then G, then B, h x w each.
 * Frame f of the export starts at dst + f * frame_bytes.
 *
 * Streams: `stream` (a cudaStream_t) NULL means the session stream (separate variant: the luma
 * session's); the legacy default stream is named by cudaStreamLegacy.  For every session stream other than the launch stream the export waits for the work
 * queued there so far, and that stream waits for the export: the export reads the planes of the
 * solve queued before it, and a later upload / reset / iterate of the session cannot overwrite them
 * first.  Asynchronous: the host never blocks.
 *
 * J2P_ERR_ARG: null dst or o, nframes == 0 or frames out of range, w or h 0 or larger than a plane's
 * frame, unknown sample or layout, frame_bytes smaller than one image, a joint export of a session
 * whose nchannel != 3, a strip session; separate sessions that do not have nchannel == 1, have
 * different frame counts, or live on different devices. */
enum { J2P_LAYOUT_HWC = 0, J2P_LAYOUT_CHW = 1 };
struct j2p_image_out {
        unsigned w, h;        /* visible image (struct j2p_jpeg w,h); <= every plane's frame  */
        unsigned sample;      /* 8: uint8, 16: uint16 (native endian), 32: float             */
        unsigned layout;      /* J2P_LAYOUT_HWC (interleaved) or J2P_LAYOUT_CHW (planar)      */
        size_t frame_bytes;   /* distance between consecutive frames in dst, >= one image     */
};
/* joint (nchannel == 3) whole-frame sessions, single or batch */
int j2p_session_export(j2p_session *s, unsigned frame0, unsigned nframes,
                       const struct j2p_image_out *o, void *dst, void *stream);
/* separate mode (-s): three nchannel == 1 sessions (Y, Cb, Cr) on one device with equal frame
 * counts; each plane is read with its own session's frame size */
int j2p_session_export_separate(j2p_session *y, j2p_session *cb, j2p_session *cr, unsigned frame0,
                                unsigned nframes, const struct j2p_image_out *o, void *dst,
                                void *stream);
/* gray: one sample per pixel from plane 0 alone, x = clamp(float((double)(Y + 128))), which is the
 * R (= G = B) sample of the RGB export for that luma with zero chroma; the same sample types, and
 * HWC and CHW are the same bytes ((h, w, 1) or (1, h, w)).  `s`: a whole-frame session with one
 * plane (a gray file, or a separate-mode luma session) or three (joint mode: its luma).  Streams
 * and refusals as j2p_session_export, the refusal of nchannel being "not 1 or 3". */
int j2p_session_export_gray(j2p_session *s, unsigned frame0, unsigned nframes,
                            const struct j2p_image_out *o, void *dst, void *stream);
/* oriented: the export of j2p_session_export (nsessions 1, channels 3), j2p_session_export_gray
 * (nsessions 1, channels 1) or j2p_session_export_separate (nsessions 3: Y, Cb, Cr; channels 3),
 * with frame frame0 + i flipped or rotated by its EXIF orientation orientation[i] as Pillow's
 * ImageOps.exif_transpose does it: 2 FLIP_LEFT_RIGHT, 3 ROTATE_180, 4 FLIP_TOP_BOTTOM, 5 TRANSPOSE,
 * 6 ROTATE_270, 7 TRANSVERSE, 8 ROTATE_90.
 *   orientation: device pointer to nframes bytes on the sessions' device (values outside 1..8 are
 *                written as 1); NULL = every frame 1.
 * o->w x o->h is the stored (unrotated) image.  Frames with orientation 5..8 are o->h wide and o->w
 * tall in dst, so HWC is (w, h, c) and CHW (c, w, h) for them; frame_bytes, the sample types and the
 * channel order are as j2p_session_export.  The samples are bit-identical to the unoriented export;
 * only their addresses change.  One launch for any mix of orientations.  Streams and refusals as
 * the export each combination stands for, and J2P_ERR_ARG for a null `sessions` or session, a
 * nsessions / channels combination that is none of the three, orientation memory that is not device
 * memory on the sessions' device, and o->h above 2097120 (65535 rows of 32-pixel tiles). */
int j2p_session_export_oriented(j2p_session *const *sessions, unsigned nsessions, unsigned channels,
                                unsigned frame0, unsigned nframes, const unsigned char *orientation,
                                const struct j2p_image_out *o, void *dst, void *stream);
/* Four-component JPEGs (Adobe CMYK and YCCK files): the frames of `nframes` files from file frame0 on,
 * one launch on `stream` ordered with the sessions as the exports above.  The four planes of a file
 * come from `sessions` in channel order; session k holds q_k planes of every file, q_k = its nchannel
 * times its frames over the file count N, and the q_k add up to 4 (N: the sessions' planes over 4).
 * So four nchannel == 1 sessions of N frames, one of 4N frames (file f's plane c is its frame
 * 4f + c), or for YCCK an nchannel == 3 session of N frames followed by a nchannel == 1 one.
 * kind J2P_FOUR_CMYK: channel c = the inverse of plane c's gray sample (the gray export's sample g,
 * 255 - g at 8 bits, 65535 - g at 16, 255.f - g at 32).  J2P_FOUR_YCCK: channels 0-2 the RGB
 * samples of planes 0-2, channel 3 the inverse of plane 3's gray sample.  channels 4 writes these;
 * channels 3 (sample 8 only) writes Pillow's CMYK -> RGB of the 8-bit samples: nk = 255 - K,
 * t = x * nk + 128, each of R, G, B = clip(nk - ((t + (t >> 8)) >> 8), 0, 255).
 * orientation: NULL writes every frame upright as j2p_session_export does; otherwise per-file EXIF
 * orientations in device memory, as j2p_session_export_oriented.  Returns J2P_ERR_ARG for what the
 * other exports refuse and for a kind, channel count or session set that is none of the above. */
enum { J2P_FOUR_CMYK = 1, J2P_FOUR_YCCK = 2 };
int j2p_session_export_four(j2p_session *const *sessions, unsigned nsessions, unsigned kind, unsigned channels,
                            unsigned frame0, unsigned nframes, const unsigned char *orientation,
                            const struct j2p_image_out *o, void *dst, void *stream);

/* Iterations [first, first + count) of every frame of every session of `sessions`, in one launch chain:
 * each kernel of an iteration is launched once for all n sessions, whatever their frame sizes, on the
 * first session's stream (the grouped kernels of libj2pmixed.so, loaded on first use).  Every frame's
 * result is bit-identical to what j2p_session_iterate gives it: same CTAs, bands and tiles, its own sums
 * of g^2 folded in the same order.  Each session's FISTA state, buffer parity, iteration counter and
 * launch count advance as j2p_session_iterate would advance them, so j2p_session_iterate, the exports and
 * later groups continue from there.  The launch stream first waits for what every other session's
 * stream has queued (uploads, re-arm), and each other session's stream then waits for the group's last
 * launch.  first == 0 re-arms a session as j2p_session_iterate does.
 * Sessions join a group when they are whole-frame (batch or single-frame) sessions on one device, without
 * objective logging, with equal nchannel, equal sampling factors per plane, every plane 1x1 or 2x2, and
 * bitwise-equal weight, pweights and iterations, first is every session's next iteration, and the group
 * holds at most 65535 frames.  Everything else is J2P_ERR_ARG with a message naming the first offending
 * session; a missing libj2pmixed.so is J2P_ERR_CUDA. */
int j2p_session_iterate_group(j2p_session *const *sessions, unsigned n, unsigned first, unsigned count);

/* Objective terms of the most recent iteration, as logged by the reference (compute.c:271-272):
 * out[0]=objective, out[1]=prob_dist, out[2]=tv, out[3]=tv2.  Only tracked when logging was
 * enabled with j2p_session_set_logging(s, 1) before iterating. */
int j2p_session_set_logging(j2p_session *s, int enabled);
int j2p_session_objective(j2p_session *s, double out[4]);

/* Record the objective of every iteration on the device, for every frame of a whole-frame session
 * (single-frame or batch): the numbers j2p_session_objective gives, without a host wait per
 * iteration.  Set before iterating; re-arming (first == 0) clears the record.  Refused on strip
 * sessions and on sessions with j2p_session_set_logging on (and vice versa); a missing
 * libj2pobjective.so is J2P_ERR_CUDA.  A recording session iterates with the recording kernels of
 * libj2pobjective.so (loaded on first use): the same launches and the same iterates, bit for bit.
 * The record holds desc.iterations rows: iterating a recording session past them is J2P_ERR_ARG, and
 * so is a group (j2p_session_iterate_group) that contains one. */
int j2p_session_record_objective(j2p_session *s, int enabled);
/* Iterations [first, first+count) of every frame: out[(f * count + i) * 4 + k], k = objective,
 * prob_dist, tv, tv2.  Synchronises the session stream; one device-to-host copy.  Rows that have not
 * been recorded since the last arm are J2P_ERR_ARG. */
int j2p_session_objective_history(j2p_session *s, unsigned first, unsigned count, double *out);

/* Block the host until everything queued on the session stream has finished. */
int j2p_session_sync(j2p_session *s);

/* Make a freshly allocated host buffer resident (huge-page hint + parallel first touch).  The
 * drop-in compute() calls it for the result buffers it hands back (compute.c:458) while the device
 * is still iterating, so the page faults of 100 MB of new memory are off the download path. */
void j2p_host_prefault(void *p, size_t bytes);

/* Raw handles for callers that schedule their own work around the session (bench timing with
 * CUDA events on the launching stream; torch interop).  The stream is a cudaStream_t. */
void *j2p_session_stream(j2p_session *s);
/* Device pointer of the current iterate of `channel` (H x W floats; batch sessions: plane =
 * frame * nchannel + channel).  Null when out of range. */
void *j2p_session_plane_ptr(j2p_session *s, unsigned channel);

/* Launch counters: number of kernel launches issued by this session since creation. */
unsigned long long j2p_session_launches(const j2p_session *s);

/* Version string of the library build. */
const char *j2p_version(void);

#ifdef __cplusplus
}
#endif
#endif /* JPEG2PNG_B200_H */
