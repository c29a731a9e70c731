/* arith.h — libj2parith.so: decoding of sequential arithmetic-coded (SOF9) JPEG scans on the device.
 *
 * Input: the layouts of arithmetic-decodable files (j2p_read_jpeg_arith_layout, jpeg2png_b200/cli/
 * jpeg_reader.h).  j2p_arith_pack writes them into one packed plan: the unstuffed segments, the scan
 * and segment descriptors (with each scan's DAC conditioning and which components share statistics)
 * and one output pointer per (file, plane).  The caller uploads the plan and calls j2p_arith_decode,
 * which writes each plane's int16 coefficients as j2p_read_jpeg_mem returns them (the real block
 * grid, blocks in raster order, each block in natural order, every coefficient written) and one
 * status word per file (J2P_ARITH_OK or J2P_ARITH_BAD_CODE, arith_core.h).  A failed file's planes
 * are unspecified.
 *
 * A QM-coded segment cannot be entered in the middle (its coder state and adaptive statistics depend
 * on every decision before), so the device works on (file, scan, restart segment): one thread per
 * segment, its statistics in shared memory.  One call is one kernel launch after the status reset,
 * whatever the number of files; files without restart intervals are one serial walk each.
 */
#ifndef J2P_ARITH_H
#define J2P_ARITH_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

struct j2p_jpeg_arith_layout;

struct j2p_arith_stats {
        unsigned launches;      /* kernel launches */
        unsigned segments;      /* segments decoded (one thread each) */
};

/* Sizes of the packed plan and of the device work area (0: the decoder needs none; the argument is
 * kept so that the device decoders of decode_jpeg share one calling sequence) for `n` layouts.
 * Returns 0, or -1 (j2p_arith_last_error). */
int j2p_arith_plan_size(const struct j2p_jpeg_arith_layout *const *layouts, unsigned n, size_t *plan_bytes, size_t *work_bytes);
/* Writes the plan into `dst` (plan_bytes, 16-byte aligned).  out[3 * i + c]: where plane c of
 * file i goes (w/8 * h/8 * 64 int16, 16-byte aligned).  The empty planes 1 and 2 of a gray file are
 * never written and their out entries are not read. */
int j2p_arith_pack(const struct j2p_jpeg_arith_layout *const *layouts, unsigned n, int16_t *const *out, void *dst, size_t plan_bytes);
/* Decodes on `stream` (a cudaStream_t; NULL: the legacy default stream).  plan_host: the packed
 * plan; plan_dev: its copy in device memory (uploaded on `stream` or before it); work_dev: unused;
 * status_dev: uint32 per file.  Returns when the kernel is queued. */
int j2p_arith_decode(const void *plan_host, const void *plan_dev, void *work_dev, uint32_t *status_dev, void *stream,
                     struct j2p_arith_stats *stats);
/* The same per-segment code run serially on the host, on host memory (out pointers of the plan are
 * host memory). */
int j2p_arith_decode_host(const void *plan, void *work, uint32_t *status, struct j2p_arith_stats *stats);

const char *j2p_arith_last_error(void);

#ifdef __cplusplus
}
#endif

#endif
