/* progressive.h — libj2pprogressive.so: Huffman decoding of progressive JPEG scans on the device.
 *
 * Input: the layouts of progressive files (j2p_read_jpeg_prog_layout, jpeg2png_b200/cli/
 * jpeg_reader.h).  j2p_progressive_pack writes them into one packed plan: the unstuffed segments,
 * the step, scan, segment and subsequence descriptors, the Huffman tables and one output pointer per
 * (file, plane).  The caller uploads the plan and calls j2p_progressive_decode, which zeroes each
 * plane and writes its int16 coefficients as j2p_read_jpeg_mem returns them (the real block grid,
 * blocks in raster order, each block in natural order), and one status word per file (J2P_ENT_OK or
 * the failure kind, entropy.h, of a block of that file).  A failed file's planes are unspecified.
 *
 * Decoding runs in steps: step t decodes scan t of every file that has one, so each file's scans
 * keep their order.  The entropy-coded data of the DC first and AC first scans of all steps is
 * synchronised up front, before any step (sync rounds in groups of four as in entropy.h, one round
 * trip per group), since it does not depend on coefficients.  Launches per call: the zeroing, the
 * sync rounds, and when there are DC or AC first scans two exclusive scans and the DC differences;
 * then per step one launch for each scan kind present: the DC and AC first stores, the DC refine
 * pass, and for AC refine scans the nonzero masks and the refine walker (see DESIGN §7g).
 */
#ifndef J2P_PROGRESSIVE_H
#define J2P_PROGRESSIVE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

struct j2p_jpeg_prog_layout;

struct j2p_progressive_stats {
        unsigned rounds;           /* sync rounds launched */
        unsigned round_trips;      /* device -> host flag reads the host waited for */
        unsigned launches;         /* kernel launches */
        unsigned steps;            /* scans of the file with the most */
        unsigned subsequences;     /* of the DC first and AC first scans */
        unsigned refine_segments;  /* (file, AC refine scan, restart segment) walkers */
        unsigned step_launches;    /* of launches, those queued by the steps */
};

/* Sizes of the packed plan and of the device work area for `n` layouts at `subseq_bits` bits per
 * subsequence (a multiple of 32, at least 32).  Returns 0, or -1 (j2p_progressive_last_error). */
int j2p_progressive_plan_size(const struct j2p_jpeg_prog_layout *const *layouts, unsigned n, unsigned subseq_bits, size_t *plan_bytes,
                              size_t *work_bytes);
/* Writes the plan into `dst` (plan_bytes, 16-byte aligned).  out[3 * i + c]: where plane c of
 * file i goes (w/8 * h/8 * 64 int16, 16-byte aligned).  The empty planes 1 and 2 of a gray file
 * (J2P_READ_GRAY, w = h = 0) are never written and their out entries are not read. */
int j2p_progressive_pack(const struct j2p_jpeg_prog_layout *const *layouts, unsigned n, unsigned subseq_bits, int16_t *const *out,
                         void *dst, size_t plan_bytes);
/* Decodes on `stream` (a cudaStream_t; NULL: the legacy default stream).  plan_host: the packed
 * plan; plan_dev: its copy in device memory (uploaded on `stream` or before it); work_dev:
 * work_bytes of device memory; status_dev: uint32 per file.  Returns when the last kernel is
 * queued (after the host has read the sync flags). */
int j2p_progressive_decode(const void *plan_host, const void *plan_dev, void *work_dev, uint32_t *status_dev, void *stream,
                           struct j2p_progressive_stats *stats);
/* The same phases run serially on the host, on host memory (out pointers of the plan are host
 * memory): the testable restatement of the device decoder. */
int j2p_progressive_decode_host(const void *plan, void *work, uint32_t *status, struct j2p_progressive_stats *stats);

const char *j2p_progressive_last_error(void);

#ifdef __cplusplus
}
#endif

#endif
