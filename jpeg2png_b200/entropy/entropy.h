/* entropy.h — libj2pentropy.so: Huffman decoding of sequential JPEG scans on the device.
 *
 * Input: the layouts of device-decodable files (j2p_read_jpeg_layout, jpeg2png_b200/cli/
 * jpeg_reader.h).  j2p_entropy_pack writes them into one packed plan: the unstuffed segments, the
 * scan, segment and subsequence descriptors, the Huffman tables and one output pointer per (file,
 * plane).  The caller uploads the plan and calls j2p_entropy_decode, which writes each plane's
 * int16 coefficients as j2p_read_jpeg_mem returns them (the real block grid, blocks in raster
 * order, each block in natural order) and one status word per file (J2P_ENT_OK or the first failure
 * kind met by a block of that file).  A failed file's planes are unspecified.
 *
 * The launches of one call do not depend on the number of files: one launch per sync round, two
 * exclusive scans, the final pass and the DC pass.  Sync rounds go in groups of four, until the last
 * round of a group changed no subsequence's start state; after each group the host reads that
 * round's flag back (one round trip per group, counted in struct j2p_entropy_stats).
 */
#ifndef J2P_ENTROPY_H
#define J2P_ENTROPY_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { J2P_ENT_OK = 0, J2P_ENT_BAD_CODE = 1, J2P_ENT_BAD_MAGNITUDE = 2, J2P_ENT_BAD_INDEX = 3 };

struct j2p_jpeg_layout;
struct j2p_jpeg_layout4;

struct j2p_entropy_stats {
        unsigned rounds;        /* sync rounds launched */
        unsigned round_trips;   /* device -> host flag reads the host waited for */
        unsigned launches;      /* kernel launches */
        unsigned subsequences;
};

/* Sizes of the packed plan and of the device work area for `n` layouts at `subseq_bits` bits per
 * subsequence (a multiple of 32, at least 32).  Returns 0, or -1 (j2p_entropy_last_error). */
int j2p_entropy_plan_size(const struct j2p_jpeg_layout *const *layouts, unsigned n, unsigned subseq_bits, size_t *plan_bytes,
                          size_t *work_bytes);
/* Writes the plan into `dst` (plan_bytes, 16-byte aligned).  out[3 * i + c]: where plane c of
 * file i goes (w/8 * h/8 * 64 int16, 16-byte aligned).  The empty planes 1 and 2 of a gray file
 * (J2P_READ_GRAY, w = h = 0) are never written and their out entries are not read. */
int j2p_entropy_pack(const struct j2p_jpeg_layout *const *layouts, unsigned n, unsigned subseq_bits, int16_t *const *out,
                     void *dst, size_t plan_bytes);
/* The same for four-component files (struct j2p_jpeg_layout4 of j2p_read_jpeg_layout4, device
 * decodable): out[4 * i + c] is where plane c of file i goes.  One- and three-component layouts of
 * j2p_read_jpeg_layout4 are taken too, their empty planes' out entries not read. */
int j2p_entropy_plan_size4(const struct j2p_jpeg_layout4 *const *layouts, unsigned n, unsigned subseq_bits, size_t *plan_bytes,
                           size_t *work_bytes);
int j2p_entropy_pack4(const struct j2p_jpeg_layout4 *const *layouts, unsigned n, unsigned subseq_bits, int16_t *const *out,
                      void *dst, size_t plan_bytes);
/* Decodes on `stream` (a cudaStream_t; NULL: the legacy default stream).  plan_host: the packed
 * plan; plan_dev: its copy in device memory (uploaded on `stream` or before it); work_dev:
 * work_bytes of device memory; status_dev: uint32 per file.  Returns when the last kernel is
 * queued (after the host has read the sync flags). */
int j2p_entropy_decode(const void *plan_host, const void *plan_dev, void *work_dev, uint32_t *status_dev, void *stream,
                       struct j2p_entropy_stats *stats);
/* The same phases run serially on the host, on host memory (out pointers of the plan are host
 * memory): the testable restatement of the device decoder. */
int j2p_entropy_decode_host(const void *plan, void *work, uint32_t *status, struct j2p_entropy_stats *stats);

const char *j2p_entropy_last_error(void);

#ifdef __cplusplus
}
#endif

#endif
