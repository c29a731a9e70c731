/* jpegopt.h — libj2pjpegopt.so: RGB images in device memory to baseline JPEG files with optimized
 * Huffman tables, encoded on the device.
 *
 * The file is the one libjpeg's compressor writes with optimize_coding, as Pillow's JPEG writer
 * drives it with `optimize=True` (and quality q, subsampling s): the same segments, in the same
 * order, as libj2pjpegenc.so's files (jpegenc.h), and the same entropy-coded coefficients, but each
 * image's four DHT segments hold its own tables, built from its own symbol counts (T.81 Annex K.2
 * with libjpeg's tie rule, the K.3 limit to 16 bits; jpegopt_core.h).  A DHT lists only the
 * symbols that occur, so the header is at most the length of its set's template (jpegenc.h: 623
 * bytes for the quality tables of a colour file, 884 at most with given tables) and its length
 * varies by image.  With given quantisation tables (params->qtables, jpegenc.h) each image's DQTs
 * and SOF0 or SOF1 come from its own set, as in libj2pjpegenc.so's file.
 *
 * The images, parameters and statistics are jpegenc.h's structs, and the calls mirror its calls.
 * One call queues a memset and nine kernels, whatever the number and sizes of the images:
 * blocks, hist (symbol counts), tables (code lengths, codes, header), sizes, scan, emit, ffcount,
 * offsets, stuff.  j2p_jpegopt_encode_host runs the same steps serially on host memory and writes
 * the same bytes.
 *
 * Work-area bound: with optimized tables any code can be 16 bits long, so a block costs at most
 * 16 + 11 bits of DC and 63 x (16 + 10) of AC, J2P_JPEGOPT_BLOCK_BITS = 1665 (jpegenc.h's bound,
 * 1658, holds for the Annex K tables only).
 *
 * Gray calls (components == 1, jpegenc.h): each image counts and builds two tables, DC0 and AC0,
 * and its header is jpegenc.h's gray header with its own DHT 0x00 and 0x10.  The work-area bound
 * is the same J2P_JPEGOPT_BLOCK_BITS per block, and a call still runs the nine kernels once.
 *
 * CMYK calls (cmyk == 1, jpegenc.h): each image counts the symbols of all four components into two
 * tables, DC0 and AC0, and its header is jpegenc.h's CMYK header with its own DHT 0x00 and 0x10.
 * The bound and the nine kernels are the same.
 */
#ifndef J2P_JPEGOPT_H
#define J2P_JPEGOPT_H

#include "../jpegenc/jpegenc.h"

#ifdef __cplusplus
extern "C" {
#endif

#define J2P_JPEGOPT_BLOCK_BITS 1665u

/* As j2p_jpegenc_plan, for the optimized files. */
int j2p_jpegopt_plan(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, size_t *work_bytes,
                     size_t *out_offset);

/* As j2p_jpegenc_encode, for the optimized files (stats->launches is 9). */
int j2p_jpegopt_encode(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, void *work,
                       size_t work_bytes, void *stream, uint64_t *offsets, void *dst, size_t dst_cap, struct j2p_jpegenc_stats *stats);

/* The same steps run serially on host memory (images and work in host memory). */
int j2p_jpegopt_encode_host(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, void *work,
                            size_t work_bytes, uint64_t *offsets);

/* The table builder of one table, on host memory: counts[256] symbol counts (at least one not 0) to
 * the DHT's code counts per length bits[16] and its symbols vals[*nvals] (room for 256).  For tests. */
int j2p_jpegopt_build_table(const uint64_t *counts, uint8_t *bits, uint8_t *vals, unsigned *nvals);

const char *j2p_jpegopt_last_error(void);

#ifdef __cplusplus
}
#endif

#endif
