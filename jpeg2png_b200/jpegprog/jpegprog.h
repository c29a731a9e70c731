/* jpegprog.h — libj2pjpegprog.so: RGB images in device memory to progressive JPEG files, encoded on
 * the device.
 *
 * The file is the one libjpeg's compressor writes with jpeg_simple_progression, as Pillow's JPEG
 * writer drives it with `progressive=True` (and quality q, subsampling s; `optimize` changes no
 * byte): SOI, JFIF APP0, the DQTs of libj2pjpegenc.so's file (jpegenc.h: the image's set of
 * quantisation tables, or the two quality tables) and SOF2 (whatever their precision), then ten
 * scans, each after the DHTs of the tables it uses, then EOI.  The coefficients are the baseline
 * file's; each scan's tables are built from that scan's own symbol counts (jpegopt_core.h).  The
 * scan script and the coding rules are in jpegprog_core.h.
 *
 * The images, parameters and statistics are jpegenc.h's structs, and the calls mirror its calls.
 * Every (image, scan) pair, or every restart interval of it, is its own bit stream.  One call queues a memset and
 * J2P_JPEGPROG_LAUNCHES kernels, whatever the number and sizes of the images: blocks (and each AC
 * scan's block summaries), runs (the EOB-run state each block of an AC scan receives), hist (symbol
 * counts per image and table), tables (ten per image, and each stream's DHT and SOS header), sizes,
 * scan, emit, ffcount, offsets, stuff.  j2p_jpegprog_encode_host runs the same steps serially on
 * host memory and writes the same bytes.
 *
 * Work-area bound: a block of the AC first scan over 63 coefficients costs at most 63 x (16 + 10)
 * bits and one EOB-run emission of 16 + 14, J2P_JPEGPROG_BLOCK_BITS = 1668; every other scan's bound
 * is smaller (jpegprog_core.h), and each stream gets its own.
 *
 * Restart markers (jpegenc.h's restart fields): each scan gets the interval libjpeg gives it, in that
 * scan's MCUs (an MCU of a non-interleaved AC scan is one block of its component's own grid), and
 * its DRI, before the SOS, when the interval differs from the last DRI of the file.  Every (image,
 * scan, interval) is then its own bit stream: the EOB run and its correction bits are flushed at the
 * interval's end, and DC predictions, the run and BE restart at 0.  The per-block bounds still hold,
 * because an interval's last EOB-run emission covers at least one of its blocks; an interval adds at
 * most 7 pad bits and the 2 unstuffed bytes of its RST.  Scan headers stay per (image, scan).
 *
 * Gray calls (components == 1, jpegenc.h): SOF2 with one component, then libjpeg's six scans for
 * one component (Ss Se Ah Al: 0 0 0 1, 1 5 0 2, 6 63 0 2, 1 63 2 1, 0 0 1 0, 1 63 1 0), five
 * tables per image (the DC refine has none), every scan non-interleaved over the real block grid in
 * raster order.  Per-scan bounds: 27, 160, 1538, 1101, 1 and 1101 bits a block, all within
 * J2P_JPEGPROG_BLOCK_BITS.  Every scan has the same restart interval, so a file has one DRI.  A call
 * still runs the J2P_JPEGPROG_LAUNCHES kernels once each.
 *
 * CMYK calls (cmyk == 1, jpegenc.h): the APP14 header and DQTs of jpegenc.h's CMYK file, SOF2 with
 * the four components, then libjpeg's generic script for four components, eighteen scans: DC first
 * of all four interleaved (0 0 0 1); C, M, Y, K each 1 5 0 2, then each 6 63 0 2, then each 1 63 2
 * 1; DC refine of all four (0 0 1 0); C, M, Y, K each 1 63 1 0.  Seventeen tables per image (the
 * DC refine has none), each written as DHT 0x00 (scan 0) or 0x10.  An AC scan walks its component's
 * own block grid and counts its blocks per row for restart_marker_rows, so the interval, and a DRI,
 * can change between scans.  Per-scan bounds are the gray script's, per component.  The per-image
 * tables and symbol counts are sized by the call's kind (5, 10 or 17 slots), and a call still runs
 * the J2P_JPEGPROG_LAUNCHES kernels once each.
 */
#ifndef J2P_JPEGPROG_H
#define J2P_JPEGPROG_H

#include "../jpegenc/jpegenc.h"

#ifdef __cplusplus
extern "C" {
#endif

#define J2P_JPEGPROG_BLOCK_BITS 1668u
#define J2P_JPEGPROG_LAUNCHES 10u

/* As j2p_jpegenc_plan, for the progressive files. */
int j2p_jpegprog_plan(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, size_t *work_bytes,
                      size_t *out_offset);

/* As j2p_jpegenc_encode, for the progressive files (stats->launches is J2P_JPEGPROG_LAUNCHES). */
int j2p_jpegprog_encode(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, void *work,
                        size_t work_bytes, void *stream, uint64_t *offsets, void *dst, size_t dst_cap, struct j2p_jpegenc_stats *stats);

/* The same steps run serially on host memory (images and work in host memory). */
int j2p_jpegprog_encode_host(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, void *work,
                             size_t work_bytes, uint64_t *offsets);

const char *j2p_jpegprog_last_error(void);

#ifdef __cplusplus
}
#endif

#endif
