/* png.h — libj2ppng.so: RGB and gray images in device memory to PNG files, encoded on the device.
 *
 * Each image is 8-bit or 16-bit RGB or gray (16-bit samples in native byte order, written
 * big-endian), addressed with element strides for row, column and channel, so HWC, CHW and strided
 * views are read in place.  One call may mix RGB and gray images.  The file holds the signature,
 * IHDR (colour type 2 for RGB, 0 for gray, no interlace), one IDAT (zlib
 * header 78 01, the deflate stream, the Adler-32) and IEND.  png_core.h states the encoding.
 *
 * One call: j2p_png_plan gives the size of the device work area for a list of images;
 * j2p_png_encode queues the whole encode on a stream (after what is already queued there), reads
 * back the file offsets and, when given a host buffer, copies the files into it.  The launches of
 * one call do not depend on the number or the sizes of the images.  j2p_png_encode_host runs the
 * same steps serially on host memory and writes the same bytes.
 */
#ifndef J2P_PNG_H
#define J2P_PNG_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

struct j2p_png_image {
        const void *data;               /* first sample (R of the top-left pixel) */
        uint32_t width, height;         /* 1 .. 2^31 - 1 */
        uint32_t sample_bytes;          /* 1 (uint8) or 2 (native-endian uint16) */
        int64_t row_stride, col_stride, chan_stride;      /* in samples */
        uint32_t channels;              /* 3 (RGB) or 1 (gray; chan_stride unused); 0 reads as 3 */
};

struct j2p_png_stats {
        unsigned launches;              /* kernel launches of the call */
        unsigned pieces;                /* pieces of J2P_PNG_PIECE filtered bytes, all images */
};

/* Work area for the n images: work_bytes in all, the files at out_offset in it.  Refuses null
 * pointers, n == 0, a width or height of 0 or above 2^31 - 1, a sample size other than 1 or 2, a
 * channel count other than 0, 1 or 3, and
 * an image whose IDAT could exceed PNG's chunk limit of 2^31 - 1 bytes: the file has one IDAT, so
 * the image's worst-case deflate stream (every block stored, see j2p_png_piece_bound) plus the zlib
 * header and checksum must fit.  That admits about 2.14e9 filtered bytes, e.g. 26,700 x 26,700 RGB at
 * 8 bits or 18,900 x 18,900 at 16 bits (three times the pixels in gray).  Returns 0, or -1 (j2p_png_last_error). */
int j2p_png_plan(const struct j2p_png_image *images, unsigned n, size_t *work_bytes, size_t *out_offset);

/* Encodes on `stream` (a cudaStream_t; NULL: the legacy default stream) into `work` (device memory
 * of work_bytes on the images' device).  Writes offsets[0..n]: file i is bytes [offsets[i],
 * offsets[i+1]) of the output, which starts at work + out_offset.  If dst is not NULL the files are
 * copied there (dst_cap bytes at least offsets[n]).  Returns when the offsets (and dst) are on the
 * host.  Also refuses image data or work memory that is not device memory of one device. */
int j2p_png_encode(const struct j2p_png_image *images, unsigned n, void *work, size_t work_bytes, void *stream, uint64_t *offsets,
                   void *dst, size_t dst_cap, struct j2p_png_stats *stats);

/* The same steps run serially on host memory (images and work in host memory). */
int j2p_png_encode_host(const struct j2p_png_image *images, unsigned n, void *work, size_t work_bytes, uint64_t *offsets);

const char *j2p_png_last_error(void);

#ifdef __cplusplus
}
#endif

#endif
