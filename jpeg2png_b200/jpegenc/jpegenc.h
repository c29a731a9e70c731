/* jpegenc.h — libj2pjpegenc.so: RGB images in device memory to baseline JPEG files, encoded on the
 * device.
 *
 * Each image is 8-bit RGB addressed with element strides for row, column and channel, so HWC, CHW
 * and strided views are read in place.  The file is the one libjpeg's compressor writes with its
 * defaults, as Pillow's JPEG writer drives it (quality q, subsampling s, no other options): SOI;
 * APP0 JFIF 1.01, no units, density 1 x 1; DQT of table 0 (luma) and of table 1 (chroma), 8-bit,
 * IJG quality scaling with the baseline clamp; SOF0 with components 1, 2, 3 sampled 1x1, 2x1 or 2x2
 * for luma and 1x1 for chroma; DHT of the Annex K tables DC0, AC0, DC1, AC1; SOS of one interleaved
 * scan; the entropy-coded data; EOI.  jpegenc_core.h states each step.
 *
 * One call: j2p_jpegenc_plan gives the size of the device work area for a list of images;
 * j2p_jpegenc_encode queues the whole encode on a stream (after what is already queued there), reads
 * back the n + 1 file offsets and, when given a host buffer, copies the files into it.  The launches
 * of one call do not depend on the number or the sizes of the images.  j2p_jpegenc_encode_host runs
 * the same steps serially on host memory and writes the same bytes.
 *
 * The work area is sized from a worst-case bound, so one call needs one read-back.  The bound of a
 * block follows from the Annex K tables.  Luma: a DC difference costs at most 9 + 11 bits (category
 * 11), and each of the 63 AC coefficients at most 16 + 10 (run 0, category 10, a 16-bit code); a
 * run of zeros costs less per coefficient (ZRL is 11 bits for 16 zeros, EOB 4 bits, and a run r
 * before a coefficient at most 16 + 10 bits for r + 1 of them).  So 20 + 63 x 26 = 1658 bits.
 * Chroma: 11 + 11 for the DC and at most 22 per AC coefficient (its run 0, category 10 code is 12
 * bits), 22 + 63 x 22 = 1408.  J2P_JPEGENC_BLOCK_BITS is the larger, and stuffing at most doubles
 * the bytes.  For 64 images of 1920 x 1080 the work area is about 2.4 GB at 4:2:0, 4.7 GB at 4:4:4.
 *
 * Restart markers (restart_marker_blocks, restart_marker_rows; Pillow's keywords of the same names):
 * the scan is cut into intervals of Ri MCUs, Ri = restart_marker_blocks, or restart_marker_rows x
 * the MCUs per row capped at 65535 when that is set.  The header gets DRI (FF DD 00 04 Ri) between
 * the DHTs and the SOS.  Each interval is its own bit stream: it starts with DC predictions of 0,
 * is padded with 1-bits to a byte, and every interval but the first is preceded by RST0 + (its
 * number - 1) mod 8.  So an interval adds at most 7 pad bits and 2 unstuffed marker bytes to the
 * bound above, and each costs a stream descriptor, a 256-block tile, an 8 KiB stuffing chunk and
 * 16 bytes of rounding words of work area (jpegenc_plan.h).  Values above 65535 are refused, where
 * libjpeg would write DRI mod 65536 and count the full value (a corrupt file).
 *
 * Gray images (params->components == 1; 0 or 3 is colour): each image is one 8-bit channel, data
 * its first sample, chan_stride not read.  The file is the one libjpeg writes for a one-component
 * (Pillow 'L') image: SOI; the same APP0; DQT of table 0 only; SOF0 with component 1 and sampling
 * byte 0x11, 0x21 or 0x22 for 4:4:4, 4:2:2 and 4:2:0 (it changes no coded byte); DHT DC0 and AC0;
 * SOS of one component, 01 01 00 00 3f 00; 328 bytes before the entropy-coded data.  The scan walks
 * the component's own ceil(w/8) x ceil(h/8) block grid in raster order, one block per MCU, with no
 * dummy blocks; the samples are the pixels minus 128 (no colour conversion), the last row and
 * column repeated past the image.  With restart_marker_rows = r an interval is min(r x ceil(w/8),
 * 65535) blocks.  A block costs at most the luma bound, 1658 bits.  The kind belongs to the call,
 * so a list of gray and colour images is two calls.  Any other components value is refused.
 *
 * Given quantisation tables (params->qtables; Pillow's qtables keyword): the call takes nqtables
 * sets of 1 .. 4 tables of final values (natural order, 1 .. 8191: any parsing and quality scaling
 * is the caller's), and image i is quantised with set images[i].qtables, so files from different
 * sources keep their own tables in one call.  The components use the tables as Pillow maps them:
 * one table: Y, Cb and Cr all table 0; two: Y 0, Cb and Cr 1; three or four: Y 0, Cb 1, Cr 2 (a
 * fourth is neither written nor used); a gray image table 0.  The Huffman tables do not change (Cb
 * and Cr share DC1 / AC1 even with three quantisation tables).  The header carries one DQT per used
 * table in the order the components first use it, 16-bit (Pq = 1, 131 bytes) when one of its
 * entries exceeds 255, else 8-bit (67 bytes), and the frame is SOF1 rather than SOF0 when any DQT is
 * 16-bit (a progressive file stays SOF2).  Entries above 8191 are refused: libjpeg divides by 8q in
 * 16 bits, so they wrap and its coefficients no longer match the table its file declares.  NULL
 * qtables is the IJG tables of params->quality, one set that every image uses (the images' qtables
 * fields are not read); a zero-initialised params keeps that meaning.  The header's length is per
 * set, 623 bytes for the quality tables of a colour file, at most 884 with three 16-bit tables.
 *
 * CMYK images (params->cmyk == 1, components 0): each image is four 8-bit channels, C M Y K at
 * data, data + chan_stride, data + 2 chan_stride, data + 3 chan_stride.  The file is the one
 * libjpeg writes for a four-component JCS_CMYK image as Pillow drives it for a 'CMYK' image: SOI;
 * APP14 "Adobe" version 100, flags 0 and 0, transform 0 (FF EE 00 0E 'Adobe' 00 64 00 00 00 00 00)
 * and no APP0; the DQTs; SOF0 (SOF1 with a 16-bit table) with components 'C' 'M' 'Y' 'K' (67, 77,
 * 89, 75), C sampled 1x1, 2x1 or 2x2 and M, Y, K 1x1, as Pillow applies subsampling to component 0
 * alone; DHT DC0 and AC0 only, which every component codes with; SOS of one interleaved scan of
 * the four.  The samples are coded inverted (Pillow's raw mode CMYK;I): 255 - t for a tensor
 * sample t, so a decoder that undoes the Adobe inversion, as Pillow and decode_jpeg do, reads t
 * back.  M, Y and K are downsampled like chroma, from the inverted samples, with no colour
 * conversion; an MCU is hs x vs blocks of C and one each of M, Y and K.  The quality tables give
 * table 0 to all four components and one DQT, a 341-byte header; n given tables give component c
 * table min(c, n - 1) (one: 0 0 0 0; two: 0 1 1 1; three: 0 1 2 2; four: 0 1 2 3, the fourth
 * table written and used by K) and one DQT each.  The longest header, four 16-bit DQTs, is 804
 * bytes.  A block costs at most the luma bound, 1658 bits.  Any other cmyk value is refused, and
 * so is cmyk = 1 with a components value other than 0.
 */
#ifndef J2P_JPEGENC_H
#define J2P_JPEGENC_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define J2P_JPEGENC_BLOCK_BITS 1658u

enum j2p_jpegenc_sampling { J2P_JPEGENC_444 = 0, J2P_JPEGENC_422 = 1, J2P_JPEGENC_420 = 2 };

struct j2p_jpegenc_image {
        const void *data;               /* first sample (R, gray or C of the top-left pixel), uint8 */
        uint32_t width, height;         /* 1 .. 65535 */
        int64_t row_stride, col_stride, chan_stride;      /* in samples */
        uint32_t qtables;               /* the image's set of params->qtables; not read when that is NULL */
};

/* One set of quantisation tables: final values, natural (row-major) order. */
struct j2p_jpegenc_qtables {
        uint16_t table[4][64];          /* 1 .. 8191 */
        uint32_t ntables;               /* 1 .. 4 */
};

struct j2p_jpegenc_params {
        int quality;                    /* 1 .. 100 */
        int sampling;                   /* enum j2p_jpegenc_sampling */
        int restart_marker_blocks;      /* 0 .. 65535: a restart interval of this many MCUs in every scan; 0 none */
        int restart_marker_rows;        /* 0 .. 65535: one of this many MCU rows per scan (capped at 65535
                                           MCUs); overrides restart_marker_blocks; 0 none */
        int components;                 /* 0 or 3: RGB images, YCbCr files; 1: gray images, one-component files */
        const struct j2p_jpegenc_qtables *qtables;        /* nqtables sets, or NULL: the IJG tables of quality */
        unsigned nqtables;
        int cmyk;                       /* 0: as components says; 1: CMYK images, Adobe CMYK files (components 0) */
};

struct j2p_jpegenc_stats {
        unsigned launches;              /* kernel launches of the call */
        uint64_t blocks;                /* 8 x 8 blocks coded, dummy blocks included, all images */
};

/* Work area for the n images: work_bytes in all, the files at out_offset in it.  Refuses null
 * pointers, n == 0, a width or height of 0 or above 65535 (SOF's 16-bit fields), a quality outside
 * 1 .. 100, an unknown sampling, a restart field outside 0 .. 65535, components other than 0, 1
 * or 3, cmyk other than 0 or 1 or with components not 0, and given tables with nqtables == 0, a set with ntables outside 1 .. 4 or an entry of 0 or
 * above 8191, or an image whose set is not below nqtables.  Returns 0, or -1 (j2p_jpegenc_last_error). */
int j2p_jpegenc_plan(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, size_t *work_bytes,
                     size_t *out_offset);

/* Encodes on `stream` (a cudaStream_t; NULL: the legacy default stream) into `work` (device memory
 * of work_bytes on the images' device).  Writes offsets[0..n]: file i is bytes [offsets[i],
 * offsets[i+1]) of the output, which starts at work + out_offset.  If dst is not NULL the files are
 * copied there (dst_cap bytes at least offsets[n]).  Returns when the offsets (and dst) are on the
 * host.  Also refuses image data or work memory that is not device memory of one device. */
int j2p_jpegenc_encode(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, void *work,
                       size_t work_bytes, void *stream, uint64_t *offsets, void *dst, size_t dst_cap, struct j2p_jpegenc_stats *stats);

/* The same steps run serially on host memory (images and work in host memory). */
int j2p_jpegenc_encode_host(const struct j2p_jpegenc_image *images, unsigned n, const struct j2p_jpegenc_params *params, void *work,
                            size_t work_bytes, uint64_t *offsets);

const char *j2p_jpegenc_last_error(void);

#ifdef __cplusplus
}
#endif

#endif
