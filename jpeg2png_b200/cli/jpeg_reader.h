/* jpeg_reader.h — JPEG file -> quantised DCT coefficients, without libjpeg.
 *
 * Replaces reference jpeg.c:22-80 (read_jpeg, built on libjpeg's jpeg_read_coefficients, which is
 * not available on the build box): same output contract — three `struct coef` with
 *   w,h            = width_in_blocks*8, height_in_blocks*8 of the component, NOT padded to whole
 *                    MCUs (jpeg.c:52-53)
 *   w_samp,h_samp  = max_h/h_i, max_v/v_i (jpeg.c:57-58)
 *   data           = int16 [blocks][64], natural (row-major) order, blocks in raster order
 *   quant_table    = natural order (jpeg.c:46)
 * and the same rejections: not exactly 3 components (jpeg.c:34), a zero quantisation entry
 * (jpeg.c:41-45), component sizes that do not match the sampling factors (jpeg.c:59-64).
 *
 * Supported: baseline and extended sequential Huffman (SOF0, SOF1), progressive Huffman (SOF2),
 * sequential and progressive arithmetic coding (SOF9, SOF10, with DAC conditioning), 8-bit
 * precision, restart intervals, interleaved and non-interleaved scans.  Not supported: lossless,
 * hierarchical, 12-bit (SOF3, SOF5-7, SOF11, SOF13-15: "unsupported jpeg: SOFn ...").
 *
 * Arithmetic coding follows libjpeg's jdarith.c (the QM decoder and sequential block step are
 * ../arith/arith_core.h).  DAC segments are refused where libjpeg's get_dac refuses them: an odd
 * length, a table index of 32 or more, L > U; any Kx byte is accepted.  One difference: libjpeg
 * accepts arithmetic table selectors up to 15, this reader refuses selectors above 3 for every
 * scan ("bad table selector").  Another: a segment's bytes end at the first FF not followed by 00,
 * as for Huffman scans, where libjpeg's arithmetic decoder skips FF fill bytes and reads FF FF 00
 * as one FF (encoders do not write that sequence inside entropy-coded data).  A magnitude category reaching 2^15 or a zero run or refinement past
 * the band's end is "corrupt jpeg: bad arithmetic code" where libjpeg warns and stops decoding.
 */
#ifndef J2P_JPEG_READER_H
#define J2P_JPEG_READER_H

#include <stddef.h>
#include <stdint.h>

#include "../../include/jpeg2png_b200.h"

struct j2p_jpeg {
        unsigned w, h;              /* image size in pixels */
        struct coef coefs[3];       /* data malloc'd (caller frees), fdata NULL */
        unsigned ncomp;             /* 3, or 1 (J2P_READ_GRAY): coefs[1..2] empty (w = h = 0, data NULL) */
};

/* Returns 0 on success; on failure returns non-zero and writes a message into err (if non-NULL).
 * The messages for the reference's own rejections are the reference's (jpeg.c:34,43,60,63). */
int j2p_read_jpeg_mem(const uint8_t *buf, size_t len, struct j2p_jpeg *out, char *err, size_t errlen);

/* Flags of the _ex entry points; the plain ones pass 0.
 * J2P_READ_GRAY: accept one-component (grayscale) files as well as three-component ones, and refuse
 * every other count with "only 1 and 3 component jpegs are supported".  A gray file's plane is
 * coefs[0] with w_samp = h_samp = 1 (whatever sampling factor its SOF gives it) and its scans are
 * non-interleaved over the plane's real block grid; coefs[1..2] stay empty. */
enum { J2P_READ_GRAY = 1u, J2P_READ_CMYK = 2u };
int j2p_read_jpeg_mem_ex(const uint8_t *buf, size_t len, unsigned flags, struct j2p_jpeg *out, char *err, size_t errlen);

/* ---- four-component files (Adobe CMYK and YCCK) ----
 * J2P_READ_CMYK: accept one-, three- and four-component files, and refuse every other count with
 * "only 1, 3 and 4 component jpegs are supported".  struct j2p_jpeg has room for three planes, so
 * j2p_read_jpeg_mem_ex ignores the flag; j2p_read_jpeg4_mem always applies it.  A four-component
 * file's planes keep the sampling factors of its SOF, as a colour file's do.
 * colour (four components only, else 0): libjpeg's choice, from the Adobe APP14 segment (12 data
 * bytes or more starting with "Adobe"; the last one before the first SOS counts; its transform is
 * byte 11): J2P_JPEG_CMYK without such a segment or with transform 0, J2P_JPEG_YCCK with any other
 * transform.  The three-plane layout passes report four-component files as not decodable when given
 * the flag, and refuse them with the count message without it; j2p_read_jpeg_layout4 takes them. */
enum { J2P_JPEG_CMYK = 1u, J2P_JPEG_YCCK = 2u };
struct j2p_jpeg4 {
        unsigned w, h;
        struct coef coefs[4];       /* as struct j2p_jpeg; coefs[ncomp..3] empty */
        unsigned ncomp;             /* 1, 3 or 4; on failure the frame header's count once it was read, else 0 */
        unsigned colour;            /* J2P_JPEG_CMYK or J2P_JPEG_YCCK for four components, else 0 */
};
int j2p_read_jpeg4_mem(const uint8_t *buf, size_t len, unsigned flags, struct j2p_jpeg4 *out, char *err, size_t errlen);


/* ---- layout pass: the headers and the entropy-coded data of a file, without Huffman decoding ----
 * (the _ex variant takes the J2P_READ_* flags of j2p_read_jpeg_mem_ex)
 *
 * j2p_read_jpeg_layout runs the marker loop and header checks of j2p_read_jpeg_mem (the same code)
 * and, instead of decoding each scan, cuts its entropy-coded data into segments, one per restart
 * interval, unstuffed (FF 00 -> FF), in one byte buffer.  A segment ends where the reader's bit
 * reader stops feeding bits: at the first FF not followed by 00, or at the end of the file; bits
 * past its end read as zero.  The restart markers between segments are checked by the reader's own
 * restart rule, so "missing restart marker", "out of sequence" and "truncated" fail here as there.
 *
 * device_decodable: the file is sequential Huffman (SOF0/SOF1) and each of its components is in
 * exactly one scan.  Only then are coefs (geometry and tables, data NULL), scans and segments
 * filled; for every other file the pass stops as soon as that is known (a progressive or
 * arithmetic SOF, a component's second scan) and returns 0 with device_decodable = 0: such files are for
 * j2p_read_jpeg_mem.  A non-zero return means j2p_read_jpeg_mem rejects the file too (it may name an
 * earlier error, in the entropy-coded data). */
struct j2p_jpeg_huff {
        uint8_t bits[17];           /* bits[l]: codes of length l (bits[0] unused) */
        uint8_t vals[256];
};
struct j2p_jpeg_scan {
        unsigned ncomp;             /* components in scan order */
        unsigned comp[3];           /* frame component (0..2) of each */
        unsigned bw[3], bh[3];      /* blocks per MCU of each: (h, v) when interleaved, else (1, 1) */
        unsigned mcux, mcuy;        /* MCU grid: the frame's MCUs when interleaved, else the component's real block grid */
        unsigned restart_interval;  /* MCUs per segment, 0: one segment */
        struct j2p_jpeg_huff dc[3], ac[3];  /* the tables in force at this SOS */
        unsigned seg0, nseg;        /* its segments */
};
struct j2p_jpeg_segment {
        size_t off, len;            /* unstuffed bytes in data */
        unsigned mcus;              /* MCUs it codes */
};
struct j2p_jpeg_layout {
        unsigned w, h;
        struct coef coefs[3];       /* as struct j2p_jpeg, but data NULL */
        unsigned comp_h[3], comp_v[3];   /* sampling factors of the frame header */
        int device_decodable;
        unsigned nscan;
        struct j2p_jpeg_scan scan[3];
        unsigned nseg;
        struct j2p_jpeg_segment *seg;    /* malloc'd */
        uint8_t *data;                   /* malloc'd */
        size_t data_len;
        unsigned ncomp;                  /* as struct j2p_jpeg; set when device_decodable */
};
int j2p_read_jpeg_layout(const uint8_t *buf, size_t len, struct j2p_jpeg_layout *out, char *err, size_t errlen);
int j2p_read_jpeg_layout_ex(const uint8_t *buf, size_t len, unsigned flags, struct j2p_jpeg_layout *out, char *err, size_t errlen);
void j2p_free_jpeg_layout(struct j2p_jpeg_layout *l);

/* The layout pass for four-component files (J2P_READ_CMYK always on): as j2p_read_jpeg_layout_ex,
 * with room for four planes and scans of up to four components, and the colour kind.
 * device_decodable: sequential Huffman, each component in exactly one scan (what
 * libj2pentropy.so's j2p_entropy_pack4 takes).  The three-plane layout passes keep stopping at a
 * four-component frame header.  A four-component file whose interleaved scan has more than 10
 * blocks per MCU is refused by every entry point, as libjpeg refuses it. */
struct j2p_jpeg_scan4 {
        unsigned ncomp, comp[4], bw[4], bh[4];  /* as struct j2p_jpeg_scan */
        unsigned mcux, mcuy, restart_interval;
        struct j2p_jpeg_huff dc[4], ac[4];
        unsigned seg0, nseg;
};
struct j2p_jpeg_layout4 {
        unsigned w, h;
        struct coef coefs[4];
        unsigned comp_h[4], comp_v[4];
        int device_decodable;
        unsigned nscan;
        struct j2p_jpeg_scan4 scan[4];
        unsigned nseg;
        struct j2p_jpeg_segment *seg;    /* malloc'd */
        uint8_t *data;                   /* malloc'd */
        size_t data_len;
        unsigned ncomp, colour;          /* set when device_decodable; colour as struct j2p_jpeg4 */
};
int j2p_read_jpeg_layout4(const uint8_t *buf, size_t len, unsigned flags, struct j2p_jpeg_layout4 *out, char *err, size_t errlen);
void j2p_free_jpeg_layout4(struct j2p_jpeg_layout4 *l);

/* ---- progressive layout pass: every scan of a progressive file, cut as above ----
 *
 * j2p_read_jpeg_prog_layout runs the same marker loop and header checks and cuts every scan of a
 * progressive (SOF2) file into segments as j2p_read_jpeg_layout does, recording each scan's
 * spectral selection and successive approximation with the tables and restart interval in force at
 * its SOS.  A component may be in any number of scans, or none.  progressive_decodable: the file is
 * progressive and the reader accepts it up to the scan headers (coefs, scans and segments filled);
 * for every other file the pass stops as soon as that is known (a sequential SOF) and returns 0 with
 * progressive_decodable = 0.  A non-zero return means j2p_read_jpeg_mem rejects the file too. */
struct j2p_jpeg_prog_scan {
        struct j2p_jpeg_scan s;     /* components, MCU grid, tables, restart interval, segments */
        unsigned ss, se, ah, al;    /* spectral selection and successive approximation (G.1.1.1) */
};
struct j2p_jpeg_prog_layout {
        unsigned w, h;
        struct coef coefs[3];       /* as struct j2p_jpeg, but data NULL */
        unsigned comp_h[3], comp_v[3];
        int progressive_decodable;
        unsigned nscan;
        struct j2p_jpeg_prog_scan *scan;     /* malloc'd, in file order */
        unsigned nseg;
        struct j2p_jpeg_segment *seg;        /* malloc'd */
        uint8_t *data;                       /* malloc'd */
        size_t data_len;
        unsigned ncomp;                      /* as struct j2p_jpeg; set when progressive_decodable */
};
int j2p_read_jpeg_prog_layout(const uint8_t *buf, size_t len, struct j2p_jpeg_prog_layout *out, char *err, size_t errlen);
int j2p_read_jpeg_prog_layout_ex(const uint8_t *buf, size_t len, unsigned flags, struct j2p_jpeg_prog_layout *out, char *err,
                                 size_t errlen);
void j2p_free_jpeg_prog_layout(struct j2p_jpeg_prog_layout *l);

/* ---- arithmetic layout pass: a sequential arithmetic-coded file, cut as above ----
 *
 * j2p_read_jpeg_arith_layout runs the same marker loop and header checks and cuts every scan of a
 * sequential arithmetic (SOF9) file into segments as j2p_read_jpeg_layout does.  Instead of Huffman
 * tables each scan records, per component, its table selectors (components with equal selectors
 * share statistics) and the conditioning in force at its SOS: L and U of its DC table, Kx of its AC
 * table.  arith_decodable: the file is SOF9 and each of its components is in exactly one scan; every
 * other file stops as soon as that is known and returns 0 with arith_decodable = 0.  A non-zero
 * return means j2p_read_jpeg_mem rejects the file too.  The existing layout passes report SOF9 and
 * SOF10 files as not device_decodable / progressive_decodable. */
struct j2p_jpeg_arith_scan {
        unsigned ncomp, comp[3], bw[3], bh[3];  /* as struct j2p_jpeg_scan */
        unsigned mcux, mcuy, restart_interval;
        unsigned dc_tbl[3], ac_tbl[3];          /* table selectors (0..3) */
        unsigned dc_L[3], dc_U[3], ac_K[3];     /* DAC conditioning of those tables */
        unsigned seg0, nseg;
};
struct j2p_jpeg_arith_layout {
        unsigned w, h;
        struct coef coefs[3];       /* as struct j2p_jpeg, but data NULL */
        unsigned comp_h[3], comp_v[3];
        int arith_decodable;
        unsigned nscan;
        struct j2p_jpeg_arith_scan scan[3];
        unsigned nseg;
        struct j2p_jpeg_segment *seg;    /* malloc'd */
        uint8_t *data;                   /* malloc'd */
        size_t data_len;
        unsigned ncomp;                  /* set when arith_decodable */
};
int j2p_read_jpeg_arith_layout(const uint8_t *buf, size_t len, struct j2p_jpeg_arith_layout *out, char *err, size_t errlen);
int j2p_read_jpeg_arith_layout_ex(const uint8_t *buf, size_t len, unsigned flags, struct j2p_jpeg_arith_layout *out, char *err,
                                  size_t errlen);
void j2p_free_jpeg_arith_layout(struct j2p_jpeg_arith_layout *l);

/* ---- EXIF orientation ----
 * The Orientation tag (0x0112) of IFD0 in the first APP1 segment that starts with "Exif\0\0" before
 * the first SOS: 1..8 as TIFF/EXIF define it (1 = upright; 2..8 the flip or rotation that makes the
 * stored image upright, as Pillow's ImageOps.exif_transpose applies it).  Returns 1 when there is no
 * such segment or tag, when the TIFF header (II or MM, 42, the IFD0 offset) or IFD0 runs past the
 * segment or the buffer, when the tag is not one SHORT or LONG, and for values outside 1..8.
 * Reads nothing outside [data, data + len) and does not look at any other header. */
int j2p_jpeg_exif_orientation(const void *data, size_t len);

/* ---- the settings of Pillow's quality='keep' ----
 * The quantisation tables a file defines before its first SOS (natural order, bit t of present set
 * for table t: Pillow's Image.quantization) and its frame's components and sampling factors (what
 * Pillow's get_sampling reads).  The headers up to the first SOS go through the reader's own marker
 * loop and segment parsers, and the frame through its table and geometry checks, with
 * J2P_READ_GRAY and J2P_READ_CMYK: a file the reader refuses in its headers is refused with the
 * reader's message, and nothing after the first SOS is read.  Returns 0, or -1 with the message in
 * err. */
struct j2p_jpeg_keep {
        uint16_t qt[4][64];
        unsigned present;
        unsigned ncomp;             /* 1, 3 or 4 (Adobe CMYK or YCCK) */
        unsigned comp_h[4], comp_v[4];
};
int j2p_jpeg_keep_settings(const void *data, size_t len, struct j2p_jpeg_keep *out, char *err, size_t errlen);

#endif
