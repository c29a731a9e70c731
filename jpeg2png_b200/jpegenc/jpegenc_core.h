// jpegenc_core.h — every step of the JPEG encoder, written once as __host__ __device__ code: the
// kernels of jpegenc.cu and the serial host driver call the same functions, so they write the same
// bytes.  The steps are libjpeg's compressor defaults, which decide the bytes of a baseline file:
//
//   colour     16-bit fixed-point RGB -> YCbCr (SCALEBITS 16, rounding half up for Y, half down
//              for Cb and Cr), on every pixel of the image;
//   chroma     2x1 (4:2:2) or 2x2 (4:2:0) averages with the alternating rounding bias (0,1,0,1 or
//              1,2,1,2 along the output row), computed after the right edge of the full-resolution
//              rows has been replicated out to twice the component's block grid and, for 2x2, the
//              last row repeated to an even count;
//   edges      samples past the component's computed rows repeat its last row, out to the MCU row;
//              samples past its last column repeat that column, out to its block grid;
//   dummies    blocks of the MCU grid past the component's block grid: zero AC, and the DC of the
//              block to their left (right edge) or of the previous block row's last block in the
//              MCU (bottom edge), as libjpeg's coefficient controller fills them;
//   DCT        the slow-integer FDCT (CONST_BITS 13, PASS1_BITS 2), output scaled by 8;
//   quantise   libjpeg-turbo's reciprocal multiply by (q << 3), with its rounding correction;
//   coding     DC predicted along the scan order per component, the Annex K tables, ZRL and EOB,
//              the last byte padded with 1-bits, each 0xFF followed by a stuffed 0x00.
//
// A gray call (j2p_je_tables.nc == 1) is the same steps for one component: libjpeg's null gray
// conversion (the pixel minus 128), luma sampling 1 x 1 whatever the SOF declares, one block per
// MCU, so the MCU grid is the block grid, no dummies, and the DC predicted along the raster.
//
// A CMYK call (nc == 4) is the colour steps for four components with no conversion: a component's
// full-resolution sample is 255 minus the tensor's (the Adobe inversion Pillow writes), M, Y and K
// are downsampled as chroma is, from those inverted samples, and every component codes with the
// luma Huffman tables (j2p_je_htab).
#ifndef J2P_JPEGENC_CORE_H
#define J2P_JPEGENC_CORE_H

#include <stdint.h>

#include "../common/codec_host.h"       // J2P_HD
#include "jpegenc.h"

#define J2P_JE_WORDS_PER_BLOCK 52u      // 32-bit words of J2P_JPEGENC_BLOCK_BITS, rounded up
static_assert(J2P_JE_WORDS_PER_BLOCK * 32 >= J2P_JPEGENC_BLOCK_BITS && (J2P_JE_WORDS_PER_BLOCK - 1) * 32 < J2P_JPEGENC_BLOCK_BITS,
              "J2P_JE_WORDS_PER_BLOCK is J2P_JPEGENC_BLOCK_BITS in words");
// A stream (an image, or one restart interval of it) of nb blocks gets nb x J2P_JE_WORDS_PER_BLOCK
// words, whole bytes, so the 1-bits that pad its coded bits to a byte stay inside them; its RST is
// its 2-byte header, outside them.
static_assert(J2P_JE_WORDS_PER_BLOCK * 32 % 8 == 0, "the padding of a stream's last byte fits its words");
#define J2P_JE_TILE 256u                // blocks per tile of the size and emit kernels (never across images)
#define J2P_JE_CHUNK 8192u              // entropy bytes per chunk of the stuffing kernels
// A header template is SOI, APP0 (APP14 for CMYK), one DQT per used quantisation table (67 bytes
// 8-bit, 131 16-bit), SOF0 or SOF1, the DHTs and SOS; its length is its set's.  The quality tables
// give 2 + 18 + 2 x 67 + 19 + 2 x 33 + 2 x 183 + 14 = 623 bytes for a colour file, 2 + 18 + 67 + 13
// + 33 + 183 + 10 = 328 for a gray one and 2 + 16 + 67 + 22 + 33 + 183 + 16 = 341 for a CMYK one.
// SOI .. the SOF's end is longest in a colour file with three 16-bit DQTs, and in a CMYK file with
// four; the whole header is longest in the colour file, whose two DHT pairs outweigh CMYK's fourth
// DQT:
#define J2P_JE_PRE_MAX (2u + 18u + 3u * 133u + 19u)       // colour: 438
#define J2P_JE_PRE_MAX_CMYK (2u + 16u + 4u * 133u + 22u)  // CMYK: 572
#define J2P_JE_HEAD_MAX (J2P_JE_PRE_MAX + 2u * 33u + 2u * 183u + 14u)                 // 884
#define J2P_JE_HEAD_MAX_CMYK (J2P_JE_PRE_MAX_CMYK + 33u + 183u + 16u)                 // 804
static_assert(J2P_JE_HEAD_MAX_CMYK <= J2P_JE_HEAD_MAX, "a CMYK header fits the template's room");

// per image of a call, or per bit stream (host plan, read by the kernels).  A stream is an image's
// scan, or one restart interval of it; it carries its image's fields, and blk0, nblk, the tiles,
// chunks, words and output of its own blocks.
struct j2p_je_img {
        const uint8_t *src;
        int64_t s_row, s_col, s_chan;   // element strides
        uint32_t w, h;
        uint32_t mcux, mcuy;            // MCU grid
        uint64_t blk0, nblk;            // first block of the call, blocks (MCU grid, scan order)
        uint32_t tile0, ntiles;
        uint32_t chunk0, nchunks;       // stuffing chunks of the worst case
        uint64_t raw_off;               // first word of the image's entropy bits
        uint32_t img;                   // the image (its index in the call)
        uint32_t part;                  // the restart interval in the scan, 0 the first
        uint16_t ri;                    // the scan's restart interval in MCUs, 0 without restarts
        uint8_t scan;                   // the scan of the file (progressive; 0 otherwise)
        uint8_t pad_;
        uint32_t set;                   // the image's set of quantisation tables (its j2p_je_tables)
        // written by the encoder
        uint64_t bits;                  // entropy-coded bits before padding
        uint64_t file_off, file_len;
};
// one 128-byte line per descriptor: the kernels' binary searches over them touch one line a step
static_assert(sizeof(struct j2p_je_img) == 128, "a stream descriptor is one 128-byte line");

// derived Huffman codes of the four tables: DC0, AC0, DC1, AC1 (jpeg_make_c_derived_tbl)
struct j2p_je_huff {
        uint16_t code[4][256];
        uint8_t size[4][256];
};

// per set of quantisation tables of a call (the IJG tables of the call's quality are its one set):
// the reciprocals of each component's table (natural order) and the header template.  The other
// fields, the derived Huffman codes and the geometry, are the call's and the same in every set, so
// the steps that read only them take set 0.
struct j2p_je_tables {
        uint16_t recip[4][64], corr[4][64];             // per component: Y, Cb, Cr, or C, M, Y, K
        uint8_t shift[4][64];           // total right shift of the product
        struct j2p_je_huff huff;        // the Annex K tables
        uint8_t zz[64];                 // zig-zag position of each natural index
        uint32_t hs, vs;                // component 0's sampling factors (the others 1 x 1); 1 x 1 for gray
        uint32_t nc;                    // the call's kind: 3 colour, 1 gray, 4 CMYK
        uint32_t head_len, sof_at;      // the header template's length and the offset of its SOF
        uint8_t head[J2P_JE_HEAD_MAX];
};

// blocks per MCU: component 0's blocks and one of each other component, or a gray file's one block
J2P_HD uint32_t j2p_je_bpm(const struct j2p_je_tables *t) { return t->hs * t->vs + t->nc - 1; }

// the Huffman tables component comp codes with: 0 DC0 / AC0, 1 DC1 / AC1 (a colour file's chroma);
// every component of a CMYK file codes with DC0 / AC0
J2P_HD uint32_t j2p_je_htab(const struct j2p_je_tables *t, uint32_t comp) { return t->nc == 4 ? 0u : comp; }

// the identifier of component comp in the SOF and SOS: 1, 2, 3, or 'C', 'M', 'Y', 'K' in a CMYK file
J2P_HD uint32_t j2p_je_comp_id(const struct j2p_je_tables *t, uint32_t comp) {
        if (t->nc != 4) return comp + 1;
        return comp == 0 ? 'C' : comp == 1 ? 'M' : comp == 2 ? 'Y' : 'K';
}

// the end of the template's SOF (10 + 3 bytes per component) and the length of the SOS that ends it
J2P_HD uint32_t j2p_je_sof_end(const struct j2p_je_tables *t) { return t->sof_at + 10 + 3 * t->nc; }
J2P_HD uint32_t j2p_je_sos_len(const struct j2p_je_tables *t) { return 8 + 2 * t->nc; }


// ---- geometry -------------------------------------------------------------------------------------
// Where block b (scan order) of an image lies: component, its block row and column in the
// component, and the real block whose samples it is coded from (itself, or a dummy's source).
struct j2p_je_where {
        uint32_t comp;
        uint32_t row, col;              // block in the component's MCU-padded grid
        uint32_t srow, scol;            // the real block it takes its samples (or DC) from
        bool dummy;
};

J2P_HD struct j2p_je_where j2p_je_locate(const struct j2p_je_img *im, const struct j2p_je_tables *t, uint64_t b) {
        const uint32_t bpm = j2p_je_bpm(t), nl = t->hs * t->vs;
        const uint64_t mcu = b / bpm;
        const uint32_t k = (uint32_t)(b - mcu * bpm);
        const uint32_t mx = (uint32_t)(mcu % im->mcux), my = (uint32_t)(mcu / im->mcux);
        struct j2p_je_where r;
        uint32_t cw, ch, bx, by, wib, hib;
        if (k < nl) {
                r.comp = 0;
                cw = t->hs, ch = t->vs, bx = k % t->hs, by = k / t->hs;
                wib = (im->w + 7) / 8, hib = (im->h + 7) / 8;
        } else {
                r.comp = 1 + (k - nl);
                cw = ch = 1, bx = by = 0;
                wib = (im->w + 8 * t->hs - 1) / (8 * t->hs), hib = (im->h + 8 * t->vs - 1) / (8 * t->vs);
        }
        r.row = my * ch + by;
        r.col = mx * cw + bx;
        r.dummy = r.row >= hib || r.col >= wib;
        if (r.row >= hib) {             // bottom row of dummies: the previous row's last block of the MCU
                r.srow = hib - 1;
                r.scol = mx * cw + cw - 1 < wib - 1 ? mx * cw + cw - 1 : wib - 1;
        } else {                        // right-edge dummies: the last real block to the left
                r.srow = r.row;
                r.scol = r.col < wib - 1 ? r.col : wib - 1;
        }
        return r;
}

// previous block of the same component in scan order, or ~0 for the image's first
J2P_HD uint64_t j2p_je_prev(const struct j2p_je_tables *t, uint64_t b) {
        const uint32_t bpm = j2p_je_bpm(t), nl = t->hs * t->vs;
        const uint32_t k = (uint32_t)(b % bpm);
        if (k > 0 && k < nl) return b - 1;
        if (b < bpm) return ~(uint64_t)0;
        return k == 0 ? b - bpm + nl - 1 : b - bpm;
}

// ---- samples --------------------------------------------------------------------------------------
J2P_HD int j2p_je_y(int r, int g, int b) { return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16; }
J2P_HD int j2p_je_cb(int r, int g, int b) { return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16; }
J2P_HD int j2p_je_cr(int r, int g, int b) { return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16; }

J2P_HD int j2p_je_conv(int comp, int r, int g, int b) {
        return comp == 0 ? j2p_je_y(r, g, b) : comp == 1 ? j2p_je_cb(r, g, b) : j2p_je_cr(r, g, b);
}

// The sampling steps take the call's kind as K: 4 CMYK, 3 colour or gray (t->nc tells which), 0 read
// from t.  The kernels branch once per block on the kind and run K = 4 or 3, so the colour samples
// are not compiled around the CMYK ones.
template <uint32_t K>
J2P_HD bool j2p_je_is_cmyk(const struct j2p_je_tables *t) { return K == 4 || (K == 0 && t->nc == 4); }

// component comp's full-resolution sample at pixel (y, x) of the image: the colour conversion of the
// RGB pixel, or the inverted CMYK sample (Pillow's raw mode CMYK;I)
template <uint32_t K>
J2P_HD int j2p_je_full(const struct j2p_je_img *im, const struct j2p_je_tables *t, uint32_t comp, uint32_t y, uint32_t x) {
        const uint8_t *p = im->src + (int64_t)y * im->s_row + (int64_t)x * im->s_col;
        if (j2p_je_is_cmyk<K>(t)) return 255 - p[(int64_t)comp * im->s_chan];
        return j2p_je_conv((int)comp, p[0], p[im->s_chan], p[2 * im->s_chan]);
}

// Sample (y, x) of a component, in its block grid, minus 128.
template <uint32_t K = 0>
J2P_HD int j2p_je_sample(const struct j2p_je_img *im, const struct j2p_je_tables *t, uint32_t comp, uint32_t y, uint32_t x) {
        const uint32_t W = im->w - 1, H = im->h - 1;
        if (K != 4 && t->nc == 1)                       // gray: the pixel itself
                return im->src[(int64_t)(y < H ? y : H) * im->s_row + (int64_t)(x < W ? x : W) * im->s_col] - 128;
        if (comp == 0 || t->hs == 1)                    // full size
                return j2p_je_full<K>(im, t, comp, y < H ? y : H, x < W ? x : W) - 128;
        const uint32_t x0 = 2 * x < W ? 2 * x : W, x1 = 2 * x + 1 < W ? 2 * x + 1 : W;
        if (t->vs == 1) {                               // 2x1, bias 0, 1, 0, 1 along the row
                const uint32_t yy = y < H ? y : H;
                const int s = j2p_je_full<K>(im, t, comp, yy, x0) + j2p_je_full<K>(im, t, comp, yy, x1);
                return ((s + (int)(x & 1)) >> 1) - 128;
        }
        const uint32_t ylast = (im->h + 1) / 2 - 1;     // the last computed row; below it repeats
        const uint32_t yc = y < ylast ? y : ylast;
        const uint32_t y0 = 2 * yc, y1 = 2 * yc + 1 < H ? 2 * yc + 1 : H;
        const int s = j2p_je_full<K>(im, t, comp, y0, x0) + j2p_je_full<K>(im, t, comp, y0, x1) + j2p_je_full<K>(im, t, comp, y1, x0) +
                      j2p_je_full<K>(im, t, comp, y1, x1);
        return ((s + 1 + (int)(x & 1)) >> 2) - 128;     // bias 1, 2, 1, 2 along the row
}

// ---- FDCT (islow) ---------------------------------------------------------------------------------
#define J2P_JE_DESCALE(x, n) (((x) + (1 << ((n) - 1))) >> (n))

// One 1-D pass over d[0], d[s], ..., d[7s]: pass 1 (rows) scales up by PASS1_BITS, pass 2
// (columns) removes it.
template <int PASS>
J2P_HD void j2p_je_fdct_1d(int *d) {
        const int CB = 13, P1 = 2;
        const int sh = PASS == 1 ? CB - P1 : CB + P1;
        const int tmp0 = d[0] + d[7], tmp7 = d[0] - d[7];
        const int tmp1 = d[1] + d[6], tmp6 = d[1] - d[6];
        const int tmp2 = d[2] + d[5], tmp5 = d[2] - d[5];
        const int tmp3 = d[3] + d[4], tmp4 = d[3] - d[4];
        const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3;
        const int tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
        if (PASS == 1) {
                d[0] = (tmp10 + tmp11) * (1 << P1);
                d[4] = (tmp10 - tmp11) * (1 << P1);
        } else {
                d[0] = J2P_JE_DESCALE(tmp10 + tmp11, P1);
                d[4] = J2P_JE_DESCALE(tmp10 - tmp11, P1);
        }
        int z1 = (tmp12 + tmp13) * 4433;
        d[2] = J2P_JE_DESCALE(z1 + tmp13 * 6270, sh);
        d[6] = J2P_JE_DESCALE(z1 - tmp12 * 15137, sh);
        z1 = tmp4 + tmp7;
        int z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
        const int z5 = (z3 + z4) * 9633;
        const int t4 = tmp4 * 2446, t5 = tmp5 * 16819, t6 = tmp6 * 25172, t7 = tmp7 * 12299;
        z1 *= -7373;
        z2 *= -20995;
        z3 = z3 * -16069 + z5;
        z4 = z4 * -3196 + z5;
        d[7] = J2P_JE_DESCALE(t4 + z1 + z3, sh);
        d[5] = J2P_JE_DESCALE(t5 + z2 + z4, sh);
        d[3] = J2P_JE_DESCALE(t6 + z2 + z3, sh);
        d[1] = J2P_JE_DESCALE(t7 + z1 + z4, sh);
}

// Row y of a block: its 8 samples through pass 1.
template <uint32_t K = 0>
J2P_HD void j2p_je_block_row(const struct j2p_je_img *im, const struct j2p_je_tables *t, const struct j2p_je_where *w, int y, int *d) {
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
        for (int x = 0; x < 8; x++) d[x] = j2p_je_sample<K>(im, t, w->comp, w->srow * 8 + y, w->scol * 8 + x);
        j2p_je_fdct_1d<1>(d);
}

// libjpeg-turbo's quantisation of coefficient v (|v| < 2^15) of component comp at natural index i.
// (a + corr) < 2^16 and recip < 2^16 for every divisor 8q up to 65528, so the product fits 32 bits.
J2P_HD int j2p_je_quant(const struct j2p_je_tables *t, int comp, int i, int v) {
        const uint32_t a = (uint32_t)(v < 0 ? -v : v);
        const uint32_t q = ((a + t->corr[comp][i]) * (uint32_t)t->recip[comp][i]) >> t->shift[comp][i];
        return v < 0 ? -(int)q : (int)q;
}

// ---- Huffman --------------------------------------------------------------------------------------
J2P_HD int j2p_je_nbits(int v) {
        uint32_t a = (uint32_t)(v < 0 ? -v : v), n = 0;
        while (a) { n++; a >>= 1; }
        return (int)n;
}

// Walks the symbols of a block (zig-zag coefficients c, DC prediction pred) coded with the tables
// comp (j2p_je_htab: 0 DC0 / AC0, else DC1 / AC1): sym(table, symbol) for each Huffman-coded symbol
// (table 0 DC0, 1 AC0, 2 DC1, 3 AC1; the DC category, run << 4 | size, ZRL 0xF0 or EOB 0x00) and
// extra(bits, n) for each run of extra bits, in order.
#ifdef __CUDACC__
#pragma nv_exec_check_disable           // sym / extra are host lambdas in the host driver, device ones in the kernels
#endif
template <typename Sym, typename Extra>
J2P_HD void j2p_je_symbols(const int16_t *c, int pred, uint32_t comp, Sym &&sym, Extra &&extra) {
        const int dc = comp ? 2 : 0, ac = dc + 1;
        int diff = c[0] - pred, nb = j2p_je_nbits(diff);
        sym(dc, nb);
        if (nb) extra((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << nb) - 1), nb);
        int run = 0;
        for (int k = 1; k < 64; k++) {
                const int v = c[k];
                if (v == 0) { run++; continue; }
                while (run > 15) {
                        sym(ac, 0xf0);
                        run -= 16;
                }
                nb = j2p_je_nbits(v);
                sym(ac, (run << 4) + nb);
                extra((uint32_t)(v < 0 ? v - 1 : v) & ((1u << nb) - 1), nb);
                run = 0;
        }
        if (run > 0) sym(ac, 0);
}

// The block's symbols through the tables h: put(code, size) for each Huffman code and each run of
// extra bits, in order.
#ifdef __CUDACC__
#pragma nv_exec_check_disable           // put / orw are host lambdas in the host driver, device ones in the kernels
#endif
template <typename Put>
J2P_HD void j2p_je_walk(const int16_t *c, int pred, const struct j2p_je_huff *h, uint32_t comp, Put &&put) {
        j2p_je_symbols(c, pred, comp, [&](int tbl, int s) { put(h->code[tbl][s], h->size[tbl][s]); }, put);
}

J2P_HD uint32_t j2p_je_block_bits(const int16_t *c, int pred, const struct j2p_je_huff *h, uint32_t comp) {
        uint32_t n = 0;
        j2p_je_walk(c, pred, h, comp, [&](uint32_t, int s) { n += (uint32_t)s; });
        return n;
}

// Writes a block's bits at bit `pos` of a word stream (MSB first; word k holds bytes 4k .. 4k + 3
// with the first byte in the high bits).  orw(word index, bits) merges a word: only the first and
// the last word of a block can be shared with its neighbours.
template <typename Or>
struct j2p_je_writer {
        Or orw;
        uint64_t acc;                   // pending bits, left-aligned, `fill` of them
        uint32_t fill;
        uint64_t word;
#ifdef __CUDACC__
#pragma nv_exec_check_disable           // orw is a host lambda in the host driver, a device one in the kernels
#endif
        J2P_HD void operator()(uint32_t code, int s) {
                acc |= (uint64_t)code << (64 - fill - (uint32_t)s);
                fill += (uint32_t)s;
                if (fill >= 32) {
                        orw(word++, (uint32_t)(acc >> 32));
                        acc <<= 32;
                        fill -= 32;
                }
        }
};

#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <typename Or>
J2P_HD void j2p_je_emit(const int16_t *c, int pred, const struct j2p_je_huff *h, uint32_t comp, uint64_t pos, Or orw) {
        j2p_je_writer<Or> w = {orw, 0, (uint32_t)(pos & 31), pos >> 5};
        j2p_je_walk(c, pred, h, comp, w);
        if (w.fill) w.orw(w.word, (uint32_t)(w.acc >> 32));
}

// byte k of a big-endian word stream
J2P_HD uint8_t j2p_je_byte(const uint32_t *words, uint64_t k) { return (uint8_t)(words[k >> 2] >> (24 - 8 * (k & 3))); }

// 1-bits from `bits` up to the byte boundary: (word, mask) to OR in, mask 0 when none
J2P_HD uint32_t j2p_je_pad(uint64_t bits, uint64_t *word) {
        const uint32_t r = (uint32_t)(bits & 7);
        *word = bits >> 5;
        if (!r) return 0;
        const uint32_t at = (uint32_t)(bits & 31), n = 8 - r;          // n bits from position at
        return (0xffffffffu >> at) & ~(n + at >= 32 ? 0u : 0xffffffffu >> (at + n));
}

// the header with the image's size in its SOF
J2P_HD uint8_t j2p_je_head_byte(const struct j2p_je_tables *t, const struct j2p_je_img *im, uint32_t k) {
        const uint32_t s = t->sof_at;
        if (k == s + 5) return (uint8_t)(im->h >> 8);
        if (k == s + 6) return (uint8_t)im->h;
        if (k == s + 7) return (uint8_t)(im->w >> 8);
        if (k == s + 8) return (uint8_t)im->w;
        return t->head[k];
}

#endif
