// png.cu — libj2ppng.so: the plan of a call, the device encoder (filter, pieces, assembly, copy)
// and the serial host driver of the same steps.  See png.h and png_core.h.
#include <string.h>

#include "../common/codec_host.h"
#include "png_core.h"

extern "C" const char *j2p_png_last_error(void) { return g_err; }

static const uint32_t kSlot = J2P_PNG_SLOT;     // output slot of a piece

struct PieceResult {
    uint32_t len, adler, crc;
    uint32_t shift;                     // x^(8 len) modulo the CRC polynomial: joins crc onto what precedes it
    uint64_t dst;                       // offset of the piece's bytes in its file
};

// ---- plan --------------------------------------------------------------------------------------
// work: [images][piece -> image][crc table][x^(2^k)] [filtered streams] [piece slots]
//       [piece results] [offsets] [files]
struct Layout {
    uint32_t n, npieces;
    uint64_t rows;
    size_t off_imgs, off_pmap, off_tab, off_x2k, off_filt, off_slots, off_res, off_offs, off_out, total;
};

static int make_plan(const struct j2p_png_image *im, unsigned n, Layout *L, struct j2p_png_img *imgs) {
    if (!im) return fail("null argument: images");
    if (n == 0) return fail("no images");
    uint64_t pieces = 0, filt = 0, out = 0, rows = 0;
    for (unsigned i = 0; i < n; i++) {
        const struct j2p_png_image *x = &im[i];
        if (!x->data) return fail("image %u: null data pointer", i);
        if (x->width == 0 || x->height == 0 || x->width > 0x7fffffffu || x->height > 0x7fffffffu)
            return fail("image %u: width and height must be 1 .. 2^31 - 1 (got %u x %u)", i, x->width, x->height);
        if (x->sample_bytes != 1 && x->sample_bytes != 2) return fail("image %u: unknown sample size %u (1 or 2 bytes)", i, x->sample_bytes);
        if (x->channels != 0 && x->channels != 1 && x->channels != 3) return fail("image %u: %u channels (1 or 3)", i, x->channels);
        const uint32_t nc = x->channels == 1 ? 1 : 3;
        const uint64_t len = (uint64_t)x->height * (1 + (uint64_t)x->width * nc * x->sample_bytes);
        const uint64_t np = (len + J2P_PNG_PIECE - 1) / J2P_PNG_PIECE;
        // PNG caps a chunk at 2^31 - 1 bytes and the file has one IDAT: refuse an image whose
        // IDAT could exceed it (every piece at its bound), before anything is sized from it
        const uint64_t idat_bound = 6 + (np - 1) * (uint64_t)j2p_png_piece_bound(J2P_PNG_PIECE) +
                                    j2p_png_piece_bound((uint32_t)(len - (np - 1) * J2P_PNG_PIECE));
        if (len > J2P_PNG_MAX_IDAT || idat_bound > J2P_PNG_MAX_IDAT)
            return fail("image %u: %u x %u at %u bytes per sample is too large for one IDAT chunk (up to %llu bytes, PNG allows %u)", i,
                        x->width, x->height, x->sample_bytes, (unsigned long long)(len > J2P_PNG_MAX_IDAT ? len : idat_bound), J2P_PNG_MAX_IDAT);
        if (imgs) {
            struct j2p_png_img *g = &imgs[i];
            memset(g, 0, sizeof *g);
            g->src = (const uint8_t *)x->data;
            g->s_row = x->row_stride;
            g->s_col = x->col_stride;
            g->s_chan = x->chan_stride;
            g->w = x->width;
            g->h = x->height;
            g->sb = x->sample_bytes;
            g->nc = nc;
            g->piece0 = (uint32_t)pieces;
            g->npieces = (uint32_t)np;
            g->row0 = rows;
            g->filt_off = filt;
            g->filt_len = len;
        }
        pieces += np;
        rows += x->height;
        filt += align16(len);
        out += J2P_PNG_HEAD + J2P_PNG_TAIL - 6 + idat_bound;
    }
    if (j2p_png_piece_bound(J2P_PNG_PIECE) > J2P_PNG_SLOT) return fail("piece slot too small");
    if (pieces >= 0x7fffffffu) return fail("too many pieces for one call (%llu)", (unsigned long long)pieces);
    L->n = n;
    L->npieces = (uint32_t)pieces;
    L->rows = rows;
    size_t o = 0;
    L->off_imgs = o;  o = align16(o + n * sizeof(struct j2p_png_img));
    L->off_pmap = o;  o = align16(o + pieces * sizeof(uint32_t));
    L->off_tab = o;   o = align16(o + 256 * sizeof(uint32_t));
    L->off_x2k = o;   o = align16(o + 32 * sizeof(uint32_t));
    L->off_filt = o;  o = align16(o + filt);
    L->off_slots = o; o = align16(o + pieces * (size_t)kSlot);
    L->off_res = o;   o = align16(o + pieces * sizeof(PieceResult));
    L->off_offs = o;  o = align16(o + (n + 1) * sizeof(uint64_t));
    L->off_out = o;   o = align16(o + out);
    L->total = o;
    return 0;
}

// crc table and x^(2^k) modulo the CRC polynomial
static void crc_tables(uint32_t *tab, uint32_t *x2k) {
    for (uint32_t b = 0; b < 256; b++) {
        uint32_t c = b;
        for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ J2P_PNG_CRC_POLY : c >> 1;
        tab[b] = c;
    }
    uint32_t p = 1u << 30;              // x^1
    for (int k = 0; k < 32; k++) {
        x2k[k] = p;
        p = j2p_png_mulmod(p, p);
    }
}

// the plan region (images, piece map, tables) in host memory
static int fill_plan(const struct j2p_png_image *im, unsigned n, const Layout &L, uint8_t *p) {
    struct j2p_png_img *imgs = (struct j2p_png_img *)(p + L.off_imgs);
    Layout tmp;
    if (make_plan(im, n, &tmp, imgs) != 0) return -1;
    uint32_t *pmap = (uint32_t *)(p + L.off_pmap);
    for (unsigned i = 0; i < n; i++)
        for (uint32_t k = 0; k < imgs[i].npieces; k++) pmap[imgs[i].piece0 + k] = i;
    crc_tables((uint32_t *)(p + L.off_tab), (uint32_t *)(p + L.off_x2k));
    return 0;
}

extern "C" int j2p_png_plan(const struct j2p_png_image *images, unsigned n, size_t *work_bytes, size_t *out_offset) {
    Layout L;
    if (make_plan(images, n, &L, nullptr) != 0) return -1;
    if (work_bytes) *work_bytes = L.total;
    if (out_offset) *out_offset = L.off_out;
    return 0;
}

// CRC of "IDAT" and the zlib header, the start of every IDAT checksum
static uint32_t idat_crc0(const uint32_t *tab) {
    const uint8_t b[6] = {'I', 'D', 'A', 'T', 0x78, 0x01};
    return j2p_png_crc(0, b, 6, tab);
}

J2P_HD uint32_t piece_len(const struct j2p_png_img *im, uint32_t k) {
    const uint64_t off = (uint64_t)k * J2P_PNG_PIECE;
    return (uint32_t)(im->filt_len - off < J2P_PNG_PIECE ? im->filt_len - off : J2P_PNG_PIECE);
}

// Per image: where each piece goes in the file, the combined checksums, the file length.
J2P_HD void assemble_image(struct j2p_png_img *im, PieceResult *res, uint32_t crc0, const uint32_t *tab) {
    uint64_t total = 0;
    uint32_t a = 1, c = crc0;
    for (uint32_t k = 0; k < im->npieces; k++) {
        PieceResult *r = &res[im->piece0 + k];
        r->dst = J2P_PNG_HEAD + total;
        a = j2p_png_adler_join(a, r->adler, piece_len(im, k));
        c = j2p_png_crc_join(c, r->crc, r->shift);
        total += r->len;
    }
    im->adler = a;
    c = ~c;
    for (int s = 24; s >= 0; s -= 8) c = tab[(c ^ (a >> s)) & 0xff] ^ (c >> 8);
    im->crc = ~c;
    im->file_len = J2P_PNG_HEAD + total + J2P_PNG_TAIL;
}

J2P_HD void write_frame(uint8_t *out, const struct j2p_png_img *im, const uint32_t *tab) {
    uint8_t *o = out + im->file_off;
    j2p_png_head(o, im, (uint32_t)(im->file_len - J2P_PNG_HEAD - J2P_PNG_TAIL + 6), tab);
    j2p_png_tail(o + im->file_len - J2P_PNG_TAIL, im->adler, im->crc);
}

// ---- host driver -------------------------------------------------------------------------------
template <uint32_t NC> static void filter_host_nc(const struct j2p_png_img *im, uint8_t *filt) {
    const uint64_t rb = j2p_png_row_bytes<NC>(im);
    for (uint32_t y = 0; y < im->h; y++) {
        uint64_t sum[5] = {0, 0, 0, 0, 0};
        for (uint64_t i = 0; i < rb; i++) j2p_png_filter_sums<NC>(im, y, (int64_t)i, sum);
        const int t = j2p_png_pick(sum);
        uint8_t *o = filt + im->filt_off + (uint64_t)y * (rb + 1);
        o[0] = (uint8_t)t;
        for (uint64_t i = 0; i < rb; i++) o[1 + i] = j2p_png_filtered<NC>(im, t, y, (int64_t)i);
    }
}

static void filter_host(const struct j2p_png_img *im, uint8_t *filt) {
    if (im->nc == 1) filter_host_nc<1>(im, filt);
    else filter_host_nc<3>(im, filt);
}

static void piece_host(const uint8_t *src, uint32_t n, bool last, uint32_t *out, const uint32_t *tab, const uint32_t *x2k, PieceResult *res,
                       uint32_t (*hist)[288], struct j2p_png_block *blk, struct j2p_png_scratch *sc) {
    memset(out, 0, kSlot);
    memset(hist, 0, J2P_PNG_MAX_BLOCKS * 288 * sizeof(uint32_t));
    uint32_t nsym = 0;
    j2p_png_walk(src, 0, n, 0, n, [&](uint32_t pos, uint32_t sym) {
        const uint32_t b = nsym / J2P_PNG_BLOCK_SYMS;
        uint32_t eb, ev;
        hist[b][sym < 256 ? sym : j2p_png_len_code(sym - 256, &eb, &ev)]++;
        if (nsym % J2P_PNG_BLOCK_SYMS == 0) blk[b].byte0 = pos;
        nsym++;
    });
    const uint32_t nb = (nsym + J2P_PNG_BLOCK_SYMS - 1) / J2P_PNG_BLOCK_SYMS;
    for (uint32_t b = 0; b < nb; b++) {
        blk[b].byte1 = b + 1 < nb ? blk[b + 1].byte0 : n;
        hist[b][256] = 1;
        memset(blk[b].len, 0, sizeof blk[b].len);
        uint32_t m = 0;
        for (uint32_t s = 0; s < J2P_PNG_NLIT; s++)
            if (hist[b][s]) {
                const uint32_t k = j2p_png_key(hist[b][s], s);
                uint32_t j = m++;
                while (j > 0 && sc->key[j - 1] > k) { sc->key[j] = sc->key[j - 1]; j--; }
                sc->key[j] = k;
            }
        j2p_png_lengths(sc->key, m, 15, sc, blk[b].len);
        j2p_png_choose(&blk[b], hist[b], sc);
    }
    const uint32_t nbytes = j2p_png_layout(blk, nb, last);
    for (uint32_t b = 0; b < nb; b++) j2p_png_put_block_frame(out, &blk[b], last && b + 1 == nb);
    if (!last) j2p_png_put_flush(out, nbytes);
    uint32_t isym = 0, pos = 0;
    j2p_png_walk(src, 0, n, 0, n, [&](uint32_t, uint32_t sym) {
        const uint32_t b = isym / J2P_PNG_BLOCK_SYMS;
        if (isym % J2P_PNG_BLOCK_SYMS == 0) pos = blk[b].data_bit0;
        isym++;
        if (blk[b].type == J2P_BT_STORED) return;
        j2p_png_put_sym(out, pos, &blk[b], sym);
        pos += j2p_png_sym_bits(&blk[b], sym);
    });
    uint8_t *ob = (uint8_t *)out;
    for (uint32_t b = 0; b < nb; b++)
        if (blk[b].type == J2P_BT_STORED)
            for (uint32_t j = 0; j < blk[b].byte1 - blk[b].byte0; j++) ob[j2p_png_stored_at(&blk[b], j)] = src[blk[b].byte0 + j];
    res->len = nbytes;
    res->adler = j2p_png_adler(1, src, n);
    res->crc = j2p_png_crc(0, ob, nbytes, tab);
    res->shift = j2p_png_shift(nbytes, x2k);
}

extern "C" int j2p_png_encode_host(const struct j2p_png_image *images, unsigned n, void *work, size_t work_bytes, uint64_t *offsets) {
    Layout L;
    if (make_plan(images, n, &L, nullptr) != 0) return -1;
    if (!work || !offsets) return fail("null argument");
    if (work_bytes < L.total) return fail("work area of %zu bytes is smaller than the plan's %zu", work_bytes, L.total);
    uint8_t *w = (uint8_t *)work;
    if (fill_plan(images, n, L, w) != 0) return -1;
    struct j2p_png_img *imgs = (struct j2p_png_img *)(w + L.off_imgs);
    const uint32_t *tab = (const uint32_t *)(w + L.off_tab), *x2k = (const uint32_t *)(w + L.off_x2k);
    uint8_t *filt = w + L.off_filt, *out = w + L.off_out;
    PieceResult *res = (PieceResult *)(w + L.off_res);
    uint32_t(*hist)[288] = (uint32_t(*)[288])malloc(J2P_PNG_MAX_BLOCKS * 288 * sizeof(uint32_t));
    struct j2p_png_block *blk = (struct j2p_png_block *)malloc(J2P_PNG_MAX_BLOCKS * sizeof(struct j2p_png_block));
    struct j2p_png_scratch *sc = (struct j2p_png_scratch *)malloc(sizeof(struct j2p_png_scratch));
    if (!hist || !blk || !sc) {
        free(hist); free(blk); free(sc);
        return fail("out of host memory");
    }
    for (unsigned i = 0; i < n; i++) {
        filter_host(&imgs[i], filt);
        for (uint32_t k = 0; k < imgs[i].npieces; k++) {
            const uint32_t p = imgs[i].piece0 + k;
            piece_host(filt + imgs[i].filt_off + (uint64_t)k * J2P_PNG_PIECE, piece_len(&imgs[i], k), k + 1 == imgs[i].npieces,
                       (uint32_t *)(w + L.off_slots + (size_t)p * kSlot), tab, x2k, &res[p], hist, blk, sc);
        }
    }
    free(hist); free(blk); free(sc);
    const uint32_t crc0 = idat_crc0(tab);
    uint64_t off = 0;
    for (unsigned i = 0; i < n; i++) {
        assemble_image(&imgs[i], res, crc0, tab);
        imgs[i].file_off = off;
        offsets[i] = off;
        off += imgs[i].file_len;
    }
    offsets[n] = off;
    for (unsigned i = 0; i < n; i++) {
        write_frame(out, &imgs[i], tab);
        for (uint32_t k = 0; k < imgs[i].npieces; k++) {
            const uint32_t p = imgs[i].piece0 + k;
            memcpy(out + imgs[i].file_off + res[p].dst, w + L.off_slots + (size_t)p * kSlot, res[p].len);
        }
    }
    return 0;
}

// ---- device ------------------------------------------------------------------------------------
static const int kFilterThreads = 256;      // a warp per row
static const int kPieceThreads = 256;       // a CTA per piece
static const int kAsmThreads = 256;
static const int kCopyThreads = 256;

__device__ __forceinline__ uint32_t find_image(const struct j2p_png_img *imgs, uint32_t n, uint64_t row) {
    uint32_t lo = 0, hi = n - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) / 2;
        if (imgs[mid].row0 <= row) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// one row on one warp; NC: the image's channel count (im.nc), the same for the whole warp
template <uint32_t NC> __device__ __forceinline__ void filter_row(const struct j2p_png_img &im, int64_t y, uint32_t lane, uint8_t *__restrict__ filt) {
    const uint64_t rb = j2p_png_row_bytes<NC>(&im);
    uint64_t sum[5] = {0, 0, 0, 0, 0};
    for (uint64_t i = lane; i < rb; i += 32) j2p_png_filter_sums<NC>(&im, y, (int64_t)i, sum);
#pragma unroll
    for (int t = 0; t < 5; t++)
#pragma unroll
        for (int d = 16; d; d >>= 1) sum[t] += __shfl_xor_sync(0xffffffffu, sum[t], d);
    const int t = j2p_png_pick(sum);
    uint8_t *o = filt + im.filt_off + (uint64_t)y * (rb + 1);
    if (lane == 0) o[0] = (uint8_t)t;
    for (uint64_t i = lane; i < rb; i += 32) o[1 + i] = j2p_png_filtered<NC>(&im, t, y, (int64_t)i);
}

__global__ void __launch_bounds__(kFilterThreads) k_png_filter(const struct j2p_png_img *__restrict__ imgs, uint32_t n, uint64_t rows,
                                                              uint8_t *__restrict__ filt) {
    const uint64_t row = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (row >= rows) return;
    const struct j2p_png_img im = imgs[find_image(imgs, n, row)];
    const int64_t y = (int64_t)(row - im.row0);
    if (im.nc == 1) filter_row<1>(im, y, lane, filt);
    else filter_row<3>(im, y, lane, filt);
}

struct PieceShared {
    uint32_t hist[J2P_PNG_MAX_BLOCKS][288];
    struct j2p_png_block blk[J2P_PNG_MAX_BLOCKS];
    struct j2p_png_scratch sc[J2P_PNG_MAX_BLOCKS];
    uint32_t tab[256];
    int32_t sa[kPieceThreads];
    uint32_t sb[kPieceThreads], sc32[kPieceThreads];
    uint32_t pre[J2P_PNG_MAX_BLOCKS];
    uint32_t nsym, nbytes;
    uint32_t out[kSlot / 4];
};

// inclusive scans over the CTA (Hillis-Steele in shared memory)
__device__ int32_t scan_max(int32_t *s, int32_t v) {
    const int t = threadIdx.x;
    s[t] = v;
    __syncthreads();
    for (int d = 1; d < kPieceThreads; d <<= 1) {
        const int32_t x = t >= d ? s[t - d] : -1;
        __syncthreads();
        if (x > s[t]) s[t] = x;
        __syncthreads();
    }
    return s[t];
}

__device__ uint32_t scan_min_rev(uint32_t *s, uint32_t v, uint32_t none) {
    const int t = threadIdx.x;
    s[t] = v;
    __syncthreads();
    for (int d = 1; d < kPieceThreads; d <<= 1) {
        const uint32_t x = t + d < kPieceThreads ? s[t + d] : none;
        __syncthreads();
        if (x < s[t]) s[t] = x;
        __syncthreads();
    }
    return s[t];
}

__device__ uint32_t scan_add(uint32_t *s, uint32_t v, uint32_t *total) {
    const int t = threadIdx.x;
    s[t] = v;
    __syncthreads();
    for (int d = 1; d < kPieceThreads; d <<= 1) {
        const uint32_t x = t >= d ? s[t - d] : 0;
        __syncthreads();
        s[t] += x;
        __syncthreads();
    }
    const uint32_t r = s[t];
    *total = s[kPieceThreads - 1];
    __syncthreads();
    return r - v;                           // exclusive
}

__global__ void __launch_bounds__(kPieceThreads) k_png_piece(const struct j2p_png_img *__restrict__ imgs, const uint32_t *__restrict__ pmap,
                                                            const uint32_t *__restrict__ tab_g, const uint32_t *__restrict__ x2k,
                                                            const uint8_t *__restrict__ filt, uint8_t *__restrict__ slots,
                                                            PieceResult *__restrict__ res) {
    extern __shared__ __align__(16) uint8_t smem[];
    PieceShared &S = *(PieceShared *)smem;
    const uint32_t t = threadIdx.x, p = blockIdx.x;
    const struct j2p_png_img *im = &imgs[pmap[p]];
    const uint32_t k = p - im->piece0, n = piece_len(im, k);
    const bool last = k + 1 == im->npieces;
    const uint8_t *src = filt + im->filt_off + (uint64_t)k * J2P_PNG_PIECE;
    for (uint32_t j = t; j < 256; j += kPieceThreads) S.tab[j] = tab_g[j];
    for (uint32_t j = t; j < kSlot / 4; j += kPieceThreads) S.out[j] = 0;
    for (uint32_t j = t; j < J2P_PNG_MAX_BLOCKS * 288; j += kPieceThreads) (&S.hist[0][0])[j] = 0;

    // this thread's bytes, and the runs that reach into them from either side
    const uint32_t C = (n + kPieceThreads - 1) / kPieceThreads;
    const uint32_t i0 = t * C < n ? t * C : n, i1 = i0 + C < n ? i0 + C : n;
    int32_t lb = -1;
    uint32_t fb = n;
    for (uint32_t j = i0; j < i1; j++)
        if (j == 0 || src[j] != src[j - 1]) {
            if (fb == n) fb = j;
            lb = (int32_t)j;
        }
    scan_max(S.sa, lb);                     // S.sa: inclusive maxima, S.sb: inclusive minima from the right
    scan_min_rev(S.sb, fb, n);
    const uint32_t r0 = fb == i0 ? i0 : (uint32_t)(t > 0 ? S.sa[t - 1] : 0);
    const uint32_t e1 = t + 1 < kPieceThreads ? S.sb[t + 1] : n;
    __syncthreads();

    // symbols: count, then histograms per block
    uint32_t cnt = 0;
    if (i0 < i1) j2p_png_walk(src, i0, i1, r0, e1, [&](uint32_t, uint32_t) { cnt++; });
    uint32_t nsym;
    const uint32_t sym0 = scan_add(S.sc32, cnt, &nsym);
    {
        uint32_t q = sym0;
        if (i0 < i1)
            j2p_png_walk(src, i0, i1, r0, e1, [&](uint32_t pos, uint32_t sym) {
                const uint32_t b = q / J2P_PNG_BLOCK_SYMS;
                uint32_t eb, ev;
                atomicAdd(&S.hist[b][sym < 256 ? sym : j2p_png_len_code(sym - 256, &eb, &ev)], 1u);
                if (q % J2P_PNG_BLOCK_SYMS == 0) S.blk[b].byte0 = pos;
                q++;
            });
    }
    __syncthreads();
    const uint32_t nb = (nsym + J2P_PNG_BLOCK_SYMS - 1) / J2P_PNG_BLOCK_SYMS;

    // codes: warp b builds block b's
    const uint32_t warp = t >> 5, lane = t & 31;
    if (warp < nb) {
        struct j2p_png_block *b = &S.blk[warp];
        struct j2p_png_scratch *sc = &S.sc[warp];
        uint32_t *h = S.hist[warp];
        if (lane == 0) {
            b->byte1 = warp + 1 < nb ? S.blk[warp + 1].byte0 : n;
            h[256] = 1;
        }
        for (uint32_t s = lane; s < 288; s += 32) b->len[s] = 0;
        __syncwarp();
        uint32_t m = 0;
        for (uint32_t s0 = 0; s0 < J2P_PNG_NLIT; s0 += 32) m += __popc(__ballot_sync(0xffffffffu, s0 + lane < J2P_PNG_NLIT && h[s0 + lane]));
        for (uint32_t s = lane; s < J2P_PNG_NLIT; s += 32) {
            if (!h[s]) continue;
            const uint32_t key = j2p_png_key(h[s], s);
            uint32_t rank = 0;
            for (uint32_t u = 0; u < J2P_PNG_NLIT; u++) rank += h[u] && j2p_png_key(h[u], u) < key;
            sc->key[rank] = key;
        }
        __syncwarp();
        if (lane == 0) {
            j2p_png_lengths(sc->key, m, 15, sc, b->len);
            j2p_png_choose(b, h, sc);
        }
    }
    __syncthreads();
    if (t == 0) {
        S.nbytes = j2p_png_layout(S.blk, nb, last);
        uint32_t pre = 0;
        for (uint32_t b = 0; b < nb; b++) {
            S.pre[b] = pre;
            if (S.blk[b].type != J2P_BT_STORED) pre += S.blk[b].data_bits;
        }
        if (!last) j2p_png_put_flush(S.out, S.nbytes);
    }
    __syncthreads();
    if (warp < nb && lane == 0) j2p_png_put_block_frame(S.out, &S.blk[warp], last && warp + 1 == nb);

    // symbol bits: where this thread's first symbol goes, then the symbols
    uint32_t bits = 0;
    {
        uint32_t q = sym0;
        if (i0 < i1)
            j2p_png_walk(src, i0, i1, r0, e1, [&](uint32_t, uint32_t sym) {
                const struct j2p_png_block *b = &S.blk[q++ / J2P_PNG_BLOCK_SYMS];
                if (b->type != J2P_BT_STORED) bits += j2p_png_sym_bits(b, sym);
            });
    }
    uint32_t total_bits;
    uint32_t at = scan_add(S.sc32, bits, &total_bits);
    {
        uint32_t q = sym0;
        if (i0 < i1)
            j2p_png_walk(src, i0, i1, r0, e1, [&](uint32_t, uint32_t sym) {
                const uint32_t bi = q++ / J2P_PNG_BLOCK_SYMS;
                const struct j2p_png_block *b = &S.blk[bi];
                if (b->type == J2P_BT_STORED) return;
                j2p_png_put_sym(S.out, b->data_bit0 + at - S.pre[bi], b, sym);
                at += j2p_png_sym_bits(b, sym);
            });
    }
    __syncthreads();
    uint8_t *ob = (uint8_t *)S.out;
    for (uint32_t b = 0; b < nb; b++)
        if (S.blk[b].type == J2P_BT_STORED)
            for (uint32_t j = t; j < S.blk[b].byte1 - S.blk[b].byte0; j += kPieceThreads) ob[j2p_png_stored_at(&S.blk[b], j)] = src[S.blk[b].byte0 + j];
    __syncthreads();

    // checksums: per thread, then joined by thread 0
    const uint32_t nbytes = S.nbytes, Co = (nbytes + kPieceThreads - 1) / kPieceThreads;
    const uint32_t o0 = t * Co < nbytes ? t * Co : nbytes, o1 = o0 + Co < nbytes ? o0 + Co : nbytes;
    const uint32_t ad = j2p_png_adler(1, src + i0, i1 - i0), cr = j2p_png_crc(0, ob + o0, o1 - o0, S.tab);
    S.sb[t] = ad;
    S.sc32[t] = cr;
    __syncthreads();
    if (t == 0) {
        uint32_t a = 1, c = 0;
        const uint32_t op = j2p_png_shift(Co, x2k);
        for (uint32_t u = 0; u < kPieceThreads; u++) {
            const uint32_t ui0 = u * C < n ? u * C : n, ui1 = ui0 + C < n ? ui0 + C : n;
            a = j2p_png_adler_join(a, S.sb[u], ui1 - ui0);
            const uint32_t u0 = u * Co < nbytes ? u * Co : nbytes, u1 = u0 + Co < nbytes ? u0 + Co : nbytes;
            if (u1 > u0) c = j2p_png_crc_join(c, S.sc32[u], u1 - u0 == Co ? op : j2p_png_shift(u1 - u0, x2k));
        }
        PieceResult r = {nbytes, a, c, j2p_png_shift(nbytes, x2k), 0};
        res[p] = r;
    }
    uint32_t *slot = (uint32_t *)(slots + (size_t)p * kSlot);
    for (uint32_t j = t; j < (nbytes + 3) / 4; j += kPieceThreads) slot[j] = S.out[j];
}

// one CTA: per image the piece offsets, checksums and file length; the file offsets; the frames
__global__ void __launch_bounds__(kAsmThreads) k_png_assemble(struct j2p_png_img *__restrict__ imgs, uint32_t n, PieceResult *__restrict__ res,
                                                             const uint32_t *__restrict__ tab, uint32_t crc0, uint64_t *__restrict__ offsets, uint8_t *__restrict__ out) {
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) assemble_image(&imgs[i], res, crc0, tab);
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t off = 0;
        for (uint32_t i = 0; i < n; i++) {
            imgs[i].file_off = off;
            offsets[i] = off;
            off += imgs[i].file_len;
        }
        offsets[n] = off;
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) write_frame(out, &imgs[i], tab);
}

__global__ void __launch_bounds__(kCopyThreads) k_png_copy(const struct j2p_png_img *__restrict__ imgs, const uint32_t *__restrict__ pmap,
                                                          const uint8_t *__restrict__ slots, const PieceResult *__restrict__ res,
                                                          uint8_t *__restrict__ out) {
    const uint32_t p = blockIdx.x;
    const PieceResult r = res[p];
    uint8_t *dst = out + imgs[pmap[p]].file_off + r.dst;
    const uint8_t *src = slots + (size_t)p * kSlot;
    for (uint32_t j = threadIdx.x; j < r.len; j += kCopyThreads) dst[j] = src[j];
}

extern "C" int j2p_png_encode(const struct j2p_png_image *images, unsigned n, void *work, size_t work_bytes, void *stream, uint64_t *offsets,
                              void *dst, size_t dst_cap, struct j2p_png_stats *stats) {
    Layout L;
    if (make_plan(images, n, &L, nullptr) != 0) return -1;
    const auto fill = [&](uint8_t *plan) { return fill_plan(images, n, L, plan); };
    const auto launch = [&](uint8_t *w, cudaStream_t st, const uint8_t *plan, auto counted) {
        struct j2p_png_img *imgs = (struct j2p_png_img *)(w + L.off_imgs);
        const uint32_t *pmap = (const uint32_t *)(w + L.off_pmap), *tab = (const uint32_t *)(w + L.off_tab), *x2k = (const uint32_t *)(w + L.off_x2k);
        PieceResult *res = (PieceResult *)(w + L.off_res);
        static const size_t smem = sizeof(PieceShared);
        const cudaError_t ea = cudaFuncSetAttribute(k_png_piece, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (ea != cudaSuccess) return fail("k_png_piece shared memory: %s", cudaGetErrorString(ea));
        const uint64_t fgrid = (L.rows * 32 + kFilterThreads - 1) / kFilterThreads;
        k_png_filter<<<(unsigned)fgrid, kFilterThreads, 0, st>>>(imgs, n, L.rows, w + L.off_filt);
        counted();
        k_png_piece<<<L.npieces, kPieceThreads, smem, st>>>(imgs, pmap, tab, x2k, w + L.off_filt, w + L.off_slots, res);
        counted();
        k_png_assemble<<<1, kAsmThreads, 0, st>>>(imgs, n, res, tab, idat_crc0((const uint32_t *)(plan + L.off_tab)), (uint64_t *)(w + L.off_offs),
                                                  w + L.off_out);
        counted();
        k_png_copy<<<L.npieces, kCopyThreads, 0, st>>>(imgs, pmap, w + L.off_slots, res, w + L.off_out);
        counted();
        return 0;
    };
    if (encode_call(images, n, L, L.off_filt, work, work_bytes, stream, offsets, dst, dst_cap, stats, fill, launch) != 0) return -1;
    if (stats) stats->pieces = L.npieces;
    return 0;
}
