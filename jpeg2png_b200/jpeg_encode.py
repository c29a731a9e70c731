"""encode_jpeg: RGB or gray CUDA tensors in, JPEG files (bytes) out, encoded on the device.

The encoder is libj2pjpegenc.so (jpeg2png_b200/jpegenc, DESIGN §7f).  It writes the file that
Pillow writes for the same pixels with `quality` and `subsampling` and no other options (libjpeg's
compressor defaults: JFIF header, IJG quality tables, slow-integer DCT, the Annex K Huffman tables,
one interleaved scan).  With `optimize=True` the encoder is libj2pjpegopt.so (jpeg2png_b200/jpegopt),
which writes Pillow's `optimize=True` file: the same coefficients, coded with Huffman tables built
per image from its own symbol counts.  With `progressive=True` the encoder is libj2pjpegprog.so
(jpeg2png_b200/jpegprog), which writes Pillow's `progressive=True` file: the same coefficients in
libjpeg's ten-scan progression, each scan with tables built from its own symbol counts.
`restart_marker_blocks` and `restart_marker_rows` add restart intervals to any of the three files,
as Pillow's keywords of the same names do (DESIGN §7i).  One-channel tensors are written as
Pillow's one-component ('L') files by the same three libraries, one call per kind (DESIGN §7k), and
with `cmyk=True` four-channel tensors as Pillow's Adobe CMYK files (DESIGN §7r).
`qtables` writes given quantisation tables, per image if need be, as Pillow's keyword of the same
name does, and `keep_settings` reads a file's tables and sampling as Pillow's quality='keep' does
(DESIGN §7n).
Colour conversion, downsampling, DCT,
quantisation, the tables, Huffman coding and byte stuffing all run on the device; only the finished
files cross PCIe.
`encode_host` runs the same steps serially on numpy arrays and gives the same bytes.

The module is not called encode_jpeg.py: importing it would make the package attribute
`encode_jpeg` the module instead of the function.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import os

import numpy as np
import torch

from . import abi
from . import batch_encode as B

JPEGENC_LIB = os.path.join(abi._PKG_DIR, 'jpegenc', 'libj2pjpegenc.so')
JPEGOPT_LIB = os.path.join(abi._PKG_DIR, 'jpegopt', 'libj2pjpegopt.so')
JPEGPROG_LIB = os.path.join(abi._PKG_DIR, 'jpegprog', 'libj2pjpegprog.so')
SAMPLINGS = {'4:4:4': 0, '4:2:2': 1, '4:2:0': 2}
MAX_SIDE = 65535                    # SOF's 16-bit height and width


class Image(C.Structure):
    """struct j2p_jpegenc_image — jpeg2png_b200/jpegenc/jpegenc.h."""
    _fields_ = [('data', C.c_void_p), ('width', C.c_uint32), ('height', C.c_uint32),
                ('row_stride', C.c_int64), ('col_stride', C.c_int64), ('chan_stride', C.c_int64), ('qtables', C.c_uint32)]


class Qtables(C.Structure):
    """struct j2p_jpegenc_qtables — jpeg2png_b200/jpegenc/jpegenc.h."""
    _fields_ = [('table', (C.c_uint16 * 64) * 4), ('ntables', C.c_uint32)]


class Params(C.Structure):
    """struct j2p_jpegenc_params — jpeg2png_b200/jpegenc/jpegenc.h."""
    _fields_ = [('quality', C.c_int), ('sampling', C.c_int), ('restart_marker_blocks', C.c_int), ('restart_marker_rows', C.c_int),
                ('components', C.c_int), ('qtables', C.POINTER(Qtables)), ('nqtables', C.c_uint), ('cmyk', C.c_int)]


class Stats(C.Structure):
    """struct j2p_jpegenc_stats — jpeg2png_b200/jpegenc/jpegenc.h."""
    _fields_ = [('launches', C.c_uint), ('blocks', C.c_uint64)]


def _declare(lib, name='jpegenc'):
    vp, sz = C.c_void_p, C.c_size_t
    imgs, par = C.POINTER(Image), C.POINTER(Params)
    fn = lambda f: getattr(lib, f'j2p_{name}_{f}')  # noqa: E731
    fn('plan').restype = C.c_int
    fn('plan').argtypes = [imgs, C.c_uint, par, C.POINTER(sz), C.POINTER(sz)]
    fn('encode').restype = C.c_int
    fn('encode').argtypes = [imgs, C.c_uint, par, vp, sz, vp, C.POINTER(C.c_uint64), vp, sz, C.POINTER(Stats)]
    fn('encode_host').restype = C.c_int
    fn('encode_host').argtypes = [imgs, C.c_uint, par, vp, sz, C.POINTER(C.c_uint64)]
    fn('last_error').restype = C.c_char_p
    fn('last_error').argtypes = []


def _declare_opt(lib):
    _declare(lib, 'jpegopt')
    u8 = C.POINTER(C.c_uint8)
    lib.j2p_jpegopt_build_table.restype = C.c_int
    lib.j2p_jpegopt_build_table.argtypes = [C.POINTER(C.c_uint64), u8, u8, C.POINTER(C.c_uint)]


def _declare_prog(lib):
    _declare(lib, 'jpegprog')


def load_jpegenc() -> C.CDLL:
    """libj2pjpegenc.so (the device JPEG encoder) from the package tree."""
    return abi.load_library(JPEGENC_LIB, 'JPEG encoder', _declare)


def load_jpegopt() -> C.CDLL:
    """libj2pjpegopt.so (the device JPEG encoder with optimized Huffman tables) from the package tree."""
    return abi.load_library(JPEGOPT_LIB, 'optimizing JPEG encoder', _declare_opt)


def load_jpegprog() -> C.CDLL:
    """libj2pjpegprog.so (the device encoder of progressive JPEG files) from the package tree."""
    return abi.load_library(JPEGPROG_LIB, 'progressive JPEG encoder', _declare_prog)


MAX_RESTART = 65535                 # DRI's 16-bit interval


def _check_restart(name, v):
    """A restart keyword: an integer (not a bool) in 0..65535.  Pillow turns -1 into DRI 65535 and
    writes a value above 65535 as its DRI mod 65536 while counting the full value between markers,
    a corrupt file; both are refused here."""
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not 0 <= v <= MAX_RESTART:
        raise ValueError(f'{name} must be an integer in 0..{MAX_RESTART}, not {v!r}')
    return int(v)


def check_quality(quality, allow_none=False):
    if quality is None and allow_none:
        return
    if isinstance(quality, bool) or not isinstance(quality, (int, np.integer)) or not 1 <= quality <= 100:
        raise ValueError(f'quality must be an integer in 1..100{" or None" if allow_none else ""}, not {quality!r}')


def check_subsampling(subsampling):
    if not isinstance(subsampling, str) or subsampling not in SAMPLINGS:
        raise ValueError(f"subsampling must be '4:4:4', '4:2:2' or '4:2:0', not {subsampling!r}")


def check_cmyk(cmyk):
    if not isinstance(cmyk, bool):
        raise ValueError(f'cmyk must be True or False, not {cmyk!r}')


def params(quality, subsampling, restart_marker_blocks=0, restart_marker_rows=0, components=3, cmyk=False) -> Params:
    """Checked call parameters: quality an integer in 1..100, subsampling '4:4:4', '4:2:2' or '4:2:0',
    the restart keywords integers in 0..65535, components 3 (RGB images, YCbCr files) or 1 (gray
    images, one-component files); cmyk=True (with components 3, the default): CMYK images, Adobe
    CMYK files."""
    check_quality(quality)
    check_subsampling(subsampling)
    blocks = _check_restart('restart_marker_blocks', restart_marker_blocks)
    rows = _check_restart('restart_marker_rows', restart_marker_rows)
    if components not in (1, 3) or isinstance(components, bool):
        raise ValueError(f'components must be 3 or 1, not {components!r}')
    check_cmyk(cmyk)
    if cmyk and components != 3:
        raise ValueError('cmyk=True writes four-component files: it does not combine with gray (components=1)')
    return Params(int(quality), SAMPLINGS[subsampling], blocks, rows, 0 if cmyk else int(components), cmyk=int(cmyk))


def _check_size(shape, h, w):
    if not (1 <= h <= MAX_SIDE and 1 <= w <= MAX_SIDE):
        raise ValueError(f'a JPEG image is 1..{MAX_SIDE} pixels high and wide; got shape {tuple(shape)}')


CODEC = B.Codec('jpegenc', lambda: load_jpegenc(), Image, _check_size)
CODEC_OPT = B.Codec('jpegopt', lambda: load_jpegopt(), Image, _check_size)
CODEC_PROG = B.Codec('jpegprog', lambda: load_jpegprog(), Image, _check_size)


def codec(p: Params, optimize=False, progressive=False, sets=None) -> B.Codec:
    """libj2pjpegenc.so, or libj2pjpegopt.so when optimize, or libj2pjpegprog.so when progressive
    (whatever optimize), for the shared driver, with the call parameters p: it takes one-channel
    images when p is gray (p.components == 1), four-channel ones when p is CMYK (p.cmyk), and
    three-channel ones otherwise.  sets: None (the IJG
    tables of p.quality), or each image's final tables in call order (lists of 64 integers in
    natural order, or None for the IJG tables of p.quality); the distinct ones become the call's
    sets, each stored once."""
    c = CODEC_PROG if progressive else CODEC_OPT if optimize else CODEC
    place = None
    if sets is not None and any(t is not None for t in sets):
        own = [tuple(map(tuple, t if t is not None else scaled_tables(IJG_TABLES, p.quality))) for t in sets]
        distinct = list(dict.fromkeys(own))
        arr = (Qtables * len(distinct))()
        for q, t in zip(arr, distinct):
            q.ntables = len(t)
            for k, row in enumerate(t):
                q.table[k][:] = row
        p.qtables, p.nqtables = arr, len(distinct)
        p.sets_ = arr                   # p, which the codec holds by reference, keeps them alive
        index = [distinct.index(t) for t in own]

        def place(d):
            for x, k in zip(d, index):
                x.qtables = k
    channels = (4,) if p.cmyk else (1,) if p.components == 1 else c.channels
    return dataclasses.replace(c, params=(C.byref(p),), channels=channels, place=place)


# ---- quantisation tables ---------------------------------------------------------------------------
# ITU-T T.81 Annex K.1 (natural order): libjpeg's tables before quality scaling
IJG_TABLES = (
    (16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
     18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100,
     103, 99),
    (17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66) + (99,) * 38)
MAX_ENTRY = 8191                    # 8q must fit libjpeg-turbo's 16-bit divisor


def scaled_tables(tables, quality):
    """Final tables as Pillow makes them from given ones: without quality (None) each entry as
    given, 0 raised to 1 and anything above 32767 lowered to it; with quality q each entry scaled as
    jpeg_quality_scaling(q) scales the IJG tables, (t s + 50) / 100 with s = 5000 / q below 50 and
    200 - 2q otherwise, then clamped to 1..255.  Raises ValueError for a final entry above 8191:
    libjpeg-turbo divides by 8q in 16 bits, so Pillow writes such a file with coefficients that do
    not match the table it declares."""
    if quality is None:
        out = [[min(max(v, 1), 32767) for v in t] for t in tables]
    else:
        s = 5000 // quality if quality < 50 else 200 - 2 * quality
        out = [[min(max((v * s + 50) // 100, 1), 255) for v in t] for t in tables]
    for k, t in enumerate(out):
        if max(t) > MAX_ENTRY:
            raise ValueError(f'quantisation table {k} has an entry of {max(t)} (quality {quality}); entries above {MAX_ENTRY} are refused: '
                             f'libjpeg divides by 8q in 16 bits, so the file would not match its own tables')
    return out


def parse_qtables(value):
    """Pillow's validate_qtables on a list, tuple or dict of 1..4 tables of 64 integers in 0..65535
    (natural order): a list of lists of ints.  A dict keeps [d[k] for k in range(len(d)) if k in d].
    Strings (Pillow's text tables and preset names) are refused."""
    if isinstance(value, str):
        raise ValueError('qtables as text or as a preset name is not supported; give a list, tuple or dict of tables')
    if isinstance(value, dict):
        value = [value[k] for k in range(len(value)) if k in value]
    elif not isinstance(value, (list, tuple, np.ndarray)):
        raise ValueError(f'qtables must be a list, tuple or dict of tables, not {type(value).__name__}')
    if not 1 <= len(value) <= 4:
        raise ValueError(f'qtables holds 1..4 tables, not {len(value)}')
    out = []
    for t in value:
        if isinstance(t, (str, bytes, dict)) or not hasattr(t, '__len__') or len(t) != 64:
            raise ValueError('a quantisation table is a sequence of 64 integers')
        for v in t:
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or not 0 <= v <= 65535:
                raise ValueError(f'quantisation table entries are integers in 0..65535, not {v!r}')
        out.append([int(v) for v in t])
    return out


def _flat(e):
    """Whether e is one table (a flat sequence), rather than an element of a per-image list."""
    return isinstance(e, (list, tuple, np.ndarray)) and not any(v is None or isinstance(v, (list, tuple, dict, np.ndarray)) for v in e)


def per_image(qtables, quality, n):
    """Each of n images' final tables, or None for the IJG tables of quality: qtables is None, one
    tables value for every image, or a list or tuple of n elements, each None or a tables value."""
    if qtables is None:
        return [None] * n
    if isinstance(qtables, (list, tuple)) and qtables and not all(_flat(e) for e in qtables):
        if len(qtables) != n:
            raise ValueError(f'a per-image qtables list has {len(qtables)} elements for {n} images')
        return [None if e is None else scaled_tables(parse_qtables(e), quality) for e in qtables]
    return [scaled_tables(parse_qtables(qtables), quality)] * n


def _subsamplings(subsampling, n):
    """Each of n images' subsampling: one value, or a list or tuple of n."""
    if isinstance(subsampling, (list, tuple)):
        if len(subsampling) != n:
            raise ValueError(f'a per-image subsampling list has {len(subsampling)} elements for {n} images')
        subs = list(subsampling)
    else:
        subs = [subsampling] * n
    for s in subs:
        check_subsampling(s)
    return subs


def _calls(quality, subsampling, optimize, progressive, restart_marker_blocks, restart_marker_rows, qtables, n, channels):
    """calls(items) for the shared driver: one library call per (channel count, subsampling) kind of
    the n images, each with the distinct tables of its images as its sets; channels(x): x's channel
    count, 3 (RGB), 1 (gray) or 4 (CMYK)."""
    check_quality(quality, allow_none=True)
    subs = _subsamplings(subsampling, n)
    sets = per_image(qtables, quality, n)
    blocks = _check_restart('restart_marker_blocks', restart_marker_blocks)
    rows = _check_restart('restart_marker_rows', restart_marker_rows)
    q = 75 if quality is None else int(quality)     # the IJG tables' quality, where an image has no tables

    def calls(items):
        kinds = {}
        for i, x in enumerate(items):
            kinds.setdefault((channels(x), subs[i]), []).append(i)
        return [(codec(params(q, s, blocks, rows, 1 if c == 1 else 3, c == 4), optimize, progressive, [sets[i] for i in idx]), idx)
                for (c, s), idx in kinds.items()]
    return calls


def _codecs(quality, subsampling, optimize, progressive, restart_marker_blocks, restart_marker_rows, cmyk=False):
    """The codec of each channel count encode_jpeg takes: {3: RGB, 1: gray}, and 4: CMYK when cmyk."""
    return {c: codec(params(quality, subsampling, restart_marker_blocks, restart_marker_rows, 1 if c == 1 else 3, c == 4), optimize, progressive)
            for c in ((3, 1, 4) if cmyk else (3, 1))}


def check_optimize(optimize):
    if not isinstance(optimize, bool):
        raise ValueError(f'optimize must be True or False, not {optimize!r}')


def check_progressive(progressive):
    if not isinstance(progressive, bool):
        raise ValueError(f'progressive must be True or False, not {progressive!r}')


def build_table(counts):
    """The optimized table of 256 symbol counts (j2p_jpegopt_build_table): (bits[16], vals), the
    DHT's code counts per length 1..16 and its symbols in order."""
    c = (C.c_uint64 * 256)(*[int(v) for v in counts])
    bits, vals, nv = (C.c_uint8 * 16)(), (C.c_uint8 * 256)(), C.c_uint()
    lib = load_jpegopt()
    if lib.j2p_jpegopt_build_table(c, bits, vals, C.byref(nv)) != 0:
        raise ValueError(lib.j2p_jpegopt_last_error().decode())
    return list(bits), list(vals)[:nv.value]


def _descs(items, layout, ptr, strides):
    """The image structs of items; ptr(x) and strides(x) give x's address and strides in elements."""
    return B.descs(CODEC, items, layout, ptr, strides)


def _work_bytes(descs, p):
    """The work area of one call on descs with the call parameters p."""
    return codec(p).plan(descs)[0]


def encode_host(images, quality=None, subsampling='4:2:0', layout='HWC', optimize=False, progressive=False, restart_marker_blocks=0,
                restart_marker_rows=0, gray=False, qtables=None, cmyk=False):
    """The serial host driver (j2p_jpegenc_encode_host, or j2p_jpegopt_encode_host when optimize,
    or j2p_jpegprog_encode_host when progressive) on numpy uint8 arrays: a list of JPEG files as
    bytes, the same bytes the device writes.  The arrays are RGB, or with gray=True all gray,
    (h, w, 1) or (1, h, w), written as one-component files, or with cmyk=True all CMYK, (h, w, 4)
    or (4, h, w), written as Adobe CMYK files.  quality, subsampling and qtables as encode_jpeg
    takes them (per-image lists included: one call per subsampling)."""
    B.check_layout(layout)
    if not isinstance(gray, bool):
        raise ValueError(f'gray must be True or False, not {gray!r}')
    check_cmyk(cmyk)
    if gray and cmyk:
        raise ValueError('gray=True and cmyk=True are different kinds of file; give one')
    check_optimize(optimize)
    check_progressive(progressive)
    for x in images:
        if x.dtype != np.uint8:
            raise ValueError(f'samples are uint8, not {x.dtype}')
    calls = _calls(quality, subsampling, optimize, progressive, restart_marker_blocks, restart_marker_rows, qtables, len(images),
                   lambda x: 1 if gray else 4 if cmyk else 3)
    out = [None] * len(images)
    for c, idx in calls(images):
        for i, f in zip(idx, B.encode_host(c, [images[i] for i in idx], layout)):
            out[i] = f
    return out


def encode_jpeg(images, *, quality=None, subsampling='4:2:0', layout='CHW', optimize=False, progressive=False, restart_marker_blocks=0,
                restart_marker_rows=0, qtables=None, cmyk=False):
    """Encode RGB, gray or CMYK CUDA tensors as baseline or progressive JPEG files on the device.

    images: one tensor or a list or tuple of them, torch.uint8, shaped (3, h, w) for layout='CHW'
    or (h, w, 3) for 'HWC', with any strides, 1..65535 pixels high and wide.  quality: an integer
    in 1..100, or None (75 without qtables); subsampling: '4:4:4', '4:2:2' or '4:2:0', or a list or
    tuple of them, one per image.  Returns the JPEG file as bytes, or a list of bytes in input
    order: byte for byte the file Pillow writes for the same pixels with `save(f, 'JPEG',
    quality=quality, subsampling=subsampling, optimize=optimize, progressive=progressive,
    restart_marker_blocks=restart_marker_blocks, restart_marker_rows=restart_marker_rows,
    qtables=qtables)` (quality=None being Pillow's default, -1).

    qtables: None (the IJG tables of quality), Pillow's form (a list, tuple or dict of 1..4 tables
    of 64 integers in 0..65535, natural order) for every image, or a list or tuple with one element
    per image, each None (the IJG tables of quality) or such a value, so that files from different
    sources keep their own tables in one call.  As in Pillow, one table serves Y, Cb and Cr, two
    serve Y and then Cb and Cr, and a third serves Cr (a fourth is not used); a gray image uses the
    first.  Without quality the entries are used as given (0 becomes 1); with quality q they are
    scaled as the IJG tables are and clamped to 1..255.  An entry that ends above 8191 is refused
    with ValueError (Pillow writes a corrupt file: libjpeg divides by 8q in 16 bits), as are
    strings (text tables and preset names).  A table with an entry above 255 is written as a 16-bit
    DQT and makes the file SOF1 (extended sequential) unless it is progressive.
    `encode_jpeg(decode_jpeg(files, mode='UNCHANGED'), **keep_settings(files))` re-encodes files
    with their own tables and sampling, as Pillow's quality='keep' does.

    A tensor with one channel, (1, h, w) or (h, w, 1) (what decode_jpeg(mode='UNCHANGED' or
    'GRAY') returns), is written as a one-component file: Pillow's file of the 'L' image, with every
    keyword applied as to a colour image.  subsampling changes no coded byte of a gray file, only
    the sampling factors its SOF declares (2 x 2 for the default '4:2:0', as Pillow writes them).
    Pillow saving an 'L' image without a subsampling keyword declares 1 x 1: that file is
    subsampling='4:4:4' here.
    Gray and RGB images mix in one list; each kind is one library call.

    cmyk: with True, a tensor with four channels, (4, h, w) or (h, w, 4) (what
    decode_jpeg(mode='UNCHANGED') returns for a CMYK file), is written as an Adobe CMYK file:
    Pillow's file of the 'CMYK' image, with every keyword applied.  The samples are stored inverted,
    as Pillow stores them, so Pillow and decode_jpeg read the tensor's values back.  As in Pillow,
    subsampling applies to the first component (C) alone and makes M, Y and K half-resolution
    planes: the default '4:2:0' halves M, Y and K in both directions.  Pillow saving a 'CMYK' image
    without a subsampling keyword samples every component 1 x 1: that file is subsampling='4:4:4'
    here.  Without qtables all four components use table 0; with n tables component c uses table
    min(c, n - 1), so a fourth table is written and used by K.  Gray, RGB and CMYK images mix in
    one list, one library call per kind.  cmyk is explicit because a four-channel tensor is more
    often RGBA, which this would write as a wrong file; without it four-channel tensors are refused.

    optimize: False writes the Annex K Huffman tables; True builds each image's tables from its own
    symbol counts, on the device, as libjpeg does for `optimize=True`: the same coefficients, files
    typically 6-9% smaller, at the cost of two more kernels per call.

    progressive: True writes libjpeg's progressive file (SOF2, its ten-scan script for YCbCr, each
    scan with Huffman tables built from its own symbol counts, as libjpeg always does for a
    progressive file): the same coefficients, shown coarse to fine as the file arrives.  optimize
    changes no byte of a progressive file, as with Pillow.

    restart_marker_blocks, restart_marker_rows: integers in 0..65535 (0, the default: no restart
    markers).  With blocks = b every scan gets a restart interval of b MCUs; with rows = r, which
    overrides b as in libjpeg, a scan gets r times its MCUs per row, capped at 65535 MCUs (in a
    progressive file the AC scans of one component count that component's blocks per row, so the
    interval can change between scans).  Each interval ends padded to a byte and is followed by an
    RST marker, and restarts its DC prediction and EOB run, so a decoder can start at any
    interval and a damaged file loses one interval.  Every interval is its own bit stream on the
    device, so very short intervals (one MCU) cost work area and time.  Unlike Pillow, negative
    values and values above 65535 are refused (Pillow writes -1 as 65535, and a value above
    65535 as a corrupt file).

    The work is queued on torch's current stream, after what is already there, so a tensor just
    written on that stream needs no synchronisation.  Images of any mix of sizes go into one call;
    a list is split into several only when the work area would not fit in a quarter of the free
    device memory.  Raises ValueError for a wrong dtype, shape, layout, quality, subsampling,
    optimize, progressive or cmyk (not a bool), restart keyword or size, and for a tensor that is not on
    a CUDA device, and RuntimeError when no CUDA device is usable.
    """
    B.check_layout(layout)
    check_optimize(optimize)
    check_progressive(progressive)
    check_cmyk(cmyk)
    n = len(images) if isinstance(images, (list, tuple)) else 1
    channels = (3, 1, 4) if cmyk else (3, 1)
    calls = _calls(quality, subsampling, optimize, progressive, restart_marker_blocks, restart_marker_rows, qtables, n,
                   lambda x: x.shape[B.axes(x.shape, layout, channels)[4]])
    codecs = _codecs(75, '4:2:0', optimize, progressive, restart_marker_blocks, restart_marker_rows, cmyk)      # the checks of the images
    return B.encode_tensors('encode_jpeg', codecs, images, layout, (torch.uint8,), calls)


def keep_settings(inputs):
    """The settings Pillow's quality='keep' re-uses for JPEG files: inputs is bytes-like, a path
    (str / os.PathLike), or a list or tuple of them, as decode_jpeg takes them.  For one input,
    {'qtables': {table id: [64 ints, natural order]}, 'subsampling': s}: the quantisation tables
    the file defines before its first scan (Pillow's Image.quantization) and its sampling as
    Pillow's get_sampling reads it, '4:4:4', '4:2:2' or '4:2:0' for those colour layouts and, for
    any other (a gray file, 4:4:0, ...), libjpeg's default that Pillow then writes: '4:2:0' for
    colour, 1 x 1 ('4:4:4' here) for gray.  A four-component file (Adobe CMYK or YCCK) is always
    '4:4:4': Pillow's get_sampling gives -1 for it, which Pillow writes as 1 x 1 for a CMYK image;
    so encode_jpeg(decode_jpeg(files, mode='UNCHANGED'), cmyk=True, **keep_settings(files)) is
    Pillow's quality='keep' re-save of CMYK files.  For a list, the same keys holding lists, which
    encode_jpeg takes per image.  The headers are read by the project's JPEG reader
    (j2p_jpeg_keep_settings): a file it refuses raises ValueError with its message."""
    from . import decode as D
    single = not isinstance(inputs, (list, tuple))
    out = {'qtables': [], 'subsampling': []}
    lib = D.load_codecs()
    for i, x in enumerate([inputs] if single else inputs):
        data, path = D._read_input(x)
        k = D.Keep()
        err = C.create_string_buffer(256)
        if lib.j2p_jpeg_keep_settings(data, len(data), C.byref(k), err, 256) != 0:
            raise ValueError(f'{D._where(i, path)}: {err.value.decode(errors="replace")}')
        out['qtables'].append({t: list(k.qt[t]) for t in range(4) if k.present >> t & 1})
        hv = tuple(v for c in range(k.ncomp) for v in (k.comp_h[c], k.comp_v[c]))
        out['subsampling'].append('4:4:4' if k.ncomp == 4 else {(1, 1, 1, 1, 1, 1): '4:4:4', (2, 1, 1, 1, 1, 1): '4:2:2',
                                                                (2, 2, 1, 1, 1, 1): '4:2:0'}.get(hv, '4:2:0' if k.ncomp == 3 else '4:4:4'))
    return {key: v[0] for key, v in out.items()} if single else out

