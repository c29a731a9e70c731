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
Pillow's one-component ('L') files by the same three libraries, one call per kind (DESIGN §7k).
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
                ('row_stride', C.c_int64), ('col_stride', C.c_int64), ('chan_stride', C.c_int64)]


class Params(C.Structure):
    """struct j2p_jpegenc_params — jpeg2png_b200/jpegenc/jpegenc.h."""
    _fields_ = [('quality', C.c_int), ('sampling', C.c_int), ('restart_marker_blocks', C.c_int), ('restart_marker_rows', C.c_int),
                ('components', C.c_int)]


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


def params(quality, subsampling, restart_marker_blocks=0, restart_marker_rows=0, components=3) -> Params:
    """Checked call parameters: quality an integer in 1..100, subsampling '4:4:4', '4:2:2' or '4:2:0',
    the restart keywords integers in 0..65535, components 3 (RGB images, YCbCr files) or 1 (gray
    images, one-component files)."""
    if isinstance(quality, bool) or not isinstance(quality, (int, np.integer)) or not 1 <= quality <= 100:
        raise ValueError(f'quality must be an integer in 1..100, not {quality!r}')
    if subsampling not in SAMPLINGS:
        raise ValueError(f"subsampling must be '4:4:4', '4:2:2' or '4:2:0', not {subsampling!r}")
    blocks = _check_restart('restart_marker_blocks', restart_marker_blocks)
    rows = _check_restart('restart_marker_rows', restart_marker_rows)
    if components not in (1, 3) or isinstance(components, bool):
        raise ValueError(f'components must be 3 or 1, not {components!r}')
    return Params(int(quality), SAMPLINGS[subsampling], blocks, rows, int(components))


def _check_size(shape, h, w):
    if not (1 <= h <= MAX_SIDE and 1 <= w <= MAX_SIDE):
        raise ValueError(f'a JPEG image is 1..{MAX_SIDE} pixels high and wide; got shape {tuple(shape)}')


CODEC = B.Codec('jpegenc', lambda: load_jpegenc(), Image, _check_size)
CODEC_OPT = B.Codec('jpegopt', lambda: load_jpegopt(), Image, _check_size)
CODEC_PROG = B.Codec('jpegprog', lambda: load_jpegprog(), Image, _check_size)


def codec(p: Params, optimize=False, progressive=False) -> B.Codec:
    """libj2pjpegenc.so, or libj2pjpegopt.so when optimize, or libj2pjpegprog.so when progressive
    (whatever optimize), for the shared driver, with the call parameters p: it takes one-channel
    images when p is gray (p.components == 1), three-channel ones otherwise."""
    c = CODEC_PROG if progressive else CODEC_OPT if optimize else CODEC
    return dataclasses.replace(c, params=(C.byref(p),), channels=(1,) if p.components == 1 else c.channels)


def _codecs(quality, subsampling, optimize, progressive, restart_marker_blocks, restart_marker_rows):
    """The codec of each channel count encode_jpeg takes: {3: RGB, 1: gray}."""
    return {c: codec(params(quality, subsampling, restart_marker_blocks, restart_marker_rows, c), optimize, progressive) for c in (3, 1)}


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


def encode_host(images, quality=75, subsampling='4:2:0', layout='HWC', optimize=False, progressive=False, restart_marker_blocks=0,
                restart_marker_rows=0, gray=False):
    """The serial host driver (j2p_jpegenc_encode_host, or j2p_jpegopt_encode_host when optimize,
    or j2p_jpegprog_encode_host when progressive) on numpy uint8 arrays: a list of JPEG files as
    bytes, the same bytes the device writes.  The arrays are RGB, or with gray=True all gray,
    (h, w, 1) or (1, h, w), written as one-component files."""
    B.check_layout(layout)
    if not isinstance(gray, bool):
        raise ValueError(f'gray must be True or False, not {gray!r}')
    p = params(quality, subsampling, restart_marker_blocks, restart_marker_rows, 1 if gray else 3)
    check_optimize(optimize)
    check_progressive(progressive)
    for x in images:
        if x.dtype != np.uint8:
            raise ValueError(f'samples are uint8, not {x.dtype}')
    return B.encode_host(codec(p, optimize, progressive), images, layout)


def encode_jpeg(images, *, quality=75, subsampling='4:2:0', layout='CHW', optimize=False, progressive=False, restart_marker_blocks=0,
                restart_marker_rows=0):
    """Encode RGB or gray CUDA tensors as baseline or progressive JPEG files on the device.

    images: one tensor or a list or tuple of them, torch.uint8, shaped (3, h, w) for layout='CHW'
    or (h, w, 3) for 'HWC', with any strides, 1..65535 pixels high and wide.  quality: an integer
    in 1..100; subsampling: '4:4:4', '4:2:2' or '4:2:0'.  Returns the JPEG file as bytes, or a list
    of bytes in input order: byte for byte the file Pillow writes for the same pixels with
    `save(f, 'JPEG', quality=quality, subsampling=subsampling, optimize=optimize,
    progressive=progressive, restart_marker_blocks=restart_marker_blocks,
    restart_marker_rows=restart_marker_rows)`.

    A tensor with one channel, (1, h, w) or (h, w, 1) (what decode_jpeg(mode='UNCHANGED' or
    'GRAY') returns), is written as a one-component file: Pillow's file of the 'L' image, with every
    keyword applied as to a colour image.  subsampling changes no coded byte of a gray file, only
    the sampling factors its SOF declares (2 x 2 for the default '4:2:0', as Pillow writes them).
    Pillow saving an 'L' image without a subsampling keyword declares 1 x 1: that file is
    subsampling='4:4:4' here.
    Gray and RGB images mix in one list; each kind is one library call.

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
    optimize or progressive (not a bool), restart keyword or size, and for a tensor that is not on
    a CUDA device, and RuntimeError when no CUDA device is usable.
    """
    B.check_layout(layout)
    codecs = _codecs(quality, subsampling, optimize, progressive, restart_marker_blocks, restart_marker_rows)
    check_optimize(optimize)
    check_progressive(progressive)
    return B.encode_tensors('encode_jpeg', codecs, images, layout, (torch.uint8,))
