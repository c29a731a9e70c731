"""encode_png: RGB or gray CUDA tensors in, PNG files (bytes) out, encoded on the device.

The encoder is libj2ppng.so (jpeg2png_b200/png, DESIGN §7e): every row gets the PNG filter with
the smallest sum of |residual|, the filtered stream is deflated in pieces of 64 KiB with zlib's
run-length parse, and the checksums are computed on the device.  Only the finished files cross
PCIe.  `encode_host` runs the same steps serially on numpy arrays and gives the same bytes.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import abi
from . import batch_encode as B

PNG_LIB = os.path.join(abi._PKG_DIR, 'png', 'libj2ppng.so')
PIECE = 65536                       # filtered bytes per piece (J2P_PNG_PIECE)

_DTYPES = (torch.uint8, torch.uint16)
_NP_DTYPES = (np.dtype(np.uint8), np.dtype(np.uint16))


class Image(C.Structure):
    """struct j2p_png_image — jpeg2png_b200/png/png.h."""
    _fields_ = [('data', C.c_void_p), ('width', C.c_uint32), ('height', C.c_uint32), ('sample_bytes', C.c_uint32),
                ('row_stride', C.c_int64), ('col_stride', C.c_int64), ('chan_stride', C.c_int64),
                ('channels', C.c_uint32)]


class Stats(C.Structure):
    """struct j2p_png_stats — jpeg2png_b200/png/png.h."""
    _fields_ = [('launches', C.c_uint), ('pieces', C.c_uint)]


def _declare(lib):
    vp, sz = C.c_void_p, C.c_size_t
    imgs = C.POINTER(Image)
    lib.j2p_png_plan.restype = C.c_int
    lib.j2p_png_plan.argtypes = [imgs, C.c_uint, C.POINTER(sz), C.POINTER(sz)]
    lib.j2p_png_encode.restype = C.c_int
    lib.j2p_png_encode.argtypes = [imgs, C.c_uint, vp, sz, vp, C.POINTER(C.c_uint64), vp, sz, C.POINTER(Stats)]
    lib.j2p_png_encode_host.restype = C.c_int
    lib.j2p_png_encode_host.argtypes = [imgs, C.c_uint, vp, sz, C.POINTER(C.c_uint64)]
    lib.j2p_png_last_error.restype = C.c_char_p
    lib.j2p_png_last_error.argtypes = []


def load_png() -> C.CDLL:
    """libj2ppng.so (the device PNG encoder) from the package tree."""
    return abi.load_library(PNG_LIB, 'PNG encoder', _declare)


def _check_size(shape, h, w):
    if h == 0 or w == 0:
        raise ValueError(f'an image needs at least one pixel; got shape {tuple(shape)}')


def _fill(d, x, channels):
    d.sample_bytes = x.itemsize
    d.channels = channels


# j2p_png_plan's refusal of an image too large for one IDAT chunk reaches the caller as a ValueError
CODEC = B.Codec('png', load_png, Image, _check_size, _fill, channels=(3, 1))


def encode_host(images, layout='HWC'):
    """The serial host driver (j2p_png_encode_host) on numpy uint8 / uint16 arrays, RGB or gray
    as encode_png takes them: a list of PNG files as bytes, the same bytes the device writes."""
    B.check_layout(layout)
    for x in images:
        if x.dtype not in _NP_DTYPES:
            raise ValueError(f'samples are uint8 or uint16, not {x.dtype}')
    return B.encode_host(CODEC, images, layout)


def encode_png(images, *, layout='CHW'):
    """Encode RGB or gray CUDA tensors as PNG files on the device.

    images: one tensor or a list or tuple of them, torch.uint8 or torch.uint16 (native-endian
    16-bit samples, written as 16-bit PNG), shaped (3, h, w) for layout='CHW' or (h, w, 3) for
    'HWC', with any strides: what decode_jpeg returns.  A tensor with one channel, (1, h, w) or
    (h, w, 1), is written as a gray PNG (colour type 0); gray and RGB images mix in one call.
    Returns the PNG file as bytes, or a list of bytes in input order.

    The work is queued on torch's current stream, after what is already there, so a tensor just
    written on that stream needs no synchronisation.  Images of any mix of sizes go into one call;
    a list is split into several only when the work areas would not fit in a quarter of the free
    device memory.  Raises ValueError for a wrong dtype, shape or layout, for a tensor that is not
    on a CUDA device, and for an image too large for PNG's chunk limit (the file has one IDAT of at
    most 2^31 - 1 bytes: about 26,700 x 26,700 pixels at 8 bits, 18,900 x 18,900 at 16), and
    RuntimeError when no CUDA device is usable.
    """
    B.check_layout(layout)
    return B.encode_tensors('encode_png', CODEC, images, layout, _DTYPES)
