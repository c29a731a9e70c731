"""encode_jpeg: RGB CUDA tensors in, baseline JPEG files (bytes) out, encoded on the device.

The encoder is libj2pjpegenc.so (jpeg2png_b200/jpegenc, DESIGN §7f).  It writes the file that
Pillow writes for the same pixels with `quality` and `subsampling` and no other options (libjpeg's
compressor defaults: JFIF header, IJG quality tables, slow-integer DCT, the Annex K Huffman tables,
one interleaved scan).  Colour conversion, downsampling, DCT, quantisation, Huffman coding and byte
stuffing all run on the device; only the finished files cross PCIe.  `encode_host` runs the same
steps serially on numpy arrays and gives the same bytes.

The module is not called encode_jpeg.py: importing it would make the package attribute
`encode_jpeg` the module instead of the function.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import abi
from .encode import _axes

JPEGENC_LIB = os.path.join(abi._PKG_DIR, 'jpegenc', 'libj2pjpegenc.so')
SAMPLINGS = {'4:4:4': 0, '4:2:2': 1, '4:2:0': 2}
MAX_SIDE = 65535                    # SOF's 16-bit height and width


class Image(C.Structure):
    """struct j2p_jpegenc_image — jpeg2png_b200/jpegenc/jpegenc.h."""
    _fields_ = [('data', C.c_void_p), ('width', C.c_uint32), ('height', C.c_uint32),
                ('row_stride', C.c_int64), ('col_stride', C.c_int64), ('chan_stride', C.c_int64)]


class Params(C.Structure):
    """struct j2p_jpegenc_params — jpeg2png_b200/jpegenc/jpegenc.h."""
    _fields_ = [('quality', C.c_int), ('sampling', C.c_int)]


class Stats(C.Structure):
    """struct j2p_jpegenc_stats — jpeg2png_b200/jpegenc/jpegenc.h."""
    _fields_ = [('launches', C.c_uint), ('blocks', C.c_uint64)]


_lib = None


def load_jpegenc() -> C.CDLL:
    """libj2pjpegenc.so (the device JPEG encoder) from the package tree."""
    global _lib
    if _lib is None:
        if not os.path.exists(JPEGENC_LIB):
            raise RuntimeError(f'{JPEGENC_LIB} is missing: the JPEG encoder has not been built '
                               '(run `python -c "import __graft_entry__ as g; g.build()"`)')
        lib = C.CDLL(JPEGENC_LIB, mode=C.RTLD_LOCAL)
        vp, sz = C.c_void_p, C.c_size_t
        imgs, par = C.POINTER(Image), C.POINTER(Params)
        lib.j2p_jpegenc_plan.restype = C.c_int
        lib.j2p_jpegenc_plan.argtypes = [imgs, C.c_uint, par, C.POINTER(sz), C.POINTER(sz)]
        lib.j2p_jpegenc_encode.restype = C.c_int
        lib.j2p_jpegenc_encode.argtypes = [imgs, C.c_uint, par, vp, sz, vp, C.POINTER(C.c_uint64), vp, sz, C.POINTER(Stats)]
        lib.j2p_jpegenc_encode_host.restype = C.c_int
        lib.j2p_jpegenc_encode_host.argtypes = [imgs, C.c_uint, par, vp, sz, C.POINTER(C.c_uint64)]
        lib.j2p_jpegenc_last_error.restype = C.c_char_p
        lib.j2p_jpegenc_last_error.argtypes = []
        _lib = lib
    return _lib


def _check(rc, error=RuntimeError):
    if rc != 0:
        raise error(load_jpegenc().j2p_jpegenc_last_error().decode())


def params(quality, subsampling) -> Params:
    """Checked call parameters: quality an integer in 1..100, subsampling '4:4:4', '4:2:2' or '4:2:0'."""
    if isinstance(quality, bool) or not isinstance(quality, (int, np.integer)) or not 1 <= quality <= 100:
        raise ValueError(f'quality must be an integer in 1..100, not {quality!r}')
    if subsampling not in SAMPLINGS:
        raise ValueError(f"subsampling must be '4:4:4', '4:2:2' or '4:2:0', not {subsampling!r}")
    return Params(int(quality), SAMPLINGS[subsampling])


def _descs(items, layout, ptr, strides):
    out = (Image * len(items))()
    for d, x in zip(out, items):
        h, w, ra, ca, ka = _axes(x.shape, layout)
        if not (1 <= h <= MAX_SIDE and 1 <= w <= MAX_SIDE):
            raise ValueError(f'a JPEG image is 1..{MAX_SIDE} pixels high and wide; got shape {tuple(x.shape)}')
        st = strides(x)
        d.data, d.width, d.height = ptr(x), w, h
        d.row_stride, d.col_stride, d.chan_stride = st[ra], st[ca], st[ka]
    return out


def encode_host(images, quality=75, subsampling='4:2:0', layout='HWC'):
    """The serial host driver (j2p_jpegenc_encode_host) on numpy uint8 arrays: a list of JPEG files
    as bytes, the same bytes the device writes."""
    if layout not in ('CHW', 'HWC'):
        raise ValueError(f"layout must be 'CHW' or 'HWC', not {layout!r}")
    p = params(quality, subsampling)
    for x in images:
        if x.dtype != np.uint8:
            raise ValueError(f'samples are uint8, not {x.dtype}')
    lib = load_jpegenc()
    d = _descs(images, layout, lambda x: x.ctypes.data, lambda x: [s // x.itemsize for s in x.strides])
    work_bytes, out_off = C.c_size_t(), C.c_size_t()
    _check(lib.j2p_jpegenc_plan(d, len(images), C.byref(p), C.byref(work_bytes), C.byref(out_off)), ValueError)
    work = np.zeros(work_bytes.value, np.uint8)
    offs = (C.c_uint64 * (len(images) + 1))()
    _check(lib.j2p_jpegenc_encode_host(d, len(images), C.byref(p), work.ctypes.data, work_bytes.value, offs))
    base = out_off.value
    return [work[base + offs[i]:base + offs[i + 1]].tobytes() for i in range(len(images))]


def _work_bytes(descs, p):
    n = C.c_size_t()
    _check(load_jpegenc().j2p_jpegenc_plan(descs, len(descs), C.byref(p), C.byref(n), None), ValueError)
    return n.value


def _chunks(descs, p, free_bytes):
    """Split the images, in order, so that each chunk's work area fits in a quarter of the free
    device memory (encode_png's rule); one chunk when everything fits."""
    budget = free_bytes // 4
    if _work_bytes(descs, p) <= budget:
        return [list(range(len(descs)))]
    chunks, cur, used = [], [], 0
    for i in range(len(descs)):
        need = _work_bytes((Image * 1)(descs[i]), p)
        if cur and used + need > budget:
            chunks.append(cur)
            cur, used = [], 0
        cur.append(i)
        used += need
    chunks.append(cur)
    return chunks


def encode_jpeg(images, *, quality=75, subsampling='4:2:0', layout='CHW'):
    """Encode RGB CUDA tensors as baseline JPEG files on the device.

    images: one tensor or a list or tuple of them, torch.uint8, shaped (3, h, w) for layout='CHW'
    or (h, w, 3) for 'HWC', with any strides, 1..65535 pixels high and wide.  quality: an integer
    in 1..100; subsampling: '4:4:4', '4:2:2' or '4:2:0'.  Returns the JPEG file as bytes, or a list
    of bytes in input order: byte for byte the file Pillow writes for the same pixels with
    `save(f, 'JPEG', quality=quality, subsampling=subsampling)`.

    The work is queued on torch's current stream, after what is already there, so a tensor just
    written on that stream needs no synchronisation.  Images of any mix of sizes go into one call;
    a list is split into several only when the work area would not fit in a quarter of the free
    device memory.  Raises ValueError for a wrong dtype, shape, layout, quality, subsampling or
    size, and for a tensor that is not on a CUDA device, and RuntimeError when no CUDA device is
    usable.
    """
    if layout not in ('CHW', 'HWC'):
        raise ValueError(f"layout must be 'CHW' or 'HWC', not {layout!r}")
    p = params(quality, subsampling)
    single = not isinstance(images, (list, tuple))
    items = [images] if single else list(images)
    for x in items:
        if not isinstance(x, torch.Tensor):
            raise ValueError(f'encode_jpeg takes torch tensors, not {type(x).__name__}')
        if x.dtype != torch.uint8:
            raise ValueError(f'encode_jpeg takes torch.uint8 tensors, not {x.dtype}')
        h, w, *_ = _axes(x.shape, layout)
        if not (1 <= h <= MAX_SIDE and 1 <= w <= MAX_SIDE):
            raise ValueError(f'a JPEG image is 1..{MAX_SIDE} pixels high and wide; got shape {tuple(x.shape)}')
        if x.device.type != 'cuda':
            raise ValueError(f'encode_jpeg encodes CUDA tensors; this one is on {x.device}')
    if not torch.cuda.is_available() or torch.cuda.device_count() <= 0:
        raise RuntimeError('encode_jpeg needs a CUDA device: the encoder has no CPU fallback')
    if not items:
        return []
    device = items[0].device
    if any(x.device != device for x in items):
        raise ValueError('all images of one call must be on the same device')
    lib = load_jpegenc()
    descs = _descs(items, layout, lambda x: x.data_ptr(), lambda x: x.stride())
    results = [None] * len(items)
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device)
        free = torch.cuda.mem_get_info(device)[0]
        for idx in _chunks(descs, p, free):
            d = (Image * len(idx))(*[descs[i] for i in idx])
            work_bytes, out_off = C.c_size_t(), C.c_size_t()
            _check(lib.j2p_jpegenc_plan(d, len(idx), C.byref(p), C.byref(work_bytes), C.byref(out_off)), ValueError)
            work = torch.empty(work_bytes.value, dtype=torch.uint8, device=device)
            offs = (C.c_uint64 * (len(idx) + 1))()
            _check(lib.j2p_jpegenc_encode(d, len(idx), C.byref(p), work.data_ptr(), work_bytes.value, stream.cuda_stream, offs,
                                          None, 0, None))
            total = offs[len(idx)]
            host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
            host.copy_(work[out_off.value:out_off.value + total])        # synchronous: the files are on the host
            view = host.numpy()
            for k, i in enumerate(idx):
                results[i] = view[offs[k]:offs[k + 1]].tobytes()
            del work
    return results[0] if single else results
