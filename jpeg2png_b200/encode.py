"""encode_png: RGB CUDA tensors in, PNG files (bytes) out, encoded on the device.

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

PNG_LIB = os.path.join(abi._PKG_DIR, 'png', 'libj2ppng.so')
PIECE = 65536                       # filtered bytes per piece (J2P_PNG_PIECE)

_DTYPES = {torch.uint8: 1, torch.uint16: 2}
_NP_DTYPES = {np.dtype(np.uint8): 1, np.dtype(np.uint16): 2}


class Image(C.Structure):
    """struct j2p_png_image — jpeg2png_b200/png/png.h."""
    _fields_ = [('data', C.c_void_p), ('width', C.c_uint32), ('height', C.c_uint32), ('sample_bytes', C.c_uint32),
                ('row_stride', C.c_int64), ('col_stride', C.c_int64), ('chan_stride', C.c_int64)]


class Stats(C.Structure):
    """struct j2p_png_stats — jpeg2png_b200/png/png.h."""
    _fields_ = [('launches', C.c_uint), ('pieces', C.c_uint)]


_png = None


def load_png() -> C.CDLL:
    """libj2ppng.so (the device PNG encoder) from the package tree."""
    global _png
    if _png is None:
        if not os.path.exists(PNG_LIB):
            raise RuntimeError(f'{PNG_LIB} is missing: the PNG encoder has not been built '
                               '(run `python -c "import __graft_entry__ as g; g.build()"`)')
        lib = C.CDLL(PNG_LIB, mode=C.RTLD_LOCAL)
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
        _png = lib
    return _png


def _check(rc, error=RuntimeError):
    if rc != 0:
        raise error(load_png().j2p_png_last_error().decode())


def _plan_check(rc):
    """j2p_png_plan refuses only what the arguments make impossible (here, once the shapes and
    dtypes are checked: an image too large for PNG's one IDAT chunk): a ValueError."""
    _check(rc, ValueError)


def _axes(shape, layout):
    """(h, w, row axis, column axis, channel axis) of a (3, h, w) CHW or (h, w, 3) HWC shape."""
    if len(shape) != 3:
        raise ValueError(f'an image is 3-dimensional, (3, h, w) or (h, w, 3); got shape {tuple(shape)}')
    if layout == 'CHW':
        if shape[0] != 3:
            raise ValueError(f"layout 'CHW' wants shape (3, h, w); got {tuple(shape)}")
        return shape[1], shape[2], 1, 2, 0
    if shape[2] != 3:
        raise ValueError(f"layout 'HWC' wants shape (h, w, 3); got {tuple(shape)}")
    return shape[0], shape[1], 0, 1, 2


def _descs(items, layout, sample_bytes, ptr, strides):
    out = (Image * len(items))()
    for d, x in zip(out, items):
        h, w, ra, ca, ka = _axes(x.shape, layout)
        if h == 0 or w == 0:
            raise ValueError(f'an image needs at least one pixel; got shape {tuple(x.shape)}')
        st = strides(x)
        d.data, d.width, d.height, d.sample_bytes = ptr(x), w, h, sample_bytes(x)
        d.row_stride, d.col_stride, d.chan_stride = st[ra], st[ca], st[ka]
    return out


def encode_host(images, layout='HWC'):
    """The serial host driver (j2p_png_encode_host) on numpy uint8 / uint16 arrays: a list of PNG
    files as bytes, the same bytes the device writes."""
    if layout not in ('CHW', 'HWC'):
        raise ValueError(f"layout must be 'CHW' or 'HWC', not {layout!r}")
    for x in images:
        if x.dtype not in _NP_DTYPES:
            raise ValueError(f'samples are uint8 or uint16, not {x.dtype}')
    lib = load_png()
    d = _descs(images, layout, lambda x: _NP_DTYPES[x.dtype], lambda x: x.ctypes.data,
               lambda x: [s // x.itemsize for s in x.strides])
    work_bytes, out_off = C.c_size_t(), C.c_size_t()
    _plan_check(lib.j2p_png_plan(d, len(images), C.byref(work_bytes), C.byref(out_off)))
    work = np.zeros(work_bytes.value, np.uint8)
    offs = (C.c_uint64 * (len(images) + 1))()
    _check(lib.j2p_png_encode_host(d, len(images), work.ctypes.data, work_bytes.value, offs))
    base = out_off.value
    return [work[base + offs[i]:base + offs[i + 1]].tobytes() for i in range(len(images))]


def _work_bytes(descs):
    n, o = C.c_size_t(), C.c_size_t()
    _plan_check(load_png().j2p_png_plan(descs, len(descs), C.byref(n), None))
    return n.value


def _chunks(descs, free_bytes):
    """Split the images, in order, so that each chunk's work area fits in a quarter of the free
    device memory (decode_jpeg's rule); one chunk when everything fits."""
    budget = free_bytes // 4
    if _work_bytes(descs) <= budget:
        return [list(range(len(descs)))]
    chunks, cur, used = [], [], 0
    for i in range(len(descs)):
        one = (Image * 1)(descs[i])
        need = _work_bytes(one)
        if cur and used + need > budget:
            chunks.append(cur)
            cur, used = [], 0
        cur.append(i)
        used += need
    chunks.append(cur)
    return chunks


def encode_png(images, *, layout='CHW'):
    """Encode RGB CUDA tensors as PNG files on the device.

    images: one tensor or a list or tuple of them, torch.uint8 or torch.uint16 (native-endian
    16-bit samples, written as 16-bit PNG), shaped (3, h, w) for layout='CHW' or (h, w, 3) for
    'HWC', with any strides: what decode_jpeg returns.  Returns the PNG file as bytes, or a list of
    bytes in input order.

    The work is queued on torch's current stream, after what is already there, so a tensor just
    written on that stream needs no synchronisation.  Images of any mix of sizes go into one call;
    a list is split into several only when the work areas would not fit in a quarter of the free
    device memory.  Raises ValueError for a wrong dtype, shape or layout, for a tensor that is not
    on a CUDA device, and for an image too large for PNG's chunk limit (the file has one IDAT of at
    most 2^31 - 1 bytes: about 26,700 x 26,700 pixels at 8 bits, 18,900 x 18,900 at 16), and
    RuntimeError when no CUDA device is usable.
    """
    if layout not in ('CHW', 'HWC'):
        raise ValueError(f"layout must be 'CHW' or 'HWC', not {layout!r}")
    single = not isinstance(images, (list, tuple))
    items = [images] if single else list(images)
    for x in items:
        if not isinstance(x, torch.Tensor):
            raise ValueError(f'encode_png takes torch tensors, not {type(x).__name__}')
        if x.dtype not in _DTYPES:
            raise ValueError(f'encode_png takes torch.uint8 or torch.uint16 tensors, not {x.dtype}')
        _axes(x.shape, layout)
        if x.device.type != 'cuda':
            raise ValueError(f'encode_png encodes CUDA tensors; this one is on {x.device}')
    if not torch.cuda.is_available() or torch.cuda.device_count() <= 0:
        raise RuntimeError('encode_png needs a CUDA device: the encoder has no CPU fallback')
    if not items:
        return []
    device = items[0].device
    if any(x.device != device for x in items):
        raise ValueError('all images of one call must be on the same device')
    lib = load_png()
    descs = _descs(items, layout, lambda x: _DTYPES[x.dtype], lambda x: x.data_ptr(), lambda x: x.stride())
    results = [None] * len(items)
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device)
        free = torch.cuda.mem_get_info(device)[0]
        for idx in _chunks(descs, free):
            d = (Image * len(idx))(*[descs[i] for i in idx])
            work_bytes, out_off = C.c_size_t(), C.c_size_t()
            _plan_check(lib.j2p_png_plan(d, len(idx), C.byref(work_bytes), C.byref(out_off)))
            work = torch.empty(work_bytes.value, dtype=torch.uint8, device=device)
            offs = (C.c_uint64 * (len(idx) + 1))()
            _check(lib.j2p_png_encode(d, len(idx), work.data_ptr(), work_bytes.value, stream.cuda_stream, offs, None, 0, None))
            total = offs[len(idx)]
            host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
            host.copy_(work[out_off.value:out_off.value + total])        # synchronous: the files are on the host
            view = host.numpy()
            for k, i in enumerate(idx):
                results[i] = view[offs[k]:offs[k + 1]].tobytes()
            del work
    return results[0] if single else results
