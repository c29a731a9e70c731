"""ctypes view of the C ABI in include/jpeg2png_b200.h (and of the reference's identical types).

This is the host-side mirror used by tests and bench.py: it builds `struct coef` arrays exactly as
the reference's decode_file does (jpeg2png.c:120-139) and hands them to a `compute()` with the
reference signature — the product's, the compiled reference's, or the oracle's.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .synth import CoefImage

_libc = C.CDLL(None)
_libc.aligned_alloc.restype = C.c_void_p
_libc.aligned_alloc.argtypes = [C.c_size_t, C.c_size_t]
_libc.malloc.restype = C.c_void_p
_libc.malloc.argtypes = [C.c_size_t]
_libc.free.restype = None
_libc.free.argtypes = [C.c_void_p]


class Coef(C.Structure):
    """struct coef — reference jpeg2png.h:7-20 / include/jpeg2png_b200.h."""
    _fields_ = [('h', C.c_uint), ('w', C.c_uint), ('h_samp', C.c_uint), ('w_samp', C.c_uint),
                ('data', C.POINTER(C.c_int16)), ('fdata', C.POINTER(C.c_float)),
                ('quant_table', C.c_uint16 * 64)]


class Logger(C.Structure):
    """struct logger — reference logger.h:6-11."""
    _fields_ = [('f', C.c_void_p), ('filename', C.c_char_p), ('channel', C.c_uint),
                ('iteration', C.c_uint)]


class ProgressBar(C.Structure):
    """struct progressbar — reference progressbar.h:4-7."""
    _fields_ = [('current', C.c_uint), ('max', C.c_uint)]


class FrameDesc(C.Structure):
    """struct j2p_frame_desc — include/jpeg2png_b200.h."""
    _fields_ = [('nchannel', C.c_uint), ('plane_w', C.c_uint * 3), ('plane_h', C.c_uint * 3),
                ('w_samp', C.c_uint * 3), ('h_samp', C.c_uint * 3), ('weight', C.c_float),
                ('pweight', C.c_float * 3), ('iterations', C.c_uint)]


LAYOUT_HWC, LAYOUT_CHW = 0, 1       # J2P_LAYOUT_HWC / J2P_LAYOUT_CHW


class ImageOut(C.Structure):
    """struct j2p_image_out — include/jpeg2png_b200.h."""
    _fields_ = [('w', C.c_uint), ('h', C.c_uint), ('sample', C.c_uint), ('layout', C.c_uint),
                ('frame_bytes', C.c_size_t)]


def alloc_floats(n: int) -> int:
    """16-byte aligned malloc-family buffer (reference alloc_simd, utils.h:89-98)."""
    nbytes = (max(n, 1) * 4 + 15) & ~15
    p = _libc.aligned_alloc(16, nbytes)
    if not p:
        raise MemoryError
    return p


def free_ptr(p) -> None:
    if p:
        _libc.free(C.cast(p, C.c_void_p))


class CoefArray:
    """Owns a C array of `struct coef` built from a CoefImage (subset of its planes).

    `fdata_planes`: list of float32 rasters (plane_h x plane_w), the conventional decode; copied
    into aligned_alloc'd memory because compute() frees it (compute.c:304-305).
    """

    def __init__(self, img: CoefImage, channels, fdata_planes=None):
        self.n = len(channels)
        self.arr = (Coef * self.n)()
        self._keep = []
        for k, ch in enumerate(channels):
            p = img.planes[ch]
            c = self.arr[k]
            c.h, c.w, c.h_samp, c.w_samp = p.h, p.w, p.h_samp, p.w_samp
            data = np.ascontiguousarray(p.data, dtype=np.int16)
            self._keep.append(data)
            c.data = data.ctypes.data_as(C.POINTER(C.c_int16))
            for j in range(64):
                c.quant_table[j] = int(p.quant[j])
            if fdata_planes is not None:
                f = np.ascontiguousarray(fdata_planes[k], dtype=np.float32).reshape(-1)
                assert f.size == p.w * p.h
                ptr = alloc_floats(f.size)
                C.memmove(ptr, f.ctypes.data, f.size * 4)
                c.fdata = C.cast(ptr, C.POINTER(C.c_float))

    def result(self, k: int) -> np.ndarray:
        """Copy of plane k's fdata as (h, w) float32 (valid after compute(): frame sized)."""
        c = self.arr[k]
        n = c.h * c.w
        out = np.empty(n, dtype=np.float32)
        C.memmove(out.ctypes.data, c.fdata, n * 4)
        return out.reshape(c.h, c.w)

    def release(self) -> None:
        for k in range(self.n):
            if self.arr[k].fdata:
                free_ptr(self.arr[k].fdata)
                self.arr[k].fdata = C.POINTER(C.c_float)()

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
PRODUCT_LIB = os.path.join(_PKG_DIR, 'csrc', 'libjpeg2png_b200.so')

_libraries = {}


def load_library(path: str, what: str, declare) -> C.CDLL:
    """The library at path (one of the package tree's helper libraries, `what` naming it in the
    error when it has not been built), loaded once and passed to declare(lib) to set its argtypes."""
    if path not in _libraries:
        if not os.path.exists(path):
            raise RuntimeError(f'{path} is missing: the {what} has not been built '
                               '(run `python -c "import __graft_entry__ as g; g.build()"`)')
        lib = C.CDLL(path, mode=C.RTLD_LOCAL)
        declare(lib)
        _libraries[path] = lib
    return _libraries[path]


def declare_product(lib: C.CDLL) -> C.CDLL:
    """Attach argtypes/restypes for every symbol include/jpeg2png_b200.h declares."""
    vp = C.c_void_p
    lib.compute.restype = None
    lib.compute.argtypes = [C.c_uint, C.POINTER(Coef), C.POINTER(Logger), C.POINTER(ProgressBar),
                            C.c_float, C.POINTER(C.c_float), C.c_uint]
    lib.j2p_last_error.restype = C.c_char_p
    lib.j2p_last_error.argtypes = []
    lib.j2p_device_count.restype = C.c_int
    lib.j2p_device_count.argtypes = []
    lib.j2p_set_thread_device.restype = C.c_int
    lib.j2p_set_thread_device.argtypes = [C.c_int]
    lib.j2p_thread_device.restype = C.c_int
    lib.j2p_thread_device.argtypes = []
    lib.j2p_session_create.restype = C.c_int
    lib.j2p_session_create.argtypes = [C.POINTER(vp), C.c_int, C.POINTER(FrameDesc)]
    lib.j2p_session_create_batch.restype = C.c_int
    lib.j2p_session_create_batch.argtypes = [C.POINTER(vp), C.c_int, C.POINTER(FrameDesc), C.c_uint]
    lib.j2p_session_frames.restype = C.c_uint
    lib.j2p_session_frames.argtypes = [vp]
    lib.j2p_session_download_frame_scanlines.restype = C.c_int
    lib.j2p_session_download_frame_scanlines.argtypes = [vp, C.c_uint, C.c_uint, C.c_uint, C.c_uint, vp]
    lib.j2p_session_export.restype = C.c_int
    lib.j2p_session_export.argtypes = [vp, C.c_uint, C.c_uint, C.POINTER(ImageOut), vp, vp]
    lib.j2p_session_export_separate.restype = C.c_int
    lib.j2p_session_export_separate.argtypes = [vp, vp, vp, C.c_uint, C.c_uint, C.POINTER(ImageOut), vp, vp]
    lib.j2p_session_export_gray.restype = C.c_int
    lib.j2p_session_export_gray.argtypes = [vp, C.c_uint, C.c_uint, C.POINTER(ImageOut), vp, vp]
    lib.j2p_session_export_oriented.restype = C.c_int
    lib.j2p_session_export_oriented.argtypes = [C.POINTER(vp), C.c_uint, C.c_uint, C.c_uint, C.c_uint, vp, C.POINTER(ImageOut), vp, vp]
    lib.j2p_session_export_four.restype = C.c_int
    lib.j2p_session_export_four.argtypes = [C.POINTER(vp), C.c_uint, C.c_uint, C.c_uint, C.c_uint, C.c_uint, vp, C.POINTER(ImageOut), vp, vp]
    lib.j2p_session_iterate_group.restype = C.c_int
    lib.j2p_session_iterate_group.argtypes = [C.POINTER(vp), C.c_uint, C.c_uint, C.c_uint]
    lib.j2p_session_create_strip.restype = C.c_int
    lib.j2p_session_create_strip.argtypes = [C.POINTER(vp), C.c_int, C.POINTER(FrameDesc), C.c_uint, C.c_uint]
    lib.j2p_session_strip_info.restype = C.c_int
    lib.j2p_session_strip_info.argtypes = [vp, C.POINTER(C.c_uint), C.POINTER(C.c_uint), C.POINTER(C.c_uint)]
    lib.j2p_session_gradient.restype = C.c_int
    lib.j2p_session_gradient.argtypes = [vp]
    lib.j2p_session_sums_ptr.restype = vp
    lib.j2p_session_sums_ptr.argtypes = [vp]
    lib.j2p_session_project.restype = C.c_int
    lib.j2p_session_project.argtypes = [vp, vp, C.c_uint]
    lib.j2p_session_halo.restype = C.c_int
    lib.j2p_session_halo.argtypes = [vp, C.c_uint, C.c_int, C.POINTER(vp), C.POINTER(vp), C.POINTER(C.c_size_t)]
    lib.j2p_session_copy_halo_to_prev.restype = C.c_int
    lib.j2p_session_copy_halo_to_prev.argtypes = [vp]
    lib.j2p_comm_unique_id.restype = C.c_int
    lib.j2p_comm_unique_id.argtypes = [vp, C.c_size_t]
    lib.j2p_comm_create.restype = C.c_int
    lib.j2p_comm_create.argtypes = [C.POINTER(vp), C.c_int, C.c_int, C.c_int, vp, C.c_size_t]
    lib.j2p_comm_destroy.restype = None
    lib.j2p_comm_destroy.argtypes = [vp]
    lib.j2p_comm_protocol.restype = C.c_int
    lib.j2p_comm_protocol.argtypes = [vp]
    lib.j2p_comm_status.restype = C.c_int
    lib.j2p_comm_status.argtypes = [vp]
    lib.j2p_session_iterate_strip.restype = C.c_int
    lib.j2p_session_iterate_strip.argtypes = [vp, vp, C.c_uint]
    lib.j2p_session_destroy.restype = None
    lib.j2p_session_destroy.argtypes = [vp]
    lib.j2p_session_width.restype = C.c_uint
    lib.j2p_session_width.argtypes = [vp]
    lib.j2p_session_height.restype = C.c_uint
    lib.j2p_session_height.argtypes = [vp]
    lib.j2p_session_upload.restype = C.c_int
    lib.j2p_session_upload.argtypes = [vp, C.c_uint, vp, vp, vp]
    lib.j2p_session_upload_device.restype = C.c_int
    lib.j2p_session_upload_device.argtypes = [vp, C.c_uint, vp, vp, vp]
    lib.j2p_session_reset.restype = C.c_int
    lib.j2p_session_reset.argtypes = [vp]
    lib.j2p_session_iterate.restype = C.c_int
    lib.j2p_session_iterate.argtypes = [vp, C.c_uint, C.c_uint]
    lib.j2p_session_profile.restype = C.c_int
    lib.j2p_session_profile.argtypes = [vp, C.c_uint, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    lib.j2p_session_wait_iteration.restype = C.c_int
    lib.j2p_session_wait_iteration.argtypes = [vp, C.c_uint]
    lib.j2p_session_download.restype = C.c_int
    lib.j2p_session_download.argtypes = [vp, C.c_uint, vp]
    lib.j2p_session_download_scanlines.restype = C.c_int
    lib.j2p_session_download_scanlines.argtypes = [vp, C.c_uint, C.c_uint, C.c_uint, vp]
    lib.j2p_session_set_logging.restype = C.c_int
    lib.j2p_session_set_logging.argtypes = [vp, C.c_int]
    lib.j2p_session_objective.restype = C.c_int
    lib.j2p_session_objective.argtypes = [vp, C.POINTER(C.c_double)]
    lib.j2p_session_record_objective.restype = C.c_int
    lib.j2p_session_record_objective.argtypes = [vp, C.c_int]
    lib.j2p_session_objective_history.restype = C.c_int
    lib.j2p_session_objective_history.argtypes = [vp, C.c_uint, C.c_uint, C.POINTER(C.c_double)]
    lib.j2p_session_sync.restype = C.c_int
    lib.j2p_session_sync.argtypes = [vp]
    lib.j2p_session_stream.restype = vp
    lib.j2p_session_stream.argtypes = [vp]
    lib.j2p_session_plane_ptr.restype = vp
    lib.j2p_session_plane_ptr.argtypes = [vp, C.c_uint]
    lib.j2p_session_launches.restype = C.c_ulonglong
    lib.j2p_session_launches.argtypes = [vp]
    lib.j2p_version.restype = C.c_char_p
    lib.j2p_version.argtypes = []
    return lib


# every symbol the header declares; tests/test_abi.py checks the .so exports all of them
HEADER_SYMBOLS = [
    'compute', 'j2p_last_error', 'j2p_device_count', 'j2p_session_create', 'j2p_session_destroy',
    'j2p_session_create_strip', 'j2p_session_strip_info', 'j2p_session_gradient', 'j2p_session_sums_ptr',
    'j2p_session_project', 'j2p_session_halo', 'j2p_session_copy_halo_to_prev',
    'j2p_comm_unique_id', 'j2p_comm_create', 'j2p_comm_destroy', 'j2p_comm_status', 'j2p_comm_protocol', 'j2p_session_iterate_strip',
    'j2p_session_width', 'j2p_session_height', 'j2p_session_upload', 'j2p_session_reset',
    'j2p_session_iterate', 'j2p_session_profile', 'j2p_session_wait_iteration', 'j2p_session_download', 'j2p_session_set_logging',
    'j2p_session_objective', 'j2p_session_sync', 'j2p_session_stream', 'j2p_session_plane_ptr',
    'j2p_session_launches', 'j2p_version', 'j2p_host_prefault', 'j2p_set_thread_device', 'j2p_thread_device', 'j2p_session_download_scanlines',
    'j2p_session_create_batch', 'j2p_session_frames', 'j2p_session_download_frame_scanlines',
    'j2p_session_export', 'j2p_session_export_separate', 'j2p_session_upload_device',
    'j2p_session_export_gray', 'j2p_session_export_oriented', 'j2p_session_export_four', 'j2p_session_iterate_group',
    'j2p_session_record_objective', 'j2p_session_objective_history',
]

_product = None


def load_product() -> C.CDLL:
    """Load libjpeg2png_b200.so from the package tree.  Fails loudly: there is no fallback."""
    global _product
    if _product is None:
        if not os.path.exists(PRODUCT_LIB):
            raise RuntimeError(
                f'{PRODUCT_LIB} is missing: the CUDA extension has not been built '
                '(run `python -c "import __graft_entry__ as g; g.build()"` or `make -C jpeg2png_b200/csrc`). '
                'There is no CPU fallback.')
        _product = declare_product(C.CDLL(PRODUCT_LIB, mode=C.RTLD_LOCAL))
    return _product


def frame_desc(img: CoefImage, channels, weight, pweight, iterations) -> FrameDesc:
    """j2p_frame_desc of planes `channels` of img; pweight: one value per entry of `channels`."""
    d = FrameDesc()
    d.nchannel = len(channels)
    for k, ch in enumerate(channels):
        p = img.planes[ch]
        d.plane_w[k], d.plane_h[k], d.w_samp[k], d.h_samp[k] = p.w, p.h, p.w_samp, p.h_samp
        d.pweight[k] = float(pweight[k])
    d.weight = float(weight)
    d.iterations = int(iterations)
    return d


class Session:
    """A resident session over the C ABI: a batch of `nframes` frames of one geometry
    (j2p_session_create_batch), or with batch=False an ordinary one-frame session
    (j2p_session_create).  Raises RuntimeError with j2p_last_error() on any failure."""

    def __init__(self, lib, desc: FrameDesc, nframes: int = 1, device: int = 0, batch: bool = True):
        self.lib, self.desc, self.nframes = lib, desc, nframes
        self.nc = int(desc.nchannel)
        self.s = C.c_void_p()
        rc = (lib.j2p_session_create_batch(C.byref(self.s), device, C.byref(desc), nframes) if batch
              else lib.j2p_session_create(C.byref(self.s), device, C.byref(desc)))
        self._check(rc)
        self.W, self.H = int(lib.j2p_session_width(self.s)), int(lib.j2p_session_height(self.s))

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(self.lib.j2p_last_error().decode())

    def upload(self, frames, channels, fdata=None):
        """Frame f of the session <- planes `channels` of frames[f]; fdata: per frame, a list of
        plane_h x plane_w conventional decodes, or None for the device decode."""
        for f, img in enumerate(frames):
            for k, ch in enumerate(channels):
                p = img.planes[ch]
                data = np.ascontiguousarray(p.data, dtype=np.int16)
                quant = np.ascontiguousarray(p.quant, dtype=np.uint16)
                fd = None if fdata is None else np.ascontiguousarray(fdata[f][k], dtype=np.float32)
                self._check(self.lib.j2p_session_upload(self.s, f * self.nc + k, data.ctypes.data, quant.ctypes.data,
                                                        None if fd is None else fd.ctypes.data))

    def iterate(self, first: int, n: int):
        self._check(self.lib.j2p_session_iterate(self.s, first, n))

    def download(self):
        """[frame][channel] -> (H, W) float32 current iterates (synchronises the session)."""
        out = []
        for f in range(self.nframes):
            planes = []
            for k in range(self.nc):
                a = np.empty((self.H, self.W), np.float32)
                self._check(self.lib.j2p_session_download(self.s, f * self.nc + k, a.ctypes.data))
                planes.append(a)
            out.append(planes)
        return out

    def sync(self):
        self._check(self.lib.j2p_session_sync(self.s))

    @property
    def launches(self) -> int:
        return int(self.lib.j2p_session_launches(self.s))

    def close(self):
        if self.s:
            self.lib.j2p_session_destroy(self.s)
            self.s = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def solve_batch(frames, channels, weight, pweight, iterations, fdata=None, device=0, lib=None):
    """Solve planes `channels` of every CoefImage in `frames` (one geometry) as ONE batch session,
    `iterations` iterations; fdata: per frame the caller's conventional decodes, or None (device
    decode).  Returns the result planes per frame: [frame][channel] -> (H, W) float32."""
    lib = lib or load_product()
    desc = frame_desc(frames[0], channels, weight, pweight, iterations)
    with Session(lib, desc, len(frames), device) as s:
        s.upload(frames, channels, fdata)
        s.iterate(0, iterations)
        return s.download()
