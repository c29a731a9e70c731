"""decode_jpeg: JPEG files in, RGB or gray CUDA tensors out, through the solver.

Every input's headers are read on the host with the JPEG reader of the command line
(libj2pcodecs.so) before any device work: sequential files whose components are each in one scan
go through its layout pass (j2p_read_jpeg_layout) and are Huffman-decoded on the device
(libj2pentropy.so, DESIGN §7d); arithmetic-coded sequential (SOF9) files of that shape go through
j2p_read_jpeg_arith_layout and, per batch, are decoded on the device one restart segment per thread
(libj2parith.so, DESIGN §7p) when that is expected to beat the host reader (arith_on_device); every other file, progressive arithmetic (SOF10)
ones included, is parsed by j2p_read_jpeg_mem.  Inputs of one geometry are solved
together in batch sessions (j2p_session_create_batch), with the conventional decode on the device as
the command line does it, and the colour conversion writes straight into one freshly allocated tensor
per chunk (j2p_session_export) on the caller's current stream.  The returned tensors of a chunk are
views of that tensor and share its storage.  With mode='UNCHANGED' or 'GRAY' the reader also takes
one-component (grayscale) files (J2P_READ_GRAY); those are solved as the luma of separate mode and,
like the luma of colour files in mode='GRAY', exported as one channel (j2p_session_export_gray).
With apply_exif_orientation=True each file's EXIF Orientation tag is read on the host
(j2p_jpeg_exif_orientation) and a chunk that holds a file with an orientation other than 1 is exported
in one call that flips or rotates every frame as it writes it (j2p_session_export_oriented, DESIGN §7l).
With mode='RGB' or 'UNCHANGED', a file the front end refuses is offered to the four-component passes:
j2p_read_jpeg_layout4 for the device decoder (four_on_device) or j2p_read_jpeg4_mem on the host; their
chunks are exported by j2p_session_export_four (DESIGN §7q).

The samples are those of the PNG the command line writes for the same file and flags:
torch.uint8 the 8-bit PNG samples, torch.uint16 the 16-bit (-1) samples in native byte order,
torch.float32 the clamped value before truncation.  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import math
import numbers
import os
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass

import numpy as np
import torch

from . import abi

CODECS_LIB = os.path.join(abi._PKG_DIR, 'cli', 'libj2pcodecs.so')
MAX_BATCH = 65535                   # frames per batch session (j2p_session_create_batch)

_SAMPLE = {torch.uint8: 8, torch.uint16: 16, torch.float32: 32}
_LAYOUT = {'HWC': abi.LAYOUT_HWC, 'CHW': abi.LAYOUT_CHW}
MODES = ('RGB', 'UNCHANGED', 'GRAY')
READ_GRAY = 1                       # J2P_READ_GRAY (jpeg_reader.h)
READ_CMYK = 2                       # J2P_READ_CMYK
CMYK, YCCK = 1, 2                   # J2P_JPEG_CMYK / J2P_JPEG_YCCK, and J2P_FOUR_CMYK / J2P_FOUR_YCCK of the export


class Jpeg(C.Structure):
    """struct j2p_jpeg — jpeg2png_b200/cli/jpeg_reader.h."""
    _fields_ = [('w', C.c_uint), ('h', C.c_uint), ('coefs', abi.Coef * 3), ('ncomp', C.c_uint)]


class Jpeg4(C.Structure):
    """struct j2p_jpeg4 — jpeg2png_b200/cli/jpeg_reader.h."""
    _fields_ = [('w', C.c_uint), ('h', C.c_uint), ('coefs', abi.Coef * 4), ('ncomp', C.c_uint), ('colour', C.c_uint)]


class Huff(C.Structure):
    """struct j2p_jpeg_huff — jpeg2png_b200/cli/jpeg_reader.h."""
    _fields_ = [('bits', C.c_uint8 * 17), ('vals', C.c_uint8 * 256)]


class Scan(C.Structure):
    """struct j2p_jpeg_scan — jpeg2png_b200/cli/jpeg_reader.h."""
    _fields_ = [('ncomp', C.c_uint), ('comp', C.c_uint * 3), ('bw', C.c_uint * 3), ('bh', C.c_uint * 3),
                ('mcux', C.c_uint), ('mcuy', C.c_uint), ('restart_interval', C.c_uint),
                ('dc', Huff * 3), ('ac', Huff * 3), ('seg0', C.c_uint), ('nseg', C.c_uint)]


class Segment(C.Structure):
    """struct j2p_jpeg_segment — jpeg2png_b200/cli/jpeg_reader.h."""
    _fields_ = [('off', C.c_size_t), ('len', C.c_size_t), ('mcus', C.c_uint)]


class Layout(C.Structure):
    """struct j2p_jpeg_layout — jpeg2png_b200/cli/jpeg_reader.h."""
    _fields_ = [('w', C.c_uint), ('h', C.c_uint), ('coefs', abi.Coef * 3), ('comp_h', C.c_uint * 3),
                ('comp_v', C.c_uint * 3), ('device_decodable', C.c_int), ('nscan', C.c_uint), ('scan', Scan * 3),
                ('nseg', C.c_uint), ('seg', C.POINTER(Segment)), ('data', C.POINTER(C.c_uint8)),
                ('data_len', C.c_size_t), ('ncomp', C.c_uint)]


class Scan4(C.Structure):
    """struct j2p_jpeg_scan4 — jpeg2png_b200/cli/jpeg_reader.h."""
    _fields_ = [('ncomp', C.c_uint), ('comp', C.c_uint * 4), ('bw', C.c_uint * 4), ('bh', C.c_uint * 4),
                ('mcux', C.c_uint), ('mcuy', C.c_uint), ('restart_interval', C.c_uint),
                ('dc', Huff * 4), ('ac', Huff * 4), ('seg0', C.c_uint), ('nseg', C.c_uint)]


class Layout4(C.Structure):
    """struct j2p_jpeg_layout4 — jpeg2png_b200/cli/jpeg_reader.h."""
    _fields_ = [('w', C.c_uint), ('h', C.c_uint), ('coefs', abi.Coef * 4), ('comp_h', C.c_uint * 4),
                ('comp_v', C.c_uint * 4), ('device_decodable', C.c_int), ('nscan', C.c_uint), ('scan', Scan4 * 4),
                ('nseg', C.c_uint), ('seg', C.POINTER(Segment)), ('data', C.POINTER(C.c_uint8)),
                ('data_len', C.c_size_t), ('ncomp', C.c_uint), ('colour', C.c_uint)]


class ProgScan(C.Structure):
    """struct j2p_jpeg_prog_scan — jpeg2png_b200/cli/jpeg_reader.h."""
    _fields_ = [('s', Scan), ('ss', C.c_uint), ('se', C.c_uint), ('ah', C.c_uint), ('al', C.c_uint)]


class ProgLayout(C.Structure):
    """struct j2p_jpeg_prog_layout — jpeg2png_b200/cli/jpeg_reader.h."""
    _fields_ = [('w', C.c_uint), ('h', C.c_uint), ('coefs', abi.Coef * 3), ('comp_h', C.c_uint * 3),
                ('comp_v', C.c_uint * 3), ('progressive_decodable', C.c_int), ('nscan', C.c_uint),
                ('scan', C.POINTER(ProgScan)), ('nseg', C.c_uint), ('seg', C.POINTER(Segment)),
                ('data', C.POINTER(C.c_uint8)), ('data_len', C.c_size_t), ('ncomp', C.c_uint)]


class ArithScan(C.Structure):
    """struct j2p_jpeg_arith_scan — jpeg2png_b200/cli/jpeg_reader.h."""
    _fields_ = [('ncomp', C.c_uint), ('comp', C.c_uint * 3), ('bw', C.c_uint * 3), ('bh', C.c_uint * 3),
                ('mcux', C.c_uint), ('mcuy', C.c_uint), ('restart_interval', C.c_uint),
                ('dc_tbl', C.c_uint * 3), ('ac_tbl', C.c_uint * 3), ('dc_L', C.c_uint * 3), ('dc_U', C.c_uint * 3),
                ('ac_K', C.c_uint * 3), ('seg0', C.c_uint), ('nseg', C.c_uint)]


class ArithLayout(C.Structure):
    """struct j2p_jpeg_arith_layout — jpeg2png_b200/cli/jpeg_reader.h."""
    _fields_ = [('w', C.c_uint), ('h', C.c_uint), ('coefs', abi.Coef * 3), ('comp_h', C.c_uint * 3),
                ('comp_v', C.c_uint * 3), ('arith_decodable', C.c_int), ('nscan', C.c_uint), ('scan', ArithScan * 3),
                ('nseg', C.c_uint), ('seg', C.POINTER(Segment)), ('data', C.POINTER(C.c_uint8)),
                ('data_len', C.c_size_t), ('ncomp', C.c_uint)]


class ArithStats(C.Structure):
    """struct j2p_arith_stats — jpeg2png_b200/arith/arith.h."""
    _fields_ = [('launches', C.c_uint), ('segments', C.c_uint)]


class EntropyStats(C.Structure):
    """struct j2p_entropy_stats — jpeg2png_b200/entropy/entropy.h."""
    _fields_ = [('rounds', C.c_uint), ('round_trips', C.c_uint), ('launches', C.c_uint), ('subsequences', C.c_uint)]


class ProgressiveStats(C.Structure):
    """struct j2p_progressive_stats — jpeg2png_b200/progressive/progressive.h."""
    _fields_ = [('rounds', C.c_uint), ('round_trips', C.c_uint), ('launches', C.c_uint), ('steps', C.c_uint),
                ('subsequences', C.c_uint), ('refine_segments', C.c_uint), ('step_launches', C.c_uint)]


PROGRESSIVE_LIB = os.path.join(abi._PKG_DIR, 'progressive', 'libj2pprogressive.so')
ENTROPY_LIB = os.path.join(abi._PKG_DIR, 'entropy', 'libj2pentropy.so')
SUBSEQ_BITS = 1024                  # bits per subsequence of the device decoder (DESIGN §7d)
ENT_FAILURES = {1: 'bad huffman code', 2: 'bad magnitude category', 3: 'coefficient index out of range'}
ARITH_LIB = os.path.join(abi._PKG_DIR, 'arith', 'libj2parith.so')
ARITH_FAILURES = {1: 'bad arithmetic code'}
# The routing rule of arithmetic-coded files (DESIGN §7p, arith_on_device).  One device call decodes
# every segment of a chunk at once, one thread each, so it lasts about as long as the serial walk of
# the chunk's longest segment; the host reader pays for every byte of every file, on the threads of
# decode_jpeg's pool.  Both rates measured on an H100 80GB HBM3 and its host (tools/arith_bench.py).
ARITH_DEVICE_NS_PER_BYTE = 3800     # one device thread walking a segment
ARITH_HOST_NS_PER_BYTE = 190        # j2p_read_jpeg_mem on one host thread

class Keep(C.Structure):
    """struct j2p_jpeg_keep — jpeg2png_b200/cli/jpeg_reader.h."""
    _fields_ = [('qt', (C.c_uint16 * 64) * 4), ('present', C.c_uint), ('ncomp', C.c_uint), ('comp_h', C.c_uint * 4),
                ('comp_v', C.c_uint * 4)]


def _declare_codecs(lib):
    lib.j2p_read_jpeg_mem.restype = C.c_int
    lib.j2p_read_jpeg_mem.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(Jpeg), C.c_char_p, C.c_size_t]
    lib.j2p_read_jpeg_layout.restype = C.c_int
    lib.j2p_read_jpeg_layout.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(Layout), C.c_char_p, C.c_size_t]
    lib.j2p_free_jpeg_layout.restype = None
    lib.j2p_free_jpeg_layout.argtypes = [C.POINTER(Layout)]
    lib.j2p_read_jpeg_prog_layout.restype = C.c_int
    lib.j2p_read_jpeg_prog_layout.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(ProgLayout), C.c_char_p, C.c_size_t]
    lib.j2p_read_jpeg_mem_ex.restype = C.c_int
    lib.j2p_read_jpeg_mem_ex.argtypes = [C.c_char_p, C.c_size_t, C.c_uint, C.POINTER(Jpeg), C.c_char_p, C.c_size_t]
    lib.j2p_read_jpeg_layout_ex.restype = C.c_int
    lib.j2p_read_jpeg_layout_ex.argtypes = [C.c_char_p, C.c_size_t, C.c_uint, C.POINTER(Layout), C.c_char_p, C.c_size_t]
    lib.j2p_read_jpeg_prog_layout_ex.restype = C.c_int
    lib.j2p_read_jpeg_prog_layout_ex.argtypes = [C.c_char_p, C.c_size_t, C.c_uint, C.POINTER(ProgLayout), C.c_char_p, C.c_size_t]
    lib.j2p_free_jpeg_prog_layout.restype = None
    lib.j2p_free_jpeg_prog_layout.argtypes = [C.POINTER(ProgLayout)]
    lib.j2p_jpeg_exif_orientation.restype = C.c_int
    lib.j2p_jpeg_exif_orientation.argtypes = [C.c_char_p, C.c_size_t]
    lib.j2p_read_jpeg_arith_layout_ex.restype = C.c_int
    lib.j2p_read_jpeg_arith_layout_ex.argtypes = [C.c_char_p, C.c_size_t, C.c_uint, C.POINTER(ArithLayout), C.c_char_p, C.c_size_t]
    lib.j2p_free_jpeg_arith_layout.restype = None
    lib.j2p_free_jpeg_arith_layout.argtypes = [C.POINTER(ArithLayout)]
    lib.j2p_jpeg_keep_settings.restype = C.c_int
    lib.j2p_read_jpeg_layout4.restype = C.c_int
    lib.j2p_read_jpeg_layout4.argtypes = [C.c_char_p, C.c_size_t, C.c_uint, C.POINTER(Layout4), C.c_char_p, C.c_size_t]
    lib.j2p_free_jpeg_layout4.restype = None
    lib.j2p_free_jpeg_layout4.argtypes = [C.POINTER(Layout4)]
    lib.j2p_read_jpeg4_mem.restype = C.c_int
    lib.j2p_read_jpeg4_mem.argtypes = [C.c_char_p, C.c_size_t, C.c_uint, C.POINTER(Jpeg4), C.c_char_p, C.c_size_t]
    lib.j2p_jpeg_keep_settings.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(Keep), C.c_char_p, C.c_size_t]


def load_codecs() -> C.CDLL:
    """libj2pcodecs.so (the command line's JPEG reader) from the package tree."""
    return abi.load_library(CODECS_LIB, 'command line', _declare_codecs)


def _declare_entropy(lib):
    vp, lay = C.c_void_p, C.POINTER(C.POINTER(Layout))
    lib.j2p_entropy_plan_size.restype = C.c_int
    lib.j2p_entropy_plan_size.argtypes = [lay, C.c_uint, C.c_uint, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    lib.j2p_entropy_pack.restype = C.c_int
    lib.j2p_entropy_pack.argtypes = [lay, C.c_uint, C.c_uint, C.POINTER(vp), vp, C.c_size_t]
    lay4 = C.POINTER(C.POINTER(Layout4))
    lib.j2p_entropy_plan_size4.restype = C.c_int
    lib.j2p_entropy_plan_size4.argtypes = [lay4, C.c_uint, C.c_uint, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    lib.j2p_entropy_pack4.restype = C.c_int
    lib.j2p_entropy_pack4.argtypes = [lay4, C.c_uint, C.c_uint, C.POINTER(vp), vp, C.c_size_t]
    lib.j2p_entropy_decode.restype = C.c_int
    lib.j2p_entropy_decode.argtypes = [vp, vp, vp, vp, vp, C.POINTER(EntropyStats)]
    lib.j2p_entropy_decode_host.restype = C.c_int
    lib.j2p_entropy_decode_host.argtypes = [vp, vp, vp, C.POINTER(EntropyStats)]
    lib.j2p_entropy_last_error.restype = C.c_char_p
    lib.j2p_entropy_last_error.argtypes = []


def load_entropy() -> C.CDLL:
    """libj2pentropy.so (the device entropy decoder) from the package tree."""
    return abi.load_library(ENTROPY_LIB, 'entropy decoder', _declare_entropy)


def _declare_arith(lib):
    vp, lay = C.c_void_p, C.POINTER(C.POINTER(ArithLayout))
    lib.j2p_arith_plan_size.restype = C.c_int
    lib.j2p_arith_plan_size.argtypes = [lay, C.c_uint, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    lib.j2p_arith_pack.restype = C.c_int
    lib.j2p_arith_pack.argtypes = [lay, C.c_uint, C.POINTER(vp), vp, C.c_size_t]
    lib.j2p_arith_decode.restype = C.c_int
    lib.j2p_arith_decode.argtypes = [vp, vp, vp, vp, vp, C.POINTER(ArithStats)]
    lib.j2p_arith_decode_host.restype = C.c_int
    lib.j2p_arith_decode_host.argtypes = [vp, vp, vp, C.POINTER(ArithStats)]
    lib.j2p_arith_last_error.restype = C.c_char_p
    lib.j2p_arith_last_error.argtypes = []


def load_arith() -> C.CDLL:
    """libj2parith.so (the device decoder of sequential arithmetic-coded files) from the package tree."""
    return abi.load_library(ARITH_LIB, 'arithmetic decoder', _declare_arith)


def _declare_progressive(lib):
    vp, lay = C.c_void_p, C.POINTER(C.POINTER(ProgLayout))
    lib.j2p_progressive_plan_size.restype = C.c_int
    lib.j2p_progressive_plan_size.argtypes = [lay, C.c_uint, C.c_uint, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    lib.j2p_progressive_pack.restype = C.c_int
    lib.j2p_progressive_pack.argtypes = [lay, C.c_uint, C.c_uint, C.POINTER(vp), vp, C.c_size_t]
    lib.j2p_progressive_decode.restype = C.c_int
    lib.j2p_progressive_decode.argtypes = [vp, vp, vp, vp, vp, C.POINTER(ProgressiveStats)]
    lib.j2p_progressive_decode_host.restype = C.c_int
    lib.j2p_progressive_decode_host.argtypes = [vp, vp, vp, C.POINTER(ProgressiveStats)]
    lib.j2p_progressive_last_error.restype = C.c_char_p
    lib.j2p_progressive_last_error.argtypes = []


def load_progressive() -> C.CDLL:
    """libj2pprogressive.so (the progressive device entropy decoder) from the package tree."""
    return abi.load_library(PROGRESSIVE_LIB, 'progressive decoder', _declare_progressive)


class FileLayout:
    """A file's layout (j2p_read_jpeg_layout_ex with the J2P_READ_* `flags`); frees the C buffers
    when collected.  planes: one per component of a device-decodable file."""

    def __init__(self, data: bytes, flags: int = 0):
        lib = load_codecs()
        self.lay = Layout()
        err = C.create_string_buffer(256)
        if lib.j2p_read_jpeg_layout_ex(data, len(data), flags, C.byref(self.lay), err, 256) != 0:
            raise ValueError(err.value.decode(errors='replace'))
        self.device_decodable = bool(self.lay.device_decodable)
        self.w, self.h = int(self.lay.w), int(self.lay.h)
        self.compressed = int(self.lay.data_len)
        self.planes = [Plane(int(c.w), int(c.h), int(c.w_samp), int(c.h_samp), None,
                             np.array(list(c.quant_table), np.uint16)) for c in self.lay.coefs[:self.lay.ncomp]]

    def key(self):
        return Parsed.key(self)

    def __del__(self):
        try:
            load_codecs().j2p_free_jpeg_layout(C.byref(self.lay))
        except Exception:
            pass


class FileLayout4:
    """A four-component file's layout (j2p_read_jpeg_layout4 with the J2P_READ_* `flags`); frees the C
    buffers when collected.  device_decodable: sequential Huffman, each component in one scan."""
    planes_per_file = 4

    def __init__(self, data: bytes, flags: int = 0):
        lib = load_codecs()
        self.lay = Layout4()
        err = C.create_string_buffer(256)
        if lib.j2p_read_jpeg_layout4(data, len(data), flags, C.byref(self.lay), err, 256) != 0:
            raise ValueError(err.value.decode(errors='replace'))
        self.device_decodable = bool(self.lay.device_decodable)
        self.w, self.h = int(self.lay.w), int(self.lay.h)
        self.colour = int(self.lay.colour)
        self.compressed = int(self.lay.data_len)
        self.planes = [Plane(int(c.w), int(c.h), int(c.w_samp), int(c.h_samp), None,
                             np.array(list(c.quant_table), np.uint16)) for c in self.lay.coefs[:self.lay.ncomp]]

    def key(self):
        return Parsed.key(self)

    def __del__(self):
        try:
            load_codecs().j2p_free_jpeg_layout4(C.byref(self.lay))
        except Exception:
            pass


class ProgFileLayout:
    """A progressive file's layout (j2p_read_jpeg_prog_layout_ex with the J2P_READ_* `flags`); frees
    the C buffers when collected."""

    def __init__(self, data: bytes, flags: int = 0):
        lib = load_codecs()
        self.lay = ProgLayout()
        err = C.create_string_buffer(256)
        if lib.j2p_read_jpeg_prog_layout_ex(data, len(data), flags, C.byref(self.lay), err, 256) != 0:
            raise ValueError(err.value.decode(errors='replace'))
        self.progressive_decodable = bool(self.lay.progressive_decodable)
        self.w, self.h = int(self.lay.w), int(self.lay.h)
        self.compressed = int(self.lay.data_len)
        self.planes = [Plane(int(c.w), int(c.h), int(c.w_samp), int(c.h_samp), None,
                             np.array(list(c.quant_table), np.uint16)) for c in self.lay.coefs[:self.lay.ncomp]]

    def key(self):
        return Parsed.key(self)

    def __del__(self):
        try:
            load_codecs().j2p_free_jpeg_prog_layout(C.byref(self.lay))
        except Exception:
            pass


class ArithFileLayout:
    """A sequential arithmetic-coded file's layout (j2p_read_jpeg_arith_layout_ex with the J2P_READ_*
    `flags`); frees the C buffers when collected.  longest_segment: the bytes of its longest segment
    (0 when not arith_decodable)."""

    def __init__(self, data: bytes, flags: int = 0):
        lib = load_codecs()
        self.lay = ArithLayout()
        err = C.create_string_buffer(256)
        if lib.j2p_read_jpeg_arith_layout_ex(data, len(data), flags, C.byref(self.lay), err, 256) != 0:
            raise ValueError(err.value.decode(errors='replace'))
        self.arith_decodable = bool(self.lay.arith_decodable)
        self.w, self.h = int(self.lay.w), int(self.lay.h)
        self.compressed = int(self.lay.data_len)
        self.longest_segment = max((int(self.lay.seg[k].len) for k in range(self.lay.nseg)), default=0)
        self.planes = [Plane(int(c.w), int(c.h), int(c.w_samp), int(c.h_samp), None,
                             np.array(list(c.quant_table), np.uint16)) for c in self.lay.coefs[:self.lay.ncomp]]

    def key(self):
        return Parsed.key(self)

    def __del__(self):
        try:
            load_codecs().j2p_free_jpeg_arith_layout(C.byref(self.lay))
        except Exception:
            pass


def arith_on_device(layouts, workers: int) -> bool:
    """Whether one device call on the ArithFileLayouts of a chunk is expected to beat the host reader
    running on min(workers, len(layouts)) threads: the serial walk of the longest segment against
    the host's share of all their bytes.  Files without restart intervals are one segment each, so a
    chunk of them goes to the device only when it holds many more files than there are threads; a
    file cut into many restart intervals goes there even alone."""
    longest = max(lay.longest_segment for lay in layouts)
    total = sum(lay.compressed for lay in layouts)
    threads = max(1, min(int(workers), len(layouts)))
    return longest * ARITH_DEVICE_NS_PER_BYTE < total * ARITH_HOST_NS_PER_BYTE / threads


def _layout_ptrs(layouts):
    return (C.POINTER(Layout) * len(layouts))(*[C.pointer(x.lay) for x in layouts])


def entropy_plan(layouts, outs, subseq_bits=SUBSEQ_BITS, pinned=False):
    """Pack `layouts` (FileLayout) into a plan for libj2pentropy.so; outs[3 * i + c]: address of
    file i's plane c (any value for the planes a gray file does not have).  Returns (plan buffer: a pinned uint8 tensor or a numpy array, its address,
    plan bytes, work bytes)."""
    lib = load_entropy()
    ptrs = _layout_ptrs(layouts)
    plan_bytes, work_bytes = C.c_size_t(), C.c_size_t()
    if lib.j2p_entropy_plan_size(ptrs, len(layouts), subseq_bits, C.byref(plan_bytes), C.byref(work_bytes)) != 0:
        raise RuntimeError(lib.j2p_entropy_last_error().decode())
    if pinned:
        buf = torch.empty(plan_bytes.value, dtype=torch.uint8, pin_memory=True)
        addr = buf.data_ptr()
    else:
        buf = np.zeros(plan_bytes.value + 16, np.uint8)
        addr = (buf.ctypes.data + 15) & ~15
    if addr % 16:
        raise RuntimeError('plan buffer is not 16-byte aligned')
    o = (C.c_void_p * len(outs))(*outs)
    if lib.j2p_entropy_pack(ptrs, len(layouts), subseq_bits, o, addr, plan_bytes.value) != 0:
        raise RuntimeError(lib.j2p_entropy_last_error().decode())
    return buf, addr, plan_bytes.value, work_bytes.value


def entropy_plan4(layouts, outs, subseq_bits=SUBSEQ_BITS, pinned=False):
    """entropy_plan for FileLayout4s (j2p_entropy_pack4); outs[4 * i + c]: file i's plane c."""
    lib = load_entropy()
    ptrs = (C.POINTER(Layout4) * len(layouts))(*[C.pointer(x.lay) for x in layouts])
    plan_bytes, work_bytes = C.c_size_t(), C.c_size_t()
    if lib.j2p_entropy_plan_size4(ptrs, len(layouts), subseq_bits, C.byref(plan_bytes), C.byref(work_bytes)) != 0:
        raise RuntimeError(lib.j2p_entropy_last_error().decode())
    if pinned:
        buf = torch.empty(plan_bytes.value, dtype=torch.uint8, pin_memory=True)
        addr = buf.data_ptr()
    else:
        buf = np.zeros(plan_bytes.value + 16, np.uint8)
        addr = (buf.ctypes.data + 15) & ~15
    o = (C.c_void_p * len(outs))(*outs)
    if lib.j2p_entropy_pack4(ptrs, len(layouts), subseq_bits, o, addr, plan_bytes.value) != 0:
        raise RuntimeError(lib.j2p_entropy_last_error().decode())
    return buf, addr, plan_bytes.value, work_bytes.value


def progressive_plan(layouts, outs, subseq_bits=SUBSEQ_BITS, pinned=False):
    """entropy_plan for ProgFileLayouts and libj2pprogressive.so."""
    lib = load_progressive()
    ptrs = (C.POINTER(ProgLayout) * len(layouts))(*[C.pointer(x.lay) for x in layouts])
    plan_bytes, work_bytes = C.c_size_t(), C.c_size_t()
    if lib.j2p_progressive_plan_size(ptrs, len(layouts), subseq_bits, C.byref(plan_bytes), C.byref(work_bytes)) != 0:
        raise RuntimeError(lib.j2p_progressive_last_error().decode())
    if pinned:
        buf = torch.empty(plan_bytes.value, dtype=torch.uint8, pin_memory=True)
        addr = buf.data_ptr()
    else:
        buf = np.zeros(plan_bytes.value + 16, np.uint8)
        addr = (buf.ctypes.data + 15) & ~15
    o = (C.c_void_p * len(outs))(*outs)
    if lib.j2p_progressive_pack(ptrs, len(layouts), subseq_bits, o, addr, plan_bytes.value) != 0:
        raise RuntimeError(lib.j2p_progressive_last_error().decode())
    return buf, addr, plan_bytes.value, work_bytes.value


def arith_plan(layouts, outs, subseq_bits=None, pinned=False):
    """entropy_plan for ArithFileLayouts and libj2parith.so (subseq_bits: unused, the decoder works
    per segment)."""
    lib = load_arith()
    ptrs = (C.POINTER(ArithLayout) * len(layouts))(*[C.pointer(x.lay) for x in layouts])
    plan_bytes, work_bytes = C.c_size_t(), C.c_size_t()
    if lib.j2p_arith_plan_size(ptrs, len(layouts), C.byref(plan_bytes), C.byref(work_bytes)) != 0:
        raise RuntimeError(lib.j2p_arith_last_error().decode())
    if pinned:
        buf = torch.empty(plan_bytes.value, dtype=torch.uint8, pin_memory=True)
        addr = buf.data_ptr()
    else:
        buf = np.zeros(plan_bytes.value + 16, np.uint8)
        addr = (buf.ctypes.data + 15) & ~15
    o = (C.c_void_p * len(outs))(*outs)
    if lib.j2p_arith_pack(ptrs, len(layouts), o, addr, plan_bytes.value) != 0:
        raise RuntimeError(lib.j2p_arith_last_error().decode())
    return buf, addr, plan_bytes.value, work_bytes.value


@dataclass
class Plane:
    w: int
    h: int
    w_samp: int
    h_samp: int
    data: np.ndarray        # int16 [blocks][64], natural order
    quant: np.ndarray       # uint16[64], natural order


@dataclass
class Parsed:
    """One parsed JPEG: the visible size and its coefficient planes (three, one for a gray file,
    four for a CMYK or YCCK file, whose kind is `colour`)."""
    w: int
    h: int
    planes: list
    colour: int = 0             # CMYK or YCCK for four planes

    def key(self):
        """Inputs with equal keys are solved in one batch session; a four-component file's key also
        holds its kind."""
        k = (self.w, self.h, tuple((p.w, p.h, p.w_samp, p.h_samp) for p in self.planes))
        return k + (self.colour,) if len(self.planes) == 4 else k


def parse_jpeg(data: bytes, flags: int = 0) -> Parsed:
    """Parse JPEG bytes with j2p_read_jpeg_mem_ex and the J2P_READ_* `flags`; ValueError carries the
    reader's message."""
    lib = load_codecs()
    j = Jpeg()
    err = C.create_string_buffer(256)
    if lib.j2p_read_jpeg_mem_ex(data, len(data), flags, C.byref(j), err, 256) != 0:
        raise ValueError(err.value.decode(errors='replace'))
    planes = []
    for c in j.coefs[:j.ncomp]:
        n = c.w * c.h
        d = np.ctypeslib.as_array(c.data, shape=(n,)).copy() if n else np.zeros(0, np.int16)
        abi.free_ptr(c.data)
        planes.append(Plane(int(c.w), int(c.h), int(c.w_samp), int(c.h_samp), d, np.array(list(c.quant_table), np.uint16)))
    return Parsed(int(j.w), int(j.h), planes)


def parse_jpeg4(data: bytes, flags: int = 0) -> Parsed:
    """Parse JPEG bytes with j2p_read_jpeg4_mem, which takes four-component files (J2P_READ_CMYK is
    always on); a four-component Parsed has its colour kind.  The ValueError carries the reader's
    message and, as .ncomp, the frame header's component count (0 when it was not read)."""
    lib = load_codecs()
    j = Jpeg4()
    err = C.create_string_buffer(256)
    if lib.j2p_read_jpeg4_mem(data, len(data), flags, C.byref(j), err, 256) != 0:
        e = ValueError(err.value.decode(errors='replace'))
        e.ncomp = int(j.ncomp)
        raise e
    planes = []
    for c in j.coefs[:j.ncomp]:
        n = c.w * c.h
        d = np.ctypeslib.as_array(c.data, shape=(n,)).copy() if n else np.zeros(0, np.int16)
        abi.free_ptr(c.data)
        planes.append(Plane(int(c.w), int(c.h), int(c.w_samp), int(c.h_samp), d, np.array(list(c.quant_table), np.uint16)))
    return Parsed(int(j.w), int(j.h), planes, int(j.colour))


def exif_orientation(data: bytes) -> int:
    """The EXIF Orientation of JPEG bytes (j2p_jpeg_exif_orientation): 1..8, 1 without a usable tag."""
    return int(load_codecs().j2p_jpeg_exif_orientation(data, len(data)))


def oriented_shape(shape, layout_id, orientation):
    """The (c, h, w) or (h, w, c) shape of a frame of `shape` written with an EXIF orientation."""
    if orientation < 5:
        return shape
    c, h, w = shape if layout_id == abi.LAYOUT_CHW else (shape[2], shape[0], shape[1])
    return (c, w, h) if layout_id == abi.LAYOUT_CHW else (w, h, c)


def solver_flags(iterations, weight, pweight, separate):
    """The command line's flags (reference jpeg2png.c:206-244): returns per-plane iterations,
    weights and pweights.  A scalar weight sets luma only (chroma 0); three weights or three
    iteration counts need separate mode."""
    def three(v):
        return isinstance(v, (list, tuple))

    if three(weight):
        if len(weight) != 3:
            raise ValueError('invalid weight')
        if not separate:
            raise ValueError('different weights are only possible when using separated components')
        weights = tuple(float(x) for x in weight)
    else:
        weights = (float(weight), 0.0, 0.0)
    if three(pweight):
        if len(pweight) != 3:
            raise ValueError('invalid probability weight')
        pweights = tuple(float(x) for x in pweight)
    else:
        pweights = (float(pweight),) * 3
    if three(iterations):
        if len(iterations) != 3:
            raise ValueError('invalid number of iterations')
        if not separate:
            raise ValueError('different iteration counts are only possible when using separated components')
        iters = tuple(iterations)
    else:
        iters = (iterations,) * 3
    for n in iters:
        if not isinstance(n, numbers.Integral) or isinstance(n, bool) or not 0 <= n <= 0xffffffff:
            raise ValueError('invalid number of iterations')
    return tuple(int(n) for n in iters), weights, pweights


def solved_planes(key, separate: bool, mode: str = 'RGB'):
    """(planes solved, output channels) of a frame of `key` in `mode`: a gray file's one plane and
    one channel; for a colour file all three planes and three channels, or one channel in mode
    'GRAY', from the luma alone when separate; for a four-component file all four planes, and four
    channels, or three in mode 'RGB'."""
    planes = key[2]
    if len(planes) == 1:
        return 1, 1
    if len(planes) == 4:
        return 4, (3 if mode == 'RGB' else 4)
    if mode == 'GRAY':
        return (1 if separate else 3), 1
    return 3, 3


def frame_footprint(key, separate: bool, sample_bytes: int, mode: str = 'RGB', record_rows: int = 0) -> int:
    """Estimated device bytes one frame of `key` takes in its batch session(s) (DESIGN §4: x, xp, g,
    gp at frame size per plane; coefficients int16 and the conventional decode fp32 at plane size;
    the reduction state) plus its part of the output tensor, for the planes solved and the channels
    written in `mode` (solved_planes).  record_rows: iterations the frame's sessions record
    (return_objective), five fp64 sums each (DESIGN §7o), plus the projection's partials."""
    w, h, planes = key[:3]
    nsolved, nout = solved_planes(key, separate, mode)
    planes = planes[:nsolved]

    def session(pl):
        W = max(pw * ws for pw, ph, ws, hs in pl)
        H = max(ph * hs for pw, ph, ws, hs in pl)
        ps = (W * H + 63) // 64 * 64
        n = 4 * 4 * ps * len(pl)
        for pw, ph, ws, hs in pl:
            n += (pw * ph + 127) // 128 * 128 * 2 + (pw * ph + 63) // 64 * 64 * 4
        return n + (16 << 10)

    if len(planes) == 4:        # CMYK: every plane alone; YCCK: Y, Cb, Cr as a colour file, K alone
        total = (sum(session([p]) for p in planes) if separate or key[3] == CMYK else
                 session(list(planes[:3])) + session([planes[3]]))
    else:
        total = sum(session([p]) for p in planes) if separate else session(list(planes))
    if record_rows:
        total += 40 * record_rows + 3 * 8 * sum((pw // 8) * (ph // 8) for pw, ph, _, _ in planes)
    return total + w * h * nout * sample_bytes


def max_files(key) -> int:
    """Files per chunk of `key` its sessions can hold: MAX_BATCH, or MAX_BATCH // 4 for a CMYK key
    whose four planes share one grid, solved in one batch session of four frames per file."""
    planes = key[2]
    if len(planes) == 4 and key[3] == CMYK and len(set(planes)) == 1:
        return MAX_BATCH // 4
    return MAX_BATCH


def chunk_frames(key, separate: bool, sample_bytes: int, max_frames, free_bytes: int, mode: str = 'RGB') -> int:
    """Frames per batch of `key`: max_frames, or as many as keep the estimated footprint of two
    chunks in flight (one solving while the next is uploaded) under half of `free_bytes`; never more
    than max_files(key)."""
    if max_frames is not None:
        return min(int(max_frames), max_files(key))
    per = frame_footprint(key, separate, sample_bytes, mode)
    return max(1, min(max_files(key), free_bytes // 4 // per))


def plan(keys, frames_for_key):
    """Group input indices by key (groups in order of first appearance, indices in input order)
    and split each group into chunks of at most frames_for_key(key) inputs.
    Returns [(key, [input index, ...]), ...]."""
    groups = {}
    for i, k in enumerate(keys):
        groups.setdefault(k, []).append(i)
    chunks = []
    for k, idx in groups.items():
        n = frames_for_key(k)
        if n < 1:
            raise ValueError('a chunk needs at least one frame')
        chunks.extend((k, idx[j:j + n]) for j in range(0, len(idx), n))
    return chunks


# Grouping (internal switch; tools/mixed_bench.py and the tests compare the two): chunks of different
# geometries whose frames are small are iterated together, one j2p_session_iterate_group call per pack
# (DESIGN §7m).  False solves every chunk on its own, as before grouping existed.
_group_chunks = True
# Frames up to this many pixels are grouped.  Measured on an H100 (DESIGN §7m): a group of 64 sizes
# around 256² (65 536 px) is faster than its chunks one after another; at 512² (4:4:4) and at 1080p
# the group's flat grids are slower than the per-size launches, so those chunks keep their own.
GROUP_MAX_PIXELS = 1 << 17


def group_class(key, separate: bool, mode: str = 'RGB'):
    """The class of a chunk of `key` for grouping, or None when it is solved on its own: chunks of one
    class may share a group (the join rules of j2p_session_iterate_group: one session per chunk, equal
    plane count and sampling factors, every plane 1x1 or 2x2), and only frames of at most
    GROUP_MAX_PIXELS pixels are grouped.  Separate-mode colour chunks (a session per plane) and
    four-component chunks are not."""
    w, h, planes = key[:3]
    nsolved, _ = solved_planes(key, separate, mode)
    if (separate and len(planes) > 1) or len(planes) == 4:
        return None
    solved = planes[:nsolved]
    if any((ws, hs) not in ((1, 1), (2, 2)) for _, _, ws, hs in solved):
        return None
    W = max(pw * ws for pw, _, ws, _ in solved)
    H = max(ph * hs for _, ph, _, hs in solved)
    if W * H > GROUP_MAX_PIXELS:
        return None
    return (nsolved, tuple((ws, hs) for _, _, ws, hs in solved))


def pack(chunks, class_of, bytes_of, cap_bytes):
    """Packs of the chunks of plan(): lists of chunk indices, each list in order and the packs in
    order of their first chunk.  A chunk whose class_of(key) is None is a pack of its own.  Chunks of
    one class share a pack while it holds no other chunk of their key, at most MAX_BATCH frames and at
    most cap_bytes of bytes_of(key, frames) (a chunk alone may exceed it, as it does today)."""
    packs, open_ = [], {}
    for j, (key, idx) in enumerate(chunks):
        cls = class_of(key)
        if cls is None:
            packs.append([j])
            continue
        cur = open_.get(cls)
        if cur is not None:
            p, keys, frames, nbytes = cur
            b = bytes_of(key, len(idx))
            if key not in keys and frames + len(idx) <= MAX_BATCH and nbytes + b <= cap_bytes:
                p.append(j)
                open_[cls] = (p, keys | {key}, frames + len(idx), nbytes + b)
                continue
        p = [j]
        packs.append(p)
        open_[cls] = (p, {key}, len(idx), bytes_of(key, len(idx)))
    return packs


def _read_input(x):
    if isinstance(x, (bytes, bytearray, memoryview)):
        return bytes(x), None
    if isinstance(x, (str, os.PathLike)):
        path = os.fspath(x)
        with open(path, 'rb') as f:
            return f.read(), path
    raise TypeError(f'decode_jpeg inputs are bytes-like objects or paths, not {type(x).__name__}')


def _frame_desc(parsed: Parsed, channels, weight, pweights, iterations) -> abi.FrameDesc:
    d = abi.FrameDesc()
    d.nchannel = len(channels)
    for k, c in enumerate(channels):
        p = parsed.planes[c]
        d.plane_w[k], d.plane_h[k], d.w_samp[k], d.h_samp[k] = p.w, p.h, p.w_samp, p.h_samp
        d.pweight[k] = pweights[c]
    d.weight = weight
    d.iterations = iterations
    return d


class _DeviceCoefs:
    """The coefficients of a chunk's device-decodable files, Huffman-decoded on the device by
    libj2pentropy.so into one int16 tensor: the packed plan goes up in one pinned copy on `stream`,
    the decoder runs there, and the constructor waits for the decode only.  status[i]: J2P_ENT_OK
    or the failure kind of file i."""

    per = 3                     # planes per file in ptrs

    def __init__(self, device, layouts, stream, subseq_bits=SUBSEQ_BITS):
        self._decode(device, layouts, stream, subseq_bits, entropy_plan, load_entropy(), 'entropy', EntropyStats())

    def _decode(self, device, layouts, stream, subseq_bits, make_plan, lib, name, stats):
        dev = torch.device('cuda', device)
        # `per` planes per file, the ones a gray file does not have empty
        sizes = [lay.planes[c].w * lay.planes[c].h if c < len(lay.planes) else 0 for lay in layouts for c in range(self.per)]
        offs = np.concatenate([[0], np.cumsum(sizes, dtype=np.int64)])
        with torch.cuda.stream(stream):
            self.coefs = torch.empty(max(int(offs[-1]), 1), dtype=torch.int16, device=dev)
            base = self.coefs.data_ptr()
            self.ptrs = [base + 2 * int(o) for o in offs[:-1]]           # planes are whole 128-byte blocks
            self.plan, addr, plan_bytes, work_bytes = make_plan(layouts, self.ptrs, subseq_bits, pinned=True)
            self.plan_dev = torch.empty(plan_bytes, dtype=torch.uint8, device=dev)
            self.plan_dev.copy_(self.plan, non_blocking=True)
            self.work = torch.empty(max(work_bytes, 16), dtype=torch.uint8, device=dev)
            status = torch.empty(len(layouts), dtype=torch.int32, device=dev)
            self.stats = stats
            if getattr(lib, f'j2p_{name}_decode')(addr, self.plan_dev.data_ptr(), self.work.data_ptr(), status.data_ptr(),
                                                  stream.cuda_stream, C.byref(self.stats)) != 0:
                raise RuntimeError(getattr(lib, f'j2p_{name}_last_error')().decode())
            stream.record_event().synchronize()
            self.status = status.cpu().numpy()
        self.plan = self.work = self.plan_dev = None

    def plane(self, i, c):
        return self.ptrs[self.per * i + c]

    def plane_tensor(self, i, c):
        """A view of file i's plane c in the coefficient tensor (int16, blocks * 64)."""
        k = self.per * i + c
        start = (self.ptrs[k] - self.coefs.data_ptr()) // 2
        end = (self.ptrs[k + 1] - self.coefs.data_ptr()) // 2 if k + 1 < len(self.ptrs) else self.coefs.numel()
        return self.coefs[start:end]


class _DeviceCoefs4(_DeviceCoefs):
    """_DeviceCoefs for four-component files (FileLayout4), four planes per file, decoded by
    libj2pentropy.so through j2p_entropy_pack4."""
    per = 4

    def __init__(self, device, layouts, stream, subseq_bits=SUBSEQ_BITS):
        self._decode(device, layouts, stream, subseq_bits, entropy_plan4, load_entropy(), 'entropy', EntropyStats())


class _ProgCoefs(_DeviceCoefs):
    """_DeviceCoefs for progressive files (ProgFileLayout), decoded by libj2pprogressive.so."""

    def __init__(self, device, layouts, stream, subseq_bits=SUBSEQ_BITS):
        self._decode(device, layouts, stream, subseq_bits, progressive_plan, load_progressive(), 'progressive',
                     ProgressiveStats())


class _ArithCoefs(_DeviceCoefs):
    """_DeviceCoefs for sequential arithmetic-coded files (ArithFileLayout), decoded by libj2parith.so."""

    def __init__(self, device, layouts, stream, subseq_bits=None):
        self._decode(device, layouts, stream, subseq_bits, arith_plan, load_arith(), 'arith', ArithStats())


class _Chunk:
    """The batch session(s) of one chunk: created, uploaded, iterated and exported by the
    constructor; close() waits for them and returns their blocks to the device cache.
    coefs: {item index: (_DeviceCoefs, its file index)} for items whose coefficients are on the
    device (uploaded with j2p_session_upload_device after `coef_stream`).  A gray file is solved as
    the luma of separate mode; the output has the channels solved_planes gives for `mode`.
    orientations: the EXIF orientation of each item, or None.  When one of them is not 1 the chunk is
    exported by j2p_session_export_oriented into an (n, c * h * w) tensor; frame(j) is item j's
    tensor either way."""

    def __init__(self, lib, device, items, flags, separate, dtype, layout, coefs=None, coef_stream=None, mode='RGB',
                 orientations=None, grouped=False, record=False):
        """grouped: create and upload only; the caller iterates the sessions in a group, then calls export().
        record: the sessions record the objective (j2p_session_record_objective); logs[j] is item j's
        log after the solve (decode_jpeg's return_objective)."""
        iters, weights, pweights = flags
        self.lib, self.sessions, self.coefs = lib, [], coefs or {}
        first, n = items[0], len(items)
        nsolved, nout = solved_planes(first.key(), separate, mode)
        # work: (descriptor, the planes a session holds of every file, iterations); a session has
        # n * len(planes) / nchannel frames, file f's plane planes[k] in its plane f * len(planes) + k
        self.four = first.colour if nsolved == 4 else 0
        if self.four == CMYK:           # each plane alone with the luma's flags (DESIGN §7q)
            pw = (pweights[0],) * 4
            if len({(p.w, p.h, p.w_samp, p.h_samp) for p in first.planes}) == 1:
                work = [(_frame_desc(first, [0], weights[0], pw, iters[0]), [0, 1, 2, 3], iters[0])]
            else:
                work = [(_frame_desc(first, [c], weights[0], pw, iters[0]), [c], iters[0]) for c in range(4)]
        else:
            pw = tuple(pweights) + (pweights[0],)
            ncolour = 3 if self.four else nsolved
            if ncolour == 1 or separate:
                work = [(_frame_desc(first, [c], weights[c], pw, iters[c]), [c], iters[c]) for c in range(ncolour)]
            else:
                work = [(_frame_desc(first, [0, 1, 2], weights[0], pw, iters[0]), [0, 1, 2], iters[0])]
            if self.four:               # YCCK: K alone with the luma's flags
                work.append((_frame_desc(first, [3], weights[0], pw, iters[0]), [3], iters[0]))
        try:
            for desc, channels, _ in work:
                s = C.c_void_p()
                self._check(lib.j2p_session_create_batch(C.byref(s), device, C.byref(desc), n * len(channels) // desc.nchannel))
                self.sessions.append(s)
                if record:
                    self._check(lib.j2p_session_record_objective(s, 1))
            for s, (_, channels, it) in zip(self.sessions, work):
                for f, parsed in enumerate(items):
                    for k, c in enumerate(channels):
                        p = parsed.planes[c]
                        if f in self.coefs:
                            dc, i = self.coefs[f]
                            self._check(lib.j2p_session_upload_device(s, f * len(channels) + k, dc.plane(i, c),
                                                                      p.quant.ctypes.data, coef_stream.cuda_stream))
                        else:
                            self._check(lib.j2p_session_upload(s, f * len(channels) + k, p.data.ctypes.data,
                                                               p.quant.ctypes.data, None))     # conventional decode on the device
                if not grouped:
                    self._check(lib.j2p_session_iterate(s, 0, it))
            self.iterations = work[0][2]
            self.logs = None
            if record:
                # one read per session after its solve; the key is the command line's CSV channel
                self.logs = [{} for _ in range(n)]
                for s, (_, channels, it) in zip(self.sessions, work):
                    hist = np.zeros((n, it, 4), dtype=np.float64)
                    self._check(lib.j2p_session_objective_history(s, 0, it, hist.ctypes.data_as(C.POINTER(C.c_double))))
                    key = 3 if len(channels) == 3 else channels[0]
                    for f in range(n):
                        self.logs[f][key] = torch.from_numpy(hist[f].copy())
            self._export_args = (device, items, dtype, layout, nout, separate, orientations)
            if not grouped:
                self.export()
        except BaseException:
            self.close()
            raise

    def export(self):
        """The chunk's tensor, written on the current torch stream after the sessions' solve."""
        device, items, dtype, layout, nout, separate, orientations = self._export_args
        lib, first, n = self.lib, items[0], len(items)
        try:
            w, h = first.w, first.h
            shape = (nout, h, w) if layout == abi.LAYOUT_CHW else (h, w, nout)
            cuda = torch.device('cuda', device)
            self.shapes = None
            if orientations is not None and any(k != 1 for k in orientations):
                self.shapes = [oriented_shape(shape, layout, k) for k in orientations]
                self.out = torch.empty((n, nout * h * w), dtype=dtype, device=cuda)
            else:
                self.out = torch.empty((n,) + shape, dtype=dtype, device=cuda)
            o = abi.ImageOut(w, h, _SAMPLE[dtype], layout, nout * h * w * self.out.element_size())
            # torch's default stream is handle 0, which the ABI reads as "the session stream":
            # name it cudaStreamLegacy (1) instead
            stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream or 1)
            dst = C.c_void_p(self.out.data_ptr())
            if self.four:
                orient = None
                if self.shapes is not None:
                    self.orient = torch.tensor(orientations, dtype=torch.uint8).to(cuda)
                    orient = C.c_void_p(self.orient.data_ptr())
                ss = self.sessions
                self._check(lib.j2p_session_export_four((C.c_void_p * len(ss))(*ss), len(ss), self.four, nout, 0, n, orient,
                                                        C.byref(o), dst, stream))
            elif self.shapes is not None:
                # uploaded on the current stream, which the export runs on
                self.orient = torch.tensor(orientations, dtype=torch.uint8).to(cuda)
                ss = self.sessions[:1] if nout == 1 else self.sessions
                self._check(lib.j2p_session_export_oriented((C.c_void_p * len(ss))(*ss), len(ss), nout, 0, n,
                                                            C.c_void_p(self.orient.data_ptr()), C.byref(o), dst, stream))
            elif nout == 1:
                self._check(lib.j2p_session_export_gray(self.sessions[0], 0, n, C.byref(o), dst, stream))
            elif separate:
                self._check(lib.j2p_session_export_separate(*self.sessions, 0, n, C.byref(o), dst, stream))
            else:
                self._check(lib.j2p_session_export(self.sessions[0], 0, n, C.byref(o), dst, stream))
        except BaseException:
            self.close()
            raise

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(self.lib.j2p_last_error().decode())

    def frame(self, j):
        """Item j's tensor: a view of out[j]."""
        return self.out[j] if self.shapes is None else self.out[j].view(self.shapes[j])

    def close(self):
        for s in self.sessions:
            self.lib.j2p_session_destroy(s)
        self.sessions = []
        self.coefs = {}             # the session streams are idle: the coefficient tensor can go


# The front end (internal switch; tools/entropy_bench.py compares the two): with a device, files
# that are device-decodable (j2p_read_jpeg_layout) are Huffman-decoded there and every other file is
# parsed by j2p_read_jpeg_mem; True sends every file to j2p_read_jpeg_mem.
_host_front_end = False


def _where(i, path):
    return f'input {i} ({path})' if path is not None else f'input {i}'


def _front_end(data, device_ok, progressive=False, flags=0):
    """The host part of one input: a FileLayout for the device decoder, an ArithFileLayout for the
    arithmetic device decoder (a SOF9 file whose components are each in one scan; decode_jpeg sends
    a chunk's ArithFileLayouts back to the host reader when arith_on_device says so), a ProgFileLayout for the progressive device decoder (progressive=True), a Parsed from the host
    reader, or the ValueError (always the host reader's message) or RuntimeError to raise.  flags:
    J2P_READ_*, for every reader."""
    if not device_ok or _host_front_end:
        try:
            return parse_jpeg(data, flags)
        except ValueError as e:
            return e
    try:
        lay = FileLayout(data, flags)
    except ValueError:
        try:
            parse_jpeg(data, flags)
        except ValueError as e:
            return e
        return RuntimeError('the layout pass rejected a file the host reader accepts')
    if lay.device_decodable:
        return lay
    try:
        ari = ArithFileLayout(data, flags)
    except ValueError:
        try:
            parse_jpeg(data, flags)
        except ValueError as e:
            return e
        return RuntimeError('the arithmetic layout pass rejected a file the host reader accepts')
    if ari.arith_decodable:
        return ari
    if progressive:
        try:
            prog = ProgFileLayout(data, flags)
        except ValueError:
            try:
                parse_jpeg(data, flags)
            except ValueError as e:
                return e
            return RuntimeError('the progressive layout pass rejected a file the host reader accepts')
        if prog.progressive_decodable:
            return prog
    try:
        return parse_jpeg(data, flags)
    except ValueError as e:
        return e


# Four-component files on the device decoder (DESIGN §7q): a decoder state at a subsequence boundary
# is (bit, block within the MCU).  When every component of an interleaved scan uses the same Huffman
# tables (Pillow's and libjpeg's CMYK files), a guessed state finds the bit alignment but not the
# block's place in the MCU, so each sync round corrects one more subsequence of a segment: such a
# file goes to the device only when its longest segment is at most FOUR_SYNC_SUBSEQ subsequences.
# Measured on an H100 (tools/cmyk_bench.py, 64 1080p Pillow CMYK files): segments of 80 subsequences
# (one restart interval per MCU row) decode in 2.9 ms per image on the device against 10.9 on the
# host, one segment of about 8000 in 44.7 against 12.1; the limit lies between the two.
FOUR_SYNC_SUBSEQ = 512


def four_on_device(lay) -> bool:
    """Whether a device-decodable FileLayout4 goes to the device decoder (see FOUR_SYNC_SUBSEQ)."""
    same_tables = False
    for k in range(lay.lay.nscan):
        sc = lay.lay.scan[k]
        tabs = {(bytes(sc.dc[s]), bytes(sc.ac[s])) for s in range(sc.ncomp)}
        same_tables |= sc.ncomp > 1 and len(tabs) == 1
    if not same_tables:
        return True
    longest = max((int(lay.lay.seg[k].len) for k in range(lay.lay.nseg)), default=0)
    return -(-longest * 8 // SUBSEQ_BITS) <= FOUR_SYNC_SUBSEQ


def _front_end_four(data, device_ok, progressive=False, flags=0):
    """_front_end, and for a file it refuses, the four-component reader (parse_jpeg4): a four-component
    file's Parsed, or the four-component reader's error for a four-component file; every other file's
    result is _front_end's.  With a device, a four-component sequential Huffman file whose components
    are each in one scan is a FileLayout4 for the device decoder when four_on_device says so; other
    four-component files are parsed on the host (DESIGN §7q)."""
    p = _front_end(data, device_ok, progressive, flags)
    if not isinstance(p, ValueError):
        return p
    if device_ok and not _host_front_end:
        try:
            lay = FileLayout4(data, flags)
        except ValueError:
            lay = None          # the four-component reader below gives the message
        if lay is not None and lay.device_decodable and len(lay.planes) == 4 and four_on_device(lay):
            return lay
    try:
        q = parse_jpeg4(data, flags)
    except ValueError as e:
        return e if e.ncomp == 4 else p
    return q if len(q.planes) == 4 else p


def decode_jpeg(inputs, *, iterations=50, weight=0.3, pweight=0.001, separate=False,
                dtype=torch.uint8, layout='CHW', device=None, max_frames=None, progressive_on_device=False,
                mode='RGB', apply_exif_orientation=False, return_objective=False):
    """Decode JPEG files into RGB or gray tensors on a CUDA device, deblocked by the solver.

    inputs: bytes-like, a path (str / os.PathLike), or a list or tuple of them.  A single input
    returns one tensor, a list returns a list in input order.  Each tensor is (c, h, w) for
    layout='CHW' or (h, w, c) for 'HWC' at the image's visible size, on `device` (default: the
    current CUDA device).  dtype: torch.uint8 (the 8-bit PNG samples), torch.uint16 (the 16-bit
    PNG samples) or torch.float32 (the clamped samples before truncation).

    mode: 'RGB' (c = 3; a grayscale file is refused with the reader's "only 3 component jpegs are
    supported"), 'UNCHANGED' (c = 1 for a grayscale file, 3 for a colour file, 4 for a CMYK or YCCK
    file) or 'GRAY' (c = 1 for every file; four-component files are refused with the reader's "only 1
    and 3 component jpegs are supported").  A one-channel sample is the RGB sample of its luma with zero chroma, so a gray
    tensor t gives the RGB image as t.expand(3, -1, -1) (CHW).  A grayscale file is solved as the
    luma of separate mode, with the first of three iterations, weights and pweights, so its result
    does not depend on `separate`.  For a colour file, mode='GRAY' gives the luma of the joint solve,
    or with separate=True the luma solve alone: its chroma planes are neither uploaded nor solved.

    Four-component files (Adobe CMYK and YCCK, DESIGN §7q): the kind is libjpeg's, from the last
    Adobe APP14 segment before the first SOS (none or transform 0: CMYK, any other transform: YCCK).
    mode='UNCHANGED' gives Pillow's CMYK samples, which are inverted: channel c of a CMYK file is
    255 - g (uint8), 65535 - g (uint16) or 255.0 - g (float32), with g the gray sample of plane c,
    each plane solved alone as a grayscale file is, whatever `separate` is.  A YCCK file's channels
    0-2 are the RGB samples of its Y, Cb, Cr solved as a colour file's planes (`separate` applies),
    and channel 3 is its K plane inverted, solved alone.  mode='RGB' with torch.uint8 gives Pillow's
    Image.convert('RGB') of the uint8 samples; with uint16 or float32 it raises ValueError (use
    mode='UNCHANGED').  Sequential ones whose components are each in one scan are Huffman-decoded
    on the device (j2p_read_jpeg_layout4, libj2pentropy.so), except files whose components all share
    one Huffman table and whose longest segment is over FOUR_SYNC_SUBSEQ subsequences
    (four_on_device); progressive and arithmetic ones go to the host reader whatever
    progressive_on_device.  return_objective=True refuses them.

    iterations, weight, pweight, separate: the command line's -i, -w, -p and -s.  Scalars as there:
    a scalar weight sets luma only; three weights or three iteration counts need separate=True.

    Inputs with the same geometry are solved together, max_frames per batch (default: as many as
    fit in a quarter of the free device memory).  Batches of different small geometries (up to
    GROUP_MAX_PIXELS pixels per frame, joint or gray) are iterated together in one group.  The
    tensors of one batch are views of one allocation and share its storage.  The result is written on the current torch stream and can
    be used there without synchronising.

    Sequential (baseline or extended) files whose components are each coded in one scan are
    Huffman-decoded on the device: only their compressed bytes are uploaded.  Arithmetic-coded files
    (SOF9, SOF10, as `jpegtran -arithmetic` writes them) give the pixels of their Huffman originals:
    SOF9 files of that shape are decoded on the device (libj2parith.so, DESIGN §7p) when one device
    call on the batch's arithmetic files is expected to beat the host reader (arith_on_device: their
    longest restart segment against all their bytes), the others on the host.  progressive_on_device:
    progressive files are Huffman-decoded on the device too (libj2pprogressive.so, DESIGN §7g);
    by default they are parsed on the host, as is every other file.  Raises ValueError for bad arguments and
    unreadable files, with the host reader's message: header errors before any device work, errors
    in a device-decoded file's entropy-coded data once its batch has been decoded, before that batch
    is solved.  Raises RuntimeError when no CUDA device is usable.

    apply_exif_orientation: True or False (default).  With True, a file whose EXIF Orientation tag
    (0x0112 of IFD0 in its first "Exif" APP1 segment) is 2..8 comes back flipped or rotated as
    Pillow's ImageOps.exif_transpose shows it, at its rotated visible size: orientations 5..8 swap h
    and w, giving (c, w, h) or (w, h, c).  Files without a usable tag read as 1 and are unchanged.
    The samples are those of the unrotated decode, written to their rotated places by the export
    itself; mode, separate, dtype, layout, max_frames and progressive_on_device work as without it,
    and files of one geometry share a batch whatever their orientation.  Every tensor is contiguous.

    return_objective: True or False (default).  With True the call returns (images, logs), or
    (tensor, log) for a single input: each file's objective at every iteration, as the command line's
    -c log has it.  A log is a dict keyed by the log's channel: {3: t} for a joint solve, {0: t0, 1: t1,
    2: t2} with separate=True, {0: t} for a grayscale file and for mode='GRAY' with separate=True.
    Each t is a CPU float64 tensor of shape (iterations, 4): objective, prob_dist, tv, tv2.  The
    objective is recorded on the device (j2p_session_record_objective) and read once per batch after
    its solve; the images are those of return_objective=False.  Batches are then solved one by one,
    not grouped.  write_objective_csv writes the logs as the command line's CSV file.
    """
    flags = solver_flags(iterations, weight, pweight, separate)
    if not isinstance(mode, str) or mode not in MODES:
        raise ValueError(f"mode must be 'RGB', 'UNCHANGED' or 'GRAY', not {mode!r}")
    read_flags = 0 if mode == 'RGB' else READ_GRAY
    if apply_exif_orientation is not True and apply_exif_orientation is not False:
        raise ValueError(f'apply_exif_orientation must be True or False, not {apply_exif_orientation!r}')
    if return_objective is not True and return_objective is not False:
        raise ValueError(f'return_objective must be True or False, not {return_objective!r}')
    if dtype not in _SAMPLE:
        raise ValueError(f'dtype must be torch.uint8, torch.uint16 or torch.float32, not {dtype}')
    if layout not in _LAYOUT:
        raise ValueError(f"layout must be 'CHW' or 'HWC', not {layout!r}")
    if max_frames is not None and (not isinstance(max_frames, numbers.Integral) or max_frames < 1):
        raise ValueError('max_frames must be a positive integer or None')
    dev = torch.device('cuda' if device is None else device) if not isinstance(device, int) else torch.device('cuda', device)
    if dev.type != 'cuda':
        raise ValueError(f'decode_jpeg writes CUDA tensors; device {dev} is not a CUDA device')

    single = not isinstance(inputs, (list, tuple))
    read = [_read_input(x) for x in ([inputs] if single else inputs)]
    if not read:
        return ([], []) if return_objective else []

    # Without a device the host reader reads every input (its errors first), as the solver needs a
    # device anyway.  With one, the layout pass runs instead and only non-device-decodable files are
    # parsed on the host.  Either runs without the GIL (ctypes), many files in parallel.
    device_ok = torch.cuda.is_available()
    workers = min(len(read), os.cpu_count() or 1, 16)
    front_end = _front_end if mode == 'GRAY' else _front_end_four
    if workers > 1:
        with ThreadPoolExecutor(workers) as pool:
            parsed = list(pool.map(lambda d: front_end(d, device_ok, progressive_on_device, read_flags),
                                   [data for data, _ in read]))
            orientations = (list(pool.map(exif_orientation, [data for data, _ in read]))
                            if apply_exif_orientation else None)
    else:
        parsed = [front_end(data, device_ok, progressive_on_device, read_flags) for data, _ in read]
        orientations = [exif_orientation(data) for data, _ in read] if apply_exif_orientation else None
    for i, (p, (_, path)) in enumerate(zip(parsed, read)):
        if isinstance(p, ValueError):
            raise ValueError(f'{_where(i, path)}: {p}')
        if isinstance(p, RuntimeError):
            raise RuntimeError(f'{_where(i, path)}: {p} (a decoder bug)')
        if isinstance(p, (Parsed, FileLayout4)) and len(p.planes) == 4:
            if mode == 'RGB' and dtype != torch.uint8:
                raise ValueError(f"{_where(i, path)}: a four-component (CMYK or YCCK) file has an RGB conversion for "
                                 f"torch.uint8 only; use mode='UNCHANGED' for its four channels as {dtype}")
            if return_objective:
                raise ValueError(f'{_where(i, path)}: return_objective is not available for four-component (CMYK or YCCK) files')

    lib = abi.load_product()
    if not device_ok or lib.j2p_device_count() <= 0:
        raise RuntimeError('decode_jpeg needs a CUDA device: the solver has no CPU fallback')
    index = dev.index if dev.index is not None else torch.cuda.current_device()
    sample_bytes = _SAMPLE[dtype] // 8
    free = torch.cuda.mem_get_info(index)[0] if max_frames is None else 0
    # the rows a frame's sessions record (return_objective): per session, its iteration count
    if return_objective:
        def record_rows(k):
            nsolved = solved_planes(k, separate, mode)[0]
            return sum(flags[0][c] for c in range(nsolved)) if (separate or nsolved == 1) else flags[0][0]
        chunks = plan([p.key() for p in parsed],
                      lambda k: (min(int(max_frames), MAX_BATCH) if max_frames is not None else
                                 max(1, min(MAX_BATCH, free // 4 // frame_footprint(k, separate, sample_bytes, mode, record_rows(k))))))
    else:
        chunks = plan([p.key() for p in parsed],
                      lambda k: chunk_frames(k, separate, sample_bytes, max_frames, free, mode))

    # A chunk's arithmetic files are one device call, as long as the walk of their longest segment:
    # where the host reader is expected to be faster (arith_on_device) they are parsed there instead.
    # Their headers were read by the layout pass; errors in their entropy-coded data come here, before
    # any device work.
    to_host = []
    for _, idx in chunks:
        ari = [i for i in idx if isinstance(parsed[i], ArithFileLayout)]
        if ari and not arith_on_device([parsed[i] for i in ari], workers):
            to_host.extend(ari)
    if to_host:
        def host_parse(i):
            try:
                return parse_jpeg(read[i][0], read_flags)
            except ValueError as e:
                return e
        if min(workers, len(to_host)) > 1:
            with ThreadPoolExecutor(min(workers, len(to_host))) as pool:
                reparsed = list(pool.map(host_parse, to_host))
        else:
            reparsed = [host_parse(i) for i in to_host]
        for i, p in zip(to_host, reparsed):
            if isinstance(p, ValueError):
                raise ValueError(f'{_where(i, read[i][1])}: {p}')
            parsed[i] = p

    # packs of chunks iterated in one group; a pack of one chunk is solved as the chunk alone.  Groups
    # refuse recording sessions: with return_objective every chunk is solved alone.
    if _group_chunks and not return_objective:
        cap = (free if max_frames is None else torch.cuda.mem_get_info(index)[0]) // 4
        packs = pack(chunks, lambda k: group_class(k, separate, mode),
                     lambda k, n: n * frame_footprint(k, separate, sample_bytes, mode), cap)
    else:
        packs = [[j] for j in range(len(chunks))]

    results = [None] * len(parsed)
    logs = [None] * len(parsed)
    layout_id = _LAYOUT[layout]
    previous = []
    try:
        with torch.cuda.device(index):
            # the entropy decoder's own stream: waiting for a chunk's decode does not wait for the
            # solve of the chunk before it
            coef_stream = torch.cuda.Stream(index)

            def chunk_coefs(idx):
                coefs = {}
                for kind, decoder, failures in ((FileLayout, _DeviceCoefs, ENT_FAILURES), (FileLayout4, _DeviceCoefs4, ENT_FAILURES),
                                                (ProgFileLayout, _ProgCoefs, ENT_FAILURES),
                                                (ArithFileLayout, _ArithCoefs, ARITH_FAILURES)):
                    on_dev = [j for j, i in enumerate(idx) if isinstance(parsed[i], kind)]
                    if not on_dev:
                        continue
                    dc = decoder(index, [parsed[idx[j]] for j in on_dev], coef_stream)
                    for k, j in enumerate(on_dev):
                        if dc.status[k] != 0:
                            i = idx[j]
                            where = _where(i, read[i][1])
                            try:
                                (parse_jpeg4 if kind is FileLayout4 else parse_jpeg)(read[i][0], read_flags)
                            except ValueError as e:
                                raise ValueError(f'{where}: {e}') from None
                            raise RuntimeError(f'{where}: the device entropy decoder failed '
                                               f'({failures.get(int(dc.status[k]), int(dc.status[k]))}) on a file '
                                               'the host reader accepts (a decoder bug)')
                        coefs[j] = (dc, k)
                return coefs

            for p in packs:
                made = []
                try:
                    for j in p:
                        idx = chunks[j][1]
                        made.append(_Chunk(lib, index, [parsed[i] for i in idx], flags, separate, dtype, layout_id,
                                           chunk_coefs(idx), coef_stream, mode,
                                           None if orientations is None else [orientations[i] for i in idx],
                                           grouped=len(p) > 1, record=return_objective))
                    if len(p) > 1:
                        ss = [c.sessions[0] for c in made]
                        if lib.j2p_session_iterate_group((C.c_void_p * len(ss))(*ss), len(ss), 0, made[0].iterations) != 0:
                            raise RuntimeError(lib.j2p_last_error().decode())
                        for c in made:
                            c.export()
                except BaseException:
                    for c in made:
                        c.close()
                    raise
                for j, c in zip(p, made):
                    for k, i in enumerate(chunks[j][1]):
                        results[i] = c.frame(k)
                        if return_objective:
                            logs[i] = c.logs[k]
                for c in previous:              # this pack is queued: let the previous one finish
                    c.close()
                previous = made
    finally:
        for c in previous:
            c.close()
    if return_objective:
        return (results[0], logs[0]) if single else (results, logs)
    return results[0] if single else results


def _glibc_f(v: float) -> str:
    """v as glibc's printf("%f") prints it, NaN and infinity included."""
    if math.isnan(v):
        return '-nan' if math.copysign(1.0, v) < 0 else 'nan'
    if math.isinf(v):
        return '-inf' if v < 0 else 'inf'
    return '%f' % v


def write_objective_csv(file, names, logs):
    """Write the logs decode_jpeg(..., return_objective=True) returns as the command line's -c file:
    the header "filename,channel,iteration,objective,prob_dist,tv,tv2", then one row per file,
    channel and iteration, formatted "%s,%u,%u,%f,%f,%f,%f" (logger.c).  A file's rows are written
    together, its channels in order and each channel's iterations in order.

    file: a path or a text file object.  names: the filename column, one per log."""
    names, logs = list(names), list(logs)
    if len(names) != len(logs):
        raise ValueError(f'{len(names)} names for {len(logs)} logs')
    lines = ['filename,channel,iteration,objective,prob_dist,tv,tv2\n']
    for name, log in zip(names, logs):
        for channel in sorted(log):
            t = log[channel]
            rows = t.tolist() if hasattr(t, 'tolist') else list(t)
            for i, row in enumerate(rows):
                if len(row) != 4:
                    raise ValueError(f'a log row holds objective, prob_dist, tv, tv2; got {len(row)} values')
                lines.append(f'{name},{int(channel)},{i},' + ','.join(_glibc_f(float(v)) for v in row) + '\n')
    text = ''.join(lines)
    if hasattr(file, 'write'):
        file.write(text)
    else:
        with open(file, 'w', newline='') as f:
            f.write(text)
