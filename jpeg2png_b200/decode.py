"""decode_jpeg: JPEG files in, RGB CUDA tensors out, through the solver.

Every input is parsed on the host with the JPEG coefficient reader of the command line
(libj2pcodecs.so, j2p_read_jpeg_mem) before any device work.  Inputs of one geometry are solved
together in batch sessions (j2p_session_create_batch), with the conventional decode on the device as
the command line does it, and the colour conversion writes straight into one freshly allocated tensor
per chunk (j2p_session_export) on the caller's current stream.  The returned tensors of a chunk are
views of that tensor and share its storage.

The samples are those of the PNG the command line writes for the same file and flags:
torch.uint8 the 8-bit PNG samples, torch.uint16 the 16-bit (-1) samples in native byte order,
torch.float32 the clamped value before truncation.  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
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


class Jpeg(C.Structure):
    """struct j2p_jpeg — jpeg2png_b200/cli/jpeg_reader.h."""
    _fields_ = [('w', C.c_uint), ('h', C.c_uint), ('coefs', abi.Coef * 3)]


_codecs = None


def load_codecs() -> C.CDLL:
    """libj2pcodecs.so (the command line's JPEG reader) from the package tree."""
    global _codecs
    if _codecs is None:
        if not os.path.exists(CODECS_LIB):
            raise RuntimeError(f'{CODECS_LIB} is missing: the command line has not been built '
                               '(run `python -c "import __graft_entry__ as g; g.build()"`)')
        lib = C.CDLL(CODECS_LIB, mode=C.RTLD_LOCAL)
        lib.j2p_read_jpeg_mem.restype = C.c_int
        lib.j2p_read_jpeg_mem.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(Jpeg), C.c_char_p, C.c_size_t]
        _codecs = lib
    return _codecs


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
    """One parsed JPEG: the visible size and its three coefficient planes."""
    w: int
    h: int
    planes: list

    def key(self):
        """Inputs with equal keys are solved in one batch session."""
        return (self.w, self.h, tuple((p.w, p.h, p.w_samp, p.h_samp) for p in self.planes))


def parse_jpeg(data: bytes) -> Parsed:
    """Parse JPEG bytes with j2p_read_jpeg_mem; ValueError carries the reader's message."""
    lib = load_codecs()
    j = Jpeg()
    err = C.create_string_buffer(256)
    if lib.j2p_read_jpeg_mem(data, len(data), C.byref(j), err, 256) != 0:
        raise ValueError(err.value.decode(errors='replace'))
    planes = []
    for c in j.coefs:
        n = c.w * c.h
        d = np.ctypeslib.as_array(c.data, shape=(n,)).copy() if n else np.zeros(0, np.int16)
        abi.free_ptr(c.data)
        planes.append(Plane(int(c.w), int(c.h), int(c.w_samp), int(c.h_samp), d, np.array(list(c.quant_table), np.uint16)))
    return Parsed(int(j.w), int(j.h), planes)


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


def frame_footprint(key, separate: bool, sample_bytes: int) -> int:
    """Estimated device bytes one frame of `key` takes in its batch session(s) (DESIGN §4: x, xp, g,
    gp at frame size per plane; coefficients int16 and the conventional decode fp32 at plane size;
    the reduction state) plus its part of the output tensor."""
    w, h, planes = key

    def session(pl):
        W = max(pw * ws for pw, ph, ws, hs in pl)
        H = max(ph * hs for pw, ph, ws, hs in pl)
        ps = (W * H + 63) // 64 * 64
        n = 4 * 4 * ps * len(pl)
        for pw, ph, ws, hs in pl:
            n += (pw * ph + 127) // 128 * 128 * 2 + (pw * ph + 63) // 64 * 64 * 4
        return n + (16 << 10)

    total = sum(session([p]) for p in planes) if separate else session(list(planes))
    return total + w * h * 3 * sample_bytes


def chunk_frames(key, separate: bool, sample_bytes: int, max_frames, free_bytes: int) -> int:
    """Frames per batch of `key`: max_frames, or as many as keep the estimated footprint of two
    chunks in flight (one solving while the next is uploaded) under half of `free_bytes`."""
    if max_frames is not None:
        return min(int(max_frames), MAX_BATCH)
    per = frame_footprint(key, separate, sample_bytes)
    return max(1, min(MAX_BATCH, free_bytes // 4 // per))


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


class _Chunk:
    """The batch session(s) of one chunk: created, uploaded, iterated and exported by the
    constructor; close() waits for them and returns their blocks to the device cache."""

    def __init__(self, lib, device, items, flags, separate, dtype, layout):
        iters, weights, pweights = flags
        self.lib, self.sessions = lib, []
        first, n = items[0], len(items)
        if separate:
            work = [(_frame_desc(first, [c], weights[c], pweights, iters[c]), [c], iters[c]) for c in range(3)]
        else:
            work = [(_frame_desc(first, [0, 1, 2], weights[0], pweights, iters[0]), [0, 1, 2], iters[0])]
        try:
            for desc, _, _ in work:
                s = C.c_void_p()
                self._check(lib.j2p_session_create_batch(C.byref(s), device, C.byref(desc), n))
                self.sessions.append(s)
            for s, (_, channels, it) in zip(self.sessions, work):
                for f, parsed in enumerate(items):
                    for k, c in enumerate(channels):
                        p = parsed.planes[c]
                        self._check(lib.j2p_session_upload(s, f * len(channels) + k, p.data.ctypes.data,
                                                           p.quant.ctypes.data, None))     # conventional decode on the device
                self._check(lib.j2p_session_iterate(s, 0, it))
            w, h = first.w, first.h
            shape = (n, 3, h, w) if layout == abi.LAYOUT_CHW else (n, h, w, 3)
            self.out = torch.empty(shape, dtype=dtype, device=torch.device('cuda', device))
            o = abi.ImageOut(w, h, _SAMPLE[dtype], layout, 3 * h * w * self.out.element_size())
            # torch's default stream is handle 0, which the ABI reads as "the session stream":
            # name it cudaStreamLegacy (1) instead
            stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream or 1)
            dst = C.c_void_p(self.out.data_ptr())
            if separate:
                self._check(lib.j2p_session_export_separate(*self.sessions, 0, n, C.byref(o), dst, stream))
            else:
                self._check(lib.j2p_session_export(self.sessions[0], 0, n, C.byref(o), dst, stream))
        except BaseException:
            self.close()
            raise

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(self.lib.j2p_last_error().decode())

    def close(self):
        for s in self.sessions:
            self.lib.j2p_session_destroy(s)
        self.sessions = []


def decode_jpeg(inputs, *, iterations=50, weight=0.3, pweight=0.001, separate=False,
                dtype=torch.uint8, layout='CHW', device=None, max_frames=None):
    """Decode JPEG files into RGB tensors on a CUDA device, deblocked by the solver.

    inputs: bytes-like, a path (str / os.PathLike), or a list or tuple of them.  A single input
    returns one tensor, a list returns a list in input order.  Each tensor is (3, h, w) for
    layout='CHW' or (h, w, 3) for 'HWC' at the image's visible size, on `device` (default: the
    current CUDA device).  dtype: torch.uint8 (the 8-bit PNG samples), torch.uint16 (the 16-bit
    PNG samples) or torch.float32 (the clamped samples before truncation).

    iterations, weight, pweight, separate: the command line's -i, -w, -p and -s.  Scalars as there:
    a scalar weight sets luma only; three weights or three iteration counts need separate=True.

    Inputs with the same geometry are solved together, max_frames per batch (default: as many as
    fit in a quarter of the free device memory).  The tensors of one batch are views of one
    allocation and share its storage.  The result is written on the current torch stream and can
    be used there without synchronising.  Raises ValueError for bad arguments and unreadable
    files (before any device work) and RuntimeError when no CUDA device is usable.
    """
    flags = solver_flags(iterations, weight, pweight, separate)
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
        return []

    def parse(data):
        try:
            return parse_jpeg(data)
        except ValueError as e:
            return e

    # the reader runs without the GIL (ctypes): a 1080p file takes about as long to parse on the host
    # as to solve on the device, so many files are parsed in parallel
    workers = min(len(read), os.cpu_count() or 1, 16)
    if workers > 1:
        with ThreadPoolExecutor(workers) as pool:
            parsed = list(pool.map(parse, [data for data, _ in read]))
    else:
        parsed = [parse(data) for data, _ in read]
    for i, (p, (_, path)) in enumerate(zip(parsed, read)):
        if isinstance(p, ValueError):
            where = f'input {i} ({path})' if path is not None else f'input {i}'
            raise ValueError(f'{where}: {p}')

    lib = abi.load_product()
    if not torch.cuda.is_available() or lib.j2p_device_count() <= 0:
        raise RuntimeError('decode_jpeg needs a CUDA device: the solver has no CPU fallback')
    index = dev.index if dev.index is not None else torch.cuda.current_device()
    sample_bytes = _SAMPLE[dtype] // 8
    free = torch.cuda.mem_get_info(index)[0] if max_frames is None else 0
    chunks = plan([p.key() for p in parsed],
                  lambda k: chunk_frames(k, separate, sample_bytes, max_frames, free))

    results = [None] * len(parsed)
    layout_id = _LAYOUT[layout]
    previous = None
    try:
        with torch.cuda.device(index):
            for _, idx in chunks:
                chunk = _Chunk(lib, index, [parsed[i] for i in idx], flags, separate, dtype, layout_id)
                for j, i in enumerate(idx):
                    results[i] = chunk.out[j]
                if previous is not None:        # this chunk is queued: let the previous one finish
                    previous.close()
                previous = chunk
    finally:
        if previous is not None:
            previous.close()
    return results[0] if single else results
