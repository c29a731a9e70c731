"""CPU strip backend for jpeg2png_b200.strips: the oracle's strip interface behind the same
methods as ProductStrip, so the orchestration (all-gather of the sums, halo exchange) can run
under gloo with world size 2 on a machine without GPUs."""
import contextlib
import ctypes as C

import numpy as np
import torch

from jpeg2png_b200.strips import plane_rows_of_strip
from tests import helpers as H


def _lib():
    lib = H.load_oracle()
    U3 = C.POINTER(C.c_uint)
    lib.oracle_strip_create.restype = C.c_void_p
    lib.oracle_strip_create.argtypes = [C.c_uint, U3, U3, U3, U3, C.c_float, C.POINTER(C.c_float), C.c_uint, C.c_uint, C.c_uint]
    lib.oracle_strip_destroy.argtypes = [C.c_void_p]
    lib.oracle_strip_width.restype = C.c_uint
    lib.oracle_strip_width.argtypes = [C.c_void_p]
    lib.oracle_strip_owned_rows.restype = C.c_uint
    lib.oracle_strip_owned_rows.argtypes = [C.c_void_p]
    lib.oracle_strip_upload.argtypes = [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.oracle_strip_gradient.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.oracle_strip_project.argtypes = [C.c_void_p, C.c_void_p, C.c_uint]
    lib.oracle_strip_halo.restype = C.c_void_p
    lib.oracle_strip_halo.argtypes = [C.c_void_p, C.c_uint, C.c_int, C.c_int, C.POINTER(C.c_size_t)]
    lib.oracle_strip_copy_halo_to_prev.argtypes = [C.c_void_p]
    lib.oracle_strip_download.argtypes = [C.c_void_p, C.c_uint, C.c_void_p]
    return lib


class OracleStrip:
    """The channel count is the frame's (1..3); fdata_full: the conventional decode of the whole frame."""

    def __init__(self, img, weight, pweight, iterations, row0, rows, fdata_full):
        self.lib = _lib()
        n = self.nc = len(img.planes)
        arr = lambda vals: (C.c_uint * 3)(*vals)
        pw = (C.c_float * 3)(*pweight)
        self.s = self.lib.oracle_strip_create(n, arr([p.w for p in img.planes]), arr([p.h for p in img.planes]),
                                              arr([p.w_samp for p in img.planes]), arr([p.h_samp for p in img.planes]),
                                              C.c_float(weight), pw, iterations, row0, rows)
        for c, p in enumerate(img.planes):
            cy0, cy1 = plane_rows_of_strip(p.h, p.h_samp, row0, rows)
            bw = p.w // 8
            data = np.ascontiguousarray(p.data.reshape(-1, 64)[(cy0 // 8) * bw:(cy1 // 8) * bw].reshape(-1))
            quant = np.ascontiguousarray(p.quant)
            fd = np.ascontiguousarray(fdata_full[c][cy0:cy1])
            self.lib.oracle_strip_upload(self.s, c, data.ctypes.data, quant.ctypes.data, fd.ctypes.data)
        self.width = self.lib.oracle_strip_width(self.s)
        self.owned_rows = self.lib.oracle_strip_owned_rows(self.s)
        self._sums = np.zeros(3, np.float64)

    def gradient(self):
        self.lib.oracle_strip_gradient(self.s, self._sums.ctypes.data, None)
        return torch.from_numpy(self._sums)

    def new_gather_buffer(self, world):
        return torch.zeros(3 * world, dtype=torch.float64)

    def project(self, gathered, world):
        g = np.ascontiguousarray(gathered.numpy())
        self.lib.oracle_strip_project(self.s, g.ctypes.data, world)

    def halo(self, c, side):
        cnt = C.c_size_t()
        send = self.lib.oracle_strip_halo(self.s, c, side, 0, C.byref(cnt))
        if not send or cnt.value == 0:
            return None
        recv = self.lib.oracle_strip_halo(self.s, c, side, 1, C.byref(cnt))
        mk = lambda p: torch.from_numpy(np.ctypeslib.as_array((C.c_float * cnt.value).from_address(p)))
        return mk(send), mk(recv)

    def copy_halo_to_prev(self):
        self.lib.oracle_strip_copy_halo_to_prev(self.s)

    def download(self, c):
        out = np.empty((self.owned_rows, self.width), np.float32)
        self.lib.oracle_strip_download(self.s, c, out.ctypes.data)
        return out

    def stream_context(self):
        return contextlib.nullcontext()

    def close(self):
        self.lib.oracle_strip_destroy(self.s)


# ---------------------------------------------------------------------------------------------
# lock-step driver: every strip of a frame in one process (and, for product strips, on one device)
# ---------------------------------------------------------------------------------------------
def cuts_to_strips(frame_h, cuts):
    """Explicit cut rows (strictly increasing, inside the frame) -> [(row0, rows)]."""
    edges = [0] + list(cuts) + [frame_h]
    assert all(a < b for a, b in zip(edges, edges[1:])), f'bad cuts {cuts} for {frame_h} rows'
    return [(a, b - a) for a, b in zip(edges, edges[1:])]


class LockStep:
    """Drives N strips of one frame through the iteration the ranks of strips.solve_strips run, but
    from one process: the sums are gathered in rank order into one fp64 buffer, the border rows are
    copied between neighbours directly.  `sync` is called at every exchange (a full device sync for
    product strips: ordering must not be in doubt; nothing for oracle strips).  The sessions are
    never bound to a communicator, so their kernels never wait on flags."""

    def __init__(self, strips, sync=lambda: None, device=None):
        self.strips, self.sync, self.device = strips, sync, device
        self.nc = strips[0].nc

    def exchange(self):
        """Border rows of the current iterate into the neighbours' halo rows.  The pointers are
        queried again every time: the iterate buffers swap with every projection."""
        self.sync()
        for upper, lower in zip(self.strips, self.strips[1:]):
            for c in range(self.nc):
                up, lo = upper.halo(c, 1), lower.halo(c, 0)
                assert up is not None and lo is not None, 'neighbouring strips without halo rows'
                lo[1].copy_(up[0])
                up[1].copy_(lo[0])
        self.sync()

    def start(self):
        """After (re)arming: halo rows of the initial iterate, then x_{-1} = x_0 there too."""
        self.exchange()
        for s in self.strips:
            s.copy_halo_to_prev()
        self.sync()

    def gradient(self):
        """First half of an iteration on every strip: the sums of g^2 in rank order, [3 * N] fp64
        on the strips' device (a copy: the strips' own sums buffers are rewritten next iteration)."""
        sums = [s.gradient() for s in self.strips]
        self.sync()
        gathered = torch.cat(sums)
        self.sync()
        return gathered

    def project(self, gathered):
        """Second half on every strip with the given rank-ordered sums, then the halo exchange."""
        g = gathered.to(self.device) if self.device is not None else gathered
        self.sync()
        for s in self.strips:
            s.project(g, len(self.strips))
        self.exchange()

    def download(self):
        """The owned rows of every strip, concatenated: one (H, W) array per plane."""
        self.sync()
        return [np.concatenate([s.download(c) for s in self.strips], axis=0) for c in range(self.nc)]


def fold(gathered, nranks, c):
    """sqrtf((float)sum) of channel c over the ranks' sums, added in rank order from 0 as
    k_fold_sums and oracle_strip_project add them."""
    s = 0.0
    for r in range(nranks):
        s += float(gathered[3 * r + c])
    return np.sqrt(np.float32(s), dtype=np.float32)
