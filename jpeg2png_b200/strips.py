"""Row-strip tiling of one frame over several ranks (SURVEY.md §8e, BASELINE config 4).

One process per GPU.  Every rank owns a horizontal strip of the frame, aligned to the tallest
coefficient block (8 * max h_samp rows).  The projection and the DCT-distance term are block-local,
so the only data that ever crosses ranks is

  * three fp64 numbers per rank and iteration — the strip's sums of g^2 — all-gathered and folded
    in RANK ORDER on every rank (deterministic, independent of the collective's internal order;
    reference semantics: one norm per channel over the whole frame, compute.c:200-216), and
  * the two rows of x_{k+1} on each side of every strip border, per channel and iteration
    (the stencil reach of the TV/TGV gather, SURVEY.md §8a): neighbour-only send/recv.

The orchestration below is backend-agnostic: on GPUs the backend is a strip session of
libjpeg2png_b200.so and torch.distributed runs over NCCL/NVLink; in the CPU tests the backend is
the oracle's strip interface and torch.distributed runs over gloo — same code path, world size 2.
"""
from __future__ import annotations

import ctypes as C

import numpy as np


def plan_strips(frame_h: int, mcu_rows: int, world: int):
    """Split `frame_h` rows into `world` strips of whole MCU rows (mcu_rows = 8 * max h_samp), as
    evenly as possible, larger strips first: [(row0, rows)] * world.  Raises if there are fewer MCU
    rows than ranks."""
    n_mcu = -(-frame_h // mcu_rows)
    if world > n_mcu:
        raise ValueError(f'{world} ranks but only {n_mcu} MCU rows of {mcu_rows} frame rows')
    base, extra = divmod(n_mcu, world)
    out, row = [], 0
    for r in range(world):
        m = base + (1 if r < extra else 0)
        rows = min(m * mcu_rows, frame_h - row)
        out.append((row, rows))
        row += rows
    assert row == frame_h
    return out


def plane_rows_of_strip(plane_h: int, h_samp: int, row0: int, rows: int):
    """Coefficient rows [cy0, cy1) of a plane that belong to frame rows [row0, row0+rows)."""
    cy0 = row0 // h_samp
    cy1 = min(-(-(row0 + rows) // h_samp), plane_h)
    return cy0, cy1


# ---------------------------------------------------------------------------------------------
# backends
# ---------------------------------------------------------------------------------------------
class _DevMem:
    """Zero-copy view of device memory for torch.as_tensor (CUDA array interface v2)."""

    def __init__(self, ptr, count, typestr):
        self.__cuda_array_interface__ = {'shape': (count,), 'typestr': typestr, 'data': (int(ptr), False), 'version': 2}


class ProductStrip:
    """A strip session of libjpeg2png_b200.so (GPU).  The channel count is the frame's (1..3).
    fdata: None to decode on the device, else the caller's conventional decode of the WHOLE frame
    (one (h, w) float32 array per plane); the strip's coefficient rows are sliced from it."""

    def __init__(self, lib, img, weight, pweight, iterations, row0, rows, device, fdata=None):
        import torch
        from . import abi
        self.torch, self.lib, self.nc = torch, lib, len(img.planes)
        d = abi.FrameDesc()
        d.nchannel = self.nc
        for c, p in enumerate(img.planes):
            d.plane_w[c], d.plane_h[c], d.w_samp[c], d.h_samp[c] = p.w, p.h, p.w_samp, p.h_samp
            d.pweight[c] = pweight[c]
        d.weight = weight
        d.iterations = iterations
        s = C.c_void_p()
        if lib.j2p_session_create_strip(C.byref(s), device, C.byref(d), row0, rows) != 0:
            raise RuntimeError(lib.j2p_last_error().decode())
        self.s = s
        for c, p in enumerate(img.planes):
            cy0, cy1 = plane_rows_of_strip(p.h, p.h_samp, row0, rows)
            bw = p.w // 8
            data = np.ascontiguousarray(p.data.reshape(-1, 64)[(cy0 // 8) * bw:(cy1 // 8) * bw].reshape(-1))
            quant = np.ascontiguousarray(p.quant)
            fd = None if fdata is None else np.ascontiguousarray(fdata[c][cy0:cy1], dtype=np.float32)
            if lib.j2p_session_upload(s, c, data.ctypes.data, quant.ctypes.data, None if fd is None else fd.ctypes.data) != 0:
                raise RuntimeError(lib.j2p_last_error().decode())
        self.width = lib.j2p_session_width(s)
        owned = C.c_uint()
        lib.j2p_session_strip_info(s, None, None, C.byref(owned))
        self.owned_rows = owned.value
        self.stream = torch.cuda.ExternalStream(lib.j2p_session_stream(s), device=torch.device('cuda', device))
        self.device = torch.device('cuda', device)
        self._views = {}

    def _view(self, ptr, count, typestr):
        key = (ptr, count, typestr)
        t = self._views.get(key)
        if t is None:
            t = self.torch.as_tensor(_DevMem(ptr, count, typestr), device=self.device)
            self._views[key] = t
        return t

    def gradient(self):
        if self.lib.j2p_session_gradient(self.s) != 0:
            raise RuntimeError(self.lib.j2p_last_error().decode())
        return self._view(self.lib.j2p_session_sums_ptr(self.s), 3, '<f8')

    def new_gather_buffer(self, world):
        return self.torch.zeros(3 * world, dtype=self.torch.float64, device=self.device)

    def project(self, gathered, world):
        if self.lib.j2p_session_project(self.s, gathered.data_ptr(), world) != 0:
            raise RuntimeError(self.lib.j2p_last_error().decode())

    def halo(self, c, side):
        send, recv, count = C.c_void_p(), C.c_void_p(), C.c_size_t()
        self.lib.j2p_session_halo(self.s, c, side, C.byref(send), C.byref(recv), C.byref(count))
        if count.value == 0:
            return None
        return self._view(send.value, count.value, '<f4'), self._view(recv.value, count.value, '<f4')

    def copy_halo_to_prev(self):
        self.lib.j2p_session_copy_halo_to_prev(self.s)

    def download(self, c):
        out = np.empty((self.owned_rows, self.width), np.float32)
        if self.lib.j2p_session_download(self.s, c, out.ctypes.data) != 0:
            raise RuntimeError(self.lib.j2p_last_error().decode())
        return out

    def stream_context(self):
        return self.torch.cuda.stream(self.stream)

    def close(self):
        self.lib.j2p_session_destroy(self.s)


# ---------------------------------------------------------------------------------------------
# orchestration
# ---------------------------------------------------------------------------------------------
def exchange_halos(backend, dist, rank, world, nchannel=3):
    """Neighbour-only exchange of the two border rows of the current iterate, all channels."""
    ops = []
    for c in range(nchannel):
        for side, peer in ((0, rank - 1), (1, rank + 1)):
            if peer < 0 or peer >= world:
                continue
            h = backend.halo(c, side)
            if h is None:
                continue
            send, recv = h
            ops.append(dist.P2POp(dist.isend, send, peer))
            ops.append(dist.P2POp(dist.irecv, recv, peer))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()


def solve_strips(backend, dist, rank, world, iterations, nchannel=3):
    """Run `iterations` solver iterations on this rank's strip.  Collective: every rank calls it."""
    with backend.stream_context():
        gathered = backend.new_gather_buffer(world)
        # halo rows of the initial iterate (aux_init only fills owned rows), x_{-1} = x_0
        exchange_halos(backend, dist, rank, world, nchannel)
        backend.copy_halo_to_prev()
        for _ in range(iterations):
            sums = backend.gradient()
            if world > 1:
                dist.all_gather_into_tensor(gathered, sums)
            else:
                gathered.copy_(sums)
            backend.project(gathered, world)
            exchange_halos(backend, dist, rank, world, nchannel)


def native_comm(backend, dist, rank, world):
    """An NCCL communicator owned by libjpeg2png_b200.so for the native strip loop.  The 128-byte
    NCCL id is made on rank 0 and handed round with torch.distributed (any backend)."""
    import torch
    lib = backend.lib
    buf = (C.c_ubyte * 128)()
    if rank == 0 and lib.j2p_comm_unique_id(buf, 128) != 0:
        raise RuntimeError(lib.j2p_last_error().decode())
    ids = [bytes(buf)]
    if world > 1:
        dist.broadcast_object_list(ids, src=0)
    raw = (C.c_ubyte * 128).from_buffer_copy(ids[0])
    comm = C.c_void_p()
    if lib.j2p_comm_create(C.byref(comm), backend.device.index, world, rank, raw, 128) != 0:
        raise RuntimeError(lib.j2p_last_error().decode())
    return comm


def solve_strips_native(backend, comm, iterations):
    """`iterations` solver iterations of this rank's strip, both exchanges queued by the library on
    the session stream through NCCL (j2p_session_iterate_strip).  Collective; asynchronous."""
    if backend.lib.j2p_session_iterate_strip(backend.s, comm, iterations) != 0:
        raise RuntimeError(backend.lib.j2p_last_error().decode())
