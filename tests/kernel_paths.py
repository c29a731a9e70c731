"""The host's kernel choice, restated in Python (no GPU, no library needed).

Given a frame (its planes' coefficient grids and sampling factors, the TGV weight) and a mode
(single session or a batch of N frames, objective logging, the J2P_GRAD_SCALAR / J2P_PROJ_TILE22 /
J2P_PROJ_TMA switches), this says which kernel instantiations one solver iteration launches and
how many launches that is.  `Mode.strip` restates a row-strip session (j2p_session_create_strip):
the same frame can launch a different gradient instantiation, group its 1x1 planes differently and
need stepped-only launches in one strip and not in another.  It follows jpeg2png_b200/csrc:

  launch_gradient / launch_gradient_packed   kernels_gradient.cu, kernels_gradient_packed.cu
  launch_project                             kernels_project.cu
  launch_project_tile / launch_project_tile22  kernels_project_tile.cu, kernels_project_tile22.cu
  grad_geometry                              kernels_gradient.cu

Names are the demangled kernel names as `cuobjdump` + `cu++filt` print them, without namespace
and arguments, and with `(int)` / `(bool)` casts dropped: `k_project<2, 1>`,
`k_gradient_packed<3, true, 0, false>`.  tests/test_kernel_coverage.py checks that the matrix
of tests/test_gpu_kernel_matrix.py reaches every kernel in the library; the matrix checks the
launch counts predicted here against `j2p_session_launches` on the GPU.
"""
from __future__ import annotations

import dataclasses
import os
import re
import shutil
import subprocess

GM_USE = 60          # output columns of one warp strip of the gradient kernel (gradient_common.cuh)
GM_WARPS = 4         # warps per gradient CTA: 240 output columns
# Resident CTAs per SM of the packed gradient kernel as documented in DESIGN.md: 2 for the
# three-channel joint builds, 5 for the one-channel builds.  The real figure is the occupancy of
# each instantiation (resident_ctas); the GPU matrix sizes its tall frames from that and from the
# device's SM count, these figures only name the cases where no device is at hand.
GRAD_CTAS_PER_SM = {1: 5, 3: 2}
H100_SMS = 132


@dataclasses.dataclass(frozen=True)
class PlaneGeom:
    cw: int          # coefficient grid in samples (multiple of 8)
    ch: int
    sw: int          # sampling factors of the plane (struct coef w_samp / h_samp)
    sh: int


@dataclasses.dataclass(frozen=True)
class Mode:
    nframes: int = 1             # 1: j2p_session_create; > 1: a batch session of that many frames
    log: bool = False            # objective logging (-c csv); refused on a batch
    grad_scalar: bool = False    # J2P_GRAD_SCALAR=1
    tile22: bool = True          # J2P_PROJ_TILE22 (0 turns it off)
    tma: bool = False            # J2P_PROJ_TMA=1
    device_decode: bool = False  # uploads without the caller's conventional decode (k_decode)
    strip: tuple | None = None   # (row0, rows): a strip session of frame rows [row0, row0 + rows)


def frame_size(planes):
    """Frame W x H (compute.c:410-416): the largest plane footprint."""
    return max(p.cw * p.sw for p in planes), max(p.ch * p.sh for p in planes)


def strip_rows(p: PlaneGeom, row0: int, rows: int) -> int:
    """Coefficient rows of plane p a strip of frame rows [row0, row0 + rows) holds
    (session.cu create_impl; strips.plane_rows_of_strip)."""
    return min(-(-(row0 + rows) // p.sh), p.ch) - row0 // p.sh


def local(planes, mode: Mode):
    """(planes as the session holds them, W, rows the solver kernels target).  A strip session holds
    the coefficient rows of its strip and targets its owned rows; a whole frame is its own strip."""
    W, H = frame_size(planes)
    if mode.strip is None:
        return tuple(planes), W, H
    row0, rows = mode.strip
    return tuple(PlaneGeom(p.cw, strip_rows(p, row0, rows), p.sw, p.sh) for p in planes), W, rows


def _b(v: bool) -> str:
    return 'true' if v else 'false'


def gradient_kernel(planes, weight, mode: Mode) -> str:
    """launch_gradient: the packed kernel unless logging or J2P_GRAD_SCALAR (single sessions only).
    In a strip the predicates see the strip's coefficient rows and its owned rows."""
    nc = len(planes)
    tgv = weight != 0.0
    planes, W, H = local(planes, mode)
    if not mode.log and (not mode.grad_scalar or mode.nframes > 1):
        full = all(p.sw == 1 and p.sh == 1 and p.cw == W and p.ch >= H for p in planes)
        c420 = (nc == 3 and planes[0].sw == 1 and planes[0].sh == 1 and planes[0].cw == W and
                all(p.sw == 2 and p.sh == 2 and 2 * p.cw == W and p.ch == planes[1].ch for p in planes[1:]))
        if full:
            return f'k_gradient_packed<{nc}, {_b(tgv)}, 1, {_b(mode.nframes > 1)}>'
        if c420:
            return f'k_gradient_packed<3, {_b(tgv)}, 2, {_b(mode.nframes > 1)}>'
        return f'k_gradient_packed<{nc}, {_b(tgv)}, 0, {_b(mode.nframes > 1)}>'
    return f'k_gradient<{nc}, {_b(mode.log)}, {_b(tgv)}>'


def projection_kernels(planes, mode: Mode):
    """launch_project: the launches of one projection, in order (a list of kernel names).  In a
    strip, grouping and the stepped-only launches go by the strip's coefficient rows and owned rows;
    `resample` stays the whole frame's."""
    _, Wf, Hf = local(planes, Mode())
    whole = planes
    planes, W, H = local(planes, mode)
    batch = mode.nframes > 1
    tma = mode.tma and not batch        # a batch has no tensor maps (session.cu)
    out = []
    c = 0
    while c < len(planes):
        P = planes[c]
        resample = not (whole[c].cw == Wf and whole[c].ch == Hf)
        if mode.log and (P.sw, P.sh) == (1, 1):
            out.append('k_project<1, 1>')              # one launch per plane, no grouping
            c += 1
            continue
        if (P.sw, P.sh) == (1, 1):
            count = 1
            while c + count < len(planes) and planes[c + count] == PlaneGeom(P.cw, P.ch, 1, 1):
                count += 1
            if tma:
                out.append(f'k_project_tma<{_b(resample)}>')
            else:
                out.append(f'k_project_tile<{_b(resample)}, {_b(batch)}>')
            for k in range(c, c + count):
                if planes[k].cw < W or planes[k].ch < H:
                    out.append(f'k_step_uncovered<{_b(batch)}>')
            c += count
            continue
        if (P.sw, P.sh) == (2, 2) and mode.tile22 and not mode.log:
            count = 1
            while c + count < len(planes) and planes[c + count] == PlaneGeom(P.cw, P.ch, 2, 2):
                count += 1
            out.append(f'k_project_tile22<{_b(batch)}>')
            for k in range(c, c + count):
                if 2 * planes[k].cw < W or 2 * planes[k].ch < H:
                    out.append(f'k_step_uncovered22<{_b(batch)}>')
            c += count
            continue
        if (P.sw, P.sh) in ((2, 2), (2, 1), (1, 2)):
            name = f'k_project<{P.sw}, {P.sh}>'
        else:
            name = 'k_project<0, 0>'
        out.extend([name] * mode.nframes)              # one launch per frame of a batch
        c += 1
    return out


def iteration(planes, weight, mode: Mode = Mode()):
    """(kernel names launched by one iteration in order, number of launches).  A strip iteration
    folds the ranks' sums (k_fold_sums, j2p_session_project) between the two halves."""
    fold = ['k_fold_sums'] if mode.strip is not None else []
    ks = [gradient_kernel(planes, weight, mode)] + fold + projection_kernels(planes, mode)
    return ks, len(ks)


def setup(planes, mode: Mode = Mode()):
    """(kernel names, launches) of uploading every plane of every frame and arming the session:
    k_decode per uploaded plane without a caller decode, k_init_plane per plane and frame."""
    n = len(planes) * mode.nframes
    ks = (['k_decode'] * n if mode.device_decode else []) + ['k_init_plane'] * n
    return ks, len(ks)


def grad_geometry(W: int, H: int, slots: int):
    """kernels_gradient.cu grad_geometry: (CTAs across, bands, rows per band)."""
    strips = -(-W // GM_USE)
    ctas_x = -(-strips // GM_WARPS)
    if slots <= 0:
        slots = H100_SMS * 3
    want = max(1, slots // ctas_x)
    rows = max(8, -(-H // want))
    return ctas_x, -(-H // rows), rows


def last_band_rows(W: int, H: int, slots: int) -> int:
    _, bands, rows = grad_geometry(W, H, slots)
    return H - (bands - 1) * rows


def short_last_band_heights(W: int, per_sm_options, lo: int, hi: int, sms: int = H100_SMS):
    """Frame heights in [lo, hi] (multiples of 16) whose last gradient band is 1..7 rows for
    every per-SM CTA count in per_sm_options."""
    return [H for H in range(lo - lo % 16, hi + 1, 16) if H >= lo and
            all(1 <= last_band_rows(W, H, sms * k) <= 7 for k in per_sm_options)]


def resident_ctas(regs: int, shared: int, threads: int = 128) -> int:
    """CTAs of one kernel resident per SM of an sm_90 device, as cudaOccupancyMaxActiveBlocksPerMultiprocessor
    counts them: 64K registers allocated per warp in units of 256, 228 KB of shared memory (`shared`
    as cuobjdump -res-usage prints it, the 1 KB reserved per CTA included), 2048 threads, 32 CTAs."""
    per_warp = -(-regs * 32 // 256) * 256
    by_regs = (65536 // per_warp) // (threads // 32)
    by_smem = 233472 // shared if shared else 32
    return min(by_regs, by_smem, 2048 // threads, 32)


def normalise(demangled: str) -> str:
    """'void j2p::k_project<(int)2, (int)1>(j2p::FrameDev, ...)' -> 'k_project<2, 1>'."""
    s = re.sub(r'^j2p::', '', re.sub(r'^void ', '', demangled.strip()))
    m = re.match(r'(\w+)(<[^>]*>)?\(', s)
    assert m, demangled
    targs = (m.group(2) or '').replace('(int)', '').replace('(bool)0', 'false').replace('(bool)1', 'true')
    return m.group(1) + targs


def library_resources(lib_path: str):
    """{kernel name: (registers, shared bytes)} of every kernel in a library, from cuobjdump -res-usage;
    None where the CUDA toolkit or the library is missing."""
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump) or not os.path.exists(lib_path):
        return None
    filt = os.path.join(os.path.dirname(cuobjdump), 'cu++filt')
    if not os.path.exists(filt):
        filt = shutil.which('cu++filt') or shutil.which('c++filt')
    txt = subprocess.run([cuobjdump, '-res-usage', lib_path], check=True, capture_output=True, text=True).stdout
    found = re.findall(r'Function (_Z\w+):\s*\n\s*REG:(\d+) STACK:\d+ SHARED:(\d+)', txt)
    names = subprocess.run([filt], input='\n'.join(m for m, _, _ in found) + '\n', check=True, capture_output=True,
                           text=True).stdout.splitlines()
    return {normalise(n): (int(r), int(sh)) for n, (_, r, sh) in zip(names, found)}
