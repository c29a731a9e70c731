"""What encode_png and encode_jpeg share (DESIGN §7e, §7f): the argument checks, the image
descriptors, the split of a list into calls whose work areas fit in a quarter of the free device
memory, the loop of device calls with the pinned read-back of the files, and the host-driver
wrapper.  An encoder describes its library with a Codec.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Callable

import numpy as np
import torch


@dataclass(frozen=True)
class Codec:
    """An encoder library as the driver sees it: j2p_<name>_plan, _encode, _encode_host and
    _last_error, which take `params` after the image count.

    image: the ctypes image struct (data, width, height and row, column and channel strides);
    check_size(shape, h, w): raises ValueError for a size the encoder refuses;
    fill(d, x, channels): sets the struct's other fields from the array or tensor x and its channel
    count, if it has any;
    channels: the channel counts the encoder accepts, in the order its messages name them;
    place(descs): sets fields of the call's structs that depend on each image's place in the call
    (the JPEG encoder's set of quantisation tables), if it has any."""
    name: str
    load: Callable[[], C.CDLL]
    image: type
    check_size: Callable
    fill: Callable | None = None
    params: tuple = ()
    channels: tuple = (3,)
    place: Callable | None = None

    def call(self, fn, descs, *args, error=RuntimeError):
        """j2p_<name>_<fn>(descs, len(descs), *params, *args); `error` with the library's message
        when it fails."""
        lib = self.load()
        if getattr(lib, f'j2p_{self.name}_{fn}')(descs, len(descs), *self.params, *args) != 0:
            raise error(getattr(lib, f'j2p_{self.name}_last_error')().decode())

    def plan(self, descs):
        """(work bytes, offset of the files in the work area) of one call on descs.  The plan
        refuses only what the arguments make impossible: a ValueError."""
        n, o = C.c_size_t(), C.c_size_t()
        self.call('plan', descs, C.byref(n), C.byref(o), error=ValueError)
        return n.value, o.value


def check_layout(layout):
    if layout not in ('CHW', 'HWC'):
        raise ValueError(f"layout must be 'CHW' or 'HWC', not {layout!r}")


def axes(shape, layout, channels=(3,)):
    """(h, w, row axis, column axis, channel axis) of a (c, h, w) CHW or (h, w, c) HWC shape, c one
    of `channels`."""
    if len(shape) != 3:
        raise ValueError(f'an image is 3-dimensional, (3, h, w) or (h, w, 3); got shape {tuple(shape)}')
    if layout == 'CHW':
        if shape[0] not in channels:
            wanted = ' or '.join(f'({c}, h, w)' for c in channels)
            raise ValueError(f"layout 'CHW' wants shape {wanted}; got {tuple(shape)}")
        return shape[1], shape[2], 1, 2, 0
    if shape[2] not in channels:
        wanted = ' or '.join(f'(h, w, {c})' for c in channels)
        raise ValueError(f"layout 'HWC' wants shape {wanted}; got {tuple(shape)}")
    return shape[0], shape[1], 0, 1, 2


def descs(codec, items, layout, ptr=lambda x: x.data_ptr(), strides=lambda x: x.stride()):
    """The codec's image structs of items, with any strides: CUDA tensors by default, or arrays
    whose address and strides in elements ptr(x) and strides(x) give."""
    out = (codec.image * len(items))()
    for d, x in zip(out, items):
        h, w, ra, ca, ka = axes(x.shape, layout, codec.channels)
        codec.check_size(x.shape, h, w)
        st = strides(x)
        d.data, d.width, d.height = ptr(x), w, h
        d.row_stride, d.col_stride, d.chan_stride = st[ra], st[ca], st[ka]
        if codec.fill:
            codec.fill(d, x, x.shape[ka])
    return out


def placed(codec, d):
    """d after the codec's place(d), when it has one."""
    if codec.place:
        codec.place(d)
    return d


def encode_host(codec, images, layout):
    """The serial host driver on numpy arrays: a list of files as bytes."""
    d = placed(codec, descs(codec, images, layout, lambda x: x.ctypes.data, lambda x: [s // x.itemsize for s in x.strides]))
    work_bytes, base = codec.plan(d)
    work = np.zeros(work_bytes, np.uint8)
    offs = (C.c_uint64 * (len(images) + 1))()
    codec.call('encode_host', d, work.ctypes.data, work_bytes, offs)
    return [work[base + offs[i]:base + offs[i + 1]].tobytes() for i in range(len(images))]


def chunks(codec, descs, free_bytes):
    """Split the images, in order, so that each chunk's work area fits in a quarter of the free
    device memory; one chunk when everything fits."""
    budget = free_bytes // 4
    if codec.plan(descs)[0] <= budget:
        return [list(range(len(descs)))]
    out, cur, used = [], [], 0
    for i in range(len(descs)):
        need = codec.plan((codec.image * 1)(descs[i]))[0]
        if cur and used + need > budget:
            out.append(cur)
            cur, used = [], 0
        cur.append(i)
        used += need
    out.append(cur)
    return out


def encode_device(codec, descs, device):
    """Encode descs on `device` after what torch's current stream has queued: a list of files as
    bytes, in input order."""
    results = [None] * len(descs)
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device)
        free = torch.cuda.mem_get_info(device)[0]
        for idx in chunks(codec, descs, free):
            d = (codec.image * len(idx))(*[descs[i] for i in idx])
            work_bytes, base = codec.plan(d)
            work = torch.empty(work_bytes, dtype=torch.uint8, device=device)
            offs = (C.c_uint64 * (len(idx) + 1))()
            codec.call('encode', d, work.data_ptr(), work_bytes, stream.cuda_stream, offs, None, 0, None)
            total = offs[len(idx)]
            host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
            host.copy_(work[base:base + total])        # synchronous: the files are on the host
            view = host.numpy()
            for k, i in enumerate(idx):
                results[i] = view[offs[k]:offs[k + 1]].tobytes()
            del work
    return results


def by_codec(codecs, items, layout):
    """The calls a list of images makes when each channel count has its codec, codecs = {channel
    count: Codec}: [(codec, indices of its images, in input order)], a codec that several counts
    share taking all their images."""
    groups = {}
    for i, x in enumerate(items):
        c = codecs[x.shape[axes(x.shape, layout, tuple(codecs))[4]]]
        groups.setdefault(id(c), (c, []))[1].append(i)
    return list(groups.values())


def encode_tensors(fn, codec, images, layout, dtypes, calls=None):
    """The body of the public encoder `fn` once its own arguments are checked: images is one CUDA
    tensor or a list or tuple of them, of one of `dtypes`.  codec: a Codec, or {channel count:
    Codec} for an encoder whose library call takes one kind of image (the images of each kind go
    to their own calls).  calls(items), when given, replaces that split: [(Codec, indices of its
    images, in input order)], once codec's checks have accepted the images.  Returns bytes or a
    list of bytes, in input order."""
    codecs = codec if isinstance(codec, dict) else {c: codec for c in codec.channels}
    channels = tuple(codecs)
    single = not isinstance(images, (list, tuple))
    items = [images] if single else list(images)
    for x in items:
        if not isinstance(x, torch.Tensor):
            raise ValueError(f'{fn} takes torch tensors, not {type(x).__name__}')
        if x.dtype not in dtypes:
            raise ValueError(f'{fn} takes {" or ".join(map(str, dtypes))} tensors, not {x.dtype}')
        h, w, *_ = axes(x.shape, layout, channels)
        codecs[channels[0]].check_size(x.shape, h, w)
        if x.device.type != 'cuda':
            raise ValueError(f'{fn} encodes CUDA tensors; this one is on {x.device}')
    if not torch.cuda.is_available() or torch.cuda.device_count() <= 0:
        raise RuntimeError(f'{fn} needs a CUDA device: the encoder has no CPU fallback')
    if not items:
        return []
    device = items[0].device
    if any(x.device != device for x in items):
        raise ValueError('all images of one call must be on the same device')
    results = [None] * len(items)
    for c, idx in (calls or (lambda x: by_codec(codecs, x, layout)))(items):
        for i, r in zip(idx, encode_device(c, placed(c, descs(c, [items[i] for i in idx], layout)), device)):
            results[i] = r
    return results[0] if single else results
