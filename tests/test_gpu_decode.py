"""decode_jpeg and j2p_session_export on the GPU: the tensors equal the checker pipeline (reader
coefficients -> oracle solver -> +128 on luma -> reference colour conversion) at 8 and 16 bits, the
float samples equal a numpy restatement of the conversion, mixed lists come back in input order
equal to decoding each file alone, the export is ordered with the session streams, and every
refusal of the export calls returns J2P_ERR_ARG."""
import ctypes as C

import numpy as np
import pytest
import torch

from jpeg2png_b200 import abi, decode_jpeg, synth
from tests import helpers as H
from tests import jpeg_synth
from tests.test_codecs import codecs, make_jpeg, read_jpeg  # noqa: F401  (codecs is a fixture)
from tests.test_gpu_cli import expected_rgb

pytestmark = pytest.mark.gpu


def _pillow(w, h, q, ss, prog):
    return lambda: make_jpeg(w, h, q, ss, prog, seed=5 * w + h)


def _synth(w, h, sampling):
    def make():
        planes, quants = jpeg_synth.random_planes(w, h, sampling, seed=w * 7 + h)
        return jpeg_synth.encode_baseline(w, h, sampling, planes, quants)
    return make


# the files of tests/test_gpu_cli.py: maker, joint flags (iterations, weight), separate flags
FILES = {
    'pillow_420': (_pillow(160, 120, 20, '4:2:0', False), (20, 0.3), ((20, 20, 20), (0.3, 0.0, 0.0))),
    'progressive_444_97x61': (_pillow(97, 61, 50, '4:4:4', True), (15, 0.5), ((15, 15, 15), (0.5, 0.0, 0.0))),
    'separate_12_8_6': (_pillow(120, 88, 30, '4:2:0', False), (12, 0.3), ((12, 8, 6), (0.3, 0.1, 0.0))),
    'synth_422': (_synth(95, 33, [(2, 1), (1, 1), (1, 1)]), (9, 0.3), ((9, 7, 5), (0.3, 0.0, 0.2))),
    'synth_440': (_synth(40, 72, [(1, 2), (1, 1), (1, 1)]), (9, 0.3), ((9, 7, 5), (0.3, 0.0, 0.2))),
    'synth_mixed_41_21_11': (_synth(48, 40, [(4, 1), (2, 1), (1, 1)]), (9, 0.3), ((9, 7, 5), (0.3, 0.0, 0.2))),
    'synth_mixed_41_21_12': (_synth(36, 40, [(4, 1), (2, 1), (1, 2)]), (9, 0.3), ((9, 7, 5), (0.3, 0.0, 0.2))),
}
PW = [0.001] * 3


def _case(name, sep):
    make, (it, w), (its, ws) = FILES[name]
    data = make()
    if sep:
        return data, dict(iterations=its, weight=ws, separate=True), list(its), list(ws)
    return data, dict(iterations=it, weight=w), [it] * 3, [w, w, w]


def expected_rgb16(img, joint, iterations, weight, pweights):
    """expected_rgb at 16 bits: the checker's big-endian samples as integers, (h, w, 3) uint16."""
    ora = H.load_oracle()
    if joint:
        planes = H.run_compute('oracle', img, [0, 1, 2], weight[0], pweights, iterations[0])
    else:
        planes = [H.run_compute('oracle', img, [c], weight[c], [pweights[c]], iterations[c])[0] for c in range(3)]
    planes[0] = planes[0] + np.float32(128.0)
    out = np.zeros(img.width * img.height * 6, np.uint8)
    p = [np.ascontiguousarray(x, np.float32) for x in planes]
    ora.oracle_ycc_to_rgb(img.width, img.height, 16, p[0].ctypes.data, p[0].shape[1], p[1].ctypes.data, p[1].shape[1],
                          p[2].ctypes.data, p[2].shape[1], out.ctypes.data)
    return out.view('>u2').astype(np.uint16).reshape(img.height, img.width, 3)


def _hwc(t, layout):
    a = t.cpu().numpy()
    return a.transpose(1, 2, 0) if layout == 'CHW' else a


@pytest.mark.parametrize('sep', [False, True], ids=['joint', 'separate'])
@pytest.mark.parametrize('name', list(FILES))
def test_uint8_equals_checker_pipeline(codecs, name, sep):  # noqa: F811
    data, kw, iters, weights = _case(name, sep)
    img, err = read_jpeg(codecs, data)
    assert img is not None, err
    want = expected_rgb(img, not sep, iters, weights, PW)
    for layout in ('CHW', 'HWC'):
        got = decode_jpeg(data, layout=layout, **kw)
        assert got.dtype == torch.uint8 and got.device.type == 'cuda'
        assert tuple(got.shape) == ((3, img.height, img.width) if layout == 'CHW' else (img.height, img.width, 3))
        got = _hwc(got, layout)
        assert (got == want).all(), f'{layout}: {int((got != want).sum())} of {got.size} samples differ'


@pytest.mark.parametrize('sep', [False, True], ids=['joint', 'separate'])
@pytest.mark.parametrize('name', list(FILES))
def test_uint16_equals_checker_pipeline(codecs, name, sep):  # noqa: F811
    data, kw, iters, weights = _case(name, sep)
    img, err = read_jpeg(codecs, data)
    assert img is not None, err
    want = expected_rgb16(img, not sep, iters, weights, PW)
    for layout in ('CHW', 'HWC'):
        got = _hwc(decode_jpeg(data, layout=layout, dtype=torch.uint16, **kw), layout)
        assert got.dtype == np.uint16
        assert (got == want).all(), f'{layout}: {int((got != want).sum())} of {got.size} samples differ'


def _big_coefficient_session(lib):
    """The frame of test_device_scanlines_match_reference_conversion: 203x117 in a 208x128 4:2:0
    frame, coefficients tripled so that the samples leave [0, 255] on both sides."""
    img = synth.synth_coefs(203, 117, 8, '4:2:0', seed=11)
    for pl in img.planes:
        pl.data[:] = np.clip(pl.data.astype(np.int32) * 3, -1000, 1000).astype(np.int16)
    desc = abi.frame_desc(img, [0, 1, 2], 0.3, PW, 6)
    s = abi.Session(lib, desc, 1, 0, batch=False)
    s.upload([img], [0, 1, 2])
    s.iterate(0, 6)
    return img, s


def _export(lib, s, w, h, dtype, layout, stream=None, frame0=0, n=1):
    out = torch.empty((n, 3, h, w) if layout == 'CHW' else (n, h, w, 3), dtype=dtype, device='cuda')
    o = abi.ImageOut(w, h, {torch.uint8: 8, torch.uint16: 16, torch.float32: 32}[dtype],
                     abi.LAYOUT_CHW if layout == 'CHW' else abi.LAYOUT_HWC, out[0].numel() * out.element_size())
    rc = lib.j2p_session_export(s, frame0, n, C.byref(o), C.c_void_p(out.data_ptr()), stream)
    assert rc == 0, lib.j2p_last_error()
    return out


def test_float_export_equals_numpy_restatement():
    lib = abi.load_product()
    img, s = _big_coefficient_session(lib)
    with s:
        planes = s.download()[0]
        w, h = img.width, img.height
        got = {}
        for layout in ('CHW', 'HWC'):
            for dt in (torch.float32, torch.uint8, torch.uint16):
                t = _export(lib, s.s, w, h, dt, layout)
                torch.cuda.synchronize()
                got[layout, dt] = _hwc(t[0], layout)
    # png.c:39-47 in numpy: float64 products and sums (round to nearest, no contraction), narrowed
    # to float32, compared with the double bounds
    y = (planes[0][:h, :w] + np.float32(128.0)).astype(np.float64)
    cb, cr = planes[1][:h, :w].astype(np.float64), planes[2][:h, :w].astype(np.float64)
    rgb = [y + 1.402 * cr, (y - 0.34414 * cb) - 0.71414 * cr, y + 1.772 * cb]
    want = []
    for v in rgb:
        x = v.astype(np.float32)
        x = np.where(x.astype(np.float64) > 255.0, np.float32(255.0), np.where(x.astype(np.float64) < 0.0, np.float32(0.0), x))
        want.append(x.astype(np.float32))
    want = np.stack(want, axis=-1)
    assert want.min() == 0 and want.max() == 255, 'the case is meant to hit both clamps'
    for layout in ('CHW', 'HWC'):
        f = got[layout, torch.float32]
        assert (f.view(np.uint32) == want.view(np.uint32)).all(), f'{layout}: {int((f != want).sum())} samples differ'
        assert (got[layout, torch.uint8] == np.trunc(f).astype(np.uint8)).all()
        assert (got[layout, torch.uint16] == np.trunc(f * np.float32(256.0)).astype(np.uint16)).all()


def _mixed_inputs():
    a = [make_jpeg(120, 88, 40, '4:2:0', seed=s) for s in (1, 2, 3)]
    b = [make_jpeg(118, 86, 40, '4:2:0', seed=s) for s in (4, 5)]            # a's planes, another visible size
    c = [make_jpeg(64, 64, 60, '4:4:4', progressive=True, seed=s) for s in (6, 7)]
    d = [make_jpeg(96, 80, 50, '4:2:2', seed=s) for s in (8, 9)]
    return [a[0], b[0], c[0], d[0], a[1], c[1], b[1], a[2], d[1]], a


@pytest.mark.parametrize('sep', [False, True], ids=['joint', 'separate'])
def test_mixed_list_equals_each_file_alone(sep):
    inputs, _ = _mixed_inputs()
    kw = dict(iterations=(10, 8, 6), weight=(0.3, 0.1, 0.0), separate=True) if sep else dict(iterations=10)
    got = decode_jpeg(inputs, **kw)
    assert isinstance(got, list) and len(got) == len(inputs)
    for i, (data, t) in enumerate(zip(inputs, got)):
        alone = decode_jpeg(data, **kw)
        assert t.shape == alone.shape, i
        assert torch.equal(t, alone), f'input {i} differs from decoding it alone'
    # inputs 0, 4 and 7 share a geometry: one batch, views of one tensor
    assert got[0].untyped_storage().data_ptr() == got[4].untyped_storage().data_ptr() == got[7].untyped_storage().data_ptr()
    assert got[1].shape[1:] == (86, 118) and got[0].shape[1:] == (88, 120)


def test_max_frames_splits_a_group_without_changing_results():
    _, a = _mixed_inputs()
    five = a + [make_jpeg(120, 88, 40, '4:2:0', seed=s) for s in (10, 11)]
    whole = decode_jpeg(five, iterations=10, dtype=torch.float32, layout='HWC')
    split = decode_jpeg(five, iterations=10, dtype=torch.float32, layout='HWC', max_frames=2)
    for x, y in zip(whole, split):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    ptrs = [t.untyped_storage().data_ptr() for t in split]
    assert ptrs[0] == ptrs[1] != ptrs[2] == ptrs[3] != ptrs[4]


def test_decode_on_a_side_stream_needs_no_synchronisation():
    data = make_jpeg(160, 120, 20, '4:2:0', seed=5 * 160 + 120)
    want = decode_jpeg(data, iterations=20)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)                       # the side stream is busy when the call queues its work
        got = decode_jpeg(data, iterations=20)
        copy = got.clone()                                  # consumed on `side`, no synchronisation
        total = got.to(torch.int64).sum()
    side.synchronize()
    assert torch.equal(copy, want)
    assert int(total) == int(want.to(torch.int64).sum())


def test_session_stream_waits_for_an_export_on_another_stream():
    """Export frame 0 on a side stream that is still busy, then immediately upload other
    coefficients into the same session and iterate: the export still sees the first solve."""
    lib = abi.load_product()
    img1 = synth.synth_coefs(256, 256, 30, '4:2:0', seed=1)
    img2 = synth.synth_coefs(256, 256, 30, '4:2:0', seed=2)
    desc = abi.frame_desc(img1, [0, 1, 2], 0.3, PW, 20)

    def solved(img):
        with abi.Session(lib, desc, 1, 0, batch=False) as s:
            s.upload([img], [0, 1, 2])
            s.iterate(0, 20)
            out = _export(lib, s.s, 256, 256, torch.uint8, 'HWC')
            s.sync()
            return out

    want1, want2 = solved(img1), solved(img2)
    assert not torch.equal(want1, want2)
    side = torch.cuda.Stream()
    with abi.Session(lib, desc, 1, 0, batch=False) as s:
        s.upload([img1], [0, 1, 2])
        s.iterate(0, 20)
        with torch.cuda.stream(side):
            torch.cuda._sleep(100_000_000)                  # holds the export back
            got = _export(lib, s.s, 256, 256, torch.uint8, 'HWC', stream=C.c_void_p(side.cuda_stream))
        s.upload([img2], [0, 1, 2])                          # re-arms the session: overwrites the iterates
        s.iterate(0, 20)
        s.sync()
        torch.cuda.synchronize()
        assert torch.equal(got, want1), 'the session overwrote its planes before the export read them'
        again = _export(lib, s.s, 256, 256, torch.uint8, 'HWC')
        s.sync()
        assert torch.equal(again, want2)


def test_export_refusals():
    lib = abi.load_product()
    img = synth.synth_coefs(64, 64, 30, '4:4:4', seed=3)
    joint = abi.frame_desc(img, [0, 1, 2], 0.3, PW, 2)
    one = abi.frame_desc(img, [0], 0.3, PW, 2)
    dst = torch.empty(64 * 64 * 3 * 4 * 2, dtype=torch.uint8, device='cuda')
    p = C.c_void_p(dst.data_ptr())

    def out(w=64, h=64, sample=8, layout=abi.LAYOUT_CHW, frame_bytes=None):
        fb = w * h * 3 * max(sample // 8, 1) if frame_bytes is None else frame_bytes
        return C.byref(abi.ImageOut(w, h, sample, layout, fb))

    def refused(rc):
        msg = lib.j2p_last_error()
        return rc == -1 and len(msg) > 0

    with abi.Session(lib, joint, 1, 0, batch=False) as s, abi.Session(lib, joint, 2, 0) as b, \
            abi.Session(lib, one, 1, 0, batch=False) as y, abi.Session(lib, one, 1, 0, batch=False) as cb, \
            abi.Session(lib, one, 2, 0) as cr2:
        for x in (s, b):
            x.upload([img] * x.nframes, [0, 1, 2])
            x.iterate(0, 2)
        for x in (y, cb, cr2):
            x.upload([img] * x.nframes, [0])
            x.iterate(0, 2)
        ex = lib.j2p_session_export
        assert ex(s.s, 0, 1, out(), p, None) == 0, lib.j2p_last_error()          # the valid call
        assert ex(b.s, 0, 2, out(), p, None) == 0, lib.j2p_last_error()
        assert refused(ex(s.s, 0, 1, out(), None, None))                         # null dst
        assert refused(ex(s.s, 0, 1, None, p, None))                             # null description
        assert refused(ex(s.s, 0, 0, out(), p, None))                            # nframes == 0
        assert refused(ex(s.s, 1, 1, out(), p, None))                            # frame out of range
        assert refused(ex(b.s, 1, 2, out(), p, None))
        assert refused(ex(s.s, 0, 1, out(w=0), p, None))
        assert refused(ex(s.s, 0, 1, out(h=0), p, None))
        assert refused(ex(s.s, 0, 1, out(w=65), p, None))                        # larger than the frame
        assert refused(ex(s.s, 0, 1, out(h=65), p, None))
        assert refused(ex(s.s, 0, 1, out(sample=12), p, None))                   # unknown sample
        assert refused(ex(s.s, 0, 1, out(layout=2), p, None))                    # unknown layout
        assert refused(ex(s.s, 0, 1, out(frame_bytes=64 * 64 * 3 - 1), p, None))  # smaller than one image
        assert refused(ex(y.s, 0, 1, out(), p, None))                            # joint export of nchannel 1
        sep = lib.j2p_session_export_separate
        assert sep(y.s, cb.s, y.s, 0, 1, out(), p, None) == 0, lib.j2p_last_error()
        assert refused(sep(y.s, s.s, cb.s, 0, 1, out(), p, None))                # nchannel != 1
        assert refused(sep(y.s, cb.s, cr2.s, 0, 1, out(), p, None))              # different frame counts
        assert refused(sep(y.s, cb.s, y.s, 0, 1, out(), None, None))             # null dst
        assert refused(sep(y.s, cb.s, y.s, 0, 1, out(w=65), p, None))
        d = C.c_void_p()
        assert lib.j2p_session_create_strip(C.byref(d), 0, C.byref(joint), 0, 32) == 0, lib.j2p_last_error()
        try:
            assert refused(ex(d, 0, 1, out(), p, None))                          # a strip session
        finally:
            lib.j2p_session_destroy(d)
        torch.cuda.synchronize()
        if lib.j2p_device_count() > 1:
            with abi.Session(lib, one, 1, 1, batch=False) as other:
                other.upload([img], [0])
                assert refused(sep(y.s, cb.s, other.s, 0, 1, out(), p, None))     # different devices
