"""Four-component (Adobe CMYK and YCCK) JPEGs in decode_jpeg on the GPU: every fixture equals the
checker pipeline (reader coefficients -> oracle solver plane by plane, joint for YCCK's Y, Cb, Cr
unless separate -> the reference conversion -> inversion, and Pillow's CMYK -> RGB restated in numpy)
at 8, 16 and 32 bits, in both layouts, joint and separate, in all eight EXIF orientations; the device
entropy decoder gives the reader's coefficients and the device and host front ends agree; mixed lists give each file what it gives alone and leave the other files' tensors
unchanged; results do not depend on max_frames or batch position; the refusals."""
import io
import os
import subprocess

import numpy as np
import pytest
import torch
from PIL import Image

from jpeg2png_b200 import decode as D
from jpeg2png_b200 import decode_jpeg, synth
from tests import cmyk_synth as S
from tests import helpers as H
from tests.test_gpu_cli import expected_rgb
from tests.test_gpu_decode import expected_rgb16
from tests.test_gpu_exif_orientation import oriented_numpy
from tests.test_gpu_gray import checker_gray

pytestmark = pytest.mark.gpu

CORPUS = S.corpus()
ITERS, WEIGHT, PW = 8, 0.3, 0.001
SEP = dict(separate=True, iterations=(ITERS, 5, 3), weight=(WEIGHT, 0.1, 0.0))
DTYPES = (torch.uint8, torch.uint16, torch.float32)


def coef_image(p, planes=None):
    return synth.CoefImage(width=p.w, height=p.h, planes=[synth.Plane(w=x.w, h=x.h, w_samp=x.w_samp, h_samp=x.h_samp,
                                                                      data=x.data, quant=x.quant)
                                                          for x in (p.planes if planes is None else planes)])


def rgb_float(img, planes):
    """The float RGB samples of solved Y, Cb, Cr planes (the reference conversion restated in numpy)."""
    h, w = img.height, img.width
    y = (planes[0][:h, :w] + np.float32(128.0)).astype(np.float64)
    cb, cr = planes[1][:h, :w].astype(np.float64), planes[2][:h, :w].astype(np.float64)
    out = []
    for v in (y + 1.402 * cr, (y - 0.34414 * cb) - 0.71414 * cr, y + 1.772 * cb):
        x = v.astype(np.float32)
        out.append(np.where(x.astype(np.float64) > 255.0, np.float32(255.0), np.where(x.astype(np.float64) < 0.0, np.float32(0.0), x)))
    return np.stack(out, axis=-1).astype(np.float32)


def checker(data, dtype, separate=False, rgb=False):
    """(h, w, 4) or, with rgb (uint8), (h, w, 3): what decode_jpeg must give for a four-component file."""
    p = D.parse_jpeg4(data)
    img = coef_image(p)
    luma = lambda c: H.run_compute('oracle', img, [c], WEIGHT, [PW], ITERS)[0]      # noqa: E731
    chans = []
    if p.colour == D.YCCK:
        img3 = coef_image(p, p.planes[:3])
        iters, weights = (list(SEP['iterations']), list(SEP['weight'])) if separate else ([ITERS] * 3, [WEIGHT] * 3)
        if dtype == torch.uint8:
            chans.append(expected_rgb(img3, not separate, iters, weights, [PW] * 3))
        elif dtype == torch.uint16:
            chans.append(expected_rgb16(img3, not separate, iters, weights, [PW] * 3))
        else:
            if separate:
                planes = [H.run_compute('oracle', img3, [c], weights[c], [PW], iters[c])[0] for c in range(3)]
            else:
                planes = H.run_compute('oracle', img3, [0, 1, 2], WEIGHT, [PW] * 3, ITERS)
            chans.append(rgb_float(img3, planes))
        planes = [3]
    else:
        planes = [0, 1, 2, 3]
    for c in planes:
        chans.append(S.invert(checker_gray(img, luma(c), dtype))[..., None])
    out = np.concatenate(chans, axis=-1)
    return S.pillow_rgb(out) if rgb else out


def hwc(t, layout):
    a = t.cpu().numpy()
    return a.transpose(1, 2, 0) if layout == 'CHW' else a


def same(a, b):
    if a.dtype == np.float32:
        return a.shape == b.shape and (a.view(np.uint32) == b.view(np.uint32)).all()
    return a.shape == b.shape and (a == b).all()


def kw(separate):
    return dict(SEP) if separate else dict(iterations=ITERS, weight=WEIGHT)


@pytest.mark.parametrize('sep', [False, True], ids=['joint', 'separate'])
@pytest.mark.parametrize('name', list(CORPUS))
def test_equals_checker_pipeline(name, sep):
    data, kind = CORPUS[name]
    assert S.pillow_opens_as_cmyk(data)
    for dtype in DTYPES:
        want = checker(data, dtype, sep)
        for layout in ('CHW', 'HWC'):
            got = decode_jpeg(data, mode='UNCHANGED', dtype=dtype, layout=layout, **kw(sep))
            assert got.dtype == dtype and got.is_contiguous()
            assert same(hwc(got, layout), want), f'{dtype} {layout}'
    want = checker(data, torch.uint8, sep, rgb=True)
    for layout in ('CHW', 'HWC'):
        assert same(hwc(decode_jpeg(data, layout=layout, **kw(sep)), layout), want), layout


def test_pillow_rgb_of_our_samples():
    """mode='RGB' is Pillow's convert('RGB') of our mode='UNCHANGED' uint8 samples."""
    files = [CORPUS[n][0] for n in ('pillow_q75_97x61', 'ycck_2211_45x35')]
    for f, u, r in zip(files, decode_jpeg(files, mode='UNCHANGED', layout='HWC', iterations=4),
                       decode_jpeg(files, layout='HWC', iterations=4)):
        u, r = u.cpu().numpy(), r.cpu().numpy()
        assert (np.asarray(Image.fromarray(u, 'CMYK').convert('RGB')) == r).all()


def _with_orientation(data, k):
    return data[:2] + S.exif_segment(k) + data[2:]


@pytest.mark.parametrize('name', ['pillow_q75_97x61', 'ycck_2211_45x35', 'cmyk_2211_t0'])
def test_every_orientation(name):
    data = CORPUS[name][0]
    assert D.exif_orientation(_with_orientation(data, 6)) == 6
    for mode, dtypes in (('UNCHANGED', DTYPES), ('RGB', (torch.uint8,))):
        for dtype in dtypes:
            for layout in ('CHW', 'HWC'):
                base = hwc(decode_jpeg(data, mode=mode, dtype=dtype, layout=layout, iterations=ITERS), layout)
                files = [_with_orientation(data, k) for k in range(1, 9)]
                got = decode_jpeg(files, mode=mode, dtype=dtype, layout=layout, iterations=ITERS, apply_exif_orientation=True)
                for k, t in zip(range(1, 9), got):
                    assert t.is_contiguous()
                    assert same(hwc(t, layout), np.ascontiguousarray(oriented_numpy(base, k))), (mode, dtype, layout, k)


def test_device_decoder_equals_reader():
    """Sequential four-component files decoded by libj2pentropy.so on the device (j2p_entropy_pack4):
    the reader's coefficients, every plane."""
    names = [n for n in CORPUS if not (n.startswith('arith') or 'progressive' in n)]
    lays = [D.FileLayout4(CORPUS[n][0]) for n in names]
    assert all(lay.device_decodable for lay in lays)
    stream = torch.cuda.Stream()
    dc = D._DeviceCoefs4(torch.cuda.current_device(), lays, stream, subseq_bits=64)
    assert (dc.status == 0).all() and dc.stats.launches > 0
    for i, n in enumerate(names):
        for c, pl in enumerate(D.parse_jpeg4(CORPUS[n][0]).planes):
            assert (dc.plane_tensor(i, c).cpu().numpy() == pl.data).all(), (n, c)


def test_front_ends_agree(monkeypatch):
    files = [d for d, _ in CORPUS.values()]
    made = []
    init = D._DeviceCoefs4.__init__

    def counting(self, device, layouts, *a, **k):
        made.append(len(layouts))
        init(self, device, layouts, *a, **k)
    monkeypatch.setattr(D._DeviceCoefs4, '__init__', counting)
    a = decode_jpeg(files, mode='UNCHANGED', dtype=torch.float32, iterations=ITERS, progressive_on_device=True)
    lays = [D.FileLayout4(f) for f in files]
    assert sum(made) == sum(1 for lay in lays if lay.device_decodable and D.four_on_device(lay)) > 0
    old = D._host_front_end
    D._host_front_end = True
    try:
        b = decode_jpeg(files, mode='UNCHANGED', dtype=torch.float32, iterations=ITERS)
    finally:
        D._host_front_end = old
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), i


def _others():
    buf = io.BytesIO()
    Image.fromarray(synth.cartoon_image(97, 61, 3).astype(np.uint8), 'RGB').save(buf, 'JPEG', quality=60, subsampling='4:4:4')
    rgb = buf.getvalue()
    buf = io.BytesIO()
    Image.fromarray(synth.cartoon_image(97, 61, 4).astype(np.uint8)[..., 1], 'L').save(buf, 'JPEG', quality=60)
    return rgb, buf.getvalue()


@pytest.mark.parametrize('sep', [False, True], ids=['joint', 'separate'])
def test_mixed_list_equals_each_file_alone(sep):
    rgb, gray = _others()
    four = [CORPUS[n][0] for n in ('pillow_q75_97x61', 'ycck_444_53x29', 'cmyk_2211_t0', 'no_app14_q75_97x61')]
    mixed = [four[0], rgb, gray, four[1], four[2], rgb, four[3], gray]
    got = decode_jpeg(mixed, mode='UNCHANGED', dtype=torch.float32, **kw(sep))
    for i, (f, t) in enumerate(zip(mixed, got)):
        alone = decode_jpeg(f, mode='UNCHANGED', dtype=torch.float32, **kw(sep))
        assert torch.equal(t.view(torch.int32), alone.view(torch.int32)), i
    without = decode_jpeg([rgb, gray, rgb, gray], mode='UNCHANGED', dtype=torch.float32, **kw(sep))
    for t, u in zip([got[1], got[2], got[5], got[7]], without):
        assert torch.equal(t.view(torch.int32), u.view(torch.int32))
    # mode='RGB' with uint8: the four-component files next to colour files
    got = decode_jpeg([four[0], rgb, four[1]], **kw(sep))
    assert torch.equal(got[1], decode_jpeg(rgb, **kw(sep)))
    assert torch.equal(got[0], decode_jpeg(four[0], **kw(sep))) and torch.equal(got[2], decode_jpeg(four[1], **kw(sep)))


@pytest.mark.parametrize('name', ['pillow_q75_97x61', 'ycck_2211_restart2', 'cmyk_2211_t0'])
def test_batch_position_and_max_frames(name):
    data, kind = CORPUS[name]
    others = [CORPUS[n][0] for n in ('pillow_q10_61x37', 'pillow_q95_40x24')]
    same_key = S.with_app14(data, S.app14(0 if kind == D.CMYK else 1))       # another file of the same batch key
    files = [data] + [same_key] * 3 + others + [data]
    whole = decode_jpeg(files, mode='UNCHANGED', dtype=torch.float32, iterations=ITERS)
    alone = decode_jpeg(data, mode='UNCHANGED', dtype=torch.float32, iterations=ITERS)
    for m in (1, 2, 3):
        split = decode_jpeg(files, mode='UNCHANGED', dtype=torch.float32, iterations=ITERS, max_frames=m)
        for i, (a, b) in enumerate(zip(whole, split)):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (m, i)
    assert torch.equal(whole[0].view(torch.int32), alone.view(torch.int32))
    assert torch.equal(whole[-1].view(torch.int32), alone.view(torch.int32))


def test_refusals():
    data = CORPUS['pillow_q75_97x61'][0]
    for dtype in (torch.uint16, torch.float32):
        with pytest.raises(ValueError, match="mode='UNCHANGED'"):
            decode_jpeg(data, dtype=dtype)
    with pytest.raises(ValueError, match='^input 0: only 1 and 3 component jpegs are supported$'):
        decode_jpeg(data, mode='GRAY')
    with pytest.raises(ValueError, match='return_objective'):
        decode_jpeg(data, mode='UNCHANGED', return_objective=True)
    # a four-component file the four-component reader refuses gives that reader's message
    bad = bytearray(data)
    dqt = next(a for m, a, _ in S.segments(data) if m == 0xDB)
    bad[dqt + 5] = 0                                    # the first entry of the first table
    with pytest.raises(ValueError, match='^input 0: invalid quantization table$'):
        decode_jpeg(bytes(bad), mode='UNCHANGED')
    # RGB mode still refuses gray files with today's message
    _, gray = _others()
    with pytest.raises(ValueError, match='^input 0: only 3 component jpegs are supported$'):
        decode_jpeg(gray)


def test_cli_refuses_cmyk(tmp_path):
    cli = os.path.join(os.path.dirname(D.CODECS_LIB), 'jpeg2png')
    if not os.path.exists(cli):
        subprocess.run(['make', '-C', os.path.dirname(D.CODECS_LIB), 'jpeg2png'], check=True, capture_output=True)
    src = tmp_path / 'in.jpg'
    src.write_bytes(CORPUS['pillow_q75_97x61'][0])
    r = subprocess.run([cli, str(src), '-o', str(tmp_path / 'out.png')], capture_output=True, text=True, timeout=120)
    assert r.returncode != 0
    assert 'only 3 component jpegs are supported' in r.stdout + r.stderr
    assert not (tmp_path / 'out.png').exists()
