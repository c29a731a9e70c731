"""End to end on the GPU box: the jpeg2png command line (own JPEG reader, device decode, solver,
own PNG writer) against the same pipeline assembled from the checker pieces — reader coefficients
-> oracle solver -> +128 on luma (jpeg2png.c:156-159) -> reference colour conversion (png.c:39-62).
The PNG pixels must be identical: this is the "bit-identical PNG" bar of the north star."""
import io
import os
import subprocess

import numpy as np
import pytest
from PIL import Image

from tests import helpers as H
from tests.test_codecs import CLI_DIR, codecs, make_jpeg, read_jpeg  # noqa: F401  (codecs is a fixture)

pytestmark = pytest.mark.gpu


def expected_rgb(img, joint, iterations, weight, pweights):
    ora = H.load_oracle()
    if joint:
        planes = H.run_compute('oracle', img, [0, 1, 2], weight[0], pweights, iterations[0])
    else:
        planes = [H.run_compute('oracle', img, [c], weight[c], [pweights[c]], iterations[c])[0] for c in range(3)]
    planes[0] = planes[0] + np.float32(128.0)
    out = np.zeros(img.width * img.height * 3, np.uint8)
    p = [np.ascontiguousarray(x, np.float32) for x in planes]
    ora.oracle_ycc_to_rgb(img.width, img.height, 8, p[0].ctypes.data, p[0].shape[1], p[1].ctypes.data, p[1].shape[1],
                          p[2].ctypes.data, p[2].shape[1], out.ctypes.data)
    return out.reshape(img.height, img.width, 3)


@pytest.mark.parametrize('w,h,q,ss,prog,args,joint,iters,weights', [
    (160, 120, 20, '4:2:0', False, ['-i', '20'], True, [20] * 3, [0.3, 0.0, 0.0]),
    (97, 61, 50, '4:4:4', True, ['-i', '15', '-w', '0.5'], True, [15] * 3, [0.5, 0.0, 0.0]),
    (120, 88, 30, '4:2:0', False, ['-s', '-i', '12,8,6', '-w', '0.3,0.1,0.0'], False, [12, 8, 6], [0.3, 0.1, 0.0]),
])
def test_cli_png_matches_reference_pipeline(codecs, tmp_path, w, h, q, ss, prog, args, joint, iters, weights):  # noqa: F811
    subprocess.run(['make', '-C', CLI_DIR, 'jpeg2png'], check=True, capture_output=True)
    data = make_jpeg(w, h, q, ss, prog, seed=5 * w + h)
    src = tmp_path / 'in.jpg'
    src.write_bytes(data)
    r = subprocess.run([os.path.join(CLI_DIR, 'jpeg2png'), '-q', *args, str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = np.asarray(Image.open(tmp_path / 'in.png'))
    img, err = read_jpeg(codecs, data)
    assert img is not None, err
    want = expected_rgb(img, joint, iters, weights, [0.001] * 3)
    assert got.shape == want.shape
    assert (got == want).all(), f'{int((got != want).sum())} of {got.size} samples differ'


@pytest.mark.parametrize('w,h,sampling', [
    (95, 33, [(2, 1), (1, 1), (1, 1)]),          # 4:2:2
    (40, 72, [(1, 2), (1, 1), (1, 1)]),          # 4:4:0
    (48, 40, [(4, 1), (2, 1), (1, 1)]),          # mixed factors: chroma planes with w_samp 2 and 4
    (36, 40, [(4, 1), (2, 1), (1, 2)]),          # mixed factors: Cb a (2,2) plane narrower than the frame
])
@pytest.mark.parametrize('sep', [False, True])
def test_cli_png_matches_reference_pipeline_for_more_layouts(codecs, tmp_path, w, h, sampling, sep):  # noqa: F811
    """Files with known coefficients (tests/jpeg_synth.py) in the layouts the Pillow-written files
    above do not have, joint and -s, against the checker pipeline."""
    from tests import jpeg_synth
    subprocess.run(['make', '-C', CLI_DIR, 'jpeg2png'], check=True, capture_output=True)
    planes, quants = jpeg_synth.random_planes(w, h, sampling, seed=w * 7 + h)
    data = jpeg_synth.encode_baseline(w, h, sampling, planes, quants)
    src = tmp_path / 'in.jpg'
    src.write_bytes(data)
    args = ['-s', '-i', '9,7,5', '-w', '0.3,0.0,0.2'] if sep else ['-i', '9', '-w', '0.3']
    r = subprocess.run([os.path.join(CLI_DIR, 'jpeg2png'), '-q', *args, str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = np.asarray(Image.open(tmp_path / 'in.png'))
    img, err = read_jpeg(codecs, data)
    assert img is not None, err
    want = expected_rgb(img, not sep, [9, 7, 5] if sep else [9] * 3, [0.3, 0.0, 0.2] if sep else [0.3] * 3, [0.001] * 3)
    assert got.shape == want.shape
    assert (got == want).all(), f'{int((got != want).sum())} of {got.size} samples differ'


def test_cli_refuses_to_overwrite_and_logs_csv(codecs, tmp_path):  # noqa: F811
    subprocess.run(['make', '-C', CLI_DIR, 'jpeg2png'], check=True, capture_output=True)
    src = tmp_path / 'pic.jpeg'
    src.write_bytes(make_jpeg(64, 64, 40, '4:2:0'))
    exe = os.path.join(CLI_DIR, 'jpeg2png')
    csv = tmp_path / 'log.csv'
    r = subprocess.run([exe, '-q', '-i', '5', '-c', str(csv), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert (tmp_path / 'pic.png').exists()
    lines = csv.read_text().strip().splitlines()
    assert lines[0] == 'filename,channel,iteration,objective,prob_dist,tv,tv2' and len(lines) == 6      # logger.c:13
    assert lines[1].split(',')[1:3] == ['3', '0']
    r = subprocess.run([exe, '-q', '-i', '5', str(src)], capture_output=True, text=True)                     # jpeg2png.c:300-303
    assert r.returncode == 1 and r.stderr.startswith('jpeg2png: not overwriting output file')
    r = subprocess.run([exe, '-q', '-i', '5', '-f', str(src)], capture_output=True, text=True)
    assert r.returncode == 0
    r = subprocess.run([exe, '-q', '-w', '0.1,0.2,0.3', str(src)], capture_output=True, text=True)           # jpeg2png.c:210-212
    assert r.returncode == 1 and 'different weights are only possible' in r.stderr


@pytest.mark.parametrize('bits', [8, 16])
def test_device_scanlines_match_reference_conversion(bits):
    """j2p_session_download_scanlines: luma + 128 (jpeg2png.c:156-159) and the colour conversion /
    truncation of png.c:39-62 on the device, against the checker's restatement applied to the
    float planes of the SAME session.  Image 203x117 in a 208x128 frame (4:2:0); a huge -w drives
    samples out of [0, 255] so the clamp is exercised."""
    import ctypes as C
    from jpeg2png_b200 import abi, synth
    lib = abi.load_product()
    img = synth.synth_coefs(203, 117, 8, '4:2:0', seed=11)
    for pl in img.planes:           # exaggerate the coefficients: results leave the displayable range
        pl.data[:] = np.clip(pl.data.astype(np.int32) * 3, -1000, 1000).astype(np.int16)
    d = abi.FrameDesc()
    d.nchannel = 3
    for c, p in enumerate(img.planes):
        d.plane_w[c], d.plane_h[c], d.w_samp[c], d.h_samp[c] = p.w, p.h, p.w_samp, p.h_samp
        d.pweight[c] = 0.001
    d.weight = 0.3
    d.iterations = 6
    s = C.c_void_p()
    assert lib.j2p_session_create(C.byref(s), 0, C.byref(d)) == 0, lib.j2p_last_error()
    try:
        for c, p in enumerate(img.planes):
            data, quant = np.ascontiguousarray(p.data), np.ascontiguousarray(p.quant)
            assert lib.j2p_session_upload(s, c, data.ctypes.data, quant.ctypes.data, None) == 0
        assert lib.j2p_session_iterate(s, 0, 6) == 0
        W, Hh = lib.j2p_session_width(s), lib.j2p_session_height(s)
        planes = []
        for c in range(3):
            out = np.empty((Hh, W), np.float32)
            assert lib.j2p_session_download(s, c, out.ctypes.data) == 0
            planes.append(out)
        w, h = img.width, img.height
        depth = bits // 8
        raw = np.full(h * (w * 3 * depth + 1), 0xAA, np.uint8)
        assert lib.j2p_session_download_scanlines(s, w, h, bits, raw.ctypes.data) == 0, lib.j2p_last_error()
        raw = raw.reshape(h, w * 3 * depth + 1)
        assert (raw[:, 0] == 0).all(), 'every scanline starts with filter type 0'
        planes[0] = planes[0] + np.float32(128.0)
        want = np.zeros(h * w * 3 * depth, np.uint8)
        H.load_oracle().oracle_ycc_to_rgb(w, h, bits, planes[0].ctypes.data, W, planes[1].ctypes.data, W, planes[2].ctypes.data, W, want.ctypes.data)
        want = want.reshape(h, w * 3 * depth)
        assert (raw[:, 1:] == want).all(), f'{int((raw[:, 1:] != want).sum())} bytes differ'
        assert want.min() == 0 and want.max() == 255, 'the case is meant to hit both clamps'
        assert lib.j2p_session_download_scanlines(s, W + 1, h, bits, raw.ctypes.data) != 0       # larger than the frame
    finally:
        lib.j2p_session_destroy(s)
