"""jpeg2png_b200.decode_jpeg without a GPU: argument rules with the command line's messages, reader
failures reported per input before any device is needed, the grouping and chunking plan, and the
error (not a fallback) when no device is present."""
import io

import numpy as np
import pytest
import torch
from PIL import Image

from jpeg2png_b200 import abi, decode as D, decode_jpeg, synth
from tests.test_codecs import make_jpeg


@pytest.fixture(scope='module')
def good():
    return make_jpeg(64, 48, 50, '4:2:0', seed=3)


def test_import_does_not_pull_in_torch():
    import subprocess
    import sys
    code = 'import sys, jpeg2png_b200; print("torch" in sys.modules)'
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, cwd=abi._PKG_DIR + '/..')
    assert r.returncode == 0 and r.stdout.strip() == 'False', r.stderr


def test_flags_follow_the_command_line():
    assert D.solver_flags(50, 0.3, 0.001, False) == ((50, 50, 50), (0.3, 0.0, 0.0), (0.001,) * 3)
    assert D.solver_flags((12, 8, 6), (0.3, 0.1, 0.0), (1e-3, 2e-3, 0.0), True) == ((12, 8, 6), (0.3, 0.1, 0.0), (1e-3, 2e-3, 0.0))
    assert D.solver_flags(7, 0.5, (0.1, 0.2, 0.3), False)[2] == (0.1, 0.2, 0.3)      # three pweights need no -s


@pytest.mark.parametrize('kw,msg', [
    (dict(weight=(0.3, 0.1, 0.0)), 'different weights are only possible when using separated components'),
    (dict(iterations=(12, 8, 6)), 'different iteration counts are only possible when using separated components'),
    (dict(weight=(0.3, 0.1)), 'invalid weight'),
    (dict(pweight=(0.1, 0.2)), 'invalid probability weight'),
    (dict(iterations=(1, 2), separate=True), 'invalid number of iterations'),
    (dict(iterations=-1), 'invalid number of iterations'),
    (dict(iterations=2.5), 'invalid number of iterations'),
    (dict(dtype=torch.int32), 'dtype must be'),
    (dict(layout='NCHW'), 'layout must be'),
    (dict(max_frames=0), 'max_frames'),
    (dict(device='cpu'), 'not a CUDA device'),
])
def test_argument_errors(good, kw, msg):
    with pytest.raises(ValueError, match=msg):
        decode_jpeg(good, **kw)


def test_inputs_must_be_bytes_or_paths():
    with pytest.raises(TypeError, match='bytes-like objects or paths'):
        decode_jpeg(12345)


def _gray_jpeg():
    buf = io.BytesIO()
    Image.fromarray(synth.cartoon_image(32, 32, 3).astype(np.uint8), 'RGB').convert('L').save(buf, 'JPEG')
    return buf.getvalue()


@pytest.mark.parametrize('bad,msg', [
    (lambda g: g[:300], 'corrupt jpeg'),                        # truncated inside the headers
    (lambda g: b'not a jpeg at all', 'no SOI marker'),
    (lambda g: _gray_jpeg(), 'only 3 component jpegs are supported'),     # jpeg.c:34
])
def test_reader_failures_name_the_input(good, tmp_path, bad, msg):
    data = bad(good)
    with pytest.raises(ValueError, match=rf'^input 0: .*{msg}'):
        decode_jpeg(data)
    with pytest.raises(ValueError, match=rf'^input 2: .*{msg}'):
        decode_jpeg([good, bytearray(good), memoryview(data), good])
    p = tmp_path / 'bad.jpg'
    p.write_bytes(data)
    with pytest.raises(ValueError, match=rf'^input 1 \({p}\): .*{msg}'):
        decode_jpeg([good, p])
    with pytest.raises(ValueError, match=rf'^input 1 \({p}\): .*{msg}'):
        decode_jpeg((good, str(p)), separate=True, dtype=torch.float32, layout='HWC')


def test_empty_list_is_an_empty_result():
    assert decode_jpeg([]) == []


def test_parse_reads_the_geometry(good):
    p = D.parse_jpeg(good)
    assert (p.w, p.h) == (64, 48)
    assert p.key() == (64, 48, ((64, 48, 1, 1), (32, 24, 2, 2), (32, 24, 2, 2)))
    assert p.planes[0].data.dtype == np.int16 and p.planes[0].data.size == 64 * 48
    assert (p.planes[1].quant == synth.quant_table(50, chroma=True)).all()


def test_plan_groups_restores_order_and_respects_max_frames():
    keys = ['a', 'b', 'a', 'c', 'a', 'b', 'a', 'a', 'c']
    chunks = D.plan(keys, lambda k: 2)
    assert chunks == [('a', [0, 2]), ('a', [4, 6]), ('a', [7]), ('b', [1, 5]), ('c', [3, 8])]
    seen = sorted(i for _, idx in chunks for i in idx)
    assert seen == list(range(len(keys)))                       # every input exactly once
    for k, idx in chunks:
        assert all(keys[i] == k for i in idx) and idx == sorted(idx)
    assert D.plan(keys, lambda k: 100) == [('a', [0, 2, 4, 6, 7]), ('b', [1, 5]), ('c', [3, 8])]
    with pytest.raises(ValueError):
        D.plan(keys, lambda k: 0)


def test_same_planes_different_visible_size_are_different_groups():
    a = D.parse_jpeg(make_jpeg(120, 88, 40, '4:2:0'))
    b = D.parse_jpeg(make_jpeg(118, 86, 40, '4:2:0'))
    assert a.key()[2] == b.key()[2] and a.key() != b.key()


def test_chunk_size_from_free_memory():
    key = (1920, 1080, ((1920, 1080, 1, 1), (960, 544, 2, 2), (960, 544, 2, 2)))
    joint = D.frame_footprint(key, False, 1)
    sep = D.frame_footprint(key, True, 1)
    # x, xp, g, gp at frame size dominate: joint, three planes in a 1920x1088 frame; separate,
    # luma in its 1920x1080 frame and each chroma plane in its own 1920x1088 frame
    assert 3 * 16 * 1920 * 1080 < joint < 3 * 16 * 1920 * 1088 + 20 * 1920 * 1080
    assert 16 * 1920 * (1080 + 2 * 1088) < sep < joint
    free = 40 << 30
    n = D.chunk_frames(key, False, 1, None, free)
    assert n * joint <= free // 4 < (n + 1) * joint                 # two chunks in flight: under half of free
    m = D.chunk_frames(key, True, 1, None, free)
    assert m * sep <= free // 4 < (m + 1) * sep
    assert D.chunk_frames(key, False, 1, None, 1000) == 1            # always at least one frame
    assert D.chunk_frames(key, False, 1, 5, free) == 5
    assert D.chunk_frames(key, False, 1, 10 ** 6, free) == D.MAX_BATCH
    tiny = (8, 8, ((8, 8, 1, 1),) * 3)
    assert D.chunk_frames(tiny, False, 4, None, 1 << 40) == D.MAX_BATCH


def test_separate_mode_plan_keeps_the_joint_grouping():
    """Separate mode splits each chunk into three single-plane batches (one per channel, with that
    channel's flags), but groups and chunks inputs exactly as joint mode does."""
    keys = [D.parse_jpeg(make_jpeg(w, h, 30, ss)).key() for w, h, ss in
            [(64, 48, '4:2:0'), (40, 40, '4:4:4'), (64, 48, '4:2:0'), (40, 40, '4:4:4'), (64, 48, '4:2:0')]]
    free = 1 << 30
    for sep in (False, True):
        chunks = D.plan(keys, lambda k: D.chunk_frames(k, sep, 1, 2, free))
        assert [idx for _, idx in chunks] == [[0, 2], [4], [1, 3]]
    iters, weights, pweights = D.solver_flags((9, 7, 5), (0.3, 0.0, 0.2), 0.001, True)
    parsed = D.parse_jpeg(make_jpeg(64, 48, 30, '4:2:0'))
    descs = [D._frame_desc(parsed, [c], weights[c], pweights, iters[c]) for c in range(3)]
    assert [(d.nchannel, d.plane_w[0], d.w_samp[0], d.iterations) for d in descs] == [(1, 64, 1, 9), (1, 32, 2, 7), (1, 32, 2, 5)]
    assert [round(d.weight, 6) for d in descs] == [0.3, 0.0, 0.2]


def test_without_gpu_a_valid_file_is_an_error_not_a_fallback(good):
    if abi.load_product().j2p_device_count() > 0 and torch.cuda.is_available():
        pytest.skip('a CUDA device is present')
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        decode_jpeg(good)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        decode_jpeg([good, good], separate=True)
