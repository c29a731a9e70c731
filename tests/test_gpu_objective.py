"""The objective recorded on the device (j2p_session_record_objective, libj2pobjective.so) and
decode_jpeg(..., return_objective=True): every recording kernel against the checker's log, iterates
bit-identical to the unrecorded solve, records independent of batching, launch counts, refusals, and
the CSV file against the command line's -c."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest
import torch
from PIL import Image

import jpeg2png_b200
from jpeg2png_b200 import abi, decode_jpeg, synth
from tests import helpers as H
from tests.objective_cases import CASES

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = dict(rtol=1e-9, atol=1e-12)          # test_gpu_parity.py::test_objective_log_matches_oracle


@pytest.fixture(scope='module')
def lib():
    lib = abi.load_product()
    assert lib.j2p_device_count() > 0, 'no CUDA device visible: the product has no CPU fallback'
    return lib


def _check(lib, rc):
    assert rc == 0, lib.j2p_last_error().decode()


def _recorded(lib, frames, channels, weight, pw, iters, runs=None):
    """A recording batch of `frames`: (planes per frame, history (n, iters, 4), launches of the solve)."""
    with abi.Session(lib, abi.frame_desc(frames[0], channels, weight, pw, iters), len(frames)) as s:
        _check(lib, lib.j2p_session_record_objective(s.s, 1))
        s.upload(frames, channels)
        s.iterate(0, 0)                        # arm
        before = s.launches
        s.iterate(0, iters)
        launches = s.launches - before
        hist = np.zeros((len(frames), iters, 4))
        _check(lib, lib.j2p_session_objective_history(s.s, 0, iters, hist.ctypes.data_as(C.POINTER(C.c_double))))
        return s.download(), hist, launches


def _unrecorded(lib, frames, channels, weight, pw, iters):
    with abi.Session(lib, abi.frame_desc(frames[0], channels, weight, pw, iters), len(frames)) as s:
        s.upload(frames, channels)
        s.iterate(0, 0)
        before = s.launches
        s.iterate(0, iters)
        return s.download(), s.launches - before


@pytest.mark.parametrize('case', sorted(CASES))
def test_recorded_batch_matches_the_checker(lib, case):
    make, channels, weight, pw, iters, _ = CASES[case]
    frames = [make(k) for k in range(3)]
    got, hist, launches = _recorded(lib, frames, channels, weight, pw, iters)
    plain, plain_launches = _unrecorded(lib, frames, channels, weight, pw, iters)
    assert launches <= plain_launches + 1, (launches, plain_launches)
    for k, img in enumerate(frames):
        want, log = H.run_compute('oracle', img, channels, weight, pw, iters, want_log=True)
        for c in range(len(channels)):
            H.assert_bit_identical(got[k][c], plain[k][c], f'{case} frame {k} plane {c}: recorded vs unrecorded')
            H.assert_bit_identical(got[k][c], want[c], f'{case} frame {k} plane {c}: recorded vs checker')
        np.testing.assert_allclose(hist[k], log, **TOL, err_msg=f'{case} frame {k}')
        assert hist[k][0][1] == 0.0                        # iteration 0: no DCT distance yet
        if weight == 0.0:
            assert (hist[k][:, 3] == 0.0).all()


@pytest.mark.parametrize('iters', [0, 1])
def test_zero_and_one_iterations(lib, iters):
    make, channels, weight, pw, _, _ = CASES['420']
    frames = [make(k) for k in range(3)]
    got, hist, _ = _recorded(lib, frames, channels, weight, pw, iters)
    assert hist.shape == (3, iters, 4)
    for k, img in enumerate(frames):
        want, log = H.run_compute('oracle', img, channels, weight, pw, iters, want_log=True)
        for c in range(3):
            H.assert_bit_identical(got[k][c], want[c], f'frame {k} plane {c}')
        np.testing.assert_allclose(hist[k], log.reshape(iters, 4), **TOL)


def test_record_does_not_depend_on_the_batch(lib):
    make, channels, weight, pw, iters, _ = CASES['420']
    frames = [make(k) for k in range(5)]
    _, alone, _ = _recorded(lib, frames[2:3], channels, weight, pw, iters)
    _, again, _ = _recorded(lib, frames[2:3], channels, weight, pw, iters)
    _, two, _ = _recorded(lib, [frames[0], frames[2]], channels, weight, pw, iters)
    _, five, _ = _recorded(lib, frames, channels, weight, pw, iters)
    _, moved, _ = _recorded(lib, [frames[2], frames[4], frames[0]], channels, weight, pw, iters)
    want = alone[0].view(np.uint64)
    for got, what in ((again[0], 'second run'), (two[1], 'batch of 2'), (five[2], 'batch of 5'), (moved[0], 'position 0')):
        assert (got.view(np.uint64) == want).all(), what
    # a single-frame session records what a batch of one does
    with abi.Session(lib, abi.frame_desc(frames[2], channels, weight, pw, iters), batch=False) as s:
        _check(lib, lib.j2p_session_record_objective(s.s, 1))
        s.upload(frames[2:3], channels)
        s.iterate(0, iters)
        h = np.zeros((iters, 4))
        _check(lib, lib.j2p_session_objective_history(s.s, 0, iters, h.ctypes.data_as(C.POINTER(C.c_double))))
    assert (h.view(np.uint64) == want).all()


def test_history_in_pieces_and_rearming(lib):
    make, channels, weight, pw, iters, _ = CASES['444']
    frames = [make(k) for k in range(2)]
    _, whole, _ = _recorded(lib, frames, channels, weight, pw, iters)
    with abi.Session(lib, abi.frame_desc(frames[0], channels, weight, pw, iters), 2) as s:
        _check(lib, lib.j2p_session_record_objective(s.s, 1))
        s.upload(frames, channels)
        for rep in range(2):                              # the second solve re-arms: the record starts again
            s.iterate(0, 3)
            s.iterate(3, iters - 3)
            h = np.zeros((2, 2, 4))
            _check(lib, lib.j2p_session_objective_history(s.s, 4, 2, h.ctypes.data_as(C.POINTER(C.c_double))))
            assert (h.view(np.uint64) == whole[:, 4:6].view(np.uint64)).all(), rep


def _refused(lib, rc, words):
    assert rc == -1, rc                                     # J2P_ERR_ARG
    msg = lib.j2p_last_error().decode()
    assert all(w in msg for w in words), msg


def test_refusals(lib):
    make, channels, weight, pw, iters, _ = CASES['444']
    img = make(0)
    d = abi.frame_desc(img, channels, weight, pw, iters)
    strip = C.c_void_p()
    _check(lib, lib.j2p_session_create_strip(C.byref(strip), 0, C.byref(d), 0, 16))
    try:
        _refused(lib, lib.j2p_session_record_objective(strip, 1), ['strip'])
    finally:
        lib.j2p_session_destroy(strip)
    with abi.Session(lib, d, batch=False) as s:
        _check(lib, lib.j2p_session_set_logging(s.s, 1))
        _refused(lib, lib.j2p_session_record_objective(s.s, 1), ['logs the objective'])
    with abi.Session(lib, d, batch=False) as s, abi.Session(lib, d, 2) as b:
        _check(lib, lib.j2p_session_record_objective(s.s, 1))
        _refused(lib, lib.j2p_session_set_logging(s.s, 1), ['records the objective'])
        s.upload([img], channels)
        b.upload([img, img], channels)
        _check(lib, lib.j2p_session_record_objective(b.s, 1))
        ss = (C.c_void_p * 2)(s.s, b.s)
        _refused(lib, lib.j2p_session_iterate_group(ss, 2, 0, 1), ['group session 0 records the objective'])
        _refused(lib, lib.j2p_session_iterate(b.s, 0, iters + 1), ['holds', str(iters)])
        s.iterate(0, 3)
        h = np.zeros(4 * 4)
        _refused(lib, lib.j2p_session_objective_history(s.s, 2, 2, h.ctypes.data_as(C.POINTER(C.c_double))), ['not been recorded'])
        _check(lib, lib.j2p_session_objective_history(s.s, 1, 2, h.ctypes.data_as(C.POINTER(C.c_double))))
        _refused(lib, lib.j2p_session_iterate(s.s, 3, iters - 2), ['holds'])


def jpeg(w, h, seed, gray=False, subsampling='4:2:0', orientation=None, progressive=False):
    im = Image.fromarray(synth.cartoon_image(w, h, seed).astype(np.uint8), 'RGB')
    if gray:
        im = im.convert('L')
    kw = {}
    if orientation is not None:
        e = Image.Exif()
        e[0x0112] = orientation
        kw['exif'] = e.tobytes()
    buf = io.BytesIO()
    im.save(buf, 'JPEG', quality=40, subsampling=subsampling, progressive=progressive, **kw)
    return buf.getvalue()


FILES = ([jpeg(w, h, 10 + k) for k, (w, h) in enumerate([(64, 48), (80, 32), (48, 64), (96, 96)])]     # sizes that would be grouped
         + [jpeg(128, 64, 20 + k) for k in range(3)]                                                  # one batch
         + [jpeg(72, 40, 30, gray=True), jpeg(96, 64, 31, progressive=True), jpeg(64, 48, 32, orientation=6)])


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)


@pytest.mark.parametrize('progressive_on_device', [False, True])
@pytest.mark.parametrize('kw', [dict(mode='UNCHANGED'), dict(mode='UNCHANGED', separate=True, iterations=[7, 5, 3], weight=[0.3, 0.0, 0.2]),
                                dict(mode='GRAY', separate=True, dtype=torch.float32, layout='HWC'), dict(mode='GRAY')])
def test_decode_jpeg_return_objective(kw, progressive_on_device):
    kw = dict(dict(iterations=6, apply_exif_orientation=True, progressive_on_device=progressive_on_device), **kw)
    plain = decode_jpeg(FILES, **kw)
    images, logs = decode_jpeg(FILES, return_objective=True, **kw)
    assert len(images) == len(logs) == len(FILES)
    for i, (a, b) in enumerate(zip(images, plain)):
        assert _same(a, b), i
    its = kw['iterations'] if isinstance(kw['iterations'], list) else [kw['iterations']] * 3
    for i, log in enumerate(logs):
        gray_file = i == 7
        if gray_file or (kw['mode'] == 'GRAY' and kw.get('separate')):
            want = {0: its[0]}
        elif kw.get('separate'):
            want = {c: its[c] for c in range(3)}
        else:
            want = {3: its[0]}
        assert sorted(log) == sorted(want), (i, sorted(log))
        for c, t in log.items():
            assert t.dtype == torch.float64 and t.device.type == 'cpu' and tuple(t.shape) == (want[c], 4), (i, c, t.shape)
    # one file alone gives the bits it gets inside the list
    for i in (0, 4, 8):
        one, log = decode_jpeg(FILES[i], return_objective=True, **kw)
        assert _same(one, images[i])
        assert sorted(log) == sorted(logs[i])
        for c in log:
            assert torch.equal(log[c].view(torch.int64), logs[i][c].view(torch.int64)), (i, c)


def test_return_objective_is_true_or_false():
    for bad in (1, 0, None, 'yes'):
        with pytest.raises(ValueError, match='return_objective'):
            decode_jpeg(FILES[0], return_objective=bad)


def _parse_csv(text):
    lines = text.strip().splitlines()
    assert lines[0] == 'filename,channel,iteration,objective,prob_dist,tv,tv2'
    rows = {}
    for line in lines[1:]:
        f = line.split(',')
        rows[(f[0], int(f[1]), int(f[2]))] = [float(v) for v in f[3:]]
    return rows


@pytest.mark.parametrize('sep', [False, True])
def test_csv_matches_the_command_line(tmp_path, sep):
    subprocess.run(['make', '-C', os.path.join(ROOT, 'jpeg2png_b200', 'cli'), 'jpeg2png'], check=True, capture_output=True)
    exe = os.path.join(ROOT, 'jpeg2png_b200', 'cli', 'jpeg2png')
    names = []
    for k, data in enumerate([FILES[0], FILES[4], FILES[5]]):          # the command line reads colour files only
        p = tmp_path / f'f{k}.jpg'
        p.write_bytes(data)
        names.append(str(p))
    args = ['-s', '-i', '9,7,5', '-w', '0.3,0.0,0.2'] if sep else ['-i', '9', '-w', '0.3']
    kw = dict(separate=True, iterations=[9, 7, 5], weight=[0.3, 0.0, 0.2]) if sep else dict(iterations=9, weight=0.3)
    cli_csv = tmp_path / 'cli.csv'
    for n in names:                                # one file per run: the rows of one file stay together
        part = tmp_path / 'part.csv'
        r = subprocess.run([exe, '-q', '-f', *args, '-c', str(part), n], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        text = part.read_text()
        cli_csv.write_text((cli_csv.read_text() if cli_csv.exists() else text.splitlines()[0] + '\n') + ''.join(l + '\n' for l in text.strip().splitlines()[1:]))
    _, logs = decode_jpeg(names, mode='UNCHANGED', return_objective=True, **kw)
    ours = tmp_path / 'ours.csv'
    jpeg2png_b200.write_objective_csv(ours, names, logs)
    want, got = _parse_csv(cli_csv.read_text()), _parse_csv(ours.read_text())
    assert sorted(got) == sorted(want)
    for key in want:
        np.testing.assert_allclose(got[key], want[key], rtol=1e-6, atol=1.5e-6, err_msg=str(key))
