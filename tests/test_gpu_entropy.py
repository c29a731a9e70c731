"""The device entropy decoder (libj2pentropy.so) and its use by decode_jpeg, on the GPU, compared
exactly with the host reader (j2p_read_jpeg_mem): Pillow and jpeg_synth files of every sampling
layout, quality and size class, multi-scan files, crafted streams, a corrupt file among many,
j2p_session_upload_device against j2p_session_upload, and decode_jpeg against its host front end."""
import numpy as np
import pytest
import torch

from jpeg2png_b200 import abi, decode_jpeg
from jpeg2png_b200 import decode as D
from tests import entropy_cases as E
from tests.test_entropy_host import CORPUS, SAMPLINGS
from tests.test_gpu_decode import FILES, PW

pytestmark = pytest.mark.gpu


def device_decode(datas, subseq_bits=D.SUBSEQ_BITS):
    """Decode files in ONE call of the device decoder: ([per file: 3 int16 arrays], statuses, stats)."""
    lays = [D.FileLayout(d) for d in datas]
    assert all(x.device_decodable for x in lays)
    dc = D._DeviceCoefs(torch.cuda.current_device(), lays, torch.cuda.Stream(), subseq_bits)
    planes = [[dc.plane_tensor(i, c).cpu().numpy() for c in range(3)] for i in range(len(lays))]
    return planes, dc.status, dc.stats


def check_equal(datas, subseq_bits=D.SUBSEQ_BITS):
    """Every file the layout pass accepts, decoded in one call, equals the reader (or fails where it
    fails); every file the layout pass rejects, the reader rejects too."""
    todo = []
    for data in datas:
        try:
            D.FileLayout(data)
        except ValueError:
            assert E.reader(data)[0] is None
            continue
        todo.append(data)
    assert todo
    planes, status, stats = device_decode(todo, subseq_bits)
    for i, data in enumerate(todo):
        want, err = E.reader(data)
        if want is None:
            assert status[i] != 0, f'file {i}: decoded, the reader says {err}'
            continue
        assert status[i] == 0, f'file {i}: status {status[i]}, the reader accepts it'
        for c in range(3):
            assert (planes[i][c] == want[c]).all(), f'file {i} plane {c}: {int((planes[i][c] != want[c]).sum())} differ'
    return stats


def _pillow_grid():
    out = []
    for q in (5, 10, 25, 50, 75, 90, 100):
        for ss in ('4:4:4', '4:2:2', '4:2:0'):
            for opt in (False, True):
                out.append(E.pillow(96 + q % 7, 64 + q % 5, q, ss, optimize=opt, seed=q))
    return out


GROUPS = {
    'pillow_quality_sampling_optimize': _pillow_grid,
    'pillow_small_sizes': lambda: [E.pillow(w, h, q, ss) for w, h in [(1, 1), (7, 9), (8, 8), (16, 16), (17, 33)]
                                   for q, ss in [(75, '4:2:0'), (90, '4:4:4')]],
    'pillow_1080p': lambda: [E.pillow(1920, 1080, 75, '4:2:0', seed=7000), E.pillow(1920, 1080, 90, '4:4:4', optimize=True)],
    'pillow_8k': lambda: [E.pillow(7680, 4320, 75, '4:2:0')],
    'pillow_strips': lambda: [E.pillow(16384, 16, 75, '4:2:0'), E.pillow(16, 16384, 75, '4:2:0')],
    'synth_sampling_restarts': lambda: [E.synth_file(48 + 8 * k, 40, s, ri) for k, s in enumerate(SAMPLINGS) for ri in (0, 1, 2, 7)],
    'multi_scan': lambda: [CORPUS[n] for n in ('three_scans_444', 'three_scans_420_ri3', 'luma_then_chroma_pair')],
    'crafted': lambda: [d for d in E.crafted().values() if _layout_ok(d)],
}


def _layout_ok(d):
    try:
        return D.FileLayout(d).device_decodable
    except ValueError:
        return False


@pytest.mark.parametrize('group', list(GROUPS))
def test_device_decoder_equals_reader(group):
    check_equal(GROUPS[group]())


def test_late_synchronisation_and_small_subsequences():
    stats = check_equal([E.crafted()['late_sync_one_bit_codes']])
    assert stats.rounds > 10 and stats.rounds == 4 * stats.round_trips
    stats = check_equal([E.pillow(640, 480, 75, '4:2:0'), CORPUS['synth_1_ri7']], subseq_bits=32)
    assert stats.rounds > 3


def test_one_corrupt_file_among_64_fails_only_its_status():
    datas = [E.pillow(64 + 8 * (i % 5), 48, 30 + i, ('4:2:0', '4:4:4', '4:2:2')[i % 3], seed=i) for i in range(63)]
    bad = E.crafted()['bad_code']
    datas.insert(40, bad)
    planes, status, stats = device_decode(datas)
    assert [i for i in range(64) if status[i]] == [40] and status[40] == 1
    for i, d in enumerate(datas):
        if i != 40:
            want = E.reader(d)[0]
            assert all((planes[i][c] == want[c]).all() for c in range(3))
    assert stats.launches == stats.rounds + 4


# ---- j2p_session_upload_device ---------------------------------------------------------------
def _solve_both(frames, lib):
    """Solve parsed frames once with j2p_session_upload and once with j2p_session_upload_device (the
    coefficients copied to the device by torch on a side stream that sleeps first)."""
    desc = D._frame_desc(frames[0], [0, 1, 2], 0.3, PW, 8)
    results = []
    for device_side in (False, True):
        with abi.Session(lib, desc, len(frames)) as s:
            keep = []
            side = torch.cuda.Stream()
            for f, p in enumerate(frames):
                for c in range(3):
                    pl = p.planes[c]
                    if device_side:
                        src = torch.from_numpy(pl.data).cuda()
                        t = torch.zeros_like(src)
                        torch.cuda.synchronize()
                        with torch.cuda.stream(side):
                            torch.cuda._sleep(20_000_000)            # the producer is late: the upload must wait
                            t.copy_(src)
                        keep += [src, t]
                        assert lib.j2p_session_upload_device(s.s, f * 3 + c, t.data_ptr(), pl.quant.ctypes.data,
                                                             side.cuda_stream) == 0, lib.j2p_last_error()
                    else:
                        assert lib.j2p_session_upload(s.s, f * 3 + c, pl.data.ctypes.data, pl.quant.ctypes.data, None) == 0
            s.iterate(0, 8)
            results.append(s.download())
    return results


@pytest.mark.parametrize('nframes', [1, 3])
def test_upload_device_equals_upload(nframes):
    lib = abi.load_product()
    frames = [D.parse_jpeg(E.pillow(72, 56, 40 + 10 * i, '4:2:0', seed=i)) for i in range(nframes)]
    host, dev = _solve_both(frames, lib)
    for f in range(nframes):
        for c in range(3):
            assert np.array_equal(host[f][c], dev[f][c]), f'frame {f} plane {c}'


def test_upload_device_refusals():
    lib = abi.load_product()
    p = D.parse_jpeg(E.pillow(32, 32, 50, '4:4:4'))
    desc = D._frame_desc(p, [0, 1, 2], 0.3, PW, 2)
    t = torch.from_numpy(p.planes[0].data).cuda()
    q = p.planes[0].quant
    zero = q.copy()
    zero[5] = 0
    host = np.zeros_like(p.planes[0].data)
    pinned = torch.from_numpy(p.planes[0].data).pin_memory()
    with abi.Session(lib, desc, 1) as s:
        ok = lambda *a: lib.j2p_session_upload_device(*a)  # noqa: E731
        assert ok(None, 0, t.data_ptr(), q.ctypes.data, None) == -1
        assert ok(s.s, 0, None, q.ctypes.data, None) == -1
        assert ok(s.s, 0, t.data_ptr(), None, None) == -1
        assert ok(s.s, 3, t.data_ptr(), q.ctypes.data, None) == -1
        assert b'out of range' in lib.j2p_last_error()
        assert ok(s.s, 0, t.data_ptr(), zero.ctypes.data, None) == -1
        assert b'quantization' in lib.j2p_last_error()
        assert ok(s.s, 0, host.ctypes.data, q.ctypes.data, None) == -1
        assert ok(s.s, 0, pinned.data_ptr(), q.ctypes.data, None) == -1
        assert b'not device memory' in lib.j2p_last_error()
        assert ok(s.s, 0, t.data_ptr(), q.ctypes.data, None) == 0


# ---- decode_jpeg: device front end against host front end ------------------------------------
def _both(data, **kw):
    got = decode_jpeg(data, **kw)
    D._host_front_end = True
    try:
        want = decode_jpeg(data, **kw)
    finally:
        D._host_front_end = False
    return got, want


@pytest.mark.parametrize('dtype', [torch.uint8, torch.uint16, torch.float32])
@pytest.mark.parametrize('sep', [False, True], ids=['joint', 'separate'])
def test_decode_jpeg_equals_host_front_end(dtype, sep):
    datas, kws = [], []
    for name, (make, (it, w), (its, ws)) in FILES.items():
        datas.append(make())
        kws.append(dict(iterations=its, weight=ws, separate=True) if sep else dict(iterations=it, weight=w))
    for data, kw in zip(datas, kws):
        got, want = _both(data, dtype=dtype, **kw)
        assert torch.equal(got, want)


def test_mixed_progressive_and_sequential_list():
    datas = [E.pillow(64, 48, 50, '4:2:0', progressive=(i % 2 == 1), seed=i) for i in range(6)]
    datas.append(CORPUS['three_scans_444'])
    got, want = _both(datas, iterations=5)
    assert len(got) == 7 and all(torch.equal(a, b) for a, b in zip(got, want))


def test_entropy_errors_name_the_input_with_the_reader_message():
    good = E.pillow(64, 48, 50, '4:2:0')
    with pytest.raises(ValueError, match=r'^input 1: corrupt jpeg: bad huffman code$'):
        decode_jpeg([good, E.crafted()['bad_code']], iterations=2)
    with pytest.raises(ValueError, match=r'^input 0: corrupt jpeg: restart marker out of sequence$'):
        decode_jpeg([E.crafted()['rst_out_of_sequence']], iterations=2)
    with pytest.raises(ValueError, match=r'^input 2: corrupt jpeg: coefficient index out of range$'):
        decode_jpeg([good, good, E.crafted()['bad_index']], iterations=2)


def test_device_rejection_of_a_readable_file_is_a_runtime_error(monkeypatch):
    real = D._DeviceCoefs.__init__

    def broken(self, *a, **k):
        real(self, *a, **k)
        self.status = self.status.copy()
        self.status[0] = 1
    monkeypatch.setattr(D._DeviceCoefs, '__init__', broken)
    with pytest.raises(RuntimeError, match=r'^input 0: the device entropy decoder failed \(bad huffman code\)'):
        decode_jpeg(E.pillow(64, 48, 50, '4:2:0'), iterations=2)


def test_front_end_routing():
    seq, prog = E.pillow(64, 48, 50, '4:2:0'), E.pillow(64, 48, 50, '4:2:0', progressive=True)
    assert isinstance(D._front_end(seq, True), D.FileLayout)
    assert isinstance(D._front_end(prog, True), D.Parsed)
    assert isinstance(D._front_end(seq, False), D.Parsed)
