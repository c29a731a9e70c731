"""The progressive device decoder (libj2pprogressive.so) and decode_jpeg(progressive_on_device=True),
on the GPU, compared exactly with the serial host driver and the host reader (j2p_read_jpeg_mem):
Pillow progressive files of every sampling, quality and size class, with restart markers, crafted
scan scripts, 1080p and 8K files, a corrupt file among 64, the launch count, and decode_jpeg against
its default (host reader) path."""
import pytest
import torch

from jpeg2png_b200 import decode_jpeg
from jpeg2png_b200 import decode as D
from tests import entropy_cases as E
from tests import progressive_cases as P
from tests.test_gpu_decode import FILES
from tests.test_progressive_host import CORPUS

pytestmark = pytest.mark.gpu


def device_decode(datas, subseq_bits=D.SUBSEQ_BITS):
    """Decode files in ONE call of the progressive device decoder: ([per file: 3 int16 arrays], statuses, stats, layouts)."""
    lays = [D.ProgFileLayout(d) for d in datas]
    assert all(x.progressive_decodable for x in lays)
    dc = D._ProgCoefs(torch.cuda.current_device(), lays, torch.cuda.Stream(), subseq_bits)
    planes = [[dc.plane_tensor(i, c).cpu().numpy() for c in range(3)] for i in range(len(lays))]
    return planes, dc.status, dc.stats, lays


def check_equal(datas, subseq_bits=D.SUBSEQ_BITS):
    """Every file the layout pass accepts, decoded in one call, equals the reader and the host driver
    (or fails where the reader fails)."""
    for d in datas:
        if P.layout(d) is None:
            assert E.reader(d)[0] is None
    todo = [d for d in datas if P.layout(d) is not None]
    assert todo
    planes, status, stats, lays = device_decode(todo, subseq_bits)
    host, hstatus, _ = P.prog_host(lays, subseq_bits)
    for i, data in enumerate(todo):
        want, err = E.reader(data)
        if want is None:
            assert status[i] != 0 and hstatus[i] != 0, f'file {i}: decoded, the reader says {err}'
            continue
        assert status[i] == 0, f'file {i}: status {status[i]}, the reader accepts it'
        for c in range(3):
            assert (planes[i][c] == want[c]).all(), f'file {i} plane {c}: {int((planes[i][c] != want[c]).sum())} differ'
            assert (host[i][c] == want[c]).all()
    return stats, lays


GROUPS = {
    'corpus': lambda: list(CORPUS.values()),
    'pillow_1080p_8k': lambda: [E.pillow(1920, 1080, 75, '4:2:0', progressive=True, seed=7000),
                                E.pillow(1920, 1080, 90, '4:4:4', optimize=True, progressive=True),
                                P.pillow_restarts(1920, 1080, 75, '4:2:0'),
                                E.pillow(7680, 4320, 75, '4:2:0', progressive=True)],
}


@pytest.mark.parametrize('group', list(GROUPS))
def test_device_decoder_equals_reader(group):
    check_equal(GROUPS[group]())


def test_small_subsequences():
    stats, _ = check_equal([E.pillow(640, 480, 75, '4:2:0', progressive=True), P.crafted()['deep_ri2']], subseq_bits=32)
    assert stats.rounds > 3 and stats.rounds == 4 * stats.round_trips


def _expected_step_launches(lays):
    n = 0
    for t in range(max(x.lay.nscan for x in lays)):
        kinds = set()
        for x in lays:
            if t < x.lay.nscan:
                s = x.lay.scan[t]
                kinds.add((s.ss > 0, s.ah > 0))
        n += ((False, False) in kinds or (True, False) in kinds) + ((False, True) in kinds) + 2 * ((True, True) in kinds)
    return n


def test_one_corrupt_file_among_64_fails_only_its_status():
    datas = [E.pillow(64 + 8 * (i % 5), 48, 30 + i, ('4:2:0', '4:4:4', '4:2:2')[i % 3], progressive=True, seed=i) for i in range(63)]
    datas.insert(40, P.crafted()['bad_code_refine'])
    planes, status, stats, lays = device_decode(datas)
    assert [i for i in range(64) if status[i]] == [40] and status[40] == 1
    for i, d in enumerate(datas):
        if i != 40:
            want = E.reader(d)[0]
            assert all((planes[i][c] == want[c]).all() for c in range(3))
    assert stats.step_launches == _expected_step_launches(lays)
    assert stats.launches == 1 + stats.rounds + 3 + stats.step_launches
    assert stats.steps == 10 and stats.refine_segments == 4 * 63 + 1


def _both(data, **kw):
    return decode_jpeg(data, progressive_on_device=True, **kw), decode_jpeg(data, **kw)


@pytest.mark.parametrize('dtype', [torch.uint8, torch.uint16, torch.float32])
@pytest.mark.parametrize('sep', [False, True], ids=['joint', 'separate'])
def test_decode_jpeg_equals_default_path(dtype, sep):
    for name, (make, (it, w), (its, ws)) in FILES.items():
        kw = dict(iterations=its, weight=ws, separate=True) if sep else dict(iterations=it, weight=w)
        data = E.pillow(96, 64, 60, '4:2:0', progressive=True, seed=len(name))
        for d in (data, make()):
            got, want = _both(d, dtype=dtype, **kw)
            assert torch.equal(got, want)


def test_mixed_sequential_progressive_and_host_routed_list():
    datas = [E.pillow(64, 48, 50, '4:2:0', progressive=(i % 2 == 1), seed=i) for i in range(6)]
    datas += [P.pillow_restarts(64, 48, 50, '4:2:0'), E.synth_file(40, 24, [(1, 1)] * 3, 0, scans=[[0, 1, 2], [0]]),
              P.crafted()['standard_random_0']]
    assert isinstance(D._front_end(datas[1], True, True), D.ProgFileLayout)
    assert isinstance(D._front_end(datas[7], True, True), D.Parsed)
    got, want = _both(datas, iterations=5)
    assert len(got) == 9 and all(torch.equal(a, b) for a, b in zip(got, want))


def test_errors_name_the_input_with_the_reader_message():
    good = E.pillow(64, 48, 50, '4:2:0', progressive=True)
    c = P.crafted()
    with pytest.raises(ValueError, match=r'^input 1: corrupt jpeg: bad huffman code$'):
        decode_jpeg([good, c['bad_code_refine']], iterations=2, progressive_on_device=True)
    with pytest.raises(ValueError, match=r'^input 2: corrupt jpeg: coefficient index out of range$'):
        decode_jpeg([good, good, c['bad_index']], iterations=2, progressive_on_device=True)
    with pytest.raises(ValueError, match=r'^input 0: corrupt jpeg: bad magnitude category$'):
        decode_jpeg([c['dc_category_17']], iterations=2, progressive_on_device=True)


def test_device_rejection_of_a_readable_file_is_a_runtime_error(monkeypatch):
    real = D._ProgCoefs.__init__

    def broken(self, *a, **k):
        real(self, *a, **k)
        self.status = self.status.copy()
        self.status[0] = 1
    monkeypatch.setattr(D._ProgCoefs, '__init__', broken)
    with pytest.raises(RuntimeError, match=r'^input 0: the device entropy decoder failed \(bad huffman code\)'):
        decode_jpeg(E.pillow(64, 48, 50, '4:2:0', progressive=True), iterations=2, progressive_on_device=True)
