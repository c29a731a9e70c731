"""GPU tests of arithmetic-coded JPEGs: the device decoder of libj2parith.so against the reader on the
SOF9 corpus, per-file statuses, decode_jpeg of each arithmetic file against decode_jpeg of its
Huffman twin (dtypes, separate, modes, EXIF orientation, return_objective, mixed lists, both sides of
the routing rule), the routing itself, and the command line's PNG against its twin's."""
import os
import subprocess

import numpy as np
import pytest
import torch

from jpeg2png_b200 import decode as D
from tests import arith_cases as AC
from tests import arith_synth as A
from tests import entropy_cases as E

pytestmark = pytest.mark.gpu

CLI_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'jpeg2png_b200', 'cli')
CORPUS = AC.corpus()
SEQUENTIAL = AC.sequential(CORPUS)


def _device_decode(datas):
    lays = [D.ArithFileLayout(d, D.READ_GRAY) for d in datas]
    assert all(l.arith_decodable for l in lays)
    stream = torch.cuda.Stream()
    dc = D._ArithCoefs(torch.cuda.current_device(), lays, stream)
    torch.cuda.synchronize()
    return lays, dc


def test_device_decoder_equals_reader():
    names = list(SEQUENTIAL)
    datas = [SEQUENTIAL[n][0] for n in names]
    coded = AC.coded_corpus()
    for n in ('large_444', 'large_420_ri3', 'large_odd_sampling'):
        names.append(n)
        datas.append(coded[n][0])
    lays, dc = _device_decode(datas)
    assert not dc.status.any()
    assert dc.stats.launches == 1 and dc.stats.segments == sum(l.lay.nseg for l in lays)
    for i, (n, d) in enumerate(zip(names, datas)):
        for c, want in enumerate(AC.reader_planes(d)):
            got = dc.plane_tensor(i, c).cpu().numpy()
            assert np.array_equal(got, want), n


def test_one_corrupt_file_in_64():
    base = [SEQUENTIAL[n][0] for n in sorted(SEQUENTIAL)]
    datas = [base[i % len(base)] for i in range(64)]
    bad = A.raw_scan(8, 8, [('dc', 0, 0), ('ac', 0, 0)] + [('ac', 3 * (k - 1) + 1, 0) for k in range(1, 64)])
    datas[37] = bad
    _, dc = _device_decode(datas)
    assert [i for i in range(64) if dc.status[i]] == [37] and dc.status[37] == 1


def test_routing_per_chunk(monkeypatch):
    """decode_jpeg asks arith_on_device once per chunk of arithmetic files and parses them on the host
    when it says no, before any device work: errors in their entropy-coded data are then the reader's,
    naming the input.  Both routes give the same images."""
    seen = []
    real = D.arith_on_device
    monkeypatch.setattr(D, 'arith_on_device', lambda lays, workers: seen.append(len(lays)) or False)
    bad = A.raw_scan(8, 8, [('dc', 0, 0), ('ac', 0, 0)] + [('ac', 3 * (k - 1) + 1, 0) for k in range(1, 64)])
    with pytest.raises(ValueError, match=r'input 1: corrupt jpeg: bad arithmetic code'):
        D.decode_jpeg([CORPUS['pillow_420_ri1'][0], bad], mode='UNCHANGED')
    assert sorted(seen) == [1, 1]                                      # two geometries, one call each
    files = [CORPUS[n][0] for n in ('pillow_420_ri1', 'pillow_420_q75', 'pillow_420_rirow', 'pillow_444_q100')]
    host = D.decode_jpeg(files, iterations=5)
    monkeypatch.setattr(D, 'arith_on_device', lambda lays, workers: True)
    _same(D.decode_jpeg(files, iterations=5), host)
    monkeypatch.setattr(D, 'arith_on_device', real)
    _same(D.decode_jpeg(files, iterations=5), host)


@pytest.fixture
def device_route(monkeypatch):
    """Every SOF9 file of the shape the device decoder takes goes there, whatever arith_on_device says
    (the host route is the reader, checked against the Huffman twins on the CPU)."""
    monkeypatch.setattr(D, 'arith_on_device', lambda lays, workers: True)


def _same(a, b):
    if isinstance(a, (list, tuple)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _same(x, y)
    elif isinstance(a, dict):
        assert a.keys() == b.keys()
        for k in a:
            _same(a[k], b[k])
    else:
        assert torch.equal(a, b)


TWINS = ['pillow_420_q75', 'pillow_444_q20', 'pillow_422_q90', 'pillow_420_rirow', 'pillow_420_components_ri7',
         'dac_nondefault', 'pillow_prog_own_sof10', 'pillow_1x1', 'pillow_7x9', 'synth_1_ri2']


@pytest.mark.parametrize('dtype', [torch.uint8, torch.uint16, torch.float32])
@pytest.mark.parametrize('separate', [False, True])
def test_decode_jpeg_equals_huffman_twin(dtype, separate, device_route):
    arith = [CORPUS[n][0] for n in TWINS]
    twins = [CORPUS[n][1] for n in TWINS]
    kw = dict(iterations=10, dtype=dtype, separate=separate)
    _same(D.decode_jpeg(arith, **kw), D.decode_jpeg(twins, **kw))


@pytest.mark.parametrize('mode', ['GRAY', 'UNCHANGED'])
def test_decode_jpeg_modes(mode, device_route):
    names = ['gray_q10_ri0', 'gray_q85_ri5', 'gray_progressive', 'pillow_420_q50', 'pillow_420_ri1']
    for separate in (False, True):
        kw = dict(iterations=8, mode=mode, separate=separate)
        _same(D.decode_jpeg([CORPUS[n][0] for n in names], **kw), D.decode_jpeg([CORPUS[n][1] for n in names], **kw))


def _exif(orientation):
    tiff = b'MM\x00\x2a\x00\x00\x00\x08' + b'\x00\x01' + b'\x01\x12\x00\x03\x00\x00\x00\x01' + bytes([0, orientation, 0, 0]) + b'\x00' * 4
    return A._seg(0xE1, b'Exif\x00\x00' + tiff)


def test_decode_jpeg_exif_orientation(device_route):
    twins = []
    for k, o in enumerate((1, 3, 6, 8)):
        src = E.pillow(64 + 8 * k, 48, 70, '4:2:0', seed=k)
        twins.append(src[:2] + _exif(o) + src[2:])
    arith = [A.transcode(t, 'sequential', 'row' if k % 2 else 0) for k, t in enumerate(twins)]
    assert [D.exif_orientation(a) for a in arith] == [1, 3, 6, 8]
    kw = dict(iterations=6, apply_exif_orientation=True)
    _same(D.decode_jpeg(arith, **kw), D.decode_jpeg(twins, **kw))


def test_decode_jpeg_return_objective(device_route):
    names = ['pillow_420_q75', 'pillow_420_ri7', 'pillow_prog_own_sof10']
    for separate in (False, True):
        kw = dict(iterations=7, return_objective=True, separate=separate)
        _same(D.decode_jpeg([CORPUS[n][0] for n in names], **kw), D.decode_jpeg([CORPUS[n][1] for n in names], **kw))


@pytest.mark.parametrize('on_device', [False, True])
def test_mixed_list_on_both_routes(monkeypatch, on_device):
    """Huffman sequential and progressive files, SOF10 files and SOF9 files with and without restart
    intervals in one call, with and without progressive_on_device, equal the call on the Huffman twins
    alone, with the SOF9 files on either route."""
    huff = E.pillow(64, 48, 60, '4:2:0', seed=9)
    hprog = E.pillow(64, 48, 60, '4:2:0', progressive=True, seed=9)
    names = ['pillow_420_ri1', 'pillow_420_q75', 'pillow_prog_own_sof10', 'pillow_420_rirow', 'pillow_444_q100']
    monkeypatch.setattr(D, 'arith_on_device', lambda lays, workers: on_device)
    arith = [huff, hprog] + [CORPUS[n][0] for n in names]
    twins = [huff, hprog] + [CORPUS[n][1] for n in names]
    for prog in (False, True):
        _same(D.decode_jpeg(arith, iterations=9, progressive_on_device=prog), D.decode_jpeg(twins, iterations=9))


def test_cli_png_byte_identical_to_twin(tmp_path):
    subprocess.run(['make', '-C', CLI_DIR, 'jpeg2png'], check=True, capture_output=True)
    for n in ('pillow_420_q75', 'pillow_prog_own_sof10', 'pillow_420_ri7'):
        arith, twin = CORPUS[n]
        pngs = []
        for tag, data in (('a', arith), ('h', twin)):
            src = tmp_path / f'{n}_{tag}.jpg'
            src.write_bytes(data)
            r = subprocess.run([os.path.join(CLI_DIR, 'jpeg2png'), '-q', '-i', '12', str(src)], capture_output=True, text=True)
            assert r.returncode == 0, r.stderr
            pngs.append((tmp_path / f'{n}_{tag}.png').read_bytes())
        assert pngs[0] == pngs[1], n
