"""CPU tests of the device entropy decoder's host side: the layout pass (j2p_read_jpeg_layout) against
the host reader (j2p_read_jpeg_mem), the serial host driver of the decoder's phases
(j2p_entropy_decode_host, the same per-block and per-subsequence code as the kernels) bit for bit
against the reader at subsequence sizes down to 32 bits, a mutation fuzz of both in a child process,
and the kernel inventory of libj2pentropy.so."""
import os
import subprocess
import sys

import numpy as np
import pytest

from jpeg2png_b200 import decode as D
from tests import codec_checks as CK
from tests import entropy_cases as E

# kernel -> the GPU test that reaches it (every call of j2p_entropy_decode launches all four)
KERNELS = {
    'k_ent_sync': 'tests/test_gpu_entropy.py::test_device_decoder_equals_reader (sync rounds)',
    'k_ent_scan': 'tests/test_gpu_entropy.py::test_device_decoder_equals_reader (block counts and DC sums)',
    'k_ent_final': 'tests/test_gpu_entropy.py::test_device_decoder_equals_reader (coefficients, statuses)',
    'k_ent_dc': 'tests/test_gpu_entropy.py::test_device_decoder_equals_reader (DC predictions)',
}

SAMPLINGS = [[(1, 1)] * 3, [(2, 2), (1, 1), (1, 1)], [(2, 1), (1, 1), (1, 1)], [(4, 1), (2, 1), (1, 1)],
             [(1, 2), (1, 1), (1, 1)], [(4, 1), (2, 1), (1, 2)]]


def corpus():
    """name -> bytes: the Pillow files of the CLI and decode tests, jpeg_synth files in every
    sampling layout with restart intervals, multi-scan files and the crafted streams."""
    files = {
        'pillow_420_q20': E.pillow(160, 120, 20, '4:2:0', seed=3),
        'pillow_444_q50_opt': E.pillow(97, 61, 50, '4:4:4', optimize=True),
        'pillow_422_q90': E.pillow(96, 80, 90, '4:2:2'),
        'pillow_420_odd_q5': E.pillow(73, 59, 5, '4:2:0'),
        'pillow_1x1': E.pillow(1, 1, 75, '4:2:0'),
        'pillow_7x9_q100': E.pillow(7, 9, 100, '4:4:4'),
        'pillow_progressive': E.pillow(64, 48, 60, '4:2:0', progressive=True),
    }
    for k, s in enumerate(SAMPLINGS):
        for ri in (0, 1, 2, 7):
            files[f'synth_{k}_ri{ri}'] = E.synth_file(48 + 8 * k, 40, s, ri)
    files['three_scans_444'] = E.synth_file(40, 24, [(1, 1)] * 3, 0, scans=[[0], [1], [2]])
    files['three_scans_420_ri3'] = E.synth_file(70, 50, [(2, 2), (1, 1), (1, 1)], 3, scans=[[0], [1], [2]])
    files['luma_then_chroma_pair'] = E.synth_file(70, 50, [(2, 2), (1, 1), (1, 1)], 0, scans=[[0], [1, 2]])
    files['twice_scanned'] = E.synth_file(40, 24, [(1, 1)] * 3, 0, scans=[[0, 1, 2], [0]])
    files['never_scanned'] = E.synth_file(40, 24, [(1, 1)] * 3, 0, scans=[[0], [1]])
    files.update(E.crafted())
    return files


CORPUS = corpus()


@pytest.mark.parametrize('name', list(CORPUS))
def test_layout_pass_matches_reader(name):
    data = CORPUS[name]
    want, err = E.reader(data)
    try:
        lay = D.FileLayout(data)
    except ValueError as e:
        assert want is None, f'the layout pass rejects ({e}) a file the reader accepts'
        return
    if not lay.device_decodable:
        return
    p = D.parse_jpeg(data) if want is not None else None
    if p is not None:
        assert (lay.w, lay.h) == (p.w, p.h)
        for a, b in zip(lay.planes, p.planes):
            assert (a.w, a.h, a.w_samp, a.h_samp) == (b.w, b.h, b.w_samp, b.h_samp)
            assert (a.quant == b.quant).all()
    # the segments re-decode to the reader's coefficients, or fail where it fails
    arrs, status, _ = E.entropy_host([lay], 1024)
    if want is None:
        assert status[0] != 0, f'decoded a file the reader rejects: {err}'
    else:
        assert status[0] == 0
        for c in range(3):
            assert (arrs[0][c] == want[c]).all(), f'plane {c}'


def test_routing_rule():
    dd = {name: D.FileLayout(CORPUS[name]).device_decodable for name in
          ['pillow_420_q20', 'pillow_progressive', 'three_scans_444', 'three_scans_420_ri3', 'luma_then_chroma_pair',
           'twice_scanned', 'never_scanned', 'synth_1_ri7']}
    assert dd == {'pillow_420_q20': True, 'pillow_progressive': False, 'three_scans_444': True,
                  'three_scans_420_ri3': True, 'luma_then_chroma_pair': True, 'twice_scanned': False,
                  'never_scanned': False, 'synth_1_ri7': True}
    # the reader does decode the host-routed ones (never_scanned: its third plane stays zero)
    assert E.reader(CORPUS['twice_scanned'])[0] is not None and E.reader(CORPUS['never_scanned'])[0] is not None


def test_layout_segments_follow_restart_intervals():
    lay = D.FileLayout(CORPUS['synth_1_ri7'])
    sc = lay.lay.scan[0]
    total = sc.mcux * sc.mcuy
    assert sc.restart_interval == 7 and sc.nseg == -(-total // 7) == lay.lay.nseg
    mcus = [lay.lay.seg[k].mcus for k in range(sc.nseg)]
    assert sum(mcus) == total and all(m == 7 for m in mcus[:-1])
    segs = [lay.lay.seg[k] for k in range(sc.nseg)]
    assert [g.off for g in segs] == list(np.cumsum([0] + [g.len for g in segs[:-1]]))
    assert sum(g.len for g in segs) == lay.lay.data_len
    three = D.FileLayout(CORPUS['three_scans_420_ri3']).lay
    assert three.nscan == 3 and [three.scan[k].comp[0] for k in range(3)] == [0, 1, 2]
    assert (three.scan[0].mcux, three.scan[1].mcux) == (9, 5)          # non-interleaved: the real block grid


@pytest.mark.parametrize('subseq_bits', [32, 64, 96, 256, 1024, 4096])
def test_host_driver_equals_reader_bit_for_bit(subseq_bits):
    names = [n for n in CORPUS if E.reader(CORPUS[n])[0] is not None]
    lays, wants = [], []
    for n in names:
        lay = D.FileLayout(CORPUS[n])
        if lay.device_decodable:
            lays.append(lay)
            wants.append(E.reader(CORPUS[n])[0])
    assert len(lays) > 30
    arrs, status, stats = E.entropy_host(lays, subseq_bits)      # all files in one call
    assert (status == 0).all()
    for lay, got, want in zip(lays, arrs, wants):
        for c in range(3):
            assert (got[c] == want[c]).all()
    if subseq_bits <= 64:
        assert stats.rounds > 3            # small subsequences: synchronisation took several rounds


def test_one_corrupt_file_fails_only_its_status():
    names = ['pillow_420_q20', 'bad_code', 'synth_2_ri2', 'bad_index', 'bad_magnitude', 'three_scans_444']
    lays = [D.FileLayout(CORPUS[n]) for n in names]
    arrs, status, _ = E.entropy_host(lays, 64)
    assert list(status) == [0, 1, 0, 3, 2, 0]
    for n, got, st in zip(names, arrs, status):
        if st == 0:
            want = E.reader(CORPUS[n])[0]
            assert all((got[c] == want[c]).all() for c in range(3))


def test_pack_refuses_bad_arguments():
    lay = D.FileLayout(CORPUS['pillow_420_q20'])
    with pytest.raises(RuntimeError, match='multiple of 32'):
        D.entropy_plan([lay], [0, 0, 0], 48)
    prog = D.FileLayout(CORPUS['pillow_progressive'])
    with pytest.raises(RuntimeError, match='not device-decodable'):
        D.entropy_plan([prog], [0, 0, 0])


def test_layout_and_decoder_survive_mutated_files():
    r = subprocess.run([sys.executable, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'fuzz_entropy.py'), '600', '3'],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert 'no disagreement' in r.stdout


def test_kernel_inventory_is_covered_and_does_not_spill():
    CK.check_kernel_inventory('entropy/libj2pentropy.so', KERNELS)
