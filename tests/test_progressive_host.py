"""CPU tests of the progressive device decoder's host side: the progressive layout pass
(j2p_read_jpeg_prog_layout) against the host reader (j2p_read_jpeg_mem), the serial host driver of
the decoder's passes (j2p_progressive_decode_host, the same per-block, per-subsequence and
per-segment code as the kernels) bit for bit against the reader at subsequence sizes from 32 to 4096
bits, one quirk of the reader per crafted file, a mutation fuzz in a child process, and the kernel
inventory of libj2pprogressive.so."""
import os
import subprocess
import sys

import pytest

from jpeg2png_b200 import decode as D
from tests import codec_checks as CK
from tests import entropy_cases as E
from tests import progressive_cases as P

# kernel -> the GPU test that reaches it
KERNELS = {
    'k_pg_zero': 'tests/test_gpu_progressive.py::test_device_decoder_equals_reader (every call)',
    'k_pg_sync': 'tests/test_gpu_progressive.py::test_device_decoder_equals_reader (sync rounds of DC and AC first scans)',
    'k_pg_scan': 'tests/test_gpu_progressive.py::test_device_decoder_equals_reader (block counts and DC sums)',
    'k_pg_dcdiff': 'tests/test_gpu_progressive.py::test_device_decoder_equals_reader (DC differences)',
    'k_pg_store': 'tests/test_gpu_progressive.py::test_device_decoder_equals_reader (DC predictions, AC first bands)',
    'k_pg_dcref': 'tests/test_gpu_progressive.py::test_device_decoder_equals_reader (DC refine)',
    'k_pg_mask': 'tests/test_gpu_progressive.py::test_device_decoder_equals_reader (nonzero masks)',
    'k_pg_refine': 'tests/test_gpu_progressive.py::test_device_decoder_equals_reader (AC refine walkers)',
}


def corpus():
    """name -> bytes: Pillow progressive files (with and without restart markers) and crafted scripts."""
    files = P.pillow_grid()
    for q in (10, 75):
        for ss in ('4:4:4', '4:2:2', '4:2:0'):
            files[f'pillow_restarts_q{q}_{ss}'] = P.pillow_restarts(96, 64, q, ss, seed=q)
            files[f'pillow_restarts_opt_q{q}_{ss}'] = P.pillow_restarts(64, 48, q, ss, optimize=True, seed=q + 1, rows=2)
    files.update(P.crafted())
    return files


CORPUS = corpus()


@pytest.mark.parametrize('name', list(CORPUS))
def test_layout_pass_matches_reader(name):
    data = CORPUS[name]
    want, err = E.reader(data)
    lay = P.layout(data)
    if lay is None:
        assert want is None, 'the layout pass rejects a file the reader accepts'
        return
    assert lay.progressive_decodable
    if want is not None:
        p = D.parse_jpeg(data)
        assert (lay.w, lay.h) == (p.w, p.h)
        for a, b in zip(lay.planes, p.planes):
            assert (a.w, a.h, a.w_samp, a.h_samp) == (b.w, b.h, b.w_samp, b.h_samp)
            assert (a.quant == b.quant).all()
    arrs, status, _ = P.prog_host([lay], 1024)
    if want is None:
        assert status[0] != 0, f'decoded a file the reader rejects: {err}'
    else:
        assert status[0] == 0
        for c in range(3):
            assert (arrs[0][c] == want[c]).all(), f'plane {c}'


def test_sequential_files_are_not_progressive_layouts():
    seq = E.pillow(64, 48, 50, '4:2:0')
    assert not D.ProgFileLayout(seq).progressive_decodable
    assert D.ProgFileLayout(E.pillow(64, 48, 50, '4:2:0', progressive=True)).progressive_decodable
    # the sequential layout pass still routes progressive files to the host reader
    assert not D.FileLayout(E.pillow(64, 48, 50, '4:2:0', progressive=True)).device_decodable


def test_layout_records_scans():
    keep = D.ProgFileLayout(P.pillow_restarts(96, 64, 75, '4:2:0'))
    lay = keep.lay
    assert lay.nscan == 10
    got = [(lay.scan[k].ss, lay.scan[k].se, lay.scan[k].ah, lay.scan[k].al, lay.scan[k].s.ncomp) for k in range(10)]
    assert got == [(0, 0, 0, 1, 3), (1, 5, 0, 2, 1), (1, 63, 0, 1, 1), (1, 63, 0, 1, 1), (6, 63, 0, 2, 1),
                   (1, 63, 2, 1, 1), (0, 0, 1, 0, 3), (1, 63, 1, 0, 1), (1, 63, 1, 0, 1), (1, 63, 1, 0, 1)]
    assert all(lay.scan[k].s.nseg > 1 and lay.scan[k].s.restart_interval > 0 for k in range(10))
    assert sum(lay.scan[k].s.nseg for k in range(10)) == lay.nseg


@pytest.mark.parametrize('subseq_bits', [32, 64, 96, 256, 1024, 4096])
def test_host_driver_equals_reader_bit_for_bit(subseq_bits):
    names = [n for n in CORPUS if E.reader(CORPUS[n])[0] is not None]
    lays = [D.ProgFileLayout(CORPUS[n]) for n in names]
    assert len(lays) > 100
    arrs, status, stats = P.prog_host(lays, subseq_bits)      # all files in one call
    assert (status == 0).all()
    for n, got in zip(names, arrs):
        want = E.reader(CORPUS[n])[0]
        for c in range(3):
            assert (got[c] == want[c]).all(), (n, c)
    assert stats.steps == max(x.lay.nscan for x in lays)
    if subseq_bits <= 64:
        assert stats.rounds > 3


def test_quirks_each_have_a_file():
    cases = P.crafted()
    for name in ('run_past_se', 'refine_size_2_3', 'eob_32767', 'eob_runs_cross_restarts', 'odd_0'):
        want, err = E.reader(cases[name])
        assert want is not None, (name, err)
        arrs, status, _ = P.prog_host([D.ProgFileLayout(cases[name])], 32)
        assert status[0] == 0 and all((arrs[0][c] == want[c]).all() for c in range(3)), name
    # the run lands at zig-zag 11 (natural 25), past Se = 5, and is stored there
    y = E.reader(cases['run_past_se'])[0][0]
    assert y[25] == 1 and not y[1:25].any() and not y[26:].any()
    # refine symbols of size 2 and 3 place +1 and -1 at zig-zag 1 and 2 (natural 1 and 8)
    y = E.reader(cases['refine_size_2_3'])[0][0]
    assert (y[1], y[8]) == (1, -1)
    # the odd script never scans component 2: its plane stays zero
    assert not E.reader(cases['odd_0'])[0][2].any()
    for name, code in (('bad_code', 1), ('bad_code_refine', 1), ('dc_category_17', 2), ('bad_index', 3)):
        assert E.reader(cases[name])[0] is None
        _, status, _ = P.prog_host([D.ProgFileLayout(cases[name])], 64)
        assert status[0] == code, name


def test_one_corrupt_file_fails_only_its_status():
    cases = P.crafted()
    names = ['standard_random_0', 'bad_code', 'deep_ri2', 'bad_index', 'dc_category_17', 'bad_code_refine', 'eob_32767']
    lays = [D.ProgFileLayout(cases[n]) for n in names]
    arrs, status, _ = P.prog_host(lays, 64)
    assert list(status) == [0, 1, 0, 3, 2, 1, 0]
    for n, got, st in zip(names, arrs, status):
        if st == 0:
            want = E.reader(cases[n])[0]
            assert all((got[c] == want[c]).all() for c in range(3))


def test_pack_refuses_bad_arguments():
    lay = D.ProgFileLayout(CORPUS['pillow_64x48_q50_4:2:0_std'])
    with pytest.raises(RuntimeError, match='multiple of 32'):
        D.progressive_plan([lay], [0, 0, 0], 48)
    seq = D.ProgFileLayout(E.pillow(64, 48, 50, '4:2:0'))
    with pytest.raises(RuntimeError, match='not a progressive layout'):
        D.progressive_plan([seq], [0, 0, 0])


def test_layout_and_decoder_survive_mutated_files():
    r = subprocess.run([sys.executable, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'fuzz_progressive.py'), '500', '5'],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert 'no disagreement' in r.stdout


def test_kernel_inventory_is_covered_and_does_not_spill():
    CK.check_kernel_inventory('progressive/libj2pprogressive.so', KERNELS)
