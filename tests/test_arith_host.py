"""CPU tests of arithmetic-coded JPEGs (SOF9, SOF10): the test encoder against libjpeg-turbo (Pillow),
the reader against each file's Huffman twin, the arithmetic layout pass and the routing rule of
decode_jpeg, the serial host driver of libj2parith.so (the same per-segment code as its kernel)
against the reader, the refusals, a mutation fuzz in a child process, and the kernel inventory."""
import os
import subprocess
import sys

import numpy as np
import pytest

from jpeg2png_b200 import decode as D
from tests import arith_cases as AC
from tests import arith_synth as A
from tests import codec_checks as CK
from tests import entropy_cases as E

# kernel -> the GPU test that reaches it (every call of j2p_arith_decode launches it once)
KERNELS = {
    'k_arith_decode': 'tests/test_gpu_arith.py::test_device_decoder_equals_reader (every segment of the SOF9 corpus)',
}

CORPUS = AC.corpus()
CODED = AC.coded_corpus()
SEQUENTIAL = AC.sequential(CORPUS)


@pytest.mark.parametrize('name', list(CORPUS))
def test_encoder_matches_libjpeg(name):
    """Pillow (libjpeg-turbo) decodes each arithmetic file to its Huffman twin's pixels."""
    arith, twin = CORPUS[name]
    assert np.array_equal(A.pillow_pixels(arith), A.pillow_pixels(twin))


@pytest.mark.parametrize('name', list(CODED))
def test_coded_files_decode_in_libjpeg(name):
    A.pillow_pixels(CODED[name][0])             # libjpeg-turbo reads them without an error


@pytest.mark.parametrize('name', list(CORPUS))
def test_reader_equals_huffman_twin(name):
    arith, twin = CORPUS[name]
    got, want = AC.reader_planes(arith), AC.reader_planes(twin)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


@pytest.mark.parametrize('name', list(CODED))
def test_reader_equals_coded_coefficients(name):
    data, planes = CODED[name]
    for g, p in zip(AC.reader_planes(data), planes):
        assert np.array_equal(g, p.reshape(-1))


def test_rgb_mode_reader_refuses_gray_arith():
    with pytest.raises(ValueError, match='only 3 component jpegs are supported'):
        D.parse_jpeg(CORPUS['gray_q10_ri0'][0])


@pytest.mark.parametrize('name', list(CORPUS))
def test_layout_passes(name):
    """The Huffman layout passes report arithmetic files as not decodable without failing; the
    arithmetic pass takes the SOF9 files whose components are each in one scan."""
    arith, _ = CORPUS[name]
    assert not D.FileLayout(arith, D.READ_GRAY).device_decodable
    assert not D.ProgFileLayout(arith, D.READ_GRAY).progressive_decodable
    lay = D.ArithFileLayout(arith, D.READ_GRAY)
    assert lay.arith_decodable == (name in SEQUENTIAL)
    if not lay.arith_decodable:
        return
    p = D.parse_jpeg(arith, D.READ_GRAY)
    assert (lay.w, lay.h) == (p.w, p.h) and lay.key() == p.key()
    ri = lay.lay.scan[0].restart_interval
    for k in range(lay.lay.nscan):
        sc = lay.lay.scan[k]
        mcus = sc.mcux * sc.mcuy
        assert sc.restart_interval == ri
        assert sc.nseg == (-(-mcus // ri) if ri else 1)
        segs = [lay.lay.seg[sc.seg0 + q] for q in range(sc.nseg)]
        assert sum(g.mcus for g in segs) == mcus
        assert all(g.mcus == ri for g in segs[:-1])


def test_layout_records_dac_and_tables():
    lay = D.ArithFileLayout(CORPUS['dac_nondefault'][0])
    sc = lay.lay.scan[0]
    assert list(sc.dc_tbl) == [0, 1, 1] and list(sc.ac_tbl) == [0, 1, 1]
    assert list(sc.dc_L) == [2, 3, 3] and list(sc.dc_U) == [5, 15, 15] and list(sc.ac_K) == [1, 40, 40]
    lay = D.ArithFileLayout(CORPUS['pillow_444_q75'][0])
    sc = lay.lay.scan[0]
    assert list(sc.dc_L) == [0] * 3 and list(sc.dc_U) == [1] * 3 and list(sc.ac_K) == [5] * 3


def test_huffman_files_not_arith_decodable():
    for data in (E.pillow(64, 48, 75, '4:2:0'), E.pillow(64, 48, 75, '4:2:0', progressive=True)):
        assert not D.ArithFileLayout(data).arith_decodable


def test_front_end_takes_every_arith_decodable_file():
    """_front_end: SOF9 files whose components are each in one scan become ArithFileLayouts (the
    device-or-host choice is made per chunk); SOF10 files go to the host reader, with or without
    progressive_on_device."""
    for prog in (False, True):
        for name in ('pillow_420_ri1', 'pillow_444_q100', 'pillow_opt_components'):
            assert isinstance(D._front_end(CORPUS[name][0], True, prog), D.ArithFileLayout)
        assert isinstance(D._front_end(CORPUS['pillow_prog_own_sof10'][0], True, prog), D.Parsed)
        assert isinstance(D._front_end(CORPUS['gray_q10_ri0'][0], True, prog, D.READ_GRAY), D.ArithFileLayout)
    assert isinstance(D._front_end(CORPUS['pillow_444_q100'][0], False), D.Parsed)     # without a device: the host reader
    e = D._front_end(CORPUS['gray_q10_ri0'][0], True)                 # RGB mode: the reader's message
    assert isinstance(e, ValueError) and 'only 3 component' in str(e)


class _Lay:
    def __init__(self, longest, compressed):
        self.longest_segment, self.compressed = longest, compressed


def test_arith_on_device_rule():
    """The serial walk of the longest segment against the host's share of all the bytes."""
    dev, host = D.ARITH_DEVICE_NS_PER_BYTE, D.ARITH_HOST_NS_PER_BYTE
    one_segment = _Lay(200_000, 200_000)
    assert not D.arith_on_device([one_segment], 16)                     # one file, no restart interval
    assert not D.arith_on_device([one_segment] * 64, 16)               # 64 of them on 16 threads
    n = 16 * dev // host + 16                                          # enough files to outweigh the threads
    assert D.arith_on_device([one_segment] * n, 16)
    assert not D.arith_on_device([one_segment] * n, n)
    rows = _Lay(4_000, 200_000)                                        # 50 segments of 4 KB
    assert D.arith_on_device([rows], 1) == (4_000 * dev < 200_000 * host)
    assert D.arith_on_device([rows] * 64, 16)
    mixed = [one_segment] + [rows] * 63                                # the longest segment of the chunk counts
    assert D.arith_on_device(mixed, 16) == (200_000 * dev < (200_000 + 63 * 200_000) * host / 16)


def test_longest_segment_follows_restart_interval():
    one = D.ArithFileLayout(CORPUS['pillow_420_ri1'][0])
    row = D.ArithFileLayout(CORPUS['pillow_420_rirow'][0])
    whole = D.ArithFileLayout(A.transcode(CORPUS['pillow_420_ri1'][1]))
    assert one.longest_segment < row.longest_segment < whole.longest_segment
    assert whole.longest_segment == whole.compressed


def test_host_driver_equals_reader():
    names = list(SEQUENTIAL) + ['large_444', 'large_420_ri3', 'large_odd_sampling']
    datas = [SEQUENTIAL[n][0] if n in SEQUENTIAL else CODED[n][0] for n in names]
    lays = [D.ArithFileLayout(d, D.READ_GRAY) for d in datas]
    arrs, status, stats = AC.arith_host(lays)                # all files in one call
    assert not status.any()
    assert stats.segments == sum(l.lay.nseg for l in lays) and stats.launches == 0
    for n, d, got in zip(names, datas, arrs):
        for g, w in zip(got, AC.reader_planes(d)):
            assert np.array_equal(g, w), n


def test_host_driver_flags_only_the_corrupt_file():
    good = [SEQUENTIAL[n][0] for n in ('pillow_444_q50', 'pillow_420_ri7', 'gray_q85_ri5')]
    bad = _zero_run_past_63()
    lays = [D.ArithFileLayout(d, D.READ_GRAY) for d in good[:2] + [bad] + good[2:]]
    arrs, status, _ = AC.arith_host(lays)
    assert list(status) == [0, 0, 1, 0]


def test_plan_refuses_undecodable_layouts():
    lay = D.ArithFileLayout(CORPUS['pillow_prog_own_sof10'][0])
    with pytest.raises(RuntimeError, match='not arithmetic-decodable'):
        D.arith_plan([lay], [0, 0, 0])


# ---- refusals ----------------------------------------------------------------------------------
def _zero_run_past_63():
    return A.raw_scan(8, 8, [('dc', 0, 0), ('ac', 0, 0)] + [('ac', 3 * (k - 1) + 1, 0) for k in range(1, 64)])


def _dc_overflow():
    return A.raw_scan(8, 8, [('dc', 0, 1), ('dc', 1, 0), ('dc', 2, 1)] + [('dc', 20 + i, 1) for i in range(15)])


def _dc_category_15():
    # categories up to m = 2^14 (bins 20..33), then 14 magnitude bits on bin 48: the difference 32767
    return A.raw_scan(8, 8, [('dc', 0, 1), ('dc', 1, 0), ('dc', 2, 1)] + [('dc', 20 + i, 1) for i in range(14)]
                      + [('dc', 34, 0)] + [('dc', 48, 1)] * 13 + [('dc', 48, 0), ('ac', 0, 1)])


def _ac_overflow():
    return A.raw_scan(8, 8, [('dc', 0, 0), ('ac', 0, 0), ('ac', 1, 1), ('fixed', 0, 0), ('ac', 2, 1), ('ac', 2, 1)]
                      + [('ac', 189 + i, 1) for i in range(14)])


def _with(data, marker, body, before=b'\xff\xda'):
    i = data.find(before)
    return data[:i] + A._seg(marker, body) + data[i:]


BASE = A.transcode(E.pillow(32, 16, 75, '4:4:4'))


def _reader_error(data, flags=D.READ_GRAY):
    with pytest.raises(ValueError) as e:
        D.parse_jpeg(data, flags)
    return str(e.value)


def test_bad_arithmetic_codes():
    for data in (_zero_run_past_63(), _dc_overflow(), _ac_overflow()):
        assert _reader_error(data) == 'corrupt jpeg: bad arithmetic code'
        lay = D.ArithFileLayout(data, D.READ_GRAY)             # the layout pass does not decode
        assert lay.arith_decodable
        assert list(AC.arith_host([lay])[1]) == [1]
    p = D.parse_jpeg(_dc_category_15(), D.READ_GRAY)           # category 15 itself is fine
    assert p.planes[0].data[0] == (1 << 15) - 1 and not p.planes[0].data[1:].any()


def test_bad_refinement_past_se():
    # an AC refinement scan whose zero run passes Se
    first = [([0], 0, 0, 0, 0), ([0], 1, 63, 0, 1)]
    g = AC.pillow_gray(8, 8, 90)
    ok = A.transcode(g, first + [([0], 1, 63, 1, 0)])
    assert np.array_equal(AC.reader_planes(ok)[0], AC.reader_planes(g)[0])
    planes = [np.zeros((1, 1, 64), np.int16)]
    bad = A.write(8, 8, [A.dqt([np.ones(64, np.int64)])], [(1, 1, 1, 0)], planes, first)
    enc = A.QMEncoder()
    acst = bytearray(256)
    enc.encode(acst, 0, 0)                                     # not EOB at k = 1 (kex = 0)
    for k in range(1, 64):
        enc.encode(acst, 3 * (k - 1) + 1, 0)                  # nothing newly nonzero, up to past 63
    sos = A._seg(0xDA, bytes([1, 1, 0x00, 1, 63, 0x10]))
    bad = bad[:-2] + sos + enc.finish() + b'\xff\xd9'
    assert _reader_error(bad) == 'corrupt jpeg: bad arithmetic code'


def test_dac_refusals():
    assert _reader_error(_with(BASE, 0xCC, bytes([32, 5]))) == 'corrupt jpeg: bad DAC table index 32'
    assert _reader_error(_with(BASE, 0xCC, bytes([0, 0x12]))).startswith('corrupt jpeg: bad DAC value')
    assert _reader_error(_with(BASE, 0xCC, bytes([0, 0x11, 16]))) == 'corrupt jpeg: bad DAC length'
    for kx in (0, 1, 63, 64, 200, 255):                        # any Kx is accepted (libjpeg's get_dac)
        D.parse_jpeg(A.transcode(E.pillow(32, 16, 75, '4:4:4'), dac={16: kx, 17: kx}))
    D.parse_jpeg(_with(BASE, 0xCC, bytes([15, 0xFF, 31, 7])))    # tables 15: defined, unused


def test_sof11_and_others_refused_as_before():
    for m in (0xC3, 0xC5, 0xCB, 0xCD, 0xCF):
        data = BASE.replace(b'\xff\xc9', bytes([0xFF, m]), 1)
        assert _reader_error(data) == f'unsupported jpeg: SOF{m - 0xC0} (arithmetic, lossless or hierarchical coding)'


def test_table_selector_above_3_refused():
    i = BASE.find(b'\xff\xda')
    data = bytearray(BASE)
    data[i + 6] = 0x44                                        # the first component's Td/Ta
    assert _reader_error(bytes(data)) == 'corrupt jpeg: bad table selector'


def test_keep_settings_of_arith_file():
    import ctypes as C
    for name in ('pillow_420_q75', 'pillow_prog_own_sof10'):
        arith, twin = CORPUS[name]
        got, want = D.Keep(), D.Keep()
        lib = D.load_codecs()
        err = C.create_string_buffer(256)
        assert lib.j2p_jpeg_keep_settings(arith, len(arith), C.byref(got), err, 256) == 0, err.value
        assert lib.j2p_jpeg_keep_settings(twin, len(twin), C.byref(want), err, 256) == 0
        assert bytes(got) == bytes(want)


def test_fuzz_arith():
    r = subprocess.run([sys.executable, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'fuzz_arith.py'), '400', '5'],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]


def test_kernel_inventory():
    CK.check_kernel_inventory('arith/libj2parith.so', KERNELS)
