"""CPU tests of the optimizing JPEG encoder (libj2pjpegopt.so, encode_jpeg(..., optimize=True))
through its serial host driver, which runs the kernels' steps: Pillow's `optimize=True` bytes on
the whole corpus, the table builder against a Python restatement of T.81 K.2 / K.3 on crafted
counts, independent per-image tables in a mixed call, the files back through the project's
decoders with the default files' coefficients, the refusals, and the library's kernel inventory."""
import ctypes as C

import numpy as np
import pytest

from jpeg2png_b200 import decode as D
from jpeg2png_b200 import jpeg_encode as J
from tests import codec_checks as CK
from tests import entropy_cases as EC
from tests import jpegenc_cases as JC
from tests import jpegopt_cases as OC

# kernel -> the GPU test that reaches it (every call of j2p_jpegopt_encode launches all nine)
KERNELS = {
    'k_jo_blocks': 'tests/test_gpu_jpegopt.py::test_device_equals_host_driver (colour, DCT, quantisation: the shared body)',
    'k_jo_hist': 'tests/test_gpu_jpegopt.py::test_device_equals_host_driver (symbol counts per image and table)',
    'k_jo_tables': 'tests/test_gpu_jpegopt.py::test_device_equals_host_driver (code lengths, codes, DHT headers)',
    'k_jo_sizes': 'tests/test_gpu_jpegopt.py::test_device_equals_host_driver (bits per block with the image\'s tables)',
    'k_jo_scan': 'tests/test_gpu_jpegopt.py::test_device_equals_host_driver (tile offsets, padding)',
    'k_jo_emit': 'tests/test_gpu_jpegopt.py::test_device_equals_host_driver (the image\'s codes into the bit stream)',
    'k_jo_ffcount': 'tests/test_gpu_jpegopt.py::test_device_equals_host_driver (0xFF per chunk)',
    'k_jo_offsets': 'tests/test_gpu_jpegopt.py::test_device_equals_host_driver (per-image header lengths, file offsets)',
    'k_jo_stuff': 'tests/test_gpu_jpegopt.py::test_device_equals_host_driver (per-image headers, stuffed data, EOI)',
}

CORPUS = JC.corpus()


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
@pytest.mark.parametrize('quality', JC.QUALITIES)
def test_host_driver_equals_pillow_optimize(quality, subsampling):
    for n in CORPUS:
        lay, a, x = CORPUS[n]
        got = J.encode_host([a], quality, subsampling, lay, optimize=True)[0]
        want = OC.pillow_optimized(x, quality, subsampling)
        if got != want:
            k = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
            pytest.fail(f'{n} q{quality} {subsampling}: {len(got)} bytes against Pillow\'s {len(want)}, first difference at '
                        f'byte {k} ({JC.turbo_version()})')


@pytest.mark.parametrize('name', list(OC.crafted()))
def test_table_builder_equals_restatement(name):
    counts = OC.crafted()[name]
    bits, vals = J.build_table(counts)
    want_bits, want_vals, longest = OC.restated_table(counts)
    assert (bits, vals) == (want_bits, want_vals)
    assert sorted(vals) == [k for k in range(256) if counts[k]]
    assert sum(bits) == len(vals)
    if name in OC.LONG:
        assert longest > 16                             # the K.3 limit did the work


def test_table_builder_refuses_no_symbols():
    with pytest.raises(ValueError, match='at least one symbol'):
        J.build_table([0] * 256)


def test_a_mixed_call_equals_each_image_alone():
    names = [n for n in CORPUS if not n.startswith('1023x')]
    for q, s in ((75, '4:2:0'), (95, '4:4:4'), (10, '4:2:2')):
        hwc = [CORPUS[n][2] for n in names]
        alone = [J.encode_host([CORPUS[n][1]], q, s, CORPUS[n][0], optimize=True)[0] for n in names]
        assert J.encode_host(hwc, q, s, 'HWC', optimize=True) == alone


def _reader_takes(h, w, subsampling):
    """As tests/test_jpegenc_host.py: the sizes jpeg2png's reader takes."""
    hs, vs = {'4:4:4': (1, 1), '4:2:2': (2, 1), '4:2:0': (2, 2)}[subsampling]
    return -(-w // (8 * hs)) == (w // hs + 7) // 8 and -(-h // (8 * vs)) == (h // vs + 7) // 8


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
def test_optimized_files_hold_the_default_files_coefficients(subsampling):
    """j2p_read_jpeg_mem reads an optimized file to the default file's coefficients, the layout pass
    routes it to the device decoder, and the device decoder's host driver gives them too."""
    names = [n for n in CORPUS if not n.startswith('1023x')]
    lays, wants, taken = [], [], 0
    for n in names:
        h, w = CORPUS[n][2].shape[:2]
        if not _reader_takes(h, w, subsampling):
            continue
        for q in (1, 75, 100):
            lay_, a = CORPUS[n][0], CORPUS[n][1]
            opt = J.encode_host([a], q, subsampling, lay_, optimize=True)[0]
            want, err = EC.reader(J.encode_host([a], q, subsampling, lay_)[0])
            assert want is not None, f'{n} q{q}: {err}'
            got, err = EC.reader(opt)
            assert got is not None, f'{n} q{q}: {err}'
            for c in range(3):
                assert (got[c] == want[c]).all(), f'{n} q{q} component {c}'
            taken += 1
            lay = D.FileLayout(opt)
            assert lay.device_decodable
            lays.append(lay)
            wants.append(want)
    assert taken >= 60
    arrs, status, _ = EC.entropy_host(lays, 1024)
    assert (status == 0).all()
    for got, want in zip(arrs, wants):
        for c in range(3):
            assert (got[c] == want[c]).all()


def test_work_area_bound_is_its_own():
    """A block's worst case is 1665 bits with optimized tables, 53 words; the default plan keeps 52."""
    d = (J.Image * 1)()
    d[0].data, d[0].width, d[0].height, d[0].row_stride, d[0].col_stride, d[0].chan_stride = 1 << 20, 1024, 1024, 3072, 3, 1
    p = J.Params(75, 0)
    base = J.codec(p).plan(d)[0]
    opt = J.codec(p, True).plan(d)[0]
    blocks = 128 * 128 * 3
    assert opt - base >= blocks * 4 * 3                 # one more word per block, and twice that of files
    assert opt - base < blocks * 4 * 3 + 64 * 1024


def _descs(**kw):
    d = J.Image()
    d.data, d.width, d.height, d.row_stride, d.col_stride, d.chan_stride = 1 << 20, 4, 4, 12, 3, 1
    for k, v in kw.items():
        setattr(d, k, v)
    return (J.Image * 1)(d)


@pytest.mark.parametrize('bad,par,match', [
    (dict(data=None), (75, 2), 'null data'), (dict(width=0), (75, 2), 'width and height'),
    (dict(height=65536), (75, 2), 'width and height'), ({}, (0, 2), 'quality'), ({}, (101, 2), 'quality'),
    ({}, (75, 3), 'unknown sampling')])
def test_abi_refusals(bad, par, match):
    lib = J.load_jpegopt()
    p = J.Params(*par)
    n = C.c_size_t()
    assert lib.j2p_jpegopt_plan(_descs(**bad), 1, C.byref(p), C.byref(n), None) == -1
    assert match in lib.j2p_jpegopt_last_error().decode()
    offs = (C.c_uint64 * 2)()
    assert lib.j2p_jpegopt_encode(_descs(**bad), 1, C.byref(p), 1 << 20, 1 << 30, None, offs, None, 0, None) == -1
    assert match in lib.j2p_jpegopt_last_error().decode()
    assert lib.j2p_jpegopt_encode_host(_descs(**bad), 1, C.byref(p), 1 << 20, 1 << 30, offs) == -1
    assert match in lib.j2p_jpegopt_last_error().decode()


def test_abi_refuses_null_pointers_and_non_device_memory():
    lib = J.load_jpegopt()
    p = J.Params(75, 2)
    n = C.c_size_t()
    assert lib.j2p_jpegopt_plan(None, 1, C.byref(p), C.byref(n), None) == -1
    assert lib.j2p_jpegopt_plan(_descs(), 1, None, C.byref(n), None) == -1
    assert 'null' in lib.j2p_jpegopt_last_error().decode()
    assert lib.j2p_jpegopt_plan(_descs(), 0, C.byref(p), C.byref(n), None) == -1
    x = np.zeros((4, 4, 3), np.uint8)
    d = _descs(data=x.ctypes.data)
    assert lib.j2p_jpegopt_plan(d, 1, C.byref(p), C.byref(n), None) == 0
    work = np.zeros(n.value, np.uint8)
    offs = (C.c_uint64 * 2)()
    assert lib.j2p_jpegopt_encode(d, 1, C.byref(p), None, n.value, None, offs, None, 0, None) == -1
    assert 'null' in lib.j2p_jpegopt_last_error().decode()
    assert lib.j2p_jpegopt_encode(d, 1, C.byref(p), work.ctypes.data, n.value, None, offs, None, 0, None) == -1
    err = lib.j2p_jpegopt_last_error().decode()
    assert 'device memory' in err or 'CUDA' in err or 'driver' in err
    assert lib.j2p_jpegopt_encode_host(d, 1, C.byref(p), work.ctypes.data, n.value - 1, offs) == -1
    assert 'smaller' in lib.j2p_jpegopt_last_error().decode()
    assert lib.j2p_jpegopt_encode_host(d, 1, C.byref(p), work.ctypes.data, n.value, offs) == 0
    assert lib.j2p_jpegopt_build_table(None, None, None, None) == -1
    assert 'null' in lib.j2p_jpegopt_last_error().decode()


@pytest.mark.parametrize('bad', [1, 0, None, 'yes', np.bool_(True), 1.0])
def test_optimize_must_be_a_bool(bad):
    import torch
    from jpeg2png_b200 import encode_jpeg
    x = np.zeros((8, 8, 3), np.uint8)
    with pytest.raises(ValueError, match='optimize'):
        J.encode_host([x], optimize=bad)
    with pytest.raises(ValueError, match='optimize'):
        encode_jpeg(torch.zeros(3, 8, 8, dtype=torch.uint8), optimize=bad)


def test_kernel_inventory_is_covered_and_does_not_spill():
    CK.check_kernel_inventory('jpegopt/libj2pjpegopt.so', KERNELS)
