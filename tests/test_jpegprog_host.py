"""CPU tests of the progressive JPEG encoder (libj2pjpegprog.so, encode_jpeg(..., progressive=True))
through its serial host driver, which runs the kernels' steps: Pillow's `progressive=True` bytes on
the whole corpus, inputs crafted so that each run rule fires (with a Python restatement of the scans
that counts the events), partial-MCU sizes, independent streams in a mixed call, the files back
through the project's decoders with the default files' coefficients, the refusals, the work-area
bound and the library's kernel inventory."""
import ctypes as C

import numpy as np
import pytest

from jpeg2png_b200 import decode as D
from jpeg2png_b200 import jpeg_encode as J
from tests import codec_checks as CK
from tests import entropy_cases as EC
from tests import jpegenc_cases as JC
from tests import jpegprog_cases as PC
from tests import progressive_cases as P

_T = 'tests/test_gpu_jpegprog.py::test_device_equals_host_driver'
# kernel -> the GPU test that reaches it (every call of j2p_jpegprog_encode launches all ten)
KERNELS = {
    'k_jp_blocks': f'{_T} (colour, DCT, quantisation: the shared body; block summaries)',
    'k_jp_runs': f'{_T} (EOB-run state per AC block; long segments in test_flat_8k_equals_host_driver)',
    'k_jp_hist': f'{_T} (symbol counts per image and scan table)',
    'k_jp_tables': f'{_T} (ten tables per image, stream headers)',
    'k_jp_sizes': f'{_T} (bits per block and scan)',
    'k_jp_scan': f'{_T} (tile offsets, padding per stream)',
    'k_jp_emit': f'{_T} (codes, EOB runs and deferred correction bits)',
    'k_jp_ffcount': f'{_T} (0xFF per chunk)',
    'k_jp_offsets': f'{_T} (stream and file offsets)',
    'k_jp_stuff': f'{_T} (stream headers, stuffed data, EOI)',
}

CORPUS = JC.corpus()


def _first_difference(got, want):
    return next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))


def _check_pillow(got, x, q, s, what):
    want = PC.pillow_progressive(x, q, s)
    if got != want:
        pytest.fail(f'{what} q{q} {s}: {len(got)} bytes against Pillow\'s {len(want)}, first difference at byte '
                    f'{_first_difference(got, want)} ({JC.turbo_version()})')


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
@pytest.mark.parametrize('quality', JC.QUALITIES)
def test_host_driver_equals_pillow_progressive(quality, subsampling):
    for n in CORPUS:
        lay, a, x = CORPUS[n]
        _check_pillow(J.encode_host([a], quality, subsampling, lay, progressive=True)[0], x, quality, subsampling, n)


def test_optimize_changes_no_byte_of_a_progressive_file():
    x = next(CORPUS[n][2] for n in CORPUS if n.startswith('97x61_noise'))
    for q, s in ((90, '4:2:0'), (75, '4:4:4')):
        want = PC.pillow_progressive(x, q, s)
        assert PC.pillow_progressive(x, q, s, optimize=True) == want
        assert J.encode_host([x], q, s, 'HWC', optimize=True, progressive=True)[0] == want
        assert J.encode_host([x], q, s, 'HWC', optimize=False, progressive=True)[0] == want


@pytest.mark.parametrize('name', list(PC.crafted()))
def test_each_run_rule_fires_and_gives_pillows_bytes(name):
    x, q, s, events = PC.crafted()[name]
    _check_pillow(J.encode_host([x], q, s, 'HWC', progressive=True)[0], x, q, s, name)
    planes, err = EC.reader(J.encode_host([x], q, s, 'HWC')[0])
    assert planes is not None, err
    ev = PC.all_events(planes, x.shape[0], x.shape[1], s)
    for e in events:
        assert ev[e] > 0, (e, dict(ev))


def test_the_flat_image_has_more_than_0x7fff_blocks_in_one_component():
    x, _, s, _ = PC.crafted()['flat 1600x1600']
    (bw, bh), *_ = PC.grids(*x.shape[:2], s)[0]
    assert bw * bh > 0x7FFF
    assert max(h * w for h, w in JC.SIZES) // 64 < 0x7FFF        # the corpus alone never gets there


@pytest.mark.parametrize('h,w,subsampling', PC.partial_mcu())
def test_partial_mcu_sizes_give_pillows_bytes(h, w, subsampling):
    own, mcu = PC.grids(h, w, subsampling)
    assert own != mcu                                   # the AC scans skip the dummy blocks
    for kind in ('cartoon', 'noise'):
        x = JC.content(kind, h, w, h * w)
        for q in (50, 95):
            _check_pillow(J.encode_host([x], q, subsampling, 'HWC', progressive=True)[0], x, q, subsampling, f'{h}x{w} {kind}')


def test_a_mixed_call_equals_each_image_alone():
    names = [n for n in CORPUS if not n.startswith('1023x')]
    for q, s in ((75, '4:2:0'), (95, '4:4:4'), (10, '4:2:2')):
        hwc = [CORPUS[n][2] for n in names]
        alone = [J.encode_host([CORPUS[n][1]], q, s, CORPUS[n][0], progressive=True)[0] for n in names]
        assert J.encode_host(hwc, q, s, 'HWC', progressive=True) == alone


def _reader_takes(h, w, subsampling):
    """As tests/test_jpegenc_host.py: the sizes jpeg2png's reader takes."""
    hs, vs = {'4:4:4': (1, 1), '4:2:2': (2, 1), '4:2:0': (2, 2)}[subsampling]
    return -(-w // (8 * hs)) == (w // hs + 7) // 8 and -(-h // (8 * vs)) == (h // vs + 7) // 8


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
def test_progressive_files_hold_the_default_files_coefficients(subsampling):
    """j2p_read_jpeg_mem reads a progressive file to the default file's coefficients, the
    progressive layout pass takes it, and the progressive decoder's host driver gives them too."""
    names = [n for n in CORPUS if not n.startswith('1023x')]
    lays, wants, taken = [], [], 0
    for n in names:
        h, w = CORPUS[n][2].shape[:2]
        if not _reader_takes(h, w, subsampling):
            continue
        for q in (1, 75, 100):
            lay_, a = CORPUS[n][0], CORPUS[n][1]
            prog = J.encode_host([a], q, subsampling, lay_, progressive=True)[0]
            want, err = EC.reader(J.encode_host([a], q, subsampling, lay_)[0])
            assert want is not None, f'{n} q{q}: {err}'
            got, err = EC.reader(prog)
            assert got is not None, f'{n} q{q}: {err}'
            for c in range(3):
                assert (got[c] == want[c]).all(), f'{n} q{q} component {c}'
            taken += 1
            lay = D.ProgFileLayout(prog)
            assert lay.progressive_decodable
            lays.append(lay)
            wants.append(want)
    assert taken >= 60
    for lay, want in zip(lays, wants):
        arrs, status, _ = P.prog_host([lay], 1024)
        assert status[0] == 0
        for c in range(3):
            assert (arrs[0][c] == want[c]).all()


def test_work_area_bound():
    """Each stream gets its own bound; the worst, the AC first scan over 63 coefficients, is 1668
    bits (53 words) a block, and a 4:4:4 image's progressive work area exceeds the optimized one's
    by its eight AC streams' and two DC streams' words."""
    d = (J.Image * 1)()
    d[0].data, d[0].width, d[0].height, d[0].row_stride, d[0].col_stride, d[0].chan_stride = 1 << 20, 1024, 1024, 3072, 3, 1
    p = J.Params(75, 0)
    opt = J.codec(p, True).plan(d)[0]
    prog = J.codec(p, progressive=True).plan(d)[0]
    comp = 128 * 128
    # words per block: Y 5 + 49 + 35 + 35, Cb and Cr 53 + 35 each, the DC streams 1 per block each
    words = comp * (5 + 49 + 35 + 35 + 2 * (53 + 35)) + 2 * 3 * comp
    assert prog - opt >= (words - 3 * comp * 53) * 4 * 3      # entropy words and twice them of files
    assert prog - opt < (words - 3 * comp * 53) * 4 * 3 + 2 * comp * 3 * 4 * 4 + (1 << 20)


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
    lib = J.load_jpegprog()
    p = J.Params(*par)
    n = C.c_size_t()
    assert lib.j2p_jpegprog_plan(_descs(**bad), 1, C.byref(p), C.byref(n), None) == -1
    assert match in lib.j2p_jpegprog_last_error().decode()
    offs = (C.c_uint64 * 2)()
    assert lib.j2p_jpegprog_encode(_descs(**bad), 1, C.byref(p), 1 << 20, 1 << 30, None, offs, None, 0, None) == -1
    assert match in lib.j2p_jpegprog_last_error().decode()
    assert lib.j2p_jpegprog_encode_host(_descs(**bad), 1, C.byref(p), 1 << 20, 1 << 30, offs) == -1
    assert match in lib.j2p_jpegprog_last_error().decode()


def test_abi_refuses_null_pointers_and_non_device_memory():
    lib = J.load_jpegprog()
    p = J.Params(75, 2)
    n = C.c_size_t()
    assert lib.j2p_jpegprog_plan(None, 1, C.byref(p), C.byref(n), None) == -1
    assert lib.j2p_jpegprog_plan(_descs(), 1, None, C.byref(n), None) == -1
    assert 'null' in lib.j2p_jpegprog_last_error().decode()
    assert lib.j2p_jpegprog_plan(_descs(), 0, C.byref(p), C.byref(n), None) == -1
    x = np.zeros((4, 4, 3), np.uint8)
    d = _descs(data=x.ctypes.data)
    assert lib.j2p_jpegprog_plan(d, 1, C.byref(p), C.byref(n), None) == 0
    work = np.zeros(n.value, np.uint8)
    offs = (C.c_uint64 * 2)()
    assert lib.j2p_jpegprog_encode(d, 1, C.byref(p), None, n.value, None, offs, None, 0, None) == -1
    assert 'null' in lib.j2p_jpegprog_last_error().decode()
    assert lib.j2p_jpegprog_encode(d, 1, C.byref(p), work.ctypes.data, n.value, None, offs, None, 0, None) == -1
    err = lib.j2p_jpegprog_last_error().decode()
    assert 'device memory' in err or 'CUDA' in err or 'driver' in err
    assert lib.j2p_jpegprog_encode_host(d, 1, C.byref(p), work.ctypes.data, n.value - 1, offs) == -1
    assert 'smaller' in lib.j2p_jpegprog_last_error().decode()
    assert lib.j2p_jpegprog_encode_host(d, 1, C.byref(p), work.ctypes.data, n.value, offs) == 0


@pytest.mark.parametrize('bad', [1, 0, None, 'yes', np.bool_(True), 1.0])
def test_progressive_must_be_a_bool(bad):
    import torch
    from jpeg2png_b200 import encode_jpeg
    x = np.zeros((8, 8, 3), np.uint8)
    with pytest.raises(ValueError, match='progressive'):
        J.encode_host([x], progressive=bad)
    with pytest.raises(ValueError, match='progressive'):
        encode_jpeg(torch.zeros(3, 8, 8, dtype=torch.uint8), progressive=bad)


def test_kernel_inventory_is_covered_and_does_not_spill():
    CK.check_kernel_inventory('jpegprog/libj2pjpegprog.so', KERNELS)
