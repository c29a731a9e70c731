"""CPU tests of the JPEG encoder through its serial host driver (j2p_jpegenc_encode_host, the same
steps as the kernels of libj2pjpegenc.so): Pillow's bytes for every size, content, quality and
sampling of the corpus, the files back through the project's decoders, the refusals, and the
library's kernel inventory."""
import ctypes as C

import numpy as np
import pytest

from jpeg2png_b200 import decode as D
from jpeg2png_b200 import jpeg_encode as J
from tests import codec_checks as CK
from tests import entropy_cases as EC
from tests import jpegenc_cases as JC

# kernel -> the GPU test that reaches it (every call of j2p_jpegenc_encode launches all seven)
KERNELS = {
    'k_je_blocks': 'tests/test_gpu_jpegenc.py::test_device_equals_host_driver (colour, downsampling, edges, dummies, FDCT, quantisation)',
    'k_je_sizes': 'tests/test_gpu_jpegenc.py::test_device_equals_host_driver (bits per block, DC prediction)',
    'k_je_scan': 'tests/test_gpu_jpegenc.py::test_device_equals_host_driver (tile offsets, padding)',
    'k_je_emit': 'tests/test_gpu_jpegenc.py::test_device_equals_host_driver (Huffman codes into the bit stream)',
    'k_je_ffcount': 'tests/test_gpu_jpegenc.py::test_device_equals_host_driver (0xFF per chunk)',
    'k_je_offsets': 'tests/test_gpu_jpegenc.py::test_device_equals_host_driver (file lengths and offsets)',
    'k_je_stuff': 'tests/test_gpu_jpegenc.py::test_device_equals_host_driver (headers, stuffed data, EOI)',
}

CORPUS = JC.corpus()


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
@pytest.mark.parametrize('quality', JC.QUALITIES)
def test_host_driver_equals_pillow(quality, subsampling):
    for n in CORPUS:
        lay, a, x = CORPUS[n]
        got = J.encode_host([a], quality, subsampling, lay)[0]
        want = JC.pillow(x, quality, subsampling)
        if got != want:
            k = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
            pytest.fail(f'{n} q{quality} {subsampling}: {len(got)} bytes against Pillow\'s {len(want)}, first difference at '
                        f'byte {k} ({JC.turbo_version()})')


def test_pillow_default_is_q75_420():
    import io
    from PIL import Image
    x = JC.content('cartoon', 31, 33, 5)
    buf = io.BytesIO()
    Image.fromarray(x, 'RGB').save(buf, 'JPEG')
    assert J.encode_host([x])[0] == buf.getvalue(), JC.turbo_version()


def test_many_images_in_one_call_equal_each_alone():
    names = [n for n in CORPUS if not n.startswith('1023x')]
    for q, s in ((75, '4:2:0'), (95, '4:4:4'), (10, '4:2:2')):
        hwc = [CORPUS[n][2] for n in names]
        alone = [J.encode_host([CORPUS[n][1]], q, s, CORPUS[n][0])[0] for n in names]
        assert J.encode_host(hwc, q, s, 'HWC') == alone


def _reader_takes(h, w, subsampling):
    """jpeg2png's reader wants each chroma plane's block count to be (size // factor + 7) // 8,
    which libjpeg's ceil(size / factor / 8) misses for some odd sizes: it refuses those files
    whoever wrote them (Pillow's too, which are the same bytes)."""
    hs, vs = {'4:4:4': (1, 1), '4:2:2': (2, 1), '4:2:0': (2, 2)}[subsampling]
    return -(-w // (8 * hs)) == (w // hs + 7) // 8 and -(-h // (8 * vs)) == (h // vs + 7) // 8


@pytest.mark.parametrize('subsampling', JC.SAMPLINGS)
def test_files_go_back_through_the_decoders(subsampling):
    """j2p_read_jpeg_mem reads every file of a size it takes, the layout pass routes it to the
    device decoder, and the device decoder's host driver gives the reader's coefficients."""
    names = [n for n in CORPUS if not n.startswith('1023x')]
    lays, wants, taken = [], [], 0
    for n in names:
        h, w = CORPUS[n][2].shape[:2]
        for q in (1, 75, 100):
            data = J.encode_host([CORPUS[n][1]], q, subsampling, CORPUS[n][0])[0]
            want, err = EC.reader(data)
            if not _reader_takes(h, w, subsampling):
                assert want is None and 'invalid coef' in err, n
                continue
            assert want is not None, f'{n} q{q}: {err}'
            taken += 1
            lay = D.FileLayout(data)
            assert lay.device_decodable
            lays.append(lay)
            wants.append(want)
    assert taken >= 60
    arrs, status, _ = EC.entropy_host(lays, 1024)
    assert (status == 0).all()
    for got, want in zip(arrs, wants):
        for c in range(3):
            assert (got[c] == want[c]).all()


def _descs(**kw):
    d = J.Image()
    d.data, d.width, d.height, d.row_stride, d.col_stride, d.chan_stride = 1 << 20, 4, 4, 12, 3, 1
    for k, v in kw.items():
        setattr(d, k, v)
    return (J.Image * 1)(d)


@pytest.mark.parametrize('bad,par,match', [
    (dict(data=None), (75, 2), 'null data'), (dict(width=0), (75, 2), 'width and height'),
    (dict(height=0), (75, 2), 'width and height'), (dict(width=65536), (75, 2), 'width and height'),
    (dict(height=65536), (75, 2), 'width and height'), ({}, (0, 2), 'quality'), ({}, (101, 2), 'quality'),
    ({}, (75, 3), 'unknown sampling'), ({}, (75, -1), 'unknown sampling')])
def test_abi_refusals(bad, par, match):
    lib = J.load_jpegenc()
    p = J.Params(*par)
    n = C.c_size_t()
    assert lib.j2p_jpegenc_plan(_descs(**bad), 1, C.byref(p), C.byref(n), None) == -1
    assert match in lib.j2p_jpegenc_last_error().decode()
    offs = (C.c_uint64 * 2)()
    assert lib.j2p_jpegenc_encode(_descs(**bad), 1, C.byref(p), 1 << 20, 1 << 30, None, offs, None, 0, None) == -1
    assert match in lib.j2p_jpegenc_last_error().decode()
    assert lib.j2p_jpegenc_encode_host(_descs(**bad), 1, C.byref(p), 1 << 20, 1 << 30, offs) == -1
    assert match in lib.j2p_jpegenc_last_error().decode()


def test_abi_refuses_null_pointers_and_non_device_memory():
    lib = J.load_jpegenc()
    p = J.Params(75, 2)
    n = C.c_size_t()
    assert lib.j2p_jpegenc_plan(None, 1, C.byref(p), C.byref(n), None) == -1
    assert lib.j2p_jpegenc_plan(_descs(), 1, None, C.byref(n), None) == -1
    assert 'null' in lib.j2p_jpegenc_last_error().decode()
    assert lib.j2p_jpegenc_plan(_descs(), 0, C.byref(p), C.byref(n), None) == -1
    x = np.zeros((4, 4, 3), np.uint8)
    d = _descs(data=x.ctypes.data)
    assert lib.j2p_jpegenc_plan(d, 1, C.byref(p), C.byref(n), None) == 0
    work = np.zeros(n.value, np.uint8)
    offs = (C.c_uint64 * 2)()
    assert lib.j2p_jpegenc_encode(d, 1, C.byref(p), None, n.value, None, offs, None, 0, None) == -1
    assert 'null' in lib.j2p_jpegenc_last_error().decode()
    assert lib.j2p_jpegenc_encode(d, 1, C.byref(p), work.ctypes.data, n.value, None, None, None, 0, None) == -1
    assert lib.j2p_jpegenc_encode(d, 1, C.byref(p), work.ctypes.data, n.value, None, offs, None, 0, None) == -1
    err = lib.j2p_jpegenc_last_error().decode()
    assert 'device memory' in err or 'CUDA' in err or 'driver' in err
    assert lib.j2p_jpegenc_encode_host(d, 1, C.byref(p), work.ctypes.data, n.value - 1, offs) == -1
    assert 'smaller' in lib.j2p_jpegenc_last_error().decode()
    assert lib.j2p_jpegenc_encode_host(d, 1, C.byref(p), work.ctypes.data, n.value, offs) == 0


def test_encode_host_refusals():
    x = np.zeros((8, 8, 3), np.uint8)
    with pytest.raises(ValueError, match='quality'):
        J.encode_host([x], 0)
    with pytest.raises(ValueError, match='quality'):
        J.encode_host([x], 75.0)
    with pytest.raises(ValueError, match='subsampling'):
        J.encode_host([x], 75, '4:1:1')
    with pytest.raises(ValueError, match='uint8'):
        J.encode_host([x.astype(np.uint16)])
    with pytest.raises(ValueError, match='1..65535'):
        J.encode_host([np.lib.stride_tricks.as_strided(x, shape=(65536, 1, 3), strides=(0, 0, 1))])


def test_encode_jpeg_argument_errors():
    import torch
    from jpeg2png_b200 import encode_jpeg
    t = torch.zeros(3, 4, 4, dtype=torch.uint8)
    with pytest.raises(ValueError, match='layout'):
        encode_jpeg(t, layout='NCHW')
    with pytest.raises(ValueError, match='torch.uint8'):
        encode_jpeg(torch.zeros(3, 4, 4, dtype=torch.uint16))
    with pytest.raises(ValueError, match='CHW'):
        encode_jpeg(torch.zeros(4, 4, 3, dtype=torch.uint8))
    with pytest.raises(ValueError, match='HWC'):
        encode_jpeg(t, layout='HWC')
    with pytest.raises(ValueError, match='3-dimensional'):
        encode_jpeg([torch.zeros(4, 4, dtype=torch.uint8)])
    for q in (0, 101, 7.5, True, '75'):
        with pytest.raises(ValueError, match='quality'):
            encode_jpeg(t, quality=q)
    with pytest.raises(ValueError, match='subsampling'):
        encode_jpeg(t, subsampling='4:4:0')
    with pytest.raises(ValueError, match='1..65535'):
        encode_jpeg(torch.zeros(3, 0, 4, dtype=torch.uint8))
    with pytest.raises(ValueError, match='1..65535'):
        encode_jpeg(torch.zeros(3, 1, 1, dtype=torch.uint8).expand(3, 65536, 1))
    with pytest.raises(ValueError, match='CUDA tensors'):
        encode_jpeg([t])
    with pytest.raises(ValueError, match='torch tensors'):
        encode_jpeg(np.zeros((3, 4, 4), np.uint8))


def test_encode_jpeg_without_a_device_raises_runtime_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip('a CUDA device is present')
    from jpeg2png_b200 import encode_jpeg
    with pytest.raises(RuntimeError, match='needs a CUDA device'):
        encode_jpeg([])


def test_kernel_inventory_is_covered_and_does_not_spill():
    CK.check_kernel_inventory('jpegenc/libj2pjpegenc.so', KERNELS)
