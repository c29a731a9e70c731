"""j2p_jpeg_exif_orientation (jpeg2png_b200/cli/jpeg_reader.c) on the host: the EXIF Orientation
of Pillow-made and hand-spliced files equals what Pillow reads, every malformed or missing tag reads
as 1, and truncated or mutated files never make it read outside the buffer.  The sweeps run in a
child process, with each file ending at a guard page, so a read past the end is a failed test."""
import ctypes as C
import io
import mmap
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from jpeg2png_b200 import decode, synth  # noqa: E402

SOI = b'\xff\xd8'


def _lib():
    subprocess.run(['make', '-C', os.path.join(ROOT, 'jpeg2png_b200', 'cli'), 'libj2pcodecs.so'], check=True, capture_output=True)
    return decode.load_codecs()


def orientation(data, n=None):
    return int(_lib().j2p_jpeg_exif_orientation(data, len(data) if n is None else n))


def pillow_orientation(data):
    return Image.open(io.BytesIO(data)).getexif().get(0x0112, 1)


def plain_jpeg(mode='RGB', progressive=False, w=40, h=24, exif=None):
    rgb = synth.cartoon_image(w, h, 3).astype(np.uint8)
    im = Image.fromarray(rgb, 'RGB').convert(mode)
    buf = io.BytesIO()
    kw = {} if exif is None else {'exif': exif}
    im.save(buf, 'JPEG', quality=80, progressive=progressive, **kw)
    return buf.getvalue()


def pillow_exif_jpeg(k, **kw):
    e = Image.Exif()
    e[0x0112] = k
    return plain_jpeg(exif=e.tobytes(), **kw)


def segment(marker, payload):
    return bytes([0xFF, marker]) + struct.pack('>H', len(payload) + 2) + payload


def tiff(entries, be=False, ifd=8, count=None):
    """A TIFF structure with IFD0 at `ifd`: entries are (tag, type, count, 4 value bytes already in
    the byte order, or an int written as the type's size)."""
    e = '>' if be else '<'
    out = (b'MM' if be else b'II') + struct.pack(e + 'HI', 42, ifd) + b'\0' * (ifd - 8)
    out += struct.pack(e + 'H', len(entries) if count is None else count)
    for tag, typ, cnt, val in entries:
        if isinstance(val, int):
            val = struct.pack(e + 'H', val) + b'\0\0' if typ == 3 else struct.pack(e + 'I', val)
        out += struct.pack(e + 'HHI', tag, typ, cnt) + val
    return out + struct.pack(e + 'I', 0)


def exif_app1(entries, **kw):
    return segment(0xE1, b'Exif\0\0' + tiff(entries, **kw))


def splice(jpeg, *segments):
    """The segments right after SOI."""
    assert jpeg[:2] == SOI
    return SOI + b''.join(segments) + jpeg[2:]


XMP = segment(0xE1, b'http://ns.adobe.com/xap/1.0/\0<x:xmpmeta xmlns:x="adobe:ns:meta/"/>')
APP0 = segment(0xE0, b'JFIF\0\x01\x01\0\0\x01\0\x01\0\0')
ICC = segment(0xE2, b'ICC_PROFILE\0\x01\x01' + bytes(64))
COM = segment(0xFE, b'a comment')
OTHER_TAGS = [(0x010F, 2, 4, b'Cam\0'), (0x0110, 2, 4, b'One\0')]


def _cases(k):
    base = plain_jpeg()
    yield 'pillow', pillow_exif_jpeg(k)
    yield 'pillow_progressive', pillow_exif_jpeg(k, progressive=True)
    yield 'pillow_gray', pillow_exif_jpeg(k, mode='L')
    for be in (False, True):
        end = 'mm' if be else 'ii'
        yield f'{end}_short', splice(base, exif_app1([(0x0112, 3, 1, k)], be=be))
        yield f'{end}_not_first', splice(base, exif_app1(OTHER_TAGS + [(0x0112, 3, 1, k), (0x0131, 2, 2, b'x\0\0\0')], be=be))
        yield f'{end}_long', splice(base, exif_app1([(0x0112, 4, 1, k)], be=be))
        yield f'{end}_far_ifd', splice(base, exif_app1([(0x0112, 3, 1, k)], be=be, ifd=40))
    yield 'xmp_first', splice(base, XMP, exif_app1([(0x0112, 3, 1, k)]))
    yield 'app0_icc_com', splice(base, APP0, COM, exif_app1([(0x0112, 3, 1, k)], be=True), ICC, COM)
    yield 'gray_progressive_spliced', splice(plain_jpeg('L', True), APP0, exif_app1([(0x0112, 3, 1, k)]))


@pytest.mark.parametrize('k', range(1, 9))
def test_orientation_equals_pillow(k):
    for name, data in _cases(k):
        assert pillow_orientation(data) == k, name
        assert orientation(data) == k, name


@pytest.mark.parametrize('name,data', [
    ('no_exif', plain_jpeg()),
    ('value_0', splice(plain_jpeg(), exif_app1([(0x0112, 3, 1, 0)]))),
    ('value_9', splice(plain_jpeg(), exif_app1([(0x0112, 3, 1, 9)]))),
    ('value_65535', splice(plain_jpeg(), exif_app1([(0x0112, 3, 1, 65535)], be=True))),
    ('long_high_bits', splice(plain_jpeg(), exif_app1([(0x0112, 4, 1, 0x10006)]))),
    ('type_byte', splice(plain_jpeg(), exif_app1([(0x0112, 1, 1, b'\x06\0\0\0')]))),
    ('type_sshort', splice(plain_jpeg(), exif_app1([(0x0112, 8, 1, 6)]))),
    ('count_2', splice(plain_jpeg(), exif_app1([(0x0112, 3, 2, 6)]))),
    ('count_0', splice(plain_jpeg(), exif_app1([(0x0112, 3, 0, 6)]))),
    ('ifd_past_segment', splice(plain_jpeg(), segment(0xE1, b'Exif\0\0' + tiff([(0x0112, 3, 1, 6)])[:4] + struct.pack('<I', 4000)
                                                      + tiff([(0x0112, 3, 1, 6)])[8:]))),
    ('ifd_at_end', splice(plain_jpeg(), segment(0xE1, b'Exif\0\0' + b'II*\0' + struct.pack('<I', 8)))),
    ('entries_past_segment', splice(plain_jpeg(), exif_app1([(0x0112, 3, 1, 6)], count=2))),
    ('bad_byte_order', splice(plain_jpeg(), segment(0xE1, b'Exif\0\0IM' + tiff([(0x0112, 3, 1, 6)])[2:]))),
    ('not_42', splice(plain_jpeg(), segment(0xE1, b'Exif\0\0II\x2b\0' + tiff([(0x0112, 3, 1, 6)])[4:]))),
    ('exif_without_nuls', splice(plain_jpeg(), segment(0xE1, b'Exif' + tiff([(0x0112, 3, 1, 6)])))),
    ('only_first_exif_counts', splice(plain_jpeg(), exif_app1([(0x010F, 2, 4, b'Cam\0')]), exif_app1([(0x0112, 3, 1, 6)]))),
    ('after_sos', plain_jpeg()[:-2] + exif_app1([(0x0112, 3, 1, 6)]) + b'\xff\xd9'),
    ('not_a_jpeg', b'\x89PNG' + exif_app1([(0x0112, 3, 1, 6)])),
    ('empty', b''),
])
def test_unusable_tags_read_as_one(name, data):
    assert orientation(data) == 1


def test_len_smaller_than_the_file():
    data = splice(plain_jpeg(), APP0, exif_app1([(0x0112, 3, 1, 6)]))
    start = len(SOI) + len(APP0)
    end = start + len(exif_app1([(0x0112, 3, 1, 6)]))
    assert orientation(data) == 6 and orientation(data, end) == 6
    for n in range(0, end):
        assert orientation(data, n) == 1, n


def test_the_sweeps_never_read_outside_the_buffer():
    r = subprocess.run([sys.executable, os.path.abspath(__file__), '3000', '7'], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
    assert 'sweep ok' in r.stdout, r.stdout


def test_decode_jpeg_refuses_a_non_bool_flag():
    with pytest.raises(ValueError, match='apply_exif_orientation'):
        decode.decode_jpeg(plain_jpeg(), apply_exif_orientation=1)


class _Guarded:
    """Files placed so that their last byte is the last byte before a PROT_NONE page."""

    def __init__(self, size=1 << 16):
        page = mmap.PAGESIZE
        self.size = (size + page - 1) // page * page
        self.m = mmap.mmap(-1, self.size + page)
        self.base = C.addressof(C.c_char.from_buffer(self.m))
        libc = C.CDLL(None, use_errno=True)
        libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
        if libc.mprotect(self.base + self.size, page, 0) != 0:
            raise OSError(C.get_errno(), 'mprotect')
        self.fn = _lib().j2p_jpeg_exif_orientation
        self.fn.argtypes = [C.c_void_p, C.c_size_t]

    def __call__(self, data):
        at = self.size - len(data)
        self.m[at:self.size] = data
        return int(self.fn(self.base + at, len(data)))


def main():
    n, seed = int(sys.argv[1]), int(sys.argv[2])
    rng = np.random.default_rng(seed)
    call = _Guarded()
    seeds = [splice(plain_jpeg(), XMP, exif_app1(OTHER_TAGS + [(0x0112, 3, 1, 6)], be=True)),
             pillow_exif_jpeg(8, progressive=True), splice(plain_jpeg('L'), APP0, exif_app1([(0x0112, 4, 1, 3)]))]
    for data in seeds:                                   # every truncation, the last byte at the guard page
        assert call(data) in (6, 8, 3)
        for cut in range(len(data)):
            assert 1 <= call(data[:cut]) <= 8
    for it in range(n):                                  # seeded mutations of the headers
        data = bytearray(seeds[it % len(seeds)])
        head = min(len(data), 400)
        for _ in range(int(rng.integers(1, 6))):
            kind = rng.integers(0, 4)
            at = int(rng.integers(0, head))
            if kind == 0:
                data[at] = int(rng.integers(0, 256))
            elif kind == 1:
                data[at] ^= 1 << int(rng.integers(0, 8))
            elif kind == 2:
                data[at:at + 2] = bytes(rng.choice([b'\xff\xe1', b'\x00\x00', b'\xff\xff', b'\xff\xda', b'MM', b'II']))
            else:
                del data[at:at + int(rng.integers(1, 16))]
        if rng.integers(0, 2):
            data = data[:int(rng.integers(0, len(data) + 1))]
        v = call(bytes(data))
        assert 1 <= v <= 8, v
    print('sweep ok')


if __name__ == '__main__':
    main()
