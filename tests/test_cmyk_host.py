"""CPU tests of four-component (Adobe CMYK and YCCK) JPEGs: the reader's J2P_READ_CMYK path against
the coefficients the fixtures were written from and against Pillow's decode, the APP14 rule, the
numpy restatement of the export's samples and RGB conversion against Pillow, the layout passes'
answer for four-component files, the refusals of the old flags, decode_jpeg's keys and footprints for
four planes, and mutated files."""
import ctypes as C
import io
import os
import subprocess
import sys

import numpy as np
import pytest
from PIL import Image

from jpeg2png_b200 import decode as D
from jpeg2png_b200 import synth
from tests import cmyk_synth as S
from tests import helpers as H

CORPUS = S.corpus()
SAMPLINGS = {'444': [(1, 1)] * 4, '2211': [(2, 2), (1, 1), (1, 1), (2, 2)], '1221': [(1, 1), (2, 2), (2, 1), (1, 2)]}


@pytest.mark.parametrize('name', list(CORPUS))
def test_fixtures_open_as_cmyk_in_pillow(name):
    assert S.pillow_opens_as_cmyk(CORPUS[name][0])


def entropy_host(lay, subseq_bits=64):
    """libj2pentropy.so's serial host driver on one FileLayout4 (j2p_entropy_pack4): its four planes."""
    planes = [np.full(q.w * q.h, 0x5a5a, np.int16) for q in lay.planes]
    plan, addr, _, work_bytes = D.entropy_plan4([lay], [a.ctypes.data for a in planes], subseq_bits)
    work = np.zeros(work_bytes + 16, np.uint8)
    status = np.zeros(1, np.uint32)
    assert D.load_entropy().j2p_entropy_decode_host(addr, (work.ctypes.data + 15) & ~15, status.ctypes.data,
                                                   C.byref(D.EntropyStats())) == 0
    assert status[0] == 0
    del plan
    return planes


@pytest.mark.parametrize('interleaved', [True, False], ids=['interleaved', 'components'])
@pytest.mark.parametrize('restart', [0, 1, 3])
@pytest.mark.parametrize('transform', [None, 0, 1, 2])
@pytest.mark.parametrize('sampling', list(SAMPLINGS))
def test_reader_coefficients_equal_written(sampling, transform, restart, interleaved):
    data, planes = S.ycck_file(45, 35, SAMPLINGS[sampling], 3, restart, transform, interleaved)
    assert S.pillow_opens_as_cmyk(data)
    p = D.parse_jpeg4(data)
    assert (p.w, p.h, len(p.planes)) == (45, 35, 4)
    assert p.colour == (D.CMYK if transform in (None, 0) else D.YCCK)
    maxh = max(h for h, _ in SAMPLINGS[sampling])
    maxv = max(v for _, v in SAMPLINGS[sampling])
    for pl, want, (h, v) in zip(p.planes, planes, SAMPLINGS[sampling]):
        assert (pl.w_samp, pl.h_samp) == (maxh // h, maxv // v)
        assert (pl.data == want).all()
    # the four-plane layout pass and the entropy library's host driver give the same coefficients
    lay = D.FileLayout4(data)
    assert lay.device_decodable and lay.colour == p.colour and lay.lay.nscan == (1 if interleaved else 4)
    for bits in (32, 1024):
        assert all((a == b).all() for a, b in zip(entropy_host(lay, bits), planes))
    # the arithmetic twin decodes to the same coefficients
    q = D.parse_jpeg4(S.arith_twin(data, restart))
    assert q.colour == p.colour
    assert all((a.data == b.data).all() and (a.quant == b.quant).all() for a, b in zip(p.planes, q.planes))


def test_pillow_twins_share_coefficients():
    """APP14 removal, the arithmetic twin: the same coefficients as the file they came from."""
    for base, twins in (('pillow_q75_97x61', ('no_app14_q75_97x61', 'arith_cmyk')),
                        ('pillow_progressive_q50_97x61', ('no_app14_progressive',)),
                        ('ycck_2211_restart2', ('arith_ycck_2211',))):
        a = D.parse_jpeg4(CORPUS[base][0])
        for t in twins:
            b = D.parse_jpeg4(CORPUS[t][0])
            assert all((x.data == y.data).all() for x, y in zip(a.planes, b.planes)), t


def test_app14_rule():
    data = CORPUS['pillow_q75_97x61'][0]
    short = S.app14(0, b'Adobe' + bytes([0, 100, 0, 0, 0, 0]))             # 11 data bytes: not an Adobe segment
    other = S.app14(0, b'Adobf' + bytes([0, 100, 0, 0, 0, 0, 2]))
    cases = {
        (): D.CMYK,
        (S.app14(0),): D.CMYK,
        (S.app14(1),): D.YCCK,
        (S.app14(2),): D.YCCK,
        (S.app14(7),): D.YCCK,
        (S.app14(2), S.app14(0)): D.CMYK,                                     # the last one counts
        (S.app14(0), S.app14(2)): D.YCCK,
        (S.app14(2), short): D.YCCK,
        (short,): D.CMYK,
        (other,): D.CMYK,
        (S.app14(2, b'Adobe' + bytes([0, 100, 0, 0, 0, 0, 2, 9, 9])),): D.YCCK,   # longer is fine
    }
    want = D.parse_jpeg4(data)
    for segs, kind in cases.items():
        p = D.parse_jpeg4(S.with_app14(data, *segs))
        assert p.colour == kind, segs
        assert all((a.data == b.data).all() for a, b in zip(p.planes, want.planes))
    # an APP14 after the first SOS does not count
    late = bytearray(S.strip_app14(data))
    sos = next(a for m, a, _ in S.segments(bytes(late)) if m == 0xDA)
    eoi = len(late) - 2
    late[eoi:eoi] = S.app14(2)
    assert sos < eoi and D.parse_jpeg4(bytes(late)).colour == D.CMYK


@pytest.mark.parametrize('name', [n for n in CORPUS if n.startswith(('pillow', 'no_app14', 'arith_cmyk'))])   # Pillow's files
def test_conventional_decode_within_one_of_pillow(name):
    data = CORPUS[name][0]
    p = D.parse_jpeg4(data)
    img = synth.CoefImage(width=p.w, height=p.h, planes=[synth.Plane(w=x.w, h=x.h, w_samp=x.w_samp, h_samp=x.h_samp,
                                                                     data=x.data, quant=x.quant) for x in p.planes])
    ours = H.decode_planes(img, [0, 1, 2, 3])
    im = Image.open(io.BytesIO(data))
    assert im.mode == 'CMYK'
    theirs = np.asarray(im).astype(np.float64)
    for c in range(4):
        x = 255.0 - np.clip(np.rint(ours[c][:p.h, :p.w] + 128.0), 0, 255)
        assert np.abs(x - theirs[..., c]).max() <= 1.0, c


def test_rgb_restatement_equals_pillow():
    rng = np.random.default_rng(4)
    x = rng.integers(0, 256, (64, 96, 4), dtype=np.uint8)
    x[0, :, :] = [[a, b, 0, 0] for a, b in zip(np.arange(96) * 2 % 256, np.arange(96) * 5 % 256)]
    x[1, :, 3] = 255
    want = np.asarray(Image.fromarray(x, 'CMYK').convert('RGB'))
    assert (S.pillow_rgb(x) == want).all()
    # every (x, K) pair
    xs, ks = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8))
    full = np.dstack([xs, xs, xs, ks])
    assert (S.pillow_rgb(full) == np.asarray(Image.fromarray(full, 'CMYK').convert('RGB'))).all()


def test_inversion_restatement():
    assert (S.invert(np.array([0, 1, 255], np.uint8)) == [255, 254, 0]).all()
    assert (S.invert(np.array([0, 256, 65280], np.uint16)) == [65535, 65279, 255]).all()
    f = np.array([0.0, 0.1, 254.75, 255.0], np.float32)
    assert (S.invert(f) == np.float32(255.0) - f).all() and S.invert(f).dtype == np.float32


@pytest.mark.parametrize('name', list(CORPUS))
def test_layout_passes(name):
    """Sequential Huffman four-component files go to the device decoder (j2p_read_jpeg_layout4);
    progressive and arithmetic ones to the host reader.  The three-plane passes take none of them."""
    data = CORPUS[name][0]
    sequential = not (name.startswith('arith') or 'progressive' in name)
    lay = D.FileLayout4(data)
    assert lay.device_decodable == sequential
    front = D._front_end_four(data, True)
    assert isinstance(front, D.FileLayout4 if sequential and D.four_on_device(lay) else D.Parsed) and len(front.planes) == 4
    assert front.colour == CORPUS[name][1]
    if sequential:
        assert all((a == b.data).all() for a, b in zip(entropy_host(lay), D.parse_jpeg4(data).planes))
    flags = D.READ_GRAY | D.READ_CMYK
    assert not D.FileLayout(data, flags).device_decodable
    assert not D.ProgFileLayout(data, flags).progressive_decodable
    assert not D.ArithFileLayout(data, flags).arith_decodable
    # three-component and gray files are unchanged by the flag
    for other in (S.strip_app14(_colour()), _gray()):
        a, b = D.FileLayout(other, D.READ_GRAY), D.FileLayout(other, flags)
        assert a.device_decodable and b.device_decodable and a.lay.ncomp == b.lay.ncomp
        assert bytes(a.lay.data[:a.lay.data_len]) == bytes(b.lay.data[:b.lay.data_len])


def _colour():
    buf = io.BytesIO()
    Image.fromarray(synth.cartoon_image(40, 24, 1).astype(np.uint8), 'RGB').save(buf, 'JPEG', quality=70)
    return buf.getvalue()


def _gray():
    buf = io.BytesIO()
    Image.fromarray(synth.cartoon_image(40, 24, 1).astype(np.uint8)[..., 0], 'L').save(buf, 'JPEG', quality=70)
    return buf.getvalue()


def test_old_flags_refuse_with_todays_messages():
    data = CORPUS['pillow_q75_97x61'][0]
    for fn, name in ((D.parse_jpeg, 'pillow_q75_97x61'), (D.parse_jpeg, 'pillow_progressive_q50_97x61'), (D.parse_jpeg, 'arith_cmyk'),
                     (D.FileLayout, 'pillow_q75_97x61'), (D.ProgFileLayout, 'pillow_progressive_q50_97x61'),
                     (D.ArithFileLayout, 'arith_cmyk')):
        with pytest.raises(ValueError, match='^only 3 component jpegs are supported$'):
            fn(CORPUS[name][0])
        with pytest.raises(ValueError, match='^only 1 and 3 component jpegs are supported$'):
            fn(CORPUS[name][0], D.READ_GRAY)
    # struct j2p_jpeg has three planes: j2p_read_jpeg_mem_ex ignores J2P_READ_CMYK
    with pytest.raises(ValueError, match='^only 3 component jpegs are supported$'):
        D.parse_jpeg(data, D.READ_CMYK)
    # the new flag's message for other counts
    two = bytearray(_gray())
    sof = next(a for m, a, _ in S.segments(bytes(two)) if m == 0xC0)
    two[sof + 9] = 2
    with pytest.raises(ValueError, match='^only 1, 3 and 4 component jpegs are supported$'):
        D.parse_jpeg4(bytes(two))
    # one- and three-component files read alike through the new entry point
    for other in (_colour(), _gray()):
        a, b = D.parse_jpeg(other, D.READ_GRAY), D.parse_jpeg4(other, D.READ_GRAY)
        assert b.colour == 0 and all((x.data == y.data).all() for x, y in zip(a.planes, b.planes))


def test_truncated_and_corrupted_files_raise_value_error():
    for name in ('pillow_q75_97x61', 'ycck_2211_restart2', 'arith_ycck_2211', 'pillow_progressive_q50_97x61'):
        data = CORPUS[name][0]
        for n in (3, 40, len(data) // 3, len(data) - 40):
            with pytest.raises(ValueError) as e:
                D.parse_jpeg4(data[:n])
            assert str(e.value)


def test_reader_survives_mutated_four_component_files():
    r = subprocess.run([sys.executable, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'fuzz_cmyk.py'), '500', '7'],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert 'no crash' in r.stdout


def test_single_table_files_route_by_segment_length():
    """A CMYK file whose components share one Huffman table goes to the device decoder only when its
    longest segment is at most FOUR_SYNC_SUBSEQ subsequences; files with distinct tables always do."""
    for kw, device in (({}, False), ({'restart_marker_rows': 1}, True)):
        data = S.pillow_cmyk(1920, 1080, 75, **kw)
        lay = D.FileLayout4(data)
        assert lay.device_decodable and D.four_on_device(lay) == device
        assert isinstance(D._front_end_four(data, True), D.FileLayout4 if device else D.Parsed)
    assert D.four_on_device(D.FileLayout4(S.ycck_file(45, 35, [(1, 1)] * 4, 3)[0]))


def test_blocks_per_mcu_limit():
    """libjpeg refuses an interleaved scan of more than 10 blocks per MCU; so does the reader for
    four-component files (every entry point), and a non-interleaved file of the same sampling reads."""
    sampling = [(2, 2), (2, 1), (1, 1), (2, 2)]         # 4 + 2 + 1 + 4 = 11
    data, planes = S.ycck_file(40, 24, sampling, 5)
    for fn in (D.parse_jpeg4, D.FileLayout4):
        with pytest.raises(ValueError, match='^unsupported jpeg: 11 blocks per MCU \\(at most 10\\)$'):
            fn(data)
    data, planes = S.ycck_file(40, 24, sampling, 5, interleaved=False)
    assert all((a.data == b).all() for a, b in zip(D.parse_jpeg4(data).planes, planes))
    ten = [(2, 2), (1, 1), (1, 1), (2, 2)]
    assert len(D.parse_jpeg4(S.ycck_file(40, 24, ten, 5)[0]).planes) == 4


def test_files_per_chunk_fit_one_batch_session():
    """A CMYK chunk whose planes share a grid is one session of four frames per file: at most
    MAX_BATCH // 4 files, whatever max_frames or free memory allow."""
    cmyk = D.parse_jpeg4(S.pillow_cmyk(64, 64)).key()
    assert cmyk[3] == D.CMYK and len(set(cmyk[2])) == 1
    assert D.max_files(cmyk) == D.MAX_BATCH // 4
    for mode in ('UNCHANGED', 'RGB'):
        assert D.chunk_frames(cmyk, False, 1, 10 ** 6, 0, mode) == D.MAX_BATCH // 4
        assert D.chunk_frames(cmyk, False, 1, None, 80 << 30, mode) == D.MAX_BATCH // 4
        assert D.chunk_frames(cmyk, False, 1, 7, 0, mode) == 7
    # four sessions of n frames (planes on different grids), YCCK and colour keys: MAX_BATCH
    for name in ('cmyk_2211_t0', 'ycck_444_53x29'):
        k = D.parse_jpeg4(CORPUS[name][0]).key()
        assert D.max_files(k) == D.MAX_BATCH
        assert D.chunk_frames(k, False, 1, 10 ** 6, 0, 'UNCHANGED') == D.MAX_BATCH
    colour = cmyk[:2] + (cmyk[2][:3],)
    assert D.chunk_frames(colour, False, 1, 10 ** 6, 0) == D.MAX_BATCH


def test_keys_footprints_and_grouping():
    cmyk = D.parse_jpeg4(CORPUS['pillow_q75_97x61'][0])
    ycck = D.parse_jpeg4(CORPUS['ycck_444_53x29'][0])
    kc, ky = cmyk.key(), ycck.key()
    assert kc[3] == D.CMYK and ky[3] == D.YCCK and len(kc[2]) == 4
    # same geometry, different kind: different batches
    same = D.Parsed(cmyk.w, cmyk.h, cmyk.planes, D.YCCK)
    assert same.key() != kc and same.key()[:3] == kc[:3]
    assert D.solved_planes(kc, False, 'UNCHANGED') == (4, 4) and D.solved_planes(kc, False, 'RGB') == (4, 3)
    assert D.group_class(kc, False) is None and D.group_class(ky, False, 'UNCHANGED') is None
    for sb in (1, 2, 4):
        # every plane counted: more than the colour file of the same geometry, and the output's four channels
        colour = kc[:2] + (kc[2][:3],)
        assert D.frame_footprint(kc, False, sb, 'UNCHANGED') > D.frame_footprint(colour, True, sb, 'RGB')
        assert D.frame_footprint(kc, False, sb, 'UNCHANGED') - D.frame_footprint(kc, False, sb, 'RGB') == kc[0] * kc[1] * sb
        # CMYK solves every plane alone whatever `separate` is; YCCK's colour planes follow it
        assert D.frame_footprint(kc, False, sb, 'UNCHANGED') == D.frame_footprint(kc, True, sb, 'UNCHANGED')
        assert D.frame_footprint(ky, False, sb, 'UNCHANGED') != D.frame_footprint(ky, True, sb, 'UNCHANGED')
        assert D.chunk_frames(kc, False, sb, None, 1 << 30, 'UNCHANGED') < D.chunk_frames(colour, False, sb, None, 1 << 30)
