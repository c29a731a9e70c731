"""The arithmetic-coded corpus of tests/test_arith_host.py and tests/test_gpu_arith.py: twins of
Pillow files and of jpeg_synth files (tests/arith_synth.py), and files coded from given coefficients."""
import io

import numpy as np
from PIL import Image

from jpeg2png_b200 import decode as D, synth
from tests import arith_synth as A
from tests import entropy_cases as E
from tests import jpeg_synth as J


def pillow_gray(w, h, q, seed=1):
    rgb = synth.cartoon_image(w, h, seed).astype(np.uint8)
    buf = io.BytesIO()
    Image.fromarray(rgb, 'RGB').convert('L').save(buf, 'JPEG', quality=q)
    return buf.getvalue()


def large_planes(w, h, sampling, seed):
    """jpeg_synth.random_planes on the real block grids, with DC differences and AC values of
    magnitude category 15 in some blocks."""
    planes, quants = J.random_planes(w, h, sampling, seed)
    rng = np.random.default_rng(seed)
    maxh, maxv = max(a for a, _ in sampling), max(b for _, b in sampling)
    out = []
    for (sh, sv), p in zip(sampling, planes):
        wb, hb = -(-(-(-w * sh // maxh)) // 8), -(-(-(-h * sv // maxv)) // 8)
        p = p[:hb, :wb].astype(np.int64)
        big = rng.random(p.shape[:2]) < 0.2
        p[..., 0] = np.where(big, rng.choice([-8200, 8200], size=p.shape[:2]), p[..., 0])
        p[..., 5] = np.where(big, rng.choice([-20000, 19000, 32767], size=p.shape[:2]), p[..., 5])
        out.append(p.astype(np.int16))
    return out, quants


def coded(w, h, sampling, seed, script='sequential', ri=0, dac=None):
    """(arith bytes, planes) coded from large_planes."""
    planes, quants = large_planes(w, h, sampling, seed)
    comps = [(k + 1, sh, sv, 0 if k == 0 else 1) for k, (sh, sv) in enumerate(sampling)]
    keep = [A.dqt(quants[:2])]
    return A.write(w, h, keep, comps, planes, script, ri, dac), planes


def corpus():
    """name -> (arithmetic file, its Huffman twin): every file of the corpus that has a twin."""
    files = {}
    for q in (5, 20, 50, 75, 90, 100):
        for ss, (w, h) in (('4:4:4', (97, 61)), ('4:2:0', (73, 59)), ('4:2:2', (64, 48))):
            src = E.pillow(w, h, q, ss, seed=q)
            files[f'pillow_{ss.replace(":", "")}_q{q}'] = (A.transcode(src), src)
    opt = E.pillow(96, 80, 60, '4:2:0', optimize=True)
    files['pillow_opt_components'] = (A.transcode(opt, 'components'), opt)
    prog = E.pillow(80, 64, 70, '4:2:0', progressive=True)
    files['pillow_prog_own_sof10'] = (A.transcode(prog, 'own'), prog)
    files['pillow_prog_sof9'] = (A.transcode(prog), prog)
    progopt = E.pillow(64, 56, 40, '4:4:4', optimize=True, progressive=True)
    files['pillow_prog_opt_own_ri7_sof10'] = (A.transcode(progopt, 'own', 7), progopt)
    files['pillow_simple_progression_row_sof10'] = (A.transcode(opt, 'progressive', 'row'), opt)
    for ri in (1, 7, 'row'):
        src = E.pillow(120, 72, 75, '4:2:0', seed=5)
        files[f'pillow_420_ri{ri}'] = (A.transcode(src, 'sequential', ri), src)
        files[f'pillow_420_components_ri{ri}'] = (A.transcode(src, 'components', ri), src)
    src = E.pillow(98, 61, 30, '4:2:2', seed=7)
    files['dac_nondefault'] = (A.transcode(src, 'sequential', 0, dac={0: 0x52, 1: 0xF3, 16: 1, 17: 40}), src)
    files['dac_kx_255_l_eq_u'] = (A.transcode(src, 'components', 3, dac={0: 0x00, 1: 0x99, 16: 255, 17: 0}), src)
    files['dac_progressive'] = (A.transcode(src, 'progressive', 0, dac={0: 0x41, 16: 2, 17: 63}), src)
    files['pillow_1x1'] = (A.transcode(E.pillow(1, 1, 75, '4:4:4')), E.pillow(1, 1, 75, '4:4:4'))
    files['pillow_7x9'] = (A.transcode(E.pillow(7, 9, 100, '4:4:4')), E.pillow(7, 9, 100, '4:4:4'))
    for q, ri in ((10, 0), (85, 5)):
        g = pillow_gray(67, 45, q)
        files[f'gray_q{q}_ri{ri}'] = (A.transcode(g, 'sequential', ri), g)
    g = pillow_gray(48, 40, 60)
    files['gray_progressive'] = (A.transcode(g, 'progressive'), g)
    for k, s in enumerate([[(2, 2), (1, 1), (1, 1)], [(4, 1), (2, 1), (1, 2)], [(1, 2), (1, 1), (1, 1)]]):
        src = E.synth_file(48 + 8 * k, 40, s, 0)
        files[f'synth_{k}'] = (A.transcode(src), src)
        files[f'synth_{k}_ri2'] = (A.transcode(src, 'sequential', 2), src)
    return files


def coded_corpus():
    """name -> (arithmetic file, planes): large magnitudes and odd sampling, coded from coefficients."""
    return {
        'large_444': coded(40, 24, [(1, 1)] * 3, 1),
        'large_420_ri3': coded(70, 50, [(2, 2), (1, 1), (1, 1)], 2, ri=3),
        'large_odd_sampling': coded(52, 36, [(4, 1), (2, 1), (1, 2)], 3),
        'large_progressive': coded(40, 32, [(2, 1), (1, 1), (1, 1)], 4, script='progressive'),
    }


def frame_marker(data):
    """The SOF marker of a file (0xC9 or 0xCA for the corpus)."""
    pos = 2
    while data[pos + 1] < 0xC0 or data[pos + 1] in (0xC4, 0xCC) or data[pos + 1] >= 0xD8:
        pos += 2 + int.from_bytes(data[pos + 2:pos + 4], 'big')
    return data[pos + 1]


def sequential(files):
    """The SOF9 files of a corpus."""
    return {k: v for k, v in files.items() if frame_marker(v[0]) == 0xC9}


def reader_planes(data, flags=D.READ_GRAY):
    return [p.data for p in D.parse_jpeg(data, flags).planes]


def arith_host(layouts):
    """Decode ArithFileLayouts with the serial host driver: ([per file: int16 arrays], statuses, stats)."""
    import ctypes as C
    arrs, outs = [], []
    for lay in layouts:
        planes = []
        for p in lay.planes:
            a = np.full(p.w * p.h, 0x5a5a, np.int16)      # the decoder writes every coefficient
            planes.append(a)
            outs.append(a.ctypes.data)
        outs.extend([0] * (3 - len(lay.planes)))
        arrs.append(planes)
    buf, addr, _, _ = D.arith_plan(layouts, outs)
    status = np.zeros(max(len(layouts), 1), np.uint32)
    stats = D.ArithStats()
    lib = D.load_arith()
    assert lib.j2p_arith_decode_host(addr, None, status.ctypes.data, C.byref(stats)) == 0, lib.j2p_arith_last_error()
    return arrs, status[:len(layouts)], stats
