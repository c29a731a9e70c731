"""Mutation fuzzing of the four-component reader (j2p_read_jpeg4_mem, jpeg2png_b200/cli/jpeg_reader.c)
on CMYK and YCCK files, Huffman and arithmetic, run as a separate process by tests/test_cmyk_host.py
so that a crash shows up as a failed test.  Every mutated file must either parse (with sane plane
sizes) or be rejected with a ValueError carrying the reader's message; so must the four-plane layout
pass, and the three-plane layout passes, given the flag, must agree that a four-component file is
not theirs."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jpeg2png_b200 import decode as D  # noqa: E402
from tests import cmyk_synth as S  # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 400
    seed = int(sys.argv[2]) if len(sys.argv) > 2 else 1
    rng = np.random.default_rng(seed)
    c = S.corpus()
    seeds = [c[k][0] for k in ('pillow_q75_97x61', 'pillow_progressive_q50_97x61', 'ycck_2211_restart2', 'arith_cmyk',
                               'arith_ycck_2211')]
    parsed = rejected = 0
    for it in range(n):
        data = bytearray(seeds[it % len(seeds)])
        kind = rng.integers(0, 4)
        if kind == 0:                                   # truncate
            data = data[:int(rng.integers(2, len(data)))]
        elif kind == 1:                                 # flip a few bytes anywhere
            for _ in range(int(rng.integers(1, 8))):
                data[int(rng.integers(0, len(data)))] = int(rng.integers(0, 256))
        elif kind == 2:                                 # corrupt the header region
            for _ in range(int(rng.integers(1, 6))):
                data[int(rng.integers(2, min(len(data), 700)))] = int(rng.integers(0, 256))
        else:                                           # drop or duplicate a chunk
            a, b = sorted(int(x) for x in rng.integers(2, len(data), 2))
            data = data[:a] + data[b:] if rng.random() < 0.5 else data[:b] + data[a:b] + data[b:]
        data = bytes(data)
        try:
            p = D.parse_jpeg4(data, D.READ_GRAY)
        except ValueError as e:
            assert str(e), 'rejected without a message'
            rejected += 1
        else:
            parsed += 1
            assert 0 < p.w <= 65535 and 0 < p.h <= 65535 and len(p.planes) in (1, 3, 4)
            for pl in p.planes:
                assert pl.w % 8 == 0 and pl.h % 8 == 0 and pl.data.size == pl.w * pl.h
        try:
            lay = D.FileLayout4(data, D.READ_GRAY)
        except ValueError as e:
            assert str(e), 'rejected without a message'
        else:
            if lay.device_decodable:
                assert lay.lay.ncomp in (1, 3, 4) and lay.lay.nscan == lay.lay.ncomp or lay.lay.nscan <= lay.lay.ncomp
        for layout in (D.FileLayout, D.ProgFileLayout, D.ArithFileLayout):
            try:
                lay = layout(data, D.READ_GRAY | D.READ_CMYK)
            except ValueError:
                continue
            if lay.lay.ncomp == 4:
                raise AssertionError('a layout pass took a four-component file')
    print(f'fuzz_cmyk: {n} mutated files, {parsed} parsed, {rejected} rejected, no crash')


if __name__ == '__main__':
    main()
