"""Mutation fuzzing of the reader's arithmetic decoding (jpeg2png_b200/cli/jpeg_reader.c) and of the
arithmetic layout pass, run as a separate process by tests/test_arith_host.py so that a crash shows up
as a failed test.  Every mutated SOF9/SOF10 file must either parse (with sane plane sizes) or be
rejected with a message, by the reader and by the layout pass alike."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jpeg2png_b200 import decode as D  # noqa: E402
from tests import arith_synth as A, entropy_cases as E  # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 400
    seed = int(sys.argv[2]) if len(sys.argv) > 2 else 1
    rng = np.random.default_rng(seed)
    seeds = [A.transcode(E.pillow(64, 48, 75, '4:4:4')), A.transcode(E.pillow(72, 40, 20, '4:2:0'), 'components', 3),
             A.transcode(E.pillow(56, 64, 50, '4:2:0', progressive=True), 'own'),
             A.transcode(E.pillow(48, 48, 90, '4:2:2'), 'progressive', 'row', dac={0: 0x31, 17: 9})]
    parsed = rejected = 0
    for it in range(n):
        data = bytearray(seeds[it % len(seeds)])
        kind = rng.integers(0, 5)
        if kind == 0:                                   # truncate
            data = data[:int(rng.integers(2, len(data)))]
        elif kind == 1:                                 # flip a few bytes anywhere
            for _ in range(int(rng.integers(1, 8))):
                data[int(rng.integers(0, len(data)))] = int(rng.integers(0, 256))
        elif kind == 2:                                 # corrupt the header region (markers, lengths, tables, DAC)
            for _ in range(int(rng.integers(1, 6))):
                data[int(rng.integers(2, min(len(data), 300)))] = int(rng.integers(0, 256))
        elif kind == 3:                                 # duplicate or drop a chunk
            a, b = sorted(int(x) for x in rng.integers(2, len(data), 2))
            data = data[:a] + data[b:] if rng.random() < 0.5 else data[:b] + data[a:b] + data[b:]
        else:                                           # insert marker-like garbage
            pos = int(rng.integers(2, len(data)))
            data[pos:pos] = bytes([0xFF, int(rng.integers(0xC0, 0xFF)), 0, int(rng.integers(0, 40))])
        data = bytes(data)
        try:
            p = D.parse_jpeg(data, D.READ_GRAY)
            parsed += 1
            assert 0 < p.w <= 65535 and 0 < p.h <= 65535
            for pl in p.planes:
                assert pl.w % 8 == 0 and pl.h % 8 == 0 and pl.data.size == pl.w * pl.h
        except ValueError as e:
            rejected += 1
            assert str(e), 'rejected without a message'
        try:
            D.ArithFileLayout(data, D.READ_GRAY)
        except ValueError as e:
            assert str(e), 'the layout pass rejected without a message'
    print(f'fuzz_arith: {n} mutated files, {parsed} parsed, {rejected} rejected, no crash')


if __name__ == '__main__':
    main()
