"""Mutation fuzzing of the progressive layout pass and the progressive decoder's host driver against
the host reader, run as a separate process by tests/test_progressive_host.py so that a crash is a
failed test.  The mutations are those of tests/fuzz_entropy.py, on progressive seeds (Pillow's script
with and without restart markers, and crafted scripts).  Every mutated file must be rejected by both,
or accepted by both with identical coefficients; a file that is not progressive is left to the
reader."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jpeg2png_b200 import decode as D  # noqa: E402
from tests import entropy_cases as E  # noqa: E402
from tests import progressive_cases as P  # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 400
    seed = int(sys.argv[2]) if len(sys.argv) > 2 else 1
    rng = np.random.default_rng(seed)
    crafted = P.crafted()
    seeds = [E.pillow(64, 48, 75, '4:4:4', progressive=True), E.pillow(72, 40, 20, '4:2:0', optimize=True, progressive=True),
             P.pillow_restarts(64, 48, 50, '4:2:0'), crafted['deep_ri2'], crafted['standard_random_1']]
    both_reject = both_accept = other = 0
    for it in range(n):
        data = bytearray(seeds[it % len(seeds)])
        kind = rng.integers(0, 5)
        if kind == 0:                                   # truncate
            data = data[:int(rng.integers(2, len(data)))]
        elif kind == 1:                                 # flip a few bytes anywhere
            for _ in range(int(rng.integers(1, 8))):
                data[int(rng.integers(0, len(data)))] = int(rng.integers(0, 256))
        elif kind == 2:                                 # corrupt the header region (markers, lengths, tables)
            for _ in range(int(rng.integers(1, 6))):
                data[int(rng.integers(2, min(len(data), 700)))] = int(rng.integers(0, 256))
        elif kind == 3:                                 # duplicate or drop a chunk
            a, b = sorted(int(x) for x in rng.integers(2, len(data), 2))
            data = data[:a] + data[b:] if rng.random() < 0.5 else data[:b] + data[a:b] + data[b:]
        else:                                           # insert marker-like garbage
            pos = int(rng.integers(2, len(data)))
            data[pos:pos] = bytes([0xFF, int(rng.integers(0xC0, 0xFF)), 0, int(rng.integers(0, 40))])
        data = bytes(data)
        want, err = E.reader(data)
        try:
            lay = D.ProgFileLayout(data)
        except ValueError:
            assert want is None, f'iteration {it}: the layout pass rejects a file the reader accepts'
            both_reject += 1
            continue
        if not lay.progressive_decodable:
            other += 1
            continue
        arrs, status, _ = P.prog_host([lay], int(rng.choice([32, 64, 256, 1024])))
        if want is None:
            assert status[0] != 0, f'iteration {it}: the decoder accepts a file the reader rejects ({err})'
            both_reject += 1
        else:
            assert status[0] == 0, f'iteration {it}: the decoder rejects a file the reader accepts (status {status[0]})'
            assert all((a == b).all() for a, b in zip(arrs[0], want)), f'iteration {it}: coefficients differ'
            both_accept += 1
    print(f'fuzz_progressive: {n} mutated files, {both_accept} accepted by both, {both_reject} rejected by both, '
          f'{other} not progressive; no disagreement')


if __name__ == '__main__':
    main()
