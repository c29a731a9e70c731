"""Multi-rank row strips on CPU: world size 2 (and 3) over gloo, oracle strip backend.

What is under test is the N>1 orchestration of jpeg2png_b200/strips.py — strip planning, the
rank-ordered fold of the all-gathered sums, the neighbour halo exchange — with exactly the calls
the GPU path makes (there the backend is a strip session of libjpeg2png_b200.so and the process
group is NCCL).  The strip-parallel result must equal the single-process oracle bit for bit."""
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from jpeg2png_b200 import strips, synth
from tests import helpers as H

CASES = {
    # name: (w, h, quality, subsampling, weight, pweights, iterations)
    'c420': (96, 128, 20, '4:2:0', 0.3, [0.001] * 3, 12),
    'c444': (64, 72, 50, '4:4:4', 0.5, [0.001, 0.0, 0.002], 10),
    'luma_short': (80, 104, 30, '4:2:0', 0.3, [0.001] * 3, 8),      # frame 80x112, luma grid 104 rows
}


def _worker(rank, world, init_file, case, out_dir):
    from tests.strip_backend import OracleStrip
    w, h, q, ss, weight, pw, iters = CASES[case]
    dist.init_process_group('gloo', init_method=f'file://{init_file}', rank=rank, world_size=world)
    try:
        img = synth.synth_coefs(w, h, q, ss, seed=4242)
        fdata = H.decode_planes(img)
        mcu = 8 * max(p.h_samp for p in img.planes)
        plan = strips.plan_strips(img.frame_h, mcu, world)
        row0, rows = plan[rank]
        be = OracleStrip(img, weight, pw, iters, row0, rows, fdata)
        strips.solve_strips(be, dist, rank, world, iters)
        np.savez(os.path.join(out_dir, f'rank{rank}.npz'), row0=row0, rows=rows, **{f'p{c}': be.download(c) for c in range(3)})
        be.close()
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('case,world', [('c420', 2), ('c444', 2), ('luma_short', 2), ('c420', 3)])
def test_strips_match_single_process(case, world, tmp_path):
    H.build_oracle_libs()
    init_file = tempfile.mktemp(dir=str(tmp_path))
    mp.spawn(_worker, args=(world, init_file, case, str(tmp_path)), nprocs=world, join=True)
    w, h, q, ss, weight, pw, iters = CASES[case]
    img = synth.synth_coefs(w, h, q, ss, seed=4242)
    want = H.run_compute('oracle', img, [0, 1, 2], weight, pw, iters)
    parts = [np.load(os.path.join(str(tmp_path), f'rank{r}.npz')) for r in range(world)]
    assert sum(int(p['rows']) for p in parts) == img.frame_h
    got = [np.concatenate([p[f'p{c}'] for p in parts], axis=0) for c in range(3)]
    H.assert_bit_identical(got, want, f'{case} x{world} strips')


@pytest.mark.parametrize('world', [2, 3, 8])
@pytest.mark.parametrize('case', ['c420', 'c444'])
def test_lockstep_driver_matches_single_process(case, world):
    """The one-process lock-step driver of tests/test_gpu_strips_one_device.py, with oracle strips
    only: N strips driven by it must give the whole-frame oracle's bits, so on the GPU a difference
    is the product's and not the driver's."""
    from tests.strip_backend import LockStep, OracleStrip
    w, h, q, ss, weight, pw, iters = CASES[case]
    img = synth.synth_coefs(w, h, q, ss, seed=4242)
    fdata = H.decode_planes(img)
    plan = strips.plan_strips(img.frame_h, 8 * max(p.h_samp for p in img.planes), world)
    drv = LockStep([OracleStrip(img, weight, pw, iters, row0, rows, fdata) for row0, rows in plan])
    try:
        drv.start()
        for _ in range(iters):
            drv.project(drv.gradient())
        got = drv.download()
    finally:
        for s in drv.strips:
            s.close()
    want = H.run_compute('oracle', img, [0, 1, 2], weight, pw, iters, [p.copy() for p in fdata])
    H.assert_bit_identical(got, want, f'{case} x{world} lock-step strips')


def test_plan_strips_alignment():
    for frame_h, mcu, world in [(4320, 16, 8), (1088, 16, 8), (2160, 8, 4), (64, 16, 4), (1088, 16, 3)]:
        plan = strips.plan_strips(frame_h, mcu, world)
        assert len(plan) == world and plan[0][0] == 0
        assert sum(r for _, r in plan) == frame_h
        for (row0, rows), nxt in zip(plan, plan[1:] + [(frame_h, 0)]):
            assert row0 % mcu == 0 and rows > 0 and row0 + rows == nxt[0]
        sizes = [r for _, r in plan]
        assert max(sizes) - min(sizes) <= mcu
    with pytest.raises(ValueError):
        strips.plan_strips(32, 16, 4)


def test_plane_rows_of_strip():
    # 1080p 4:2:0: luma 1080 coefficient rows in a 1088-row frame; last strip ends at the frame bottom
    assert strips.plane_rows_of_strip(1080, 1, 944, 144) == (944, 1080)
    assert strips.plane_rows_of_strip(544, 2, 944, 144) == (472, 544)
    assert strips.plane_rows_of_strip(1080, 1, 0, 144) == (0, 144)
