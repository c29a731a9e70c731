"""Named cases of tests/test_gpu_objective.py: frames, solver settings and the kernels of
libj2pobjective.so each one reaches (the recording dispatch restated: gradient <NC, TGV, GPM>, tile
projection <RES>, 2x2 tile projection, generic projection <SW, SH>).  tests/test_objective_host.py
checks that every kernel of the library is reached by a case."""
from jpeg2png_b200 import synth

QS = [10, 35, 75, 90, 50, 20]


def _synth(w, h, sub, seed):
    return lambda k: synth.synth_coefs(w, h, QS[(seed + k) % 6], sub, seed + k)


def _rand(dims, samp, seed):
    return lambda k: synth.random_coefs(dims, samp, seed + k)


G = 'k_gradient_packed_rec<{}, {}, {}>'
TILE = 'k_project_tile_rec<{}>'
TILE22 = 'k_project_tile22_rec'
GEN = 'k_project_rec<{}, {}>'

# id: (frame k of the case, channels, weight, pweights, iterations, kernels reached)
CASES = {
    '444': (_synth(64, 48, '4:4:4', 10), [0, 1, 2], 0.7, [0.001, 0.0, 0.01], 8,
            [G.format(3, 'true', 1), TILE.format('false')]),
    '444_w0': (_synth(64, 48, '4:4:4', 20), [0, 1, 2], 0.0, [0.001, 0.002, 0.0], 8,
               [G.format(3, 'false', 1), TILE.format('false')]),
    '420': (_synth(128, 64, '4:2:0', 30), [0, 1, 2], 0.3, [0.001] * 3, 8,
            [G.format(3, 'true', 2), TILE.format('false'), TILE22]),
    '420_w0': (_synth(128, 64, '4:2:0', 40), [0, 1, 2], 0.0, [0.001, 0.0, 0.001], 8,
               [G.format(3, 'false', 2), TILE.format('false'), TILE22]),
    'short_luma': (_rand([(64, 56), (32, 32), (32, 32)], [(1, 1), (2, 2), (2, 2)], 50), [0, 1, 2], 0.3, [0.001] * 3, 8,
                   [G.format(3, 'true', 2), TILE.format('true'), TILE22]),
    '422': (_rand([(96, 48), (48, 48), (48, 48)], [(1, 1), (2, 1), (2, 1)], 60), [0, 1, 2], 0.3, [0.001] * 3, 8,
            [G.format(3, 'true', 0), TILE.format('false'), GEN.format(2, 1)]),
    '422_w0': (_rand([(96, 48), (48, 48), (48, 48)], [(1, 1), (2, 1), (2, 1)], 70), [0, 1, 2], 0.0, [0.001] * 3, 8,
               [G.format(3, 'false', 0), TILE.format('false'), GEN.format(2, 1)]),
    '440': (_rand([(48, 96), (48, 48), (48, 48)], [(1, 1), (1, 2), (1, 2)], 80), [0, 1, 2], 0.3, [0.001] * 3, 8,
            [G.format(3, 'true', 0), TILE.format('false'), GEN.format(1, 2)]),
    'odd': (_rand([(40, 24), (24, 16), (16, 8)], [(1, 1), (2, 2), (3, 4)], 90), [0, 1, 2], 0.4, [0.001] * 3, 8,
            [G.format(3, 'true', 0), TILE.format('true'), TILE22, GEN.format(0, 0)]),
    'luma': (_synth(120, 64, '4:2:0', 100), [0], 0.3, [0.001], 8, [G.format(1, 'true', 1), TILE.format('false')]),
    'luma_w0': (_synth(120, 64, '4:2:0', 110), [0], 0.0, [0.001], 8, [G.format(1, 'false', 1), TILE.format('false')]),
    'chroma': (_synth(128, 64, '4:2:0', 120), [1], 0.3, [0.001], 8, [G.format(1, 'true', 0), TILE22]),
    'chroma_w0': (_synth(128, 64, '4:2:0', 130), [2], 0.0, [0.001], 8, [G.format(1, 'false', 0), TILE22]),
    'two_444': (_synth(64, 48, '4:4:4', 140), [1, 2], 0.3, [0.001, 0.001], 8, [G.format(2, 'true', 1), TILE.format('false')]),
    'two_444_w0': (_synth(64, 48, '4:4:4', 150), [1, 2], 0.0, [0.001, 0.001], 8, [G.format(2, 'false', 1), TILE.format('false')]),
    'two_420': (_synth(128, 64, '4:2:0', 160), [1, 2], 0.3, [0.001, 0.0], 8, [G.format(2, 'true', 0), TILE22]),
    'two_420_w0': (_synth(128, 64, '4:2:0', 170), [1, 2], 0.0, [0.001, 0.001], 8, [G.format(2, 'false', 0), TILE22]),
    # tall enough for many bands of the sub-gradient, the last one short on any residency from 1 to 3 CTAs per SM
    'tall': (_synth(64, 4008, '4:4:4', 180), [0, 1, 2], 0.3, [0.001] * 3, 3, [G.format(3, 'true', 1), TILE.format('false')]),
}


def kernels_reached():
    return sorted({k for case in CASES.values() for k in case[5]})
