"""libj2pmixed.so and j2p_session_iterate_group without a GPU: the grouped kernels' inventory (each one
reached by a case of tests/test_gpu_mixed_batch.py, none spilling, none using more stack than the
solver kernel whose body it runs) and the new header symbol."""
import os
import re

from jpeg2png_b200 import abi
from tests import codec_checks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# grouped kernel -> (the solver kernel whose body it runs, the GPU case that reaches it)
KERNELS = {
    'k_gradient_packed_grouped': ('k_gradient_packed', 'test_group_frames_match_single_sessions'),
    'k_project_tile_grouped': ('k_project_tile', "test_group_frames_match_single_sessions['444', '420_short_luma']"),
    'k_project_tile22_grouped': ('k_project_tile22', "test_group_frames_match_single_sessions['420', 'sep_chroma']"),
    'k_step_uncovered_grouped': ('k_step_uncovered', "test_group_frames_match_single_sessions['420_short_luma']"),
    'k_step_uncovered22_grouped': ('k_step_uncovered22', "test_group_frames_match_single_sessions['420_short_luma']"),
}


def _by_name(lib):
    """codec_checks.kernels() keyed by the unqualified name of these j2p:: kernels (the most stack of any instantiation)."""
    out = {}
    for m, (reg, stack, local) in codec_checks.kernels(lib).items():
        n = re.match(r'_ZN3j2p(\d+)', m)
        name = m[n.end():n.end() + int(n.group(1))]
        r0, s0, l0 = out.get(name, (0, 0, 0))
        out[name] = (max(r0, reg), max(s0, stack), max(l0, local))
    return out


def test_kernel_inventory():
    mixed = _by_name(os.path.join(ROOT, 'jpeg2png_b200', 'mixed', 'libj2pmixed.so'))
    solver = _by_name(abi.PRODUCT_LIB)
    assert sorted(mixed) == sorted(KERNELS), sorted(mixed)
    for k, (reg, stack, local) in mixed.items():
        assert local == 0, f'{k} uses {local} bytes of local memory'
        assert stack <= solver[KERNELS[k][0]][1], f'{k} uses {stack} bytes of stack, {KERNELS[k][0]} {solver[KERNELS[k][0]][1]}'


def test_no_spills():
    log = open(os.path.join(ROOT, 'jpeg2png_b200', 'mixed', 'mixed.ptxas.log')).read()
    spills = re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', log)
    assert spills and all(a == '0' and b == '0' for a, b in spills), spills


def test_header_symbol():
    header = open(os.path.join(ROOT, 'include', 'jpeg2png_b200.h')).read()
    assert re.search(r'int j2p_session_iterate_group\(j2p_session \*const \*sessions, unsigned n, unsigned first, unsigned count\);', header)
    assert 'j2p_session_iterate_group' in abi.HEADER_SYMBOLS


def test_every_named_case_exists():
    """Each grouped kernel's GPU case is a test (and parameter) of tests/test_gpu_mixed_batch.py."""
    src = open(os.path.join(ROOT, 'tests', 'test_gpu_mixed_batch.py')).read()
    tests = set(re.findall(r'^def (test_\w+)', src, re.M))
    layouts = set(re.search(r"^LAYOUTS = \[(.*)\]", src, re.M).group(1).replace("'", '').replace(' ', '').split(','))
    for kernel, (_, case) in KERNELS.items():
        name, _, params = case.partition('[')
        assert name in tests, (kernel, case)
        for p in re.findall(r"'(\w+)'", params):
            assert p in layouts, (kernel, case)


# ---- decode_jpeg's packing of per-geometry chunks into groups (decode.group_class, decode.pack) ----
from jpeg2png_b200 import decode  # noqa: E402

K420 = lambda w, h: (w, h, ((w + 7) // 8 * 8, (h + 7) // 8 * 8, 1, 1), ((w + 15) // 16 * 8, (h + 15) // 16 * 8, 2, 2),  # noqa: E731
                     ((w + 15) // 16 * 8, (h + 15) // 16 * 8, 2, 2))


def key420(w, h):
    k = K420(w, h)
    return (k[0], k[1], k[2:])


def key(w, h, samp):
    return (w, h, tuple(((w + 7) // 8 * 8 // sw, (h + 7) // 8 * 8 // sh, sw, sh) for sw, sh in samp))


def test_group_class_restates_the_join_rules():
    c420 = decode.group_class(key420(64, 48), False)
    assert c420 == (3, ((1, 1), (2, 2), (2, 2)))
    assert decode.group_class(key420(200, 40), False) == c420                 # any size of one layout: one class
    assert decode.group_class(key(64, 48, [(1, 1)] * 3), False) == (3, ((1, 1),) * 3)
    assert decode.group_class(key(64, 48, [(1, 1)]), False) == (1, ((1, 1),))    # a gray file
    assert decode.group_class(key(64, 48, [(1, 1)]), True) == (1, ((1, 1),))     # solved the same with separate
    assert decode.group_class(key420(64, 48), False, 'GRAY') == c420            # joint solve, one channel out
    assert decode.group_class(key420(64, 48), True) is None                     # separate mode: a session per plane
    assert decode.group_class(key420(64, 48), True, 'GRAY') is None
    assert decode.group_class(key(64, 48, [(1, 1), (2, 1), (2, 1)]), False) is None    # 4:2:2
    assert decode.group_class(key(64, 48, [(1, 1), (1, 2), (1, 2)]), False) is None    # 4:4:0
    assert decode.group_class(key(96, 96, [(1, 1), (2, 2), (3, 4)]), False) is None    # odd factors
    assert decode.group_class(key420(352, 352), False) is not None                     # 123 904 pixels
    assert decode.group_class(key420(512, 512), False) is None                         # over GROUP_MAX_PIXELS
    assert decode.group_class(key420(1920, 1080), False) is None


def _pack(chunks, cap=1 << 40, bytes_of=lambda k, n: n):
    return decode.pack(chunks, lambda k: decode.group_class(k, False), bytes_of, cap)


def test_pack_holds_one_chunk_per_geometry_and_keeps_order():
    a, b, c = key420(64, 48), key420(80, 32), key420(48, 64)
    keys = [a, b, a, c, b, a, c]
    chunks = decode.plan(keys, lambda k: 1)                 # max_frames=1: one chunk per input
    packs = _pack(chunks)
    for p in packs:
        ks = [chunks[j][0] for j in p]
        assert len(ks) == len(set(ks)), packs
        assert p == sorted(p)
    flat = [j for p in packs for j in p]
    assert sorted(flat) == list(range(len(chunks)))          # every chunk exactly once
    assert [p[0] for p in packs] == sorted(p[0] for p in packs)
    inputs = [i for j in sorted(flat) for i in chunks[j][1]]
    assert sorted(inputs) == list(range(len(keys)))          # every input exactly once


def test_max_frames_boundaries_are_todays():
    a, b = key420(64, 48), key420(80, 32)
    keys = [a] * 5 + [b] * 3
    chunks = decode.plan(keys, lambda k: 2)
    assert [idx for _, idx in chunks] == [[0, 1], [2, 3], [4], [5, 6], [7]]
    assert _pack(chunks) == [[0], [1], [2, 3], [4]]          # a repeated geometry closes the open pack


def test_one_chunk_packs_and_ungroupable_chunks_are_alone():
    big, small, s422 = key420(1920, 1080), key420(64, 48), key(64, 48, [(1, 1), (2, 1), (2, 1)])
    chunks = decode.plan([big, small, s422, small], lambda k: 8)
    assert _pack(chunks) == [[0], [1], [2]]
    gray, colour = key(64, 48, [(1, 1)]), key420(64, 48)
    chunks = decode.plan([gray, colour, key(32, 32, [(1, 1)]), key420(32, 32)], lambda k: 8)
    assert _pack(chunks) == [[0, 2], [1, 3]]                # two classes, two packs


def test_pack_frame_and_footprint_caps():
    keys = [key420(16 + 8 * k, 16) for k in range(6)]
    chunks = [(k, list(range(30000 * j, 30000 * j + 30000))) for j, k in enumerate(keys[:3])]
    assert _pack(chunks) == [[0, 1], [2]]                    # 90 000 frames > 65535
    chunks = decode.plan(keys, lambda k: 8)
    assert _pack(chunks, cap=3) == [[0, 1, 2], [3, 4, 5]]    # one byte per frame, three per pack
    assert _pack(chunks, cap=0) == [[j] for j in range(6)]   # a chunk alone may exceed the cap
