"""Every kernel in the library is checked against the checker (CPU test, no GPU needed).

Lists the kernel instantiations of the in-tree libjpeg2png_b200.so with cuobjdump, as
test_sass_techniques.py does, and requires each of them to be launched by at least one named case
of the GPU matrix (tests/test_gpu_kernel_matrix.py), as tests/kernel_paths.py predicts the host
dispatch, or to be on the short exemption list below with the test that covers it.  A kernel added
without a matrix case fails here, by name, before anything reaches a GPU.  The seeded geometry sweep
of the matrix does not count: coverage has to come from cases whose purpose is stated.

Row-strip sessions run their own code in every solver kernel, so they are held to the same rule
separately: every kernel a strip session can launch must be reached by a named case of
tests/test_gpu_strips_one_device.py, strip by strip, as the strip mode of kernel_paths predicts.
"""
import os
import re
import shutil
import subprocess

import pytest

from tests import kernel_paths as K
from tests import test_gpu_kernel_matrix as M
from tests import test_gpu_strips_one_device as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'jpeg2png_b200', 'csrc', 'libjpeg2png_b200.so')

# kernel -> the test that compares it with the checker, and why it is not in the matrix
EXEMPT = {
    'k_halo_exchange': 'tests/test_gpu_strips.py: the halo exchange between strips over peer memory; it needs cudaIpc '
                       'mappings between the processes of two or more GPUs',
    'k_project_tma<false>': 'tests/test_gpu_parity.py::test_tma_projection_matches_oracle: opt-in J2P_PROJ_TMA=1 kernel',
    'k_project_tma<true>': 'tests/test_gpu_parity.py::test_tma_projection_matches_oracle: opt-in J2P_PROJ_TMA=1 kernel',
    'k_scanlines': 'tests/test_gpu_cli.py::test_device_scanlines_match_reference_conversion: the PNG epilogue after '
                   'a solve, not part of an iteration',
}


def library_kernels():
    """Demangled, normalised names of every kernel (every .text.* section) in the library."""
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump) or not os.path.exists(LIB):
        pytest.skip('CUDA toolkit or the built library is missing')
    filt = os.path.join(os.path.dirname(cuobjdump), 'cu++filt')
    if not os.path.exists(filt):
        filt = shutil.which('cu++filt') or shutil.which('c++filt')
    elf = subprocess.run([cuobjdump, '-elf', LIB], check=True, capture_output=True, text=True).stdout
    mangled = sorted(set(re.findall(r'\.text\.(_Z\w+)', elf)))
    assert mangled, 'no kernels found in the library?'
    out = subprocess.run([filt], input='\n'.join(mangled) + '\n', check=True, capture_output=True, text=True).stdout
    return {K.normalise(line) for line in out.splitlines() if line.strip()}


def matrix_kernels(cases):
    """kernel -> names of the cases that launch it (set-up and iteration kernels)."""
    reach = {}
    for c in cases:
        ks = K.iteration(c.planes, c.weight, c.mode())[0] + K.setup(c.planes, c.mode())[0]
        for k in ks:
            reach.setdefault(k, []).append(c.name)
    return reach


def strip_kernels(cases):
    """kernel -> names of the strip cases that launch it, strip by strip (set-up and iteration)."""
    reach = {}
    for c in cases:
        for strip in c.plan():
            m = c.mode(strip)
            for k in K.iteration(c.planes, c.weight, m)[0] + K.setup(c.planes, m)[0]:
                reach.setdefault(k, []).append(c.name)
    return reach


# what a strip session never launches: the batched instantiations, the objective-logging builds
# (logging is refused on a strip), the PNG epilogue and the peer-memory halo kernel
def _strip_launchable(k):
    batch = re.match(r'k_gradient_packed<\d, \w+, \d, true>|k_project_tile<\w+, true>|k_project_tile22<true>|'
                     r'k_step_uncovered(22)?<true>', k)
    logging = re.match(r'k_gradient<\d, true, \w+>$', k) or k == 'k_project<1, 1>'
    return not (batch or logging or k in ('k_scanlines', 'k_halo_exchange'))


def test_every_kernel_is_reached_by_a_matrix_case_or_exempt():
    lib = library_kernels()
    reached = matrix_kernels(M.NAMED)
    reached.update(strip_kernels(S.NAMED))
    missing = sorted(k for k in lib if k not in reached and k not in EXEMPT)
    assert not missing, ('kernels in the library that no named case of tests/test_gpu_kernel_matrix.py or '
                         'tests/test_gpu_strips_one_device.py launches '
                         '(add a case, or an exemption naming the test that covers it): ' + ', '.join(missing))


def test_every_strip_kernel_is_reached_by_a_named_strip_case():
    lib = library_kernels()
    want = sorted(k for k in lib if _strip_launchable(k))
    assert 'k_fold_sums' in want and 'k_project_tma<true>' in want and len(want) >= 30, want
    reached = strip_kernels(S.NAMED)
    missing = [k for k in want if k not in reached]
    assert not missing, ('kernels a strip session can launch that no named case of tests/test_gpu_strips_one_device.py '
                         'reaches: ' + ', '.join(missing))
    assert not sorted(set(reached) - set(want)), f'strip cases predicted to launch {sorted(set(reached) - set(want))}'


def test_strip_case_ids_are_unique_and_tall_strips_have_short_last_bands():
    names = [c.name for c in S.NAMED]
    assert len(names) == len(set(names))
    for c in S.NAMED:
        # what j2p_session_create_strip accepts: cuts on every plane's blocks, no strip below a plane's grid
        assert all(row0 % (8 * p.sh) == 0 and p.ch * p.sh > row0 for row0, _ in c.plan() for p in c.planes), c.describe()
        if c.tall:
            per_sm = K.GRAD_CTAS_PER_SM[len(c.planes)]
            W = K.frame_size(c.planes)[0]
            assert all(1 <= K.last_band_rows(W, rows, K.H100_SMS * per_sm) <= 7 for _, rows in c.plan()), c.describe()


def test_predicted_and_exempt_kernels_exist_in_the_library():
    """A restatement that names a kernel the library does not have is wrong, and so is a stale exemption."""
    lib = library_kernels()
    predicted = matrix_kernels(M.CASES)
    predicted.update(strip_kernels(S.NAMED))
    assert not sorted(set(predicted) - lib), f'kernel_paths predicts kernels the library lacks: {sorted(set(predicted) - lib)}'
    assert not sorted(set(EXEMPT) - lib), f'exemptions for kernels the library lacks: {sorted(set(EXEMPT) - lib)}'


def test_library_inventory_is_the_expected_size():
    # 62 instantiations when this test was written; the count moving is fine as long as the
    # coverage test above still passes, but a near-empty inventory means the parsing broke
    assert len(library_kernels()) >= 60


def test_documented_gradient_residency_follows_from_the_register_use():
    """kernel_paths.resident_ctas (what the GPU matrix sizes its tall frames with) against the figures
    DESIGN.md documents: two CTAs per SM for the three-channel joint builds, five for one channel."""
    res = K.library_resources(LIB)
    if res is None:
        pytest.skip('CUDA toolkit or the built library is missing')
    assert K.resident_ctas(*res['k_gradient_packed<3, true, 1, false>']) == 2
    assert K.resident_ctas(*res['k_gradient_packed<3, true, 2, false>']) == 2
    assert K.resident_ctas(*res['k_gradient_packed<1, true, 1, false>']) == 5


def test_case_ids_are_unique_and_tall_frames_have_short_last_bands():
    names = [c.name for c in M.CASES]
    assert len(names) == len(set(names))
    for c in M.NAMED:
        if c.name.startswith('tall_'):
            W, Hf = K.frame_size(c.planes)
            per_sm = K.GRAD_CTAS_PER_SM[3 if len(c.planes) == 3 else 1]
            assert 1 <= K.last_band_rows(W, Hf, K.H100_SMS * per_sm) <= 7, c.describe()


def test_kernel_paths_restates_the_dispatch_of_known_layouts():
    """Spot checks of the restatement against launch counts the batch tests measure on the GPU."""
    p420 = (K.PlaneGeom(1920, 1080, 1, 1), K.PlaneGeom(960, 544, 2, 2), K.PlaneGeom(960, 544, 2, 2))
    ks, n = K.iteration(p420, 0.3)
    assert ks == ['k_gradient_packed<3, true, 2, false>', 'k_project_tile<true, false>', 'k_step_uncovered<false>',
                  'k_project_tile22<false>']
    assert K.iteration(p420, 0.3, K.Mode(nframes=16))[1] == n            # the launches do not grow with a batch
    p422 = (K.PlaneGeom(96, 48, 1, 1), K.PlaneGeom(48, 48, 2, 1), K.PlaneGeom(48, 48, 2, 1))
    assert K.iteration(p422, 0.3, K.Mode(nframes=3))[0] == [
        'k_gradient_packed<3, true, 0, true>', 'k_project_tile<false, true>'] + ['k_project<2, 1>'] * 6
    assert K.iteration(p420, 0.0, K.Mode(log=True))[0] == [
        'k_gradient<3, true, false>', 'k_project<1, 1>', 'k_project<2, 2>', 'k_project<2, 2>']


def test_kernel_paths_restates_the_strip_dispatch():
    """Strip mode: one frame, different kernels per strip (launch_gradient_packed tests the strip's
    coefficient rows against its owned rows; launch_project groups and steps by the strip's rows)."""
    G = K.PlaneGeom
    three = (G(64, 48, 1, 1), G(64, 48, 1, 1), G(64, 40, 1, 1))          # plane 2 is 8 rows short
    generic_whole = ['k_gradient_packed<3, true, 0, false>', 'k_project_tile<false, false>',
                     'k_project_tile<true, false>', 'k_step_uncovered<false>']
    assert K.iteration(three, 0.3)[0] == generic_whole
    interior = K.iteration(three, 0.3, K.Mode(strip=(16, 16)))
    assert interior == (['k_gradient_packed<3, true, 1, false>', 'k_fold_sums', 'k_project_tile<false, false>'], 3)
    last = K.iteration(three, 0.3, K.Mode(strip=(32, 16)))[0]
    assert last == generic_whole[:1] + ['k_fold_sums'] + generic_whole[1:]
    # the 1080p shape: only the last strip has luma rows missing; resample stays the whole frame's
    p1080 = (G(1920, 1080, 1, 1), G(960, 544, 2, 2), G(960, 544, 2, 2))
    assert K.iteration(p1080, 0.3, K.Mode(strip=(0, 144)))[0] == [
        'k_gradient_packed<3, true, 2, false>', 'k_fold_sums', 'k_project_tile<true, false>', 'k_project_tile22<false>']
    assert K.iteration(p1080, 0.3, K.Mode(strip=(944, 144)))[0] == [
        'k_gradient_packed<3, true, 2, false>', 'k_fold_sums', 'k_project_tile<true, false>', 'k_step_uncovered<false>',
        'k_project_tile22<false>']
    # chroma grid ending inside the last strip: k_step_uncovered22 there only
    short22 = (G(64, 48, 1, 1), G(32, 16, 2, 2), G(32, 16, 2, 2))
    assert 'k_step_uncovered22<false>' not in K.iteration(short22, 0.3, K.Mode(strip=(0, 16)))[0]
    assert K.iteration(short22, 0.3, K.Mode(strip=(16, 32)))[0].count('k_step_uncovered22<false>') == 2
    assert K.strip_rows(G(32, 16, 2, 2), 16, 32) == 8 and K.strip_rows(G(64, 1080, 1, 1), 1072, 16) == 8
