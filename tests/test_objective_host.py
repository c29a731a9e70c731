"""Without a GPU: the CSV format of write_objective_csv on fixed numbers (NaN and infinity as glibc
prints them), return_objective's argument check, and that every kernel of libj2pobjective.so is
reached by a named case of tests/test_gpu_objective.py (tests/objective_cases.py)."""
import io
import os
import re
import shutil
import subprocess

import pytest
import torch

import jpeg2png_b200
from tests.objective_cases import CASES, kernels_reached

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'jpeg2png_b200', 'objective', 'libj2pobjective.so')
MAIN = os.path.join(ROOT, 'jpeg2png_b200', 'csrc', 'libjpeg2png_b200.so')


def _csv(names, logs):
    buf = io.StringIO()
    jpeg2png_b200.write_objective_csv(buf, names, logs)
    return buf.getvalue()


def test_csv_format_pinned():
    nan, inf = float('nan'), float('inf')
    logs = [{3: torch.tensor([[1.0, 0.0, 2.5, 0.125], [1234567.8912345, 1e-7, 5e-7, 0.0000015]], dtype=torch.float64)},
            {2: torch.tensor([[nan, -nan, inf, -inf]], dtype=torch.float64),
             0: torch.tensor([[-0.0, -1.5, 3.0, 1e20]], dtype=torch.float64)}]
    assert _csv(['a.jpg', 'dir/b.jpeg'], logs) == (
        'filename,channel,iteration,objective,prob_dist,tv,tv2\n'
        'a.jpg,3,0,1.000000,0.000000,2.500000,0.125000\n'
        'a.jpg,3,1,1234567.891235,0.000000,0.000000,0.000002\n'
        'dir/b.jpeg,0,0,-0.000000,-1.500000,3.000000,100000000000000000000.000000\n'
        'dir/b.jpeg,2,0,nan,-nan,inf,-inf\n')


def test_csv_to_a_path_and_empty_logs(tmp_path):
    p = tmp_path / 'log.csv'
    jpeg2png_b200.write_objective_csv(p, ['x'], [{3: torch.zeros((0, 4), dtype=torch.float64)}])
    assert p.read_text() == 'filename,channel,iteration,objective,prob_dist,tv,tv2\n'
    with pytest.raises(ValueError):
        jpeg2png_b200.write_objective_csv(p, ['x', 'y'], [{}])


def test_return_objective_is_checked_before_any_device_work():
    from jpeg2png_b200 import decode_jpeg
    for bad in (1, None, 'True'):
        with pytest.raises(ValueError, match='return_objective'):
            decode_jpeg(b'', return_objective=bad)


def _kernels(path):
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(cuobjdump) or not os.path.exists(path):
        pytest.skip('cuobjdump or the built library is missing (run __graft_entry__.build())')
    filt = os.path.join(os.path.dirname(cuobjdump), 'cu++filt')
    out = subprocess.run([cuobjdump, '-sass', path], check=True, capture_output=True, text=True).stdout
    names = re.findall(r'Function : (\S+)', out)
    dem = subprocess.run([filt], input='\n'.join(names), check=True, capture_output=True, text=True).stdout.split('\n')
    return {_short(d) for d in dem if d}


def _short(demangled):
    """'void j2p::k<(int)3, (bool)1>(args)' -> 'k<3, true>'"""
    name = re.sub(r'^(void )?j2p::', '', demangled)
    name = name[:name.index('>(') + 1] if '>(' in name else name.split('(')[0]
    name = re.sub(r'\(bool\)1', 'true', re.sub(r'\(bool\)0', 'false', name))
    return re.sub(r'\(int\)', '', name)


def test_every_recording_kernel_is_reached_by_a_named_case():
    lib = _kernels(LIB)
    reached = set(kernels_reached())
    assert sorted(lib - reached) == [], 'kernels no case reaches'
    assert sorted(reached - lib) == [], 'cases name kernels the library lacks'
    assert len(lib) == 20


def test_the_solver_library_has_no_recording_kernel():
    assert not [k for k in _kernels(MAIN) if '_rec' in k]


def test_case_ids_cover_the_settings_the_issue_names():
    assert any(c[2] == 0.0 for c in CASES.values())                    # weight 0: tv2 exactly 0
    assert any(0.0 in c[3] for c in CASES.values())                    # a plane with pweight 0
    assert {len(c[1]) for c in CASES.values()} == {1, 2, 3}
