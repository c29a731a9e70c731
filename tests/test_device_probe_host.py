"""The device probe of tests/test_gpu_device_arith.py (tests/device_probe/libj2pprobe.so) is built
and complete, and it is compiled the way the solver is: the same architecture and the same
floating-point flags as jpeg2png_b200/csrc/Makefile.  A probe built with other flags would check
other arithmetic than the kernels run, and pass without meaning it."""
import ctypes as C
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE_DIR = os.path.join(ROOT, 'tests', 'device_probe')
SOLVER_MAKEFILE = os.path.join(ROOT, 'jpeg2png_b200', 'csrc', 'Makefile')

ENTRY_POINTS = ('probe_ieee', 'probe_guards', 'probe_constants', 'probe_roots', 'probe_div', 'probe_grad_div', 'probe_dct',
                'probe_stepper', 'probe_jo_tables', 'probe_pg_nth', 'probe_pg_nth_host', 'probe_ent_word', 'probe_ent_word_host',
                'probe_last_error')

# the flags that decide what the arithmetic computes
FP_FLAG = re.compile(r'^(-fmad=|-prec-div=|-prec-sqrt=|-ftz=|--use_fast_math$|-use_fast_math$|--fmad=|--prec-div=|--prec-sqrt=|--ftz=)')


def make_vars(path):
    """name -> value of a Makefile's simple assignments, continuation lines joined, $(NAME) expanded."""
    text = open(path).read().replace('\\\n', ' ')
    raw = {}
    for line in text.splitlines():
        m = re.match(r'^([A-Za-z_][A-Za-z0-9_]*)\s*(\?=|:=|=)\s*(.*)$', line)
        if m and not line.startswith('\t'):
            raw[m.group(1)] = m.group(3).strip()

    def expand(v, depth=0):
        assert depth < 20, path
        return re.sub(r'\$\(([A-Za-z_][A-Za-z0-9_]*)\)', lambda m: expand(raw.get(m.group(1), ''), depth + 1), v)
    return {k: expand(v) for k, v in raw.items()}


def compile_flags(path):
    v = make_vars(path)
    tokens = v['NVFLAGS'].split()
    host = [t for i, t in enumerate(tokens) if i and tokens[i - 1] == '-Xcompiler']
    return {'arch': v['ARCH'].split(), 'fp': sorted(t for t in tokens if FP_FLAG.match(t)),
            'host contraction': sorted(f for h in host for f in h.split(',') if f.startswith('-ffp-contract'))}


def test_probe_library_is_built_and_exports_every_entry_point():
    path = os.path.join(PROBE_DIR, 'libj2pprobe.so')
    assert os.path.exists(path), 'build() did not build the device probe'
    lib = C.CDLL(path)
    missing = [name for name in ENTRY_POINTS if not hasattr(lib, name)]
    assert not missing, missing


def test_probe_is_compiled_with_the_solvers_arch_and_floating_point_flags():
    solver, probe = compile_flags(SOLVER_MAKEFILE), compile_flags(os.path.join(PROBE_DIR, 'Makefile'))
    assert solver['arch'] == ['-gencode', 'arch=compute_90a,code=sm_90a']
    assert solver['fp'] == sorted(['-fmad=false', '-prec-div=true', '-prec-sqrt=true', '-ftz=false']), solver['fp']
    assert probe == solver, f'the probe is built with {probe}, the solver with {solver}'


def test_probe_recipe_uses_those_flags():
    """The rule that links libj2pprobe.so passes NVFLAGS, so the flags compared above are the ones used."""
    text = open(os.path.join(PROBE_DIR, 'Makefile')).read()
    rule = re.search(r'^libj2pprobe\.so:.*\n\t(.*)$', text, re.M)
    assert rule and '$(NVFLAGS)' in rule.group(1).split(), rule and rule.group(1)
