#!/usr/bin/env python
"""sass_diff.py — compare the SASS of two builds of a shared object, kernel by kernel.

    python tools/sass_diff.py OLD.so NEW.so

Runs `cuobjdump -sass` on both, keeps each function's instruction text (addresses and encodings
dropped, so line info does not count), normalises constant-bank parameter offsets, and prints the
kernels that exist in one build only or whose instructions differ.  Exit status 0 when every kernel
is identical.  Needs the CUDA toolkit only, no GPU.
"""
import re
import shutil
import subprocess
import sys


def kernels(path):
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    out = subprocess.run([cuobjdump, '-sass', path], check=True, capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r'\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;', line)
        if m and cur is not None:
            cur.append(re.sub(r'c\[0x0\]\[0x[0-9a-f]+\]', 'c[0x0][PARAM]', m.group(1)))
    return funcs


def main():
    if len(sys.argv) != 3:
        raise SystemExit(__doc__)
    a, b = kernels(sys.argv[1]), kernels(sys.argv[2])
    only = sorted(set(a) ^ set(b))
    differ = sorted(k for k in set(a) & set(b) if a[k] != b[k])
    for k in only:
        print('only in', sys.argv[1] if k in a else sys.argv[2], k)
    for k in differ:
        print('differs', k)
    print(f'{len(set(a) & set(b))} kernels in both, {len(differ)} differ, {len(only)} in one build only')
    sys.exit(1 if only or differ else 0)


if __name__ == '__main__':
    main()
