"""Build libsparsefusion_b200.so (the C-ABI library, include/sparsefusion_b200.h) for sm_90a (H100), in tree.

    python -m sparsefusion_b200.build [--force] [--verbose]

Plain nvcc, no torch headers: the library has no torch types in its ABI.  Objects are cached under
sparsefusion_b200/csrc/_obj and rebuilt by mtime or when the flags change.  nvcc cross-compiles without a GPU.
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(CSRC, '_obj')
LIB = os.path.join(HERE, 'libsparsefusion_b200.so')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
FLAGS = ['-O3', '-std=c++17', '-lineinfo', '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr', '-Xptxas', '-v']


def _deps_mtime():
    hdrs = glob.glob(os.path.join(CSRC, '*.cuh')) + glob.glob(os.path.join(CSRC, '*.h')) + \
        glob.glob(os.path.join(os.path.dirname(HERE), 'include', '*.h'))
    return max(os.path.getmtime(h) for h in hdrs) if hdrs else 0.0


def _compile(src: str, force: bool, verbose: bool) -> str:
    obj = os.path.join(OBJ, os.path.basename(src)[:-3] + '.o')
    newest = max(os.path.getmtime(src), _deps_mtime())
    if not force and os.path.exists(obj) and os.path.getmtime(obj) >= newest:
        return obj
    cmd = [NVCC, *ARCH, *FLAGS, '-c', src, '-o', obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log = os.path.join(OBJ, os.path.basename(src)[:-3] + '.ptxas.log')
    with open(log, 'w') as f:
        f.write(r.stderr)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError(f'nvcc failed on {src}')
    if verbose:
        sys.stderr.write(r.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    # objects compiled with other flags (another architecture) are stale whatever their mtime
    stamp, flags = os.path.join(OBJ, 'flags'), ' '.join([NVCC, *ARCH, *FLAGS])
    if not os.path.exists(stamp) or open(stamp).read() != flags:
        force = True
        with open(stamp, 'w') as f:
            f.write(flags)
    srcs = sorted(glob.glob(os.path.join(CSRC, '*.cu')))
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, force, verbose), srcs))
    if force or not os.path.exists(LIB) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs):
        cmd = [NVCC, *ARCH, '-shared', '-o', LIB, *objs, '-lcudart']
        subprocess.check_call(cmd)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='--verbose' in sys.argv))
