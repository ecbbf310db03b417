"""oracle/build_ref.py -- compile the REFERENCE's own CUDA operators into oracle/_ref/ (build container only).

TEST INFRASTRUCTURE.  The sources are compiled where they lie under /root/reference (never copied):
  external/gridencoder/src/{gridencoder.cu,bindings.cpp}   -> oracle/_ref/_ref_gridencoder.so
  raymarching/src/{raymarching.cu,bindings.cpp}            -> oracle/_ref/_ref_raymarching.so
with the reference's own flags (`-O3 -U__CUDA_NO_HALF_*`, raymarching/backend.py:6-9) except the one-token
fix `-std=c++14` -> `-std=c++17` that torch >= 2.1 headers need (SURVEY.md §0.10), for sm_90a.

The resulting pybind modules are the "reference GPU build" of these operators.  They travel to the GPU box
with the repo snapshot (oracle/_ref/ is git-ignored, not gpurun-ignored) where tests/test_ref_cuda_gpu.py
checks (a) the C restatement in oracle/ngp_oracle.c and (b) our sm_90a kernels against them.
"""
from __future__ import annotations

import importlib.util
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, '_ref')
REF = '/root/reference'

MODULES = {
    '_ref_gridencoder': ['external/gridencoder/src/gridencoder.cu', 'external/gridencoder/src/bindings.cpp'],
    '_ref_raymarching': ['raymarching/src/raymarching.cu', 'raymarching/src/bindings.cpp'],
}


def so_path(name: str) -> str:
    return os.path.join(OUT, name + '.so')


def build(force: bool = False) -> None:
    if not os.path.isdir(REF):
        raise RuntimeError(f'{REF} is not present: oracle/_ref can only be built in the build container')
    os.environ.setdefault('TORCH_CUDA_ARCH_LIST', '9.0a')
    os.environ.setdefault('MAX_JOBS', '8')
    from torch.utils.cpp_extension import load
    nvcc = ['-O3', '-std=c++17', '-U__CUDA_NO_HALF_OPERATORS__', '-U__CUDA_NO_HALF_CONVERSIONS__', '-U__CUDA_NO_HALF2_OPERATORS__']
    for name, srcs in MODULES.items():
        if os.path.exists(so_path(name)) and not force:
            continue
        bdir = os.path.join(OUT, 'build_' + name)
        os.makedirs(bdir, exist_ok=True)
        load(name=name, sources=[os.path.join(REF, s) for s in srcs], extra_cflags=['-O3', '-std=c++17'], extra_cuda_cflags=nvcc,
             build_directory=bdir, is_python_module=False, verbose=False)
        os.replace(os.path.join(bdir, name + '.so'), so_path(name))
        print(f'[build_ref] {so_path(name)}')


def available() -> bool:
    return all(os.path.exists(so_path(n)) for n in MODULES)


def load_module(name: str):
    """import a prebuilt reference operator module (needs torch imported first: it links libtorch)"""
    import torch  # noqa: F401
    spec = importlib.util.spec_from_file_location(name, so_path(name))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == '__main__':
    build(force='--force' in sys.argv)
