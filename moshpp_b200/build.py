"""In-tree build of libmosh2.so (nvcc, sm_90a only) and of the oracle-side helper libraries.

``python -m moshpp_b200.build`` or ``__graft_entry__.build()``.  nvcc cross-compiles without a GPU.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libmosh2.so')
EMU_SRC = os.path.join(ROOT, 'tests', 'emu', 'mosh2_emu.cpp')
EMU_LIB = os.path.join(ROOT, 'tests', 'emu', '_build', 'libmosh2_emu.so')
TC_SRC = os.path.join(ROOT, 'tests', 'tc', 'jtj_tf32_test.cu')
TC_BIN = os.path.join(ROOT, 'tests', 'tc', '_build', 'jtj_test')
GN_SRC = os.path.join(ROOT, 'tests', 'tc', 'gauss_newton_test.cu')
GN_LIB = os.path.join(ROOT, 'tests', 'tc', '_build', 'libgn_test.so')

NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '-shared', '-Xcompiler', '-fPIC']


def _stale(target: str, sources) -> bool:
    """A source that does not exist is no reason to rebuild: a test source tree without the Gauss-Newton harness still
    builds the host build, whose source then does not include the harness's header (if it did, the compiler says so)."""
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.exists(s) and os.path.getmtime(s) > t for s in sources)


def _nvcc() -> str:
    for cand in (shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found: libmosh2.so cannot be built (there is no CPU fallback)')


def build_library(force: bool = False, verbose: bool = False) -> str:
    srcs = [os.path.join(CSRC, "mosh2.cu"), os.path.join(CSRC, "mosh2_device.cuh"), os.path.join(CSRC, "mosh2_host.h"),
            os.path.join(CSRC, "mesh_distance.cuh"), os.path.join(ROOT, 'include', 'mosh2.h')]
    if force or _stale(LIB, srcs):
        cmd = [_nvcc()] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-o', LIB, srcs[0]]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed:\n' + r.stdout + r.stderr)
        if verbose:
            print(r.stdout + r.stderr)
    return LIB


def build_emu(force: bool = False) -> str:
    """TEST-ONLY single-thread host build of the CTA program (see tests/emu/mosh2_emu.cpp)."""
    srcs = [EMU_SRC, os.path.join(CSRC, "mosh2_device.cuh"), os.path.join(CSRC, "mosh2_host.h"), os.path.join(ROOT, 'include', 'mosh2.h'),
            os.path.join(ROOT, 'tests', 'tc', 'gauss_newton_case.h')]
    if force or _stale(EMU_LIB, srcs):
        os.makedirs(os.path.dirname(EMU_LIB), exist_ok=True)
        cmd = ['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-o', EMU_LIB, EMU_SRC]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('g++ failed:\n' + r.stdout + r.stderr)
    return EMU_LIB


def build_tc_test(force: bool = False) -> str:
    """TEST-ONLY stand-alone check of the split-TF32 J^T J building block (tests/tc/jtj_tf32_test.cu)."""
    if force or _stale(TC_BIN, [TC_SRC, os.path.join(CSRC, 'mosh2_device.cuh')]):
        os.makedirs(os.path.dirname(TC_BIN), exist_ok=True)
        cmd = [_nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O2', '-std=c++17', '-o', TC_BIN, TC_SRC]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed:\n' + r.stdout + r.stderr)
    return TC_BIN


def build_gn_test(force: bool = False) -> str:
    """TEST-ONLY stand-alone harness of the device Gauss-Newton solve (tests/tc/gauss_newton_test.cu), a shared library."""
    srcs = [GN_SRC, os.path.join(ROOT, 'tests', 'tc', 'gauss_newton_case.h'), os.path.join(CSRC, 'mosh2_device.cuh'),
            os.path.join(CSRC, 'mosh2_host.h'), os.path.join(ROOT, 'include', 'mosh2.h')]
    if force or _stale(GN_LIB, srcs):
        os.makedirs(os.path.dirname(GN_LIB), exist_ok=True)
        cmd = [_nvcc()] + NVCC_FLAGS + ['-o', GN_LIB, GN_SRC]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed:\n' + r.stdout + r.stderr)
    return GN_LIB


if __name__ == '__main__':
    print(build_library(force='--force' in sys.argv, verbose='-v' in sys.argv))
