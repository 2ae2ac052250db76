"""In-tree build of libdiffsbdd_b200.so with nvcc for sm_90a (no torch dependency in the library).

The built .so stays next to this file (git-ignored); a stamp of the sources and flags it was built from sits in csrc/."""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB_NAME = 'libdiffsbdd_b200.so'
LIB_PATH = os.path.join(HERE, LIB_NAME)
SOURCES = ['dsb_api.cu', 'dsb_node.cu', 'dsb_edge.cu', 'dsb_tc.cu']
HEADERS = [os.path.join(CSRC, 'dsb_internal.cuh'), os.path.join(CSRC, 'dsb_tc.cuh'), os.path.join(CSRC, 'dsb_wgmma.cuh'),
           os.path.join(HERE, '..', 'include', 'diffsbdd_b200.h')]
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
NVCC_FLAGS = ARCH + ['-lineinfo', '-O3', '-std=c++20', '-Xcompiler', '-fPIC', '-Wno-deprecated-gpu-targets']
STAMP = os.path.join(CSRC, '.build_stamp')


def _nvcc() -> str:
    for cand in (shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found: cannot build libdiffsbdd_b200.so')


def _digest() -> str:
    h = hashlib.sha256()
    for p in [os.path.join(CSRC, s) for s in SOURCES] + HEADERS:
        with open(p, 'rb') as f:
            h.update(f.read())
    h.update(' '.join(NVCC_FLAGS).encode())
    return h.hexdigest()


def is_current() -> bool:
    """True when the library on disk was built from exactly the sources (and flags) next to it."""
    if not (os.path.exists(LIB_PATH) and os.path.exists(STAMP)):
        return False
    with open(STAMP) as f:
        return f.read().strip() == _digest()


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every CUDA translation unit for sm_90a and link the shared library. Returns its path."""
    dig = _digest()
    if not force and is_current():
        return LIB_PATH
    nvcc = _nvcc()
    objdir = os.path.join(CSRC, 'build')
    os.makedirs(objdir, exist_ok=True)
    procs = []
    objs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace('.cu', '.o'))
        objs.append(obj)
        cmd = [nvcc] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', os.path.join(CSRC, src), '-o', obj]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose and out:
            print(out, file=sys.stderr)
        if p.returncode != 0:
            raise RuntimeError('nvcc failed: %s\n%s' % (' '.join(cmd), out))
    cmd = [nvcc, '-shared'] + ARCH + ['-Wno-deprecated-gpu-targets', '-o', LIB_PATH] + objs
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed: %s\n%s' % (' '.join(cmd), r.stdout))
    with open(STAMP, 'w') as f:
        f.write(dig)
    return LIB_PATH


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
