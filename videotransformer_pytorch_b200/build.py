"""In-tree build of libvt_b200.so (hand-written sm_90a kernels + C ABI) with nvcc.

    python -m videotransformer_pytorch_b200.build [--force] [--verbose]

The shared library is written next to this file (git-ignored).  nvcc cross-compiles for sm_90a (H100) without a GPU.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
INCLUDE = os.path.join(os.path.dirname(HERE), 'include')
LIB = os.path.join(HERE, 'libvt_b200.so')
STAMP = os.path.join(HERE, '.libvt_b200.stamp')
ARCH = 'arch=compute_90a,code=sm_90a'


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cu'))


def _digest():
    h = hashlib.sha256(ARCH.encode())
    files = sources() + sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cuh'))
    files += sorted(os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE) if f.endswith('.h'))
    for f in files:
        h.update(f.encode())
        with open(f, 'rb') as fh:
            h.update(fh.read())
    return h.hexdigest()


def nvcc_path():
    for c in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if c and os.path.exists(c):
            return c
    raise RuntimeError('nvcc not found')


def build(force: bool = False, verbose: bool = False) -> str:
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP):
        with open(STAMP) as fh:
            if fh.read().strip() == dig:
                return LIB
    objs = []
    flags = ['-gencode', ARCH, '-O3', '-lineinfo', '-std=c++17',
             '-Xcompiler', '-fPIC', '-I', INCLUDE, '--use_fast_math' if False else '-DVT_BUILD']
    if verbose:
        flags += ['-Xptxas', '-v']
    procs = []
    for src in sources():
        obj = os.path.join(HERE, 'build', os.path.basename(src)[:-3] + '.o')
        os.makedirs(os.path.dirname(obj), exist_ok=True)
        cmd = [nvcc_path()] + flags + ['-c', src, '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            failed = True
            sys.stderr.write(f'--- nvcc failed for {src}\n{out}\n')
        elif verbose or out.strip():
            sys.stderr.write(out)
    if failed:
        raise RuntimeError('nvcc compilation failed')
    cmd = [nvcc_path(), '-shared', '-o', LIB] + objs + ['-gencode', ARCH]
    subprocess.check_call(cmd)
    with open(STAMP, 'w') as fh:
        fh.write(dig)
    return LIB


if __name__ == '__main__':
    path = build(force='--force' in sys.argv, verbose='--verbose' in sys.argv)
    print(path)
