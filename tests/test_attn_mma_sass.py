"""Compiler-side checks of the tensor-core attention kernels (csrc/vt_attention_mma.cu); they need nvcc / cuobjdump, no GPU.
Every instantiation loads its tiles with cp.async (LDGSTS) and its MMA fragments with ldmatrix (LDSM), none spills, and
the head-dim-64 dK / dV kernel keeps the three CTAs per SM it is launched for."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

KERNELS = ('attn_mma_fwd_kernel', 'attn_mma_dq_kernel', 'attn_mma_dkv_kernel')


def test_attention_kernels_use_cp_async_and_ldmatrix():
    from videotransformer_pytorch_b200 import build
    if not shutil.which('cuobjdump'):
        pytest.skip('cuobjdump not found')
    sass = subprocess.run(['cuobjdump', '-sass', build.build()], capture_output=True, text=True).stdout
    funcs = re.split(r'\n\s*Function : ', sass)
    found = {}
    for f in funcs:
        name = f.split('\n', 1)[0]
        for k in KERNELS:
            if k in name:
                found[name] = f
    assert len(found) == 8, sorted(found)      # fwd x {64, 96} x {lse, no lse}, dq x 2, dkv x 2
    for name, body in found.items():
        assert 'LDGSTS' in body, name
        assert 'LDSM' in body, name
        assert 'HMMA' in body, name


@pytest.fixture(scope='module')
def ptxas_stats():
    """{kernel: (spill store bytes, spill load bytes, registers)} of the tiled kernels, from ptxas -v"""
    from videotransformer_pytorch_b200 import build
    try:
        nvcc = build.nvcc_path()
    except RuntimeError:
        pytest.skip('nvcc not found')
    src = os.path.join(build.CSRC, 'vt_attention_mma.cu')
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc, '-gencode', build.ARCH, '-O3', '-std=c++17', '-I', build.INCLUDE, '-DVT_BUILD', '-Xptxas', '-v', '-c',
               src, '-o', os.path.join(tmp, 'vt_attention_mma.o')]
        res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    kernels = re.findall(r"Compiling entry function '(\w*attn_mma_\w*)'[^\n]*\n(?:[^\n]*\n)?[^\n]*?(\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads[^\n]*\n[^\n]*Used (\d+) registers", log)
    assert len(kernels) == 8, log
    return {k: (int(st), int(ld), int(regs)) for k, st, ld, regs in kernels}


def test_attention_kernels_do_not_spill(ptxas_stats):
    spilling = [k for k, (st, ld, _) in ptxas_stats.items() if st or ld]
    assert not spilling, spilling


def test_dkv_kernel_hd64_keeps_three_ctas_per_sm(ptxas_stats):
    """__launch_bounds__(128, 3): three CTAs of 128 threads share the 64K-register file, registers allocated per thread
    in multiples of 8"""
    (name, (_, _, regs)), = [(k, v) for k, v in ptxas_stats.items() if 'attn_mma_dkv_kernelILi64' in k]
    assert 3 * 128 * (-(-regs // 8) * 8) <= 65536, (name, regs)
