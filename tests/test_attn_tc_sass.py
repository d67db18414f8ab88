"""Compiler-side checks of the tensor-core attention kernels at head widths 32 and 128 (attn_tc_*, the bodies of
attn_mma_* under their own names, csrc/vt_attention_mma.cu); they need nvcc / cuobjdump, no GPU.  Each loads its tiles
with cp.async and its fragments with ldmatrix, none spills, and the width-32 dK / dV kernel keeps four CTAs per SM."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

KERNELS = ('attn_tc_fwd_kernel', 'attn_tc_dq_kernel', 'attn_tc_dkv_kernel')


def test_head_width_kernels_use_cp_async_and_ldmatrix():
    from videotransformer_pytorch_b200 import build
    if not shutil.which('cuobjdump'):
        pytest.skip('cuobjdump not found')
    sass = subprocess.run(['cuobjdump', '-sass', build.build()], capture_output=True, text=True).stdout
    found = {}
    for f in re.split(r'\n\s*Function : ', sass):
        name = f.split('\n', 1)[0]
        if any(k in name for k in KERNELS):
            found[name] = f
    assert len(found) == 8, sorted(found)      # fwd x {32, 128} x {lse, no lse}, dq x 2, dkv x 2
    for name, body in found.items():
        assert 'LDGSTS' in body and 'LDSM' in body and 'HMMA' in body, name


@pytest.fixture(scope='module')
def ptxas_stats():
    """{kernel: (spill store bytes, spill load bytes, registers)} of the attn_tc_* kernels, from ptxas -v"""
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
    kernels = re.findall(r"Compiling entry function '(\w*attn_tc_\w*)'[^\n]*\n(?:[^\n]*\n)?[^\n]*?(\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads[^\n]*\n[^\n]*Used (\d+) registers", log)
    assert len(kernels) == 8, log
    return {k: (int(st), int(ld), int(regs)) for k, st, ld, regs in kernels}


def test_head_width_kernels_do_not_spill(ptxas_stats):
    spilling = [k for k, (st, ld, _) in ptxas_stats.items() if st or ld]
    assert not spilling, spilling


def test_dkv_kernel_hd32_keeps_four_ctas_per_sm(ptxas_stats):
    (name, (_, _, regs)), = [(k, v) for k, v in ptxas_stats.items() if 'attn_tc_dkv_kernelILi32' in k]
    assert 4 * 128 * (-(-regs // 8) * 8) <= 65536, (name, regs)
