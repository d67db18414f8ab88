"""The staged GEMM epilogue (bf16 outputs written through shared memory with TMA stores) against the register epilogue.

The per-element arithmetic is the same on both paths, so every output must be bitwise equal.  VT_GEMM_STAGED_EPI=0
selects the register epilogue; vt_gemm reads it on every call.  The GPU tests are marked gpu; the SASS and ptxas checks
at the end need only nvcc / cuobjdump."""

import os
import re
import shutil
import subprocess
import tempfile

import pytest
import torch

BNS = [128, 192, 256]
FORMS = ['bf16']
SENTINEL = -12345.0


def lib():
    from videotransformer_pytorch_b200 import _lib
    return _lib


def mk(shape, seed, scale=1.0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).cuda()


def case(M, N, Kd, seed=0):
    a, b = mk((M, Kd), seed, 0.3).bfloat16(), mk((N, Kd), seed + 1, 0.3).bfloat16()
    return dict(a=a, b=b, bias=mk((N,), seed + 2), rs=mk((M,), seed + 3))


def run(form, c, M, N, Kd, bn, staged, monkeypatch, out=None):
    """the form's outputs, as a list of tensors"""
    monkeypatch.setenv('VT_GEMM_STAGED_EPI', '1' if staged else '0')
    return [lib().K.gemm(c['a'], c['b'], M, N, Kd, epi=form, bias=c['bias'], row_scale=c['rs'], force_bn=bn, out=out)]


def same(xs, ys):
    return len(xs) == len(ys) and all(torch.equal(x, y) for x, y in zip(xs, ys))


@pytest.mark.gpu
@pytest.mark.parametrize('bn', BNS)
@pytest.mark.parametrize('form', FORMS)
def test_staged_equals_register_on_edges(form, bn, monkeypatch):
    Kd = 136                                            # 3 k-blocks, the last one partial
    for M in (1, 127, 129, 12552):
        c = case(M, 2304, Kd, seed=M)
        for N in (8, 72, 200, 776, 2304):
            cn = dict(c, b=c['b'][:N].contiguous(), bias=c['bias'][:N].contiguous())
            reg = run(form, cn, M, N, Kd, bn, False, monkeypatch)
            stg = run(form, cn, M, N, Kd, bn, True, monkeypatch)
            assert same(reg, stg), (form, bn, M, N)


@pytest.mark.gpu
@pytest.mark.parametrize('bn', BNS)
@pytest.mark.parametrize('form', FORMS)
def test_guard_regions_keep_sentinel(form, bn, monkeypatch):
    """strided outputs (ldo > N) inside a larger sentinel buffer: padding columns and rows past M keep their bits"""
    M, N, Kd, PAD_C, PAD_R = 200, 200, 72, 56, 9
    c = case(M, N, Kd, seed=5)
    got = {}
    for staged in (False, True):
        buf = torch.full((M + PAD_R, N + PAD_C), SENTINEL, device='cuda').bfloat16()
        outs = run(form, c, M, N, Kd, bn, staged, monkeypatch, out=buf[:M, :N])
        bits = buf.view(torch.int16)
        sent = torch.full((), SENTINEL).bfloat16().view(torch.int16).item()
        assert bool((bits[:, N:] == sent).all()) and bool((bits[M:, :] == sent).all()), (form, bn, staged)
        got[staged] = [x.clone() for x in outs]
    assert same(got[False], got[True])


@pytest.mark.gpu
@pytest.mark.parametrize('bn', BNS)
@pytest.mark.parametrize('form', FORMS)
def test_staging_reuse_across_tiles_and_grids(form, bn, monkeypatch):
    """grids of every SM, one fewer and 64 fewer: each CTA reuses its staging buffers over several tiles"""
    M, N, Kd = 12552, 776, 200
    c = case(M, N, Kd, seed=11)
    reg = run(form, c, M, N, Kd, bn, False, monkeypatch)
    try:
        for reserve in (0, 1, 64):
            lib().set_reserved_sms(reserve)
            for _ in range(2):
                assert same(reg, run(form, c, M, N, Kd, bn, True, monkeypatch)), (form, bn, reserve)
    finally:
        lib().set_reserved_sms(0)


@pytest.mark.gpu
@pytest.mark.parametrize('form', FORMS)
def test_graph_replay_matches_eager(form, monkeypatch):
    M, N, Kd = 12552, 2304, 136
    c = case(M, N, Kd, seed=21)
    eager = run(form, c, M, N, Kd, 0, True, monkeypatch)
    outs = [torch.empty_like(x) for x in eager]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                        # warm-up outside the capture
        run(form, c, M, N, Kd, 0, True, monkeypatch, out=outs[0])
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run(form, c, M, N, Kd, 0, True, monkeypatch, out=outs[0])
    for x in outs:
        x.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert same(outs, eager)


def test_library_has_tma_stores():
    from videotransformer_pytorch_b200 import build
    if not shutil.which('cuobjdump'):
        pytest.skip('cuobjdump not found')
    sass = subprocess.run(['cuobjdump', '-sass', build.build()], capture_output=True, text=True).stdout
    assert 'UTMASTG' in sass and 'UTMALDG' in sass and 'HGMMA' in sass


def test_every_gemm_instantiation_compiles_without_spills():
    """ptxas -v for every GEMM instantiation: no spills, and no wgmma serialisation warning"""
    from videotransformer_pytorch_b200 import build
    try:
        nvcc = build.nvcc_path()
    except RuntimeError:
        pytest.skip('nvcc not found')
    src = os.path.join(build.CSRC, 'vt_gemm.cu')
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc, '-gencode', build.ARCH, '-O3', '-std=c++17', '-I', build.INCLUDE, '-DVT_BUILD', '-Xptxas', '-v', '-c',
               src, '-o', os.path.join(tmp, 'vt_gemm.o')]
        res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    assert 'serialized' not in log, log
    kernels = re.findall(r"Compiling entry function '(\w*gemm_wgmma_kernel\w*)'[^\n]*\n(?:[^\n]*\n)?[^\n]*?(\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", log)
    assert len(kernels) == 24, log
    spilling = [k for k, st, ld in kernels if int(st) or int(ld)]
    assert not spilling, spilling
