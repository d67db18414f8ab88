"""The staged fp32 GEMM epilogue (gemm_f32_kernel: residual rows loaded and result rows stored by 1-D bulk copies) against
the register epilogue.

The per-element arithmetic is the same on both paths, so every output must be bitwise equal.  VT_GEMM_STAGED_EPI=0
selects the register epilogue; vt_gemm reads it on every call.  Outputs sit in sentinel-filled buffers, so a write to a
padding column, a row past M, a dropped row or one of the stream's cls rows shows.  Which kernel ran is read from
torch.profiler.  The GPU tests are marked gpu; the SASS and ptxas checks at the end need only nvcc / cuobjdump."""

import itertools
import os
import re
import shutil
import subprocess
import tempfile

import pytest
import torch

SENTINEL = -12345.0
MS = (1, 127, 129, 12552)
NS = (8, 72, 200, 776)


def lib():
    from videotransformer_pytorch_b200 import _lib
    return _lib


def mk(shape, seed, scale=1.0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).cuda()


def gemm(staged, monkeypatch, *args, **kw):
    monkeypatch.setenv('VT_GEMM_STAGED_EPI', '1' if staged else '0')
    return lib().K.gemm(*args, epi='f32', **kw)


def gemm_kernels(fn):
    """names of the GEMM kernels fn launches"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name for e in prof.events() if 'gemm_' in e.name and 'kernel' in e.name}


def both(fn, init):
    """fn(staged, out) on a fresh copy of init for each epilogue: (register result, staged result)"""
    res = []
    for staged in (False, True):
        buf = init.clone()
        fn(staged, buf)
        torch.cuda.synchronize()
        res.append(buf)
    return res


def bits_equal(x, y):
    return torch.equal(x.view(torch.int32), y.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize('bn', [0, 128, 192])
def test_plain_rows_every_addend_combination(bn, monkeypatch):
    """aux / bias / bias2 / row_scale in every combination (bias2 needs aux), strided output inside a sentinel buffer"""
    Kd, PAD_C, PAD_R = 136, 8, 5
    for M in MS:
        a = mk((M, Kd), M, 0.3).bfloat16()
        bfull = mk((max(NS), Kd), M + 1, 0.3).bfloat16()
        for N in NS:
            b = bfull[:N].contiguous()
            bias, bias2, rs = mk((N,), 2), mk((N,), 3), mk((M,), 4)
            aux = mk((M, N + 4), 5)[:, :N]                       # strided addend (ldaux = N + 4)
            for use_aux, use_bias, use_b2, use_rs in itertools.product((0, 1), repeat=4):
                if use_b2 and not use_aux:
                    continue
                kw = dict(aux=aux if use_aux else None, bias=bias if use_bias else None,
                          bias2=bias2 if use_b2 else None, row_scale=rs if use_rs else None, force_bn=bn)
                init = torch.full((M + PAD_R, N + PAD_C), SENTINEL, device='cuda')
                reg, stg = both(lambda s, buf: gemm(s, monkeypatch, a, b, M, N, Kd, out=buf[:M, :N], **kw), init)
                tag = (M, N, bn, use_aux, use_bias, use_b2, use_rs)
                assert bits_equal(reg, stg), tag
                assert bool((stg[:, N:] == SENTINEL).all()) and bool((stg[M:] == SENTINEL).all()), tag


@pytest.mark.gpu
def test_staged_kernel_runs_and_falls_back(monkeypatch):
    M, N, Kd = 300, 200, 72
    a, b, aux = mk((M, Kd), 1).bfloat16(), mk((N, Kd), 2).bfloat16(), mk((M, N), 3)
    ran = lambda staged, bn: gemm_kernels(lambda: gemm(staged, monkeypatch, a, b, M, N, Kd, aux=aux, force_bn=bn))
    assert any('gemm_f32_kernel' in k for k in ran(True, 128)), ran(True, 128)
    assert any('gemm_f32_kernel' in k for k in ran(True, 192))
    for staged, bn in ((False, 128), (True, 256)):          # the switch, and the tile width without a staged form
        ks = ran(staged, bn)
        assert ks and not any('gemm_f32_kernel' in k for k in ks), (staged, bn, ks)


@pytest.mark.gpu
def test_aux_is_out(monkeypatch):
    """the in-place residual add: the addend is the output itself"""
    for M, N in ((12552, 776), (129, 72)):
        Kd = 200
        a, b, bias = mk((M, Kd), 7, 0.3).bfloat16(), mk((N, Kd), 8, 0.3).bfloat16(), mk((N,), 9)
        init = mk((M, N), 10)
        reg, stg = both(lambda s, buf: gemm(s, monkeypatch, a, b, M, N, Kd, aux=buf, out=buf, bias=bias, bias2=bias), init)
        assert bits_equal(reg, stg), (M, N)


def affine_case(B, T, P, D, seed):
    from videotransformer_pytorch_b200 import ops
    S = 1 + P * T
    maps, aff = ops.token_maps(B, T, P, 'cuda'), ops.affine_row_maps(B, T, P, D)
    w = mk((D, D), seed, 0.05).bfloat16()
    stream = mk((B * S + B * T, D), seed + 1)
    return S, maps, aff, w, stream


@pytest.mark.gpu
@pytest.mark.parametrize('shape', [(8, 8, 196, 768), (3, 4, 9, 136), (2, 8, 196, 96)])
def test_affine_maps(shape, monkeypatch):
    """temporal and spatial regrouping of the residual stream in place; the spatial cls replicas go to the side rows and
    the stream's own cls rows are never written"""
    B, T, P, D = shape
    S, maps, aff, w, stream = affine_case(B, T, P, D, seed=D)
    bias, bias2 = mk((D,), 1), mk((D,), 2)
    for kind in ('temporal', 'spatial'):
        M = B * P * T if kind == 'temporal' else B * T * (P + 1)
        x = mk((M, D), 3, 0.5).bfloat16()
        rs = mk((M,), 4)
        rows = dict(aux_row=maps['temporal'], out_row=maps['temporal']) if kind == 'temporal' else \
            dict(aux_row=maps['sp_aux'], out_row=maps['sp_out'])
        for bn in (0, 128, 192):
            for extra in (dict(), dict(bias=bias, bias2=bias2, row_scale=rs)):
                def run(staged, buf):
                    gemm(staged, monkeypatch, x, w, M, D, D, aux=buf, out=buf, row_map=aff[kind], force_bn=bn, **rows,
                         **extra)
                reg, stg = both(run, stream)
                assert bits_equal(reg, stg), (shape, kind, bn, sorted(extra))
                cls = torch.arange(B, device='cuda') * S
                assert bits_equal(stg[cls], stream[cls]), (shape, kind, bn)
                if kind == 'temporal':
                    assert bits_equal(stg[B * S:], stream[B * S:]), (shape, bn)
        assert any('gemm_f32_kernel' in k for k in gemm_kernels(lambda: run(True, stream.clone())))


@pytest.mark.gpu
def test_unaligned_affine_map_falls_back(monkeypatch):
    """map offsets that are even but not multiples of 4 elements: 8-byte aligned rows, which the register epilogue
    handles and the bulk copies do not take"""
    B, T, P, D, W = 2, 4, 9, 136, 140
    S = 1 + P * T
    M = B * P * T
    rmap = dict(period=P * T, skip=0, tcount=1, stride_t=W, stride_p=W, stride_b=S * W, base=W + 2)
    x, w = mk((M, D), 1, 0.5).bfloat16(), mk((D, D), 2, 0.05).bfloat16()
    init = mk((B * S + 1, W), 3)
    rows = torch.arange(M, dtype=torch.int32, device='cuda')
    def run(staged, buf):
        gemm(staged, monkeypatch, x, w, M, D, D, aux=buf, out=buf, aux_row=rows, out_row=rows, row_map=rmap)
    assert not any('gemm_f32_kernel' in k for k in gemm_kernels(lambda: run(True, init.clone())))
    reg, stg = both(run, init)
    assert bits_equal(reg, stg)


@pytest.mark.gpu
@pytest.mark.parametrize('bn', [128, 192])
def test_index_maps_with_dropped_rows_and_missing_addends(bn, monkeypatch):
    """out_row / aux_row permutations with -1 entries: dropped rows write nothing, missing addends add zero"""
    for M, N in ((12552, 776), (129, 200), (1, 8)):
        Kd, R = 72, M + 40
        a, b = mk((M, Kd), M, 0.3).bfloat16(), mk((N, Kd), M + 1, 0.3).bfloat16()
        g = torch.Generator(device='cpu').manual_seed(M)
        out_row = torch.randperm(R, generator=g)[:M].int()
        aux_row = torch.randperm(M + 7, generator=g)[:M].int()
        out_row[torch.rand(M, generator=g) < 0.1] = -1
        aux_row[torch.rand(M, generator=g) < 0.1] = -1
        out_row, aux_row = out_row.cuda(), aux_row.cuda()
        aux = mk((M + 7, N), 5)
        for use_aux in (False, True):
            kw = dict(out_row=out_row, aux_row=aux_row if use_aux else None, aux=aux if use_aux else None,
                      bias=mk((N,), 6), row_scale=mk((M,), 7), force_bn=bn)
            init = torch.full((R, N), SENTINEL, device='cuda')
            reg, stg = both(lambda s, buf: gemm(s, monkeypatch, a, b, M, N, Kd, out=buf, out_rows=R, **kw), init)
            assert bits_equal(reg, stg), (M, N, bn, use_aux)
            untouched = torch.ones(R, dtype=torch.bool, device='cuda')
            untouched[out_row[out_row >= 0].long()] = False
            assert bool((stg[untouched] == SENTINEL).all()), (M, N, bn, use_aux)


@pytest.mark.gpu
@pytest.mark.parametrize('bn', [128, 192])
def test_split_k_partials(bn, monkeypatch):
    """weight-gradient form: MN-major operands, K split into the fp32 workspace and summed by reduce_rows; the partials
    take the staged rows at BN = 128 and the register epilogue at 192"""
    M, N, Kd = 776, 200, 12552
    a, b = mk((Kd, M), 1, 0.3).bfloat16(), mk((Kd, N), 2, 0.3).bfloat16()
    for splits in (2, 5):
        def run(staged, buf):
            gemm(staged, monkeypatch, a, b, M, N, Kd, a_mn=True, b_mn=True, out=buf, split_ok=True, force_splits=splits,
                 force_bn=bn)
        reg, stg = both(run, torch.full((M, N), SENTINEL, device='cuda'))
        assert bits_equal(reg, stg), (bn, splits)
        ks = gemm_kernels(lambda: run(True, stg))
        assert ks and any('gemm_f32_kernel' in k for k in ks) == (bn == 128), (bn, ks)


@pytest.mark.gpu
def test_staging_reuse_across_tiles_and_grids(monkeypatch):
    """grids of every SM, one fewer and 64 fewer: each CTA reuses its staging rows over many tiles"""
    B, T, P, D = 8, 8, 196, 768
    _, maps, aff, w, stream = affine_case(B, T, P, D, seed=31)
    M = B * P * T
    x, bias = mk((M, D), 3, 0.5).bfloat16(), mk((D,), 4)
    def run(staged, buf):
        gemm(staged, monkeypatch, x, w, M, D, D, aux=buf, out=buf, bias=bias, aux_row=maps['temporal'],
             out_row=maps['temporal'], row_map=aff['temporal'])
    reg, _ = both(run, stream)
    try:
        for reserve in (0, 1, 64):
            lib().set_reserved_sms(reserve)
            for _ in range(2):
                _, stg = both(run, stream)
                assert bits_equal(reg, stg), reserve
    finally:
        lib().set_reserved_sms(0)


@pytest.mark.gpu
def test_graph_replay_matches_eager(monkeypatch):
    M, N, Kd = 12552, 768, 3072
    a, b, bias = mk((M, Kd), 41, 0.1).bfloat16(), mk((N, Kd), 42, 0.1).bfloat16(), mk((N,), 43)
    aux = mk((M, N), 44)
    eager = gemm(True, monkeypatch, a, b, M, N, Kd, aux=aux, bias=bias)
    out = torch.empty_like(eager)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                        # warm-up outside the capture
        gemm(True, monkeypatch, a, b, M, N, Kd, aux=aux, bias=bias, out=out)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gemm(True, monkeypatch, a, b, M, N, Kd, aux=aux, bias=bias, out=out)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert bits_equal(out, eager)
    assert bits_equal(eager, gemm(False, monkeypatch, a, b, M, N, Kd, aux=aux, bias=bias))


def _sass_functions():
    from videotransformer_pytorch_b200 import build
    sass = subprocess.run(['cuobjdump', '-sass', build.build()], capture_output=True, text=True).stdout
    return {m.group(1): m.group(2) for m in re.finditer(r'Function : (\S+)\n(.*?)(?=\n\s+Function : |\Z)', sass, re.S)}


def test_staged_f32_sass_uses_bulk_copies():
    """the new kernels move rows with bulk copies (UBLKCP) and read no residual through generic 64-bit loads"""
    if not shutil.which('cuobjdump'):
        pytest.skip('cuobjdump not found')
    funcs = {k: v for k, v in _sass_functions().items() if 'gemm_f32_kernel' in k}
    assert len(funcs) == 8, sorted(funcs)            # BN 128 / 192 x four operand layouts
    for name, body in funcs.items():
        assert 'UBLKCP.S.G' in body and 'UBLKCP.G.S' in body, name
        assert not re.search(r'\bLD\.E\.64\b', body) and not re.search(r'\bST\.E\.64\b', body), name


def test_staged_f32_kernels_do_not_spill():
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
    kernels = re.findall(r"Compiling entry function '(\w*(?:gemm_f32_kernel|gemm_e4m3_kernel)\w*)'[^\n]*\n(?:[^\n]*\n)?"
                         r"[^\n]*?(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(kernels) == 8 + 3, log
    spilling = [k for k, st, ld in kernels if int(st) or int(ld)]
    assert not spilling, spilling
