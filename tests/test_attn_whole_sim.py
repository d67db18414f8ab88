"""CPU walk-through of the whole-problem attention kernels (attn_whole_fwd_kernel / attn_whole_bwd_kernel in
csrc/vt_attention_mma.cu), no GPU needed.

1. The swizzled operands: every ldmatrix lane address the kernels form (sw_at with the lane's row offset and chunk key) is
   followed through the ldmatrix model of test_attn_fragments_sim on a [R][64] tile stored with the 16-byte chunk c of
   row r at chunk c ^ (r & 7), and the registers it delivers are compared with the mma.m16n8k16 fragments of the logical
   matrix, for every (row block, k chunk, n block) the kernels visit at N = 256.  The 8 rows of each phase fall in distinct
   bank groups and every address lies inside the rows the kernels allocate.
2. The task -> rows maps at every N in 33..256 (and the small N the tensor-core implementation takes by name): forward
   warps x rounds and backward tasks cover every output row exactly once, every row the walks read is allocated (and
   zero-filled past N), the row stats cover every index the dK / dV walk reads, and two CTAs share an SM at N = 197.
3. The SASS of the new kernels: cp.async (LDGSTS), ldmatrix (LDSM), tensor-core MMAs, and no local-memory spills.
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from tests.test_attn_fragments_sim import LANES, a_frag, b_frag, ldsm_x4

HD = 64
MT = 64
WF_WARPS, WB_WARPS = 8, 6
SMEM_PER_SM = 228 * 1024          # H100: shared memory per SM, of which 1 KB per CTA is reserved
SMEM_RESERVED = 1024


def swz(r, c):
    return r * 64 + ((c ^ (r & 7)) << 3)


def sw_at(row, key, r0, c0):
    return row + r0 * 64 + (((c0 >> 3) ^ key) << 3)


def lane_a(lane):
    """(row offset, key) of lane_a in swizzled form"""
    return (lane & 15) * HD, (lane >> 4) ^ (lane & 7)


def lane_b(lane):
    return ((lane & 7) + (lane >> 4) * 8) * HD, ((lane >> 3) & 1) ^ (lane & 7)


def swizzled_tile(R, M):
    """flat [R * 64] shared-memory image of the logical matrix M[r][c] in the swizzled layout"""
    flat = [None] * (R * 64)
    for r in range(R):
        for c in range(64):
            flat[swz(r, c >> 3) + (c & 7)] = M(r, c)
    return flat


def check_phase(R, addr):
    for j in range(4):
        offs = [addr(8 * j + i) for i in range(8)]
        for o in offs:
            assert o % 8 == 0 and 0 <= o and o + 8 <= R * 64          # 16-byte aligned, inside the allocated rows
        assert len({(o // 8) % 8 for o in offs}) == 8                # distinct 16-byte bank groups: no conflicts


def test_swizzle_is_a_permutation_of_each_row():
    for r in range(16):
        assert sorted(swz(r, c) - r * 64 for c in range(8)) == [8 * c for c in range(8)]


def test_swizzled_a_fragments():
    """Q, dO (forward, dQ) and K, V (dK / dV) as A operands at (rb, kc * 16)"""
    R = 256
    M = lambda r, c: (r, c)
    tile = swizzled_tile(R, M)
    for rb in range(0, R, 16):
        for kc in range(HD // 16):
            addr = lambda lane: sw_at(*lane_a(lane), rb, kc * 16)
            check_phase(R, addr)
            regs = ldsm_x4(tile, 64, addr, trans=False)
            for lane in LANES:
                assert regs[lane] == a_frag(M, rb, kc * 16, lane)


def test_swizzled_b_fragments_row_operand():
    """B[k][n] = T[n][k] (K in S, V in dP, Q and dO in S^T / dP^T) at (k0 + nb * 8, kc * 16) -> n blocks nb, nb + 1"""
    R = 256
    tile = swizzled_tile(R, lambda r, c: (r, c))
    B = lambda k, n: (n, k)
    for n0 in range(0, R, 16):
        for kc in range(HD // 16):
            addr = lambda lane: sw_at(*lane_b(lane), n0, kc * 16)
            check_phase(R, addr)
            regs = ldsm_x4(tile, 64, addr, trans=False)
            for lane in LANES:
                assert regs[lane][:2] == b_frag(B, kc * 16, n0, lane)
                assert regs[lane][2:] == b_frag(B, kc * 16, n0 + 8, lane)


def test_swizzled_b_fragments_trans():
    """B[k][n] = T[k][n] (V in P V, K in dS K, dO in dV, Q in dK) with .trans at (k0 + kc * 16, nb * 8)"""
    R = 256
    tile = swizzled_tile(R, lambda r, c: (r, c))
    B = lambda k, n: (k, n)
    for k0 in range(0, R, 16):
        for nb in range(0, HD // 8, 2):
            addr = lambda lane: sw_at(*lane_a(lane), k0, nb * 8)
            check_phase(R, addr)
            regs = ldsm_x4(tile, 64, addr, trans=True)
            for lane in LANES:
                assert regs[lane][:2] == b_frag(B, k0, nb * 8, lane)
                assert regs[lane][2:] == b_frag(B, k0, nb * 8 + 8, lane)


# ---- 2. task -> rows maps ----------------------------------------------------------------------------------------------
def tile_walk_rows(N, rb):
    """rows of the resident operands one 16-row group reads over the 64-row tile walk (S / dP: the n8 pairs that hold a
    valid row; second product: the k16 chunks that hold one), and the stats indices of the dK / dV walk"""
    rows, stats = set(), set()
    rows.update(range(rb, rb + 16))
    for k0 in range(0, N, MT):
        for nb in range(0, 8, 2):
            if k0 + nb * 8 >= N:
                break
            rows.update(range(k0 + nb * 8, k0 + nb * 8 + 16))
        for kc in range(4):
            if k0 + kc * 16 >= N:
                break
            rows.update(range(k0 + kc * 16, k0 + kc * 16 + 16))
        stats.update(k0 + nb * 8 + 2 * t + e for nb in range(8) for t in range(4) for e in range(2))
    return rows, stats


SIZES = list(range(1, 33, 8)) + list(range(33, 257))


@pytest.mark.parametrize('N', SIZES)
def test_forward_groups(N):
    R = (N + 15) & ~15
    rounds = (R // 16 + WF_WARPS - 1) // WF_WARPS
    written = []
    for rnd in range(rounds):
        for warp in range(WF_WARPS):
            rb = (rnd * WF_WARPS + warp) * 16
            if rb >= N:
                continue
            written += [r for r in range(rb, rb + 16) if r < N]
            rows, _ = tile_walk_rows(N, rb)
            assert max(rows) < R                                     # allocated; rows >= N are the zero-filled ones
    assert sorted(written) == list(range(N))
    # the barrier after the second group: every thread passes it once in round 0 when there are keys past 64
    assert (N > MT) == any(k0 == MT for k0 in range(0, N, MT))


@pytest.mark.parametrize('N', SIZES)
def test_backward_tasks(N):
    R = (N + 15) & ~15
    R64 = (N + MT - 1) & ~(MT - 1)
    dq, dkv = [], []
    for task in range(0, 2 * R, 16):                                 # the counter's values, times 16
        if task < R:
            dkv += [r for r in range(task, task + 16) if r < N]
            rb = task
        else:
            dq += [r for r in range(task - R, task - R + 16) if r < N]
            rb = task - R
        rows, stats = tile_walk_rows(N, rb)
        assert max(rows) < R
        assert max(stats) < R64                                      # lse = +inf, delta = 0 there
    assert sorted(dq) == list(range(N)) and sorted(dkv) == list(range(N))
    # the stats pass: pairs of threads over rows [0, R64), each row once
    seen = [r0 + tid // 2 for r0 in range(0, R64, WB_WARPS * 16) for tid in range(0, WB_WARPS * 32, 2) if r0 + tid // 2 < R64]
    assert sorted(seen) == list(range(R64))


def test_two_ctas_per_sm_at_the_spatial_shape():
    N = 197
    R, R64 = (N + 15) & ~15, (N + MT - 1) & ~(MT - 1)
    fwd = 3 * R * HD * 2
    bwd = 4 * R * HD * 2 + 2 * R64 * 4 + 16                          # + the task counter
    for smem in (fwd, bwd):
        assert 2 * (smem + SMEM_RESERVED) <= SMEM_PER_SM, smem


# ---- 3. SASS -------------------------------------------------------------------------------------------------------------
def _compile(tmp, extra):
    from videotransformer_pytorch_b200 import build
    src = os.path.join(build.CSRC, 'vt_attention_mma.cu')
    obj = os.path.join(tmp, 'vt_attention_mma.o')
    cmd = [build.nvcc_path(), '-gencode', build.ARCH, '-O3', '-std=c++17', '-I', build.INCLUDE, '-DVT_BUILD', *extra, '-c', src,
           '-o', obj]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return obj, res.stdout + res.stderr


def test_whole_kernels_sass_and_registers():
    from videotransformer_pytorch_b200 import build
    try:
        build.nvcc_path()
    except RuntimeError:
        pytest.skip('nvcc not found')
    if not shutil.which('cuobjdump'):
        pytest.skip('cuobjdump not found')
    with tempfile.TemporaryDirectory() as tmp:
        obj, log = _compile(tmp, ['-Xptxas', '-v'])
        sass = subprocess.run(['cuobjdump', '-sass', obj], capture_output=True, text=True).stdout
    stats = re.findall(r"Compiling entry function '(\w*attn_whole_\w*)'[^\n]*\n(?:[^\n]*\n)?[^\n]*?(\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads[^\n]*\n[^\n]*Used (\d+) registers", log)
    assert len(stats) == 3, log                                      # forward with / without lse, backward
    for name, st, ld, regs in stats:
        assert int(st) == 0 and int(ld) == 0, (name, st, ld)
        # two CTAs per SM: 2 x 256 threads (forward) or 2 x 192 (backward) within the 64K-register file
        threads = 192 if 'bwd' in name else 256
        assert 2 * threads * int(regs) <= 65536, (name, regs)
    funcs = {f.split('\n', 1)[0]: f for f in re.split(r'\n\s*Function : ', sass)}
    found = {n: b for n, b in funcs.items() if 'attn_whole_' in n}
    assert len(found) == 3, sorted(found)
    for name, body in found.items():
        for op in ('LDGSTS', 'LDSM', 'HMMA'):
            assert op in body, (name, op)
        assert 'LDL' not in body and 'STL' not in body, name
