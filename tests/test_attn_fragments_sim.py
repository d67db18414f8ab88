"""CPU walk-through of the data movement of the tensor-core attention kernels (csrc/vt_attention_mma.cu).

1. ldmatrix: every lane address the kernels form (lane_a / lane_b, plain and .trans) is followed through a model of
   ldmatrix.sync.m8n8.x4 on a tile of distinct values, and the registers it delivers are compared with the mma.m16n8k16
   bf16 fragment layout (PTX ISA) the MMAs assume, for head dims 64 and 96 and every (row block, k chunk, n block) the
   kernels visit.  The addresses stay inside the [64][HD + 8] tile, are 16-byte aligned, and the 8 rows of each phase
   fall in distinct banks.
2. The cp.async ring: the kernels' loops (forward / dQ with one barrier per tile, dK / dV with two) are replayed over
   1, 2, 3 and many tiles against a model of commit / wait_group and barriers: every tile is read from the stage that
   holds it, after its copy completed and a barrier passed, and no stage is overwritten while a thread may still read it.
The GPU tests (test_gpu_attention*.py) check the results; this file checks the indexing those results rest on.
"""
import pytest

MT = 64
LANES = range(32)


# ---- 1. ldmatrix fragments -----------------------------------------------------------------------------------------
def lane_a(lane, P):
    return (lane & 15) * P + (lane >> 4) * 8


def lane_b(lane, P):
    return ((lane & 7) + (lane >> 4) * 8) * P + ((lane >> 3) & 1) * 8


def ldsm_x4(tile, P, addr, trans):
    """model of ldmatrix.x4 on a flat [rows * P] tile; addr(lane) = element offset of the row that lane supplies.
    -> regs[lane][j] = (lo, hi) bf16 pair of register j"""
    mats = []
    for j in range(4):
        rows = []
        for i in range(8):
            a = addr(8 * j + i)
            rows.append([tile[a + c] for c in range(8)])
        mats.append(rows)
    regs = []
    for lane in LANES:
        r, c = lane // 4, 2 * (lane % 4)
        if trans:
            regs.append([(m[c][r], m[c + 1][r]) for m in mats])
        else:
            regs.append([(m[r][c], m[r][c + 1]) for m in mats])
    return regs


def a_frag(M, r0, c0, lane):
    """mma.m16n8k16 A fragment {a0..a3} of the 16 x 16 block (r0, c0) of M[row][col]"""
    g, t = lane >> 2, lane & 3
    return [(M(r0 + g + dr, c0 + 2 * t + dc), M(r0 + g + dr, c0 + 2 * t + dc + 1)) for dr, dc in ((0, 0), (8, 0), (0, 8), (8, 8))]


def b_frag(B, k0, n0, lane):
    """mma.m16n8k16 B fragment {b0, b1} of the 16 x 8 block (k0, n0) of B[k][n]"""
    g, t = lane >> 2, lane & 3
    return [(B(k0 + 2 * t + dk, n0 + g), B(k0 + 2 * t + dk + 1, n0 + g)) for dk in (0, 8)]


def check_addresses(P, HD, base, addr):
    for j in range(4):
        offs = [base + addr(8 * j + i) for i in range(8)]
        for o in offs:
            assert o % 8 == 0                                   # 16-byte aligned rows
            assert 0 <= o and o % P + 8 <= HD and o // P < MT   # inside the tile, never in the pad columns
        assert len({(2 * o // 16) % 8 for o in offs}) == 8      # the phase's 8 rows in distinct 16-byte bank groups


@pytest.mark.parametrize('HD', [64, 96])
def test_ldmatrix_a_fragments(HD):
    """Q (forward, dQ), dO (dQ), K and V (dK / dV) as A operands: x4 at rb * P + kc * 16 + lane_a"""
    P = HD + 8
    tile = list(range(MT * P))
    M = lambda r, c: r * P + c
    for rb in range(0, MT, 16):
        for kc in range(HD // 16):
            base = rb * P + kc * 16
            addr = lambda lane: base + lane_a(lane, P)
            check_addresses(P, HD, 0, addr)
            regs = ldsm_x4(tile, P, addr, trans=False)
            for lane in LANES:
                assert regs[lane] == a_frag(M, rb, kc * 16, lane)


@pytest.mark.parametrize('HD', [64, 96])
def test_ldmatrix_b_fragments_row_operand(HD):
    """B[k][n] = T[n][k] with T row-major (K in S = Q K^T, V in dP = dO V^T, Q and dO in S^T / dP^T of dK / dV):
    x4 at nb * 8 * P + kc * 16 + lane_b -> {b0, b1} of n blocks nb and nb + 1"""
    P = HD + 8
    tile = list(range(MT * P))
    B = lambda k, n: n * P + k
    for nb in range(0, 8, 2):
        for kc in range(HD // 16):
            base = nb * 8 * P + kc * 16
            addr = lambda lane: base + lane_b(lane, P)
            check_addresses(P, HD, 0, addr)
            regs = ldsm_x4(tile, P, addr, trans=False)
            for lane in LANES:
                assert regs[lane][:2] == b_frag(B, kc * 16, nb * 8, lane)
                assert regs[lane][2:] == b_frag(B, kc * 16, nb * 8 + 8, lane)


@pytest.mark.parametrize('HD', [64, 96])
def test_ldmatrix_b_fragments_trans(HD):
    """B[k][n] = T[k][n] with T row-major (V in P V, K in dS K, dO in dV += P^T dO, Q in dK += dS^T Q):
    x4.trans at kc * 16 * P + nb * 8 + lane_a -> {b0, b1} of n blocks nb and nb + 1"""
    P = HD + 8
    tile = list(range(MT * P))
    B = lambda k, n: k * P + n
    for kc in range(4):
        for nb in range(0, HD // 8, 2):
            base = kc * 16 * P + nb * 8
            addr = lambda lane: base + lane_a(lane, P)
            check_addresses(P, HD, 0, addr)
            regs = ldsm_x4(tile, P, addr, trans=True)
            for lane in LANES:
                assert regs[lane][:2] == b_frag(B, kc * 16, nb * 8, lane)
                assert regs[lane][2:] == b_frag(B, kc * 16, nb * 8 + 8, lane)


def test_transposed_ldmatrix_matches_the_old_transposed_copy():
    """the .trans fragment of V equals what the kernels read before from a transposed copy Vt[HD][MT + 8] with 32-bit
    loads at (nb * 8 + g) * PT + kc * 16 + 2t: the operands of P V, and so its result, are unchanged"""
    HD, P, PT = 64, 72, 72
    V = lambda k, n: 1000 * k + n
    tile = [V(i // P, i % P) for i in range(MT * P)]
    for kc in range(4):
        for nb in range(0, HD // 8, 2):
            regs = ldsm_x4(tile, P, lambda lane: kc * 16 * P + nb * 8 + lane_a(lane, P), trans=True)
            for lane in LANES:
                g, t = lane >> 2, lane & 3
                for j, n in ((0, nb), (2, nb + 1)):
                    for half in (0, 1):
                        e = (n * 8 + g) * PT + kc * 16 + 2 * t + 8 * half          # element of Vt = V[e % PT][e // PT]
                        assert regs[lane][j + half] == (V(e % PT, e // PT), V(e % PT + 1, e // PT))


# ---- 2. the cp.async ring --------------------------------------------------------------------------------------------
class Ring:
    """cp.async groups, waits and barriers of one CTA, thread-agnostic: within an epoch (between two barriers) threads run
    in any order, so a buffer must not be both written and read in one epoch, and a read must see a copy that completed
    (wait_group) before the barrier that opened the epoch."""

    def __init__(self):
        self.epoch = 0
        self.groups, self.open = [], []
        self.content, self.inflight = {}, set()
        self.last_write, self.last_read = {}, {}

    def cp(self, buf, tile):
        self._write(buf)
        self.open.append((buf, tile))
        self.inflight.add(buf)

    def store(self, buf, tile):
        self._write(buf)
        self.content[buf] = tile

    def _write(self, buf):
        assert buf not in self.inflight, f'{buf}: written while a copy into it is in flight'
        assert self.last_read.get(buf, -1) < self.epoch, f'{buf}: overwritten in the epoch that reads it'
        self.last_write[buf] = self.epoch

    def commit(self):
        self.groups.append(self.open)
        self.open = []

    def wait(self, n):
        done = self.groups[:len(self.groups) - n] if n else self.groups
        self.groups = self.groups[len(done):]
        for g in done:
            for buf, tile in g:
                self.content[buf] = tile
                self.inflight.discard(buf)

    def bar(self):
        self.epoch += 1

    def read(self, buf, tile):
        assert buf not in self.inflight, f'{buf}: read while its copy is in flight'
        assert self.last_write[buf] < self.epoch, f'{buf}: read in the epoch that writes it'
        assert self.content.get(buf) == tile, f'{buf}: holds {self.content.get(buf)}, expected {tile}'
        self.last_read[buf] = self.epoch


def walk_forward(n, dq):
    """attn_mma_fwd_kernel / attn_mma_dq_kernel over n key tiles (one barrier per tile; dQ adds dO and the row stats)"""
    r = Ring()
    stage = lambda s: (f'K{s}', f'V{s}')
    r.cp('Q', 0)
    if dq:
        r.cp('dO', 0)
    r.commit()
    for b in stage(0):
        r.cp(b, 0)
    r.commit()
    r.wait(1)
    r.bar()
    r.read('Q', 0)
    if dq:
        r.read('dO', 0)                      # row stats and fragments
        r.store('stats', 0)
        r.bar()
        r.read('stats', 0)
    for it in range(n):
        r.wait(0)
        r.bar()
        if it + 1 < n:
            for b in stage((it + 1) & 1):
                r.cp(b, it + 1)
            r.commit()
        for b in stage(it & 1):
            r.read(b, it)
    assert not r.groups and not r.inflight


def walk_dkv(n):
    """attn_mma_dkv_kernel over n query tiles (stats from the staged tile, two barriers per tile)"""
    r = Ring()
    stage = lambda s: (f'Q{s}', f'dO{s}', f'O{s}', f'lse{s}')

    def stage_tile(s, tile):
        for b in stage(s):
            r.cp(b, tile)
        r.commit()

    r.cp('K', 0)
    r.cp('V', 0)
    stage_tile(0, 0)
    for it in range(n):
        r.wait(0)
        r.bar()
        if it + 1 < n:
            stage_tile((it + 1) & 1, it + 1)
        s = it & 1
        for b in (f'dO{s}', f'O{s}', f'lse{s}'):
            r.read(b, it)
        r.store('stats', it)
        r.bar()
        r.read('stats', it)
        r.read('K', 0)
        r.read('V', 0)
        r.read(f'Q{s}', it)
        r.read(f'dO{s}', it)
    assert not r.groups and not r.inflight


@pytest.mark.parametrize('n', [1, 2, 3, 4, 7, 393])
def test_ring_walk(n):
    walk_forward(n, dq=False)
    walk_forward(n, dq=True)
    walk_dkv(n)


def test_ring_model_catches_a_missing_barrier():
    """the model is strict enough to matter: reading a stage in the epoch that refills the other one is fine, but
    refilling the stage being read is caught"""
    r = Ring()
    r.cp('K0', 0)
    r.commit()
    r.wait(0)
    r.bar()
    r.read('K0', 0)
    with pytest.raises(AssertionError):
        r.cp('K0', 1)
