// Tensor-core flash attention for sm_90a (mma.sync.m16n8k16, bf16 operands, fp32 accumulators), head dim 32, 64, 96 or
// 128 (vt_xattn_* takes 64 and 96).
// One kernel family serves both entry points: the packed-qkv attention of vt_attn_* (the 197-token spatial pass) and the
// strided pooling / long-sequence attention of vt_xattn_* (Nq != Nk).  Operands are addressed as
// base + b * bs + h * hs + n * rs (bf16 rows, 16-byte aligned), so q / k / v / dq are read and written in place.
//   forward : CTA = 64 query rows (4 warps x 16), key tiles of 64 streamed through shared memory, online softmax in
//             registers, P rounded to bf16 as the A operand of P V.
//   dQ      : CTA = 64 query rows; S = Q K^T and dP = dO V^T per key tile, dS = P (dP - delta), dQ += dS K.
//   dK / dV : CTA = 64 key rows; S^T = K Q^T and dP^T = V dO^T per query tile, dV += P^T dO, dK += dS^T Q.
// delta = rowsum(dO * O) is recomputed where it is needed, so no scratch is required and no atomics are used.
//
// Data movement: every tile is a row-major [64][HD + 8] bf16 copy of 64 rows, loaded with 16-byte cp.async into a
// two-stage ring (the next tile's loads are in flight while the current tile's MMAs run); rows past Nq / Nk are
// zero-filled by the copy (src-size 0) and never read.  MMA fragments come from ldmatrix.x4, the .trans form for operands
// used transposed (V in P V, K in dS K, Q and dO in the dK / dV MMAs).  The HD + 8 pitch puts the 8 rows read by every
// ldmatrix phase in distinct banks at every head dim (row pitch 80, 144, 208 or 272 bytes), so no swizzle is needed.  MMAs whose operands are all padding are
// skipped: a warp whose 16 rows lie past the end issues none, and on a partial last tile only the n8 blocks of S and the
// k16 chunks of the second product that hold a valid key (dK / dV: query) run; the skipped terms are exact zeros.
//
// Whole problems (attn_whole_*, the packed-qkv path at head dim 64 and N <= 256, e.g. the 197-token spatial pass): a CTA
// owns one (b, h) problem and loads each operand once into shared memory ([R][64], R = N rounded up to 16, XOR-swizzled
// 16-byte chunks instead of the pad, so two CTAs fit an SM).  Warps own 16-row groups, so at N = 197 no CTA works on a
// 5-row tile with three idle warps and no operand is streamed once per 64-row tile.
//   forward : 8 warps take the 16-row query groups in turn; K / V land in two cp.async groups (first 64 keys first).
//   backward: one launch; Q, K, V, dO resident, lse and delta computed once per problem; 6 warps take the 2 * R / 16
//             independent tasks (dK / dV of 16 keys first, then dQ of 16 queries) from a shared-memory counter.
// Both families run each warp's arithmetic through the same step functions (fwd_tile, dq_tile, dkv_tile, their stores
// and row_delta), which see an operand only through its tile type (PaddedTile, SwizzledTile), so o, lse, dq, dk and dv
// are the same bits; VT_ATTN_WHOLE=0 selects the tiled kernels instead (vt_attention.cu).  vt_xattn_* always takes the
// tiled kernels.
#include "vt_attention_mma.cuh"

namespace vt {

constexpr int MT = 64;          // rows per CTA and per staged tile
constexpr int MMA_THREADS = 128;
constexpr float MMA_LOG2E = 1.4426950408889634f;
constexpr float MMA_LN2 = 0.6931471805599453f;

__device__ __forceinline__ void mma16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t ld32(const __nv_bfloat16* p) { return *reinterpret_cast<const uint32_t*>(p); }
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
template <int N>
__device__ __forceinline__ void zero(float (&x)[N][4]) {
#pragma unroll
  for (int i = 0; i < N; ++i) x[i][0] = x[i][1] = x[i][2] = x[i][3] = 0.f;
}

// 16 (4) bytes global -> shared without passing through registers; ok = false writes zeros and reads nothing
__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool ok) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_addr(dst)), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async4(void* dst, const void* src, bool ok) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_addr(dst)), "l"(src), "r"(ok ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// four 8x8 bf16 matrices; lane l supplies the shared address of row l % 8 of matrix l / 8
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t a) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t a) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}

// Operand tiles in shared memory.  A tile type gives the shared address of the row this lane supplies to ldmatrix.x4
// (tests/test_attn_fragments_sim.py and tests/test_attn_whole_sim.py walk both layouts against the mma layout):
//   a(r0, c0): A fragment {a0..a3} of rows r0..r0+15, cols c0..c0+15; with .trans at (k0, n0) of a row-major [k][n]
//              tile -> B fragments {b0, b1} of n block n0 and {b0, b1} of n block n0 + 8 (k rows k0..k0+15).
//   b(n0, c0): of an [n][k] tile -> {b0, b1} of n block n0, then of n block n0 + 8, k cols c0..c0+15.
// That is all the per-warp step functions below see of a layout.
template <int P>
__device__ __forceinline__ int lane_a(int lane) { return (lane & 15) * P + (lane >> 4) * 8; }
template <int P>
__device__ __forceinline__ int lane_b(int lane) { return ((lane & 7) + (lane >> 4) * 8) * P + ((lane >> 3) & 1) * 8; }

// a row-major [rows][HD + 8] tile of the tiled kernels
template <int HD>
struct PaddedTile {
  static constexpr int P = HD + 8;
  uint32_t base;
  int la, lb;                                   // lane_a / lane_b in bytes
  __device__ __forceinline__ explicit PaddedTile(const __nv_bfloat16* t)
      : base(smem_addr(t)), la(2 * lane_a<P>(threadIdx.x & 31)), lb(2 * lane_b<P>(threadIdx.x & 31)) {}
  __device__ __forceinline__ uint32_t a(int r0, int c0) const { return base + (r0 * P + c0) * 2 + la; }
  __device__ __forceinline__ uint32_t b(int n0, int c0) const { return base + (n0 * P + c0) * 2 + lb; }
};

// A [R][64] operand of the whole-problem kernels, from its row r0 (r0 % 8 == 0) on.  The 16-byte chunk c of row r sits
// at chunk c ^ (r & 7) (swz), so the 8 rows of every ldmatrix phase fall in distinct bank groups without a pad.  With the
// lane's row offset ar / br and chunk key ak / bk, the fragment at (r0, c0), r0 % 8 == 0 and c0 % 16 == 0, is at element
// sw_at(row, key, r0, c0) = row + r0 * 64 + ((c0 / 8) ^ key) * 8 (c0 / 8 is even: (c0 / 8 + lc) ^ (r & 7) ==
// (c0 / 8) ^ (lc ^ (r & 7))); a() and b() return it in bytes.
__device__ __forceinline__ int swz(int r, int c) { return r * 64 + ((c ^ (r & 7)) << 3); }
struct SwizzledTile {
  uint32_t base;
  int ar, ak, br, bk;
  __device__ __forceinline__ SwizzledTile(uint32_t operand, int r0) : base(operand + r0 * 128) {
    const int lane = threadIdx.x & 31;
    ar = (lane & 15) * 128; ak = (lane >> 4) ^ (lane & 7);
    br = ((lane & 7) + (lane >> 4) * 8) * 128; bk = ((lane >> 3) & 1) ^ (lane & 7);
  }
  __device__ __forceinline__ uint32_t a(int r0, int c0) const { return base + ar + r0 * 128 + (((c0 >> 3) ^ ak) << 4); }
  __device__ __forceinline__ uint32_t b(int n0, int c0) const { return base + br + n0 * 128 + (((c0 >> 3) ^ bk) << 4); }
};

// rows [r0, r0 + MT) of a strided bf16 matrix -> dst[MT][HD + 8] in flight; rows >= limit are zero-filled
template <int HD>
__device__ __forceinline__ void stage_rows(__nv_bfloat16* dst, const __nv_bfloat16* src, long long rs, int r0, int limit) {
#pragma unroll
  for (int i = threadIdx.x; i < MT * HD / 8; i += MMA_THREADS) {
    const int r = i / (HD / 8), c = (i % (HD / 8)) * 8;
    const bool ok = r0 + r < limit;
    cp_async16(dst + r * (HD + 8) + c, ok ? src + (long long)(r0 + r) * rs + c : src, ok);
  }
}
// delta = rowsum(dO * O) of one row by a pair of threads (half = 0, 1 takes the first, second half of the columns), in
// the fmaf order of both backward families; dO2(c) reads the pair dO[c], dO[c + 1] of the row.  ok = false: 0
template <int HD, class DO2>
__device__ __forceinline__ float row_delta(bool ok, int half, DO2 dO2, const __nv_bfloat16* orow) {
  float d = 0.f;
  if (ok) {
#pragma unroll 4
    for (int c = half * (HD / 2); c < (half + 1) * (HD / 2); c += 2) {
      const float2 g = unpack_bf16x2(dO2(c));
      const float2 o = unpack_bf16x2(ld32(orow + c));
      d = fmaf(g.x, o.x, fmaf(g.y, o.y, d));
    }
  }
  return d + __shfl_xor_sync(0xffffffffu, d, 1);
}
// lse (log2 domain; +inf past the end: p = 0) and delta = rowsum(dO * O) of rows [r0, r0 + MT).  dOs is the staged dO
// tile; orow / o_rs and lrow address O and lse of row r0 (global memory, or a staged tile); delta_out is optional
template <int HD>
__device__ __forceinline__ void stage_row_stats(float* lse_s, float* del_s, const __nv_bfloat16* dOs, const __nv_bfloat16* orow,
                                                long long o_rs, const float* lrow, int r0, int limit, float* delta_out) {
  const int r = threadIdx.x >> 1, half = threadIdx.x & 1;
  const bool ok = r0 + r < limit;
  const __nv_bfloat16* g = dOs + r * (HD + 8);
  const float d = row_delta<HD>(ok, half, [=](int c) { return ld32(g + c); }, orow + r * o_rs);
  if (half == 0) {
    del_s[r] = d;
    lse_s[r] = ok ? lrow[r] * MMA_LOG2E : INFINITY;
    if (ok && delta_out) delta_out[r0 + r] = d;
  }
}

// ------------------------------------------------------------------------------------------------ per-warp steps
// One warp's arithmetic on its 16 rows, called by the tiled and the whole-problem kernels alike.  A tile argument is the
// 64-row tile of rows k0.. (q0..) of an operand with N rows (keys for K / V, queries for Q / dO), addressed from its
// first row; MMAs on n8 blocks and k16 chunks that hold no valid row are skipped.  rb of a store is the warp's first row
// in the problem; rows past the end are not written.

// A fragments of rows r0..r0+15 over the head dim
template <int KC, class Tile>
__device__ __forceinline__ void load_a(uint32_t (&f)[KC][4], const Tile& t, int r0) {
#pragma unroll
  for (int kc = 0; kc < KC; ++kc) ldsm_x4(f[kc], t.a(r0, kc * 16));
}

// the forward's running state: unnormalised o, and the max m and sum l (log2 domain) of rows g and g + 8
template <int HD>
struct FwdAcc {
  float o[HD / 8][4];
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  __device__ __forceinline__ FwdAcc() { zero(o); }
};

// forward, one key tile: S = Q K^T * scale (c = scale * log2 e), keys past N masked, online softmax, o += P V with P
// rounded to bf16
template <int HD, class Tile>
__device__ __forceinline__ void fwd_tile(FwdAcc<HD>& f, const uint32_t (&qa)[HD / 16][4], const Tile& K, const Tile& V, int k0,
                                         int N, float c) {
  constexpr int NB = HD / 8, KC = HD / 16;
  const int t = threadIdx.x & 3;
  float s[8][4];
  zero(s);
#pragma unroll
  for (int nb = 0; nb < 8; nb += 2) {
    if (k0 + nb * 8 >= N) break;                     // n8 blocks past the last key stay 0 and are masked below
    const bool hi = k0 + nb * 8 + 8 < N;
#pragma unroll
    for (int kc = 0; kc < KC; ++kc) {
      uint32_t kf[4];
      ldsm_x4(kf, K.b(nb * 8, kc * 16));
      mma16816(s[nb], qa[kc][0], qa[kc][1], qa[kc][2], qa[kc][3], kf[0], kf[1]);
      if (hi) mma16816(s[nb + 1], qa[kc][0], qa[kc][1], qa[kc][2], qa[kc][3], kf[2], kf[3]);
    }
  }
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int key = k0 + nb * 8 + 2 * t + (e & 1);
      const float v = key < N ? s[nb][e] * c : -INFINITY;
      s[nb][e] = v;
      if (e < 2) mx0 = fmaxf(mx0, v); else mx1 = fmaxf(mx1, v);
    }
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  const float mn0 = fmaxf(f.m0, mx0), mn1 = fmaxf(f.m1, mx1);  // finite: every tile holds at least one key
  const float corr0 = fast_exp2(f.m0 - mn0), corr1 = fast_exp2(f.m1 - mn1);
  f.l0 *= corr0; f.l1 *= corr1;
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) { f.o[nb][0] *= corr0; f.o[nb][1] *= corr0; f.o[nb][2] *= corr1; f.o[nb][3] *= corr1; }
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    s[nb][0] = fast_exp2(s[nb][0] - mn0); s[nb][1] = fast_exp2(s[nb][1] - mn0);
    s[nb][2] = fast_exp2(s[nb][2] - mn1); s[nb][3] = fast_exp2(s[nb][3] - mn1);
    f.l0 += s[nb][0] + s[nb][1];
    f.l1 += s[nb][2] + s[nb][3];
  }
  f.m0 = mn0; f.m1 = mn1;
#pragma unroll
  for (int kc = 0; kc < 4; ++kc) {
    if (k0 + kc * 16 >= N) break;                    // P = 0 over the whole chunk
    const uint32_t a0 = pack_bf16x2(s[2 * kc][0], s[2 * kc][1]), a1 = pack_bf16x2(s[2 * kc][2], s[2 * kc][3]);
    const uint32_t a2 = pack_bf16x2(s[2 * kc + 1][0], s[2 * kc + 1][1]), a3 = pack_bf16x2(s[2 * kc + 1][2], s[2 * kc + 1][3]);
#pragma unroll
    for (int nb = 0; nb < NB; nb += 2) {
      uint32_t vf[4];
      ldsm_x4_t(vf, V.a(kc * 16, nb * 8));
      mma16816(f.o[nb], a0, a1, a2, a3, vf[0], vf[1]);
      mma16816(f.o[nb + 1], a0, a1, a2, a3, vf[2], vf[3]);
    }
  }
}

// o / l as bf16; LSE: lse = (m + log2 l) * ln 2 (a template flag, so the forward-only form writes no lse)
template <int HD, bool LSE>
__device__ __forceinline__ void fwd_store(FwdAcc<HD>& f, const MmaAttn& p, int b, int h, int rb) {
  const int g = (threadIdx.x & 31) >> 2, t = threadIdx.x & 3;
  f.l0 += __shfl_xor_sync(0xffffffffu, f.l0, 1); f.l0 += __shfl_xor_sync(0xffffffffu, f.l0, 2);
  f.l1 += __shfl_xor_sync(0xffffffffu, f.l1, 1); f.l1 += __shfl_xor_sync(0xffffffffu, f.l1, 2);
  const float inv0 = 1.0f / f.l0, inv1 = 1.0f / f.l1;
  __nv_bfloat16* ob = p.o_out + b * p.o_bs + h * p.o_hs;
  const int r0 = rb + g, r1 = r0 + 8;
#pragma unroll
  for (int nb = 0; nb < HD / 8; ++nb) {
    if (r0 < p.Nq) *reinterpret_cast<uint32_t*>(ob + (long long)r0 * p.o_rs + nb * 8 + 2 * t) = pack_bf16x2(f.o[nb][0] * inv0, f.o[nb][1] * inv0);
    if (r1 < p.Nq) *reinterpret_cast<uint32_t*>(ob + (long long)r1 * p.o_rs + nb * 8 + 2 * t) = pack_bf16x2(f.o[nb][2] * inv1, f.o[nb][3] * inv1);
  }
  if (LSE && t == 0) {
    float* lse = p.lse + (long long)(b * p.H + h) * p.Nq;
    if (r0 < p.Nq) lse[r0] = (f.m0 + log2f(f.l0)) * MMA_LN2;
    if (r1 < p.Nq) lse[r1] = (f.m1 + log2f(f.l1)) * MMA_LN2;
  }
}

// dQ, one key tile: S = Q K^T and dP = dO V^T, dS = P (dP - delta) with P = 0 past N, dq += dS K with dS rounded to bf16.
// qa / da: the warp's Q and dO fragments; lse (log2 domain) and delta of rows g and g + 8
template <int HD, class Tile>
__device__ __forceinline__ void dq_tile(float (&dq)[HD / 8][4], const uint32_t (&qa)[HD / 16][4], const uint32_t (&da)[HD / 16][4],
                                        const Tile& K, const Tile& V, int k0, int N, float c, float lse0, float lse1, float del0, float del1) {
  constexpr int NB = HD / 8, KC = HD / 16;
  const int t = threadIdx.x & 3;
  float s[8][4], dpv[8][4];
  zero(s);
  zero(dpv);
#pragma unroll
  for (int nb = 0; nb < 8; nb += 2) {
    if (k0 + nb * 8 >= N) break;
    const bool hi = k0 + nb * 8 + 8 < N;
#pragma unroll
    for (int kc = 0; kc < KC; ++kc) {
      uint32_t kf[4], vf[4];
      ldsm_x4(kf, K.b(nb * 8, kc * 16));
      ldsm_x4(vf, V.b(nb * 8, kc * 16));
      mma16816(s[nb], qa[kc][0], qa[kc][1], qa[kc][2], qa[kc][3], kf[0], kf[1]);
      mma16816(dpv[nb], da[kc][0], da[kc][1], da[kc][2], da[kc][3], vf[0], vf[1]);
      if (hi) {
        mma16816(s[nb + 1], qa[kc][0], qa[kc][1], qa[kc][2], qa[kc][3], kf[2], kf[3]);
        mma16816(dpv[nb + 1], da[kc][0], da[kc][1], da[kc][2], da[kc][3], vf[2], vf[3]);
      }
    }
  }
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int key = k0 + nb * 8 + 2 * t + (e & 1);
      const float pr = key < N ? fast_exp2(s[nb][e] * c - (e < 2 ? lse0 : lse1)) : 0.f;
      s[nb][e] = pr * (dpv[nb][e] - (e < 2 ? del0 : del1));
    }
  }
#pragma unroll
  for (int kc = 0; kc < 4; ++kc) {
    if (k0 + kc * 16 >= N) break;                    // dS = 0 over the whole chunk
    const uint32_t a0 = pack_bf16x2(s[2 * kc][0], s[2 * kc][1]), a1 = pack_bf16x2(s[2 * kc][2], s[2 * kc][3]);
    const uint32_t a2 = pack_bf16x2(s[2 * kc + 1][0], s[2 * kc + 1][1]), a3 = pack_bf16x2(s[2 * kc + 1][2], s[2 * kc + 1][3]);
#pragma unroll
    for (int nb = 0; nb < NB; nb += 2) {
      uint32_t kf[4];
      ldsm_x4_t(kf, K.a(kc * 16, nb * 8));
      mma16816(dq[nb], a0, a1, a2, a3, kf[0], kf[1]);
      mma16816(dq[nb + 1], a0, a1, a2, a3, kf[2], kf[3]);
    }
  }
}

template <int HD>
__device__ __forceinline__ void dq_store(const float (&dq)[HD / 8][4], const MmaAttn& p, int b, int h, int rb) {
  const int g = (threadIdx.x & 31) >> 2, t = threadIdx.x & 3;
  __nv_bfloat16* dqb = p.dq + b * p.dq_bs + h * p.dq_hs;
  const int r0 = rb + g, r1 = r0 + 8;
#pragma unroll
  for (int nb = 0; nb < HD / 8; ++nb) {
    if (r0 < p.Nq)
      *reinterpret_cast<uint32_t*>(dqb + (long long)r0 * p.dq_rs + nb * 8 + 2 * t) = pack_bf16x2(dq[nb][0] * p.scale, dq[nb][1] * p.scale);
    if (r1 < p.Nq)
      *reinterpret_cast<uint32_t*>(dqb + (long long)r1 * p.dq_rs + nb * 8 + 2 * t) = pack_bf16x2(dq[nb][2] * p.scale, dq[nb][3] * p.scale);
  }
}

// dK / dV, one query tile: S^T = K Q^T and dP^T = V dO^T for the warp's key rows rb..rb+15 of K / V, P^T and
// dS^T = P^T (dP^T - delta) rounded to bf16, dv += P^T dO, dk += dS^T Q.  lse / del: the tile's log2-domain lse and
// delta (+inf / 0 past N: P = 0 there)
template <int HD, class Tile>
__device__ __forceinline__ void dkv_tile(float (&dk)[HD / 8][4], float (&dv)[HD / 8][4], const Tile& K, const Tile& V, int rb,
                                         const Tile& Q, const Tile& dO, int q0, int N, float c, const float* lse, const float* del) {
  constexpr int NB = HD / 8, KC = HD / 16;
  const int t = threadIdx.x & 3;
  float s[8][4], dpv[8][4];
  zero(s);
  zero(dpv);
#pragma unroll
  for (int kc = 0; kc < KC; ++kc) {
    uint32_t ka[4], va[4];
    ldsm_x4(ka, K.a(rb, kc * 16));
    ldsm_x4(va, V.a(rb, kc * 16));
#pragma unroll
    for (int nb = 0; nb < 8; nb += 2) {
      if (q0 + nb * 8 >= N) break;                   // n8 blocks past the last query stay 0: lse = +inf there, P = 0
      uint32_t qf[4], df[4];
      ldsm_x4(qf, Q.b(nb * 8, kc * 16));
      ldsm_x4(df, dO.b(nb * 8, kc * 16));
      mma16816(s[nb], ka[0], ka[1], ka[2], ka[3], qf[0], qf[1]);
      mma16816(dpv[nb], va[0], va[1], va[2], va[3], df[0], df[1]);
      if (q0 + nb * 8 + 8 < N) {
        mma16816(s[nb + 1], ka[0], ka[1], ka[2], ka[3], qf[2], qf[3]);
        mma16816(dpv[nb + 1], va[0], va[1], va[2], va[3], df[2], df[3]);
      }
    }
  }
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int qi = nb * 8 + 2 * t + (e & 1);
      const float pr = fast_exp2(s[nb][e] * c - lse[qi]);
      s[nb][e] = pr;
      dpv[nb][e] = pr * (dpv[nb][e] - del[qi]);
    }
  }
#pragma unroll
  for (int kc = 0; kc < 4; ++kc) {
    if (q0 + kc * 16 >= N) break;                    // P = dS = 0 over the whole chunk
    const uint32_t p0 = pack_bf16x2(s[2 * kc][0], s[2 * kc][1]), p1 = pack_bf16x2(s[2 * kc][2], s[2 * kc][3]);
    const uint32_t p2 = pack_bf16x2(s[2 * kc + 1][0], s[2 * kc + 1][1]), p3 = pack_bf16x2(s[2 * kc + 1][2], s[2 * kc + 1][3]);
    const uint32_t d0 = pack_bf16x2(dpv[2 * kc][0], dpv[2 * kc][1]), d1 = pack_bf16x2(dpv[2 * kc][2], dpv[2 * kc][3]);
    const uint32_t d2 = pack_bf16x2(dpv[2 * kc + 1][0], dpv[2 * kc + 1][1]), d3 = pack_bf16x2(dpv[2 * kc + 1][2], dpv[2 * kc + 1][3]);
#pragma unroll
    for (int nb = 0; nb < NB; nb += 2) {
      uint32_t gf[4], qf[4];
      ldsm_x4_t(gf, dO.a(kc * 16, nb * 8));
      ldsm_x4_t(qf, Q.a(kc * 16, nb * 8));
      mma16816(dv[nb], p0, p1, p2, p3, gf[0], gf[1]);
      mma16816(dv[nb + 1], p0, p1, p2, p3, gf[2], gf[3]);
      mma16816(dk[nb], d0, d1, d2, d3, qf[0], qf[1]);
      mma16816(dk[nb + 1], d0, d1, d2, d3, qf[2], qf[3]);
    }
  }
}

// dK = dk * scale and dV: fp32 [B, H, Nk, HD] (f32: p.dk32 / p.dv32) or strided bf16 (p.dk16 / p.dv16)
template <int HD>
__device__ __forceinline__ void dkv_store(const float (&dk)[HD / 8][4], const float (&dv)[HD / 8][4], const MmaAttn& p, int b, int h,
                                          int rb, bool f32) {
  const int g = (threadIdx.x & 31) >> 2, t = threadIdx.x & 3;
  const int r0 = rb + g, r1 = r0 + 8;
#pragma unroll
  for (int nb = 0; nb < HD / 8; ++nb) {
    const int col = nb * 8 + 2 * t;
    if (f32) {
      float* dkb = p.dk32 + (long long)(b * p.H + h) * p.Nk * HD;
      float* dvb = p.dv32 + (long long)(b * p.H + h) * p.Nk * HD;
      if (r0 < p.Nk) {
        *reinterpret_cast<float2*>(dkb + (long long)r0 * HD + col) = make_float2(dk[nb][0] * p.scale, dk[nb][1] * p.scale);
        *reinterpret_cast<float2*>(dvb + (long long)r0 * HD + col) = make_float2(dv[nb][0], dv[nb][1]);
      }
      if (r1 < p.Nk) {
        *reinterpret_cast<float2*>(dkb + (long long)r1 * HD + col) = make_float2(dk[nb][2] * p.scale, dk[nb][3] * p.scale);
        *reinterpret_cast<float2*>(dvb + (long long)r1 * HD + col) = make_float2(dv[nb][2], dv[nb][3]);
      }
    } else {
      __nv_bfloat16* dkb = p.dk16 + b * p.dk_bs + h * p.dk_hs;
      __nv_bfloat16* dvb = p.dv16 + b * p.dv_bs + h * p.dv_hs;
      if (r0 < p.Nk) {
        *reinterpret_cast<uint32_t*>(dkb + (long long)r0 * p.dk_rs + col) = pack_bf16x2(dk[nb][0] * p.scale, dk[nb][1] * p.scale);
        *reinterpret_cast<uint32_t*>(dvb + (long long)r0 * p.dv_rs + col) = pack_bf16x2(dv[nb][0], dv[nb][1]);
      }
      if (r1 < p.Nk) {
        *reinterpret_cast<uint32_t*>(dkb + (long long)r1 * p.dk_rs + col) = pack_bf16x2(dk[nb][2] * p.scale, dk[nb][3] * p.scale);
        *reinterpret_cast<uint32_t*>(dvb + (long long)r1 * p.dv_rs + col) = pack_bf16x2(dv[nb][2], dv[nb][3]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ forward
// shared memory: Q, then a ring of two (K, V) stages
template <int HD, bool LSE>
__device__ __forceinline__ void mma_fwd(const MmaAttn& p) {
  constexpr int TILE = MT * (HD + 8);
  extern __shared__ __align__(16) uint8_t mma_smem[];
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(mma_smem);
  __nv_bfloat16* ring = Qs + TILE;
  const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H;
  const int q0 = blockIdx.x * MT, rb = (threadIdx.x >> 5) * 16;
  const bool active = q0 + rb < p.Nq;           // warp-uniform: at least one of this warp's 16 query rows is valid
  const __nv_bfloat16* kb = p.k + b * p.k_bs + h * p.k_hs;
  const __nv_bfloat16* vb = p.v + b * p.v_bs + h * p.v_hs;
  stage_rows<HD>(Qs, p.q + b * p.q_bs + h * p.q_hs, p.q_rs, q0, p.Nq);
  cp_async_commit();
  stage_rows<HD>(ring, kb, p.k_rs, 0, p.Nk);
  stage_rows<HD>(ring + TILE, vb, p.v_rs, 0, p.Nk);
  cp_async_commit();
  cp_async_wait<1>();
  __syncthreads();
  uint32_t qa[HD / 16][4];
  load_a(qa, PaddedTile<HD>(Qs), rb);
  FwdAcc<HD> f;
  const float c = p.scale * MMA_LOG2E;
  for (int k0 = 0, it = 0; k0 < p.Nk; k0 += MT, ++it) {
    cp_async_wait<0>();
    __syncthreads();                            // tile `it` landed for every thread; stage it + 1 is no longer read
    if (k0 + MT < p.Nk) {
      __nv_bfloat16* nx = ring + ((it + 1) & 1) * 2 * TILE;
      stage_rows<HD>(nx, kb, p.k_rs, k0 + MT, p.Nk);
      stage_rows<HD>(nx + TILE, vb, p.v_rs, k0 + MT, p.Nk);
      cp_async_commit();
    }
    if (!active) continue;
    const __nv_bfloat16* Ks = ring + (it & 1) * 2 * TILE;
    fwd_tile<HD>(f, qa, PaddedTile<HD>(Ks), PaddedTile<HD>(Ks + TILE), k0, p.Nk, c);
  }
  if (active) fwd_store<HD, LSE>(f, p, b, h, q0 + rb);
}

// ------------------------------------------------------------------------------------------------ dQ
// shared memory: Q, dO, a ring of two (K, V) stages, lse and delta of the CTA's rows
template <int HD>
__device__ __forceinline__ void mma_dq(const MmaAttn& p) {
  constexpr int TILE = MT * (HD + 8);
  extern __shared__ __align__(16) uint8_t mma_smem[];
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(mma_smem);
  __nv_bfloat16* dOs = Qs + TILE;
  __nv_bfloat16* ring = dOs + TILE;
  float* lse_s = reinterpret_cast<float*>(ring + 4 * TILE);
  float* del_s = lse_s + MT;
  const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H;
  const int q0 = blockIdx.x * MT, g = (threadIdx.x & 31) >> 2, rb = (threadIdx.x >> 5) * 16;
  const bool active = q0 + rb < p.Nq;
  const __nv_bfloat16* kb = p.k + b * p.k_bs + h * p.k_hs;
  const __nv_bfloat16* vb = p.v + b * p.v_bs + h * p.v_hs;
  stage_rows<HD>(Qs, p.q + b * p.q_bs + h * p.q_hs, p.q_rs, q0, p.Nq);
  stage_rows<HD>(dOs, p.dout + b * p.o_bs + h * p.o_hs, p.o_rs, q0, p.Nq);
  cp_async_commit();
  stage_rows<HD>(ring, kb, p.k_rs, 0, p.Nk);
  stage_rows<HD>(ring + TILE, vb, p.v_rs, 0, p.Nk);
  cp_async_commit();
  cp_async_wait<1>();
  __syncthreads();
  stage_row_stats<HD>(lse_s, del_s, dOs, p.o + b * p.o_bs + h * p.o_hs + q0 * p.o_rs, p.o_rs,
                      p.lse + (long long)bh * p.Nq + q0, q0, p.Nq, p.delta ? p.delta + (long long)bh * p.Nq : nullptr);
  uint32_t qa[HD / 16][4], da[HD / 16][4];
  load_a(qa, PaddedTile<HD>(Qs), rb);
  load_a(da, PaddedTile<HD>(dOs), rb);
  __syncthreads();
  const float lse0 = lse_s[rb + g], lse1 = lse_s[rb + g + 8], del0 = del_s[rb + g], del1 = del_s[rb + g + 8];
  float dq[HD / 8][4];
  zero(dq);
  const float c = p.scale * MMA_LOG2E;
  for (int k0 = 0, it = 0; k0 < p.Nk; k0 += MT, ++it) {
    cp_async_wait<0>();
    __syncthreads();
    if (k0 + MT < p.Nk) {
      __nv_bfloat16* nx = ring + ((it + 1) & 1) * 2 * TILE;
      stage_rows<HD>(nx, kb, p.k_rs, k0 + MT, p.Nk);
      stage_rows<HD>(nx + TILE, vb, p.v_rs, k0 + MT, p.Nk);
      cp_async_commit();
    }
    if (!active) continue;
    const __nv_bfloat16* Ks = ring + (it & 1) * 2 * TILE;
    dq_tile<HD>(dq, qa, da, PaddedTile<HD>(Ks), PaddedTile<HD>(Ks + TILE), k0, p.Nk, c, lse0, lse1, del0, del1);
  }
  if (active) dq_store<HD>(dq, p, b, h, q0 + rb);
}

// ------------------------------------------------------------------------------------------------ dK / dV
// shared memory: K, V, a ring of two (Q, dO, O) stages, the ring's two lse rows, lse and delta of the current query tile.
template <int HD>
__device__ __forceinline__ void mma_dkv(const MmaAttn& p) {
  constexpr int TILE = MT * (HD + 8);
  extern __shared__ __align__(16) uint8_t mma_smem[];
  __nv_bfloat16* Ks = reinterpret_cast<__nv_bfloat16*>(mma_smem);
  __nv_bfloat16* Vs = Ks + TILE;
  __nv_bfloat16* ring = Vs + TILE;
  float* lse_ring = reinterpret_cast<float*>(ring + 6 * TILE);
  float* lse_s = lse_ring + 2 * MT;
  float* del_s = lse_s + MT;
  const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H;
  const int k0 = blockIdx.x * MT, rb = (threadIdx.x >> 5) * 16;
  const bool active = k0 + rb < p.Nk;           // warp-uniform: at least one of this warp's 16 key rows is valid
  const __nv_bfloat16* qb = p.q + b * p.q_bs + h * p.q_hs;
  const __nv_bfloat16* db = p.dout + b * p.o_bs + h * p.o_hs;
  const __nv_bfloat16* ob = p.o + b * p.o_bs + h * p.o_hs;
  const float* lse = p.lse + (long long)bh * p.Nq;
  // one query tile (Q, dO, O, lse) into ring stage st
  auto stage_tile = [&](int st, int q0) {
    __nv_bfloat16* d = ring + st * 3 * TILE;
    stage_rows<HD>(d, qb, p.q_rs, q0, p.Nq);
    stage_rows<HD>(d + TILE, db, p.o_rs, q0, p.Nq);
    stage_rows<HD>(d + 2 * TILE, ob, p.o_rs, q0, p.Nq);
    if (threadIdx.x < MT) {
      const bool ok = q0 + (int)threadIdx.x < p.Nq;
      cp_async4(lse_ring + st * MT + threadIdx.x, ok ? lse + q0 + threadIdx.x : lse, ok);
    }
    cp_async_commit();
  };
  stage_rows<HD>(Ks, p.k + b * p.k_bs + h * p.k_hs, p.k_rs, k0, p.Nk);
  stage_rows<HD>(Vs, p.v + b * p.v_bs + h * p.v_hs, p.v_rs, k0, p.Nk);
  stage_tile(0, 0);
  float dk[HD / 8][4], dv[HD / 8][4];
  zero(dk);
  zero(dv);
  const float c = p.scale * MMA_LOG2E;
  for (int q0 = 0, it = 0; q0 < p.Nq; q0 += MT, ++it) {
    cp_async_wait<0>();
    __syncthreads();                            // tile `it` landed; stage it + 1, lse_s and del_s are no longer read
    if (q0 + MT < p.Nq) stage_tile((it + 1) & 1, q0 + MT);
    const __nv_bfloat16* Qs = ring + (it & 1) * 3 * TILE;
    const __nv_bfloat16* dOs = Qs + TILE;
    stage_row_stats<HD>(lse_s, del_s, dOs, dOs + TILE, HD + 8, lse_ring + (it & 1) * MT, q0, p.Nq, nullptr);
    __syncthreads();
    if (!active) continue;
    dkv_tile<HD>(dk, dv, PaddedTile<HD>(Ks), PaddedTile<HD>(Vs), rb, PaddedTile<HD>(Qs), PaddedTile<HD>(dOs), q0, p.Nq, c,
                 lse_s, del_s);
  }
  if (active) dkv_store<HD>(dk, dv, p, b, h, k0 + rb, p.dk32 != nullptr);
}

// ------------------------------------------------------------------------------------------------ kernels
// Head dims 64 (ViT-B) and 96 (MViT) are the attn_mma_* kernels.  The packed-qkv widths 32 and 128 run the same bodies
// under their own names (attn_tc_*), so each width's resources can be checked and profiled on its own.  dK / dV: at head
// dim 64 three CTAs fit an SM (162 registers without spills, 75 KB); at 96 and 128 the register cap of more would spill;
// at 32 four fit.
template <int HD>
constexpr int dkv_min_ctas() { return HD == 32 ? 4 : HD == 64 ? 3 : 1; }

template <int HD, bool LSE>
__global__ void __launch_bounds__(MMA_THREADS) attn_mma_fwd_kernel(const MmaAttn p) { mma_fwd<HD, LSE>(p); }
template <int HD>
__global__ void __launch_bounds__(MMA_THREADS) attn_mma_dq_kernel(const MmaAttn p) { mma_dq<HD>(p); }
template <int HD>
__global__ void __launch_bounds__(MMA_THREADS, dkv_min_ctas<HD>()) attn_mma_dkv_kernel(const MmaAttn p) { mma_dkv<HD>(p); }
template <int HD, bool LSE>
__global__ void __launch_bounds__(MMA_THREADS) attn_tc_fwd_kernel(const MmaAttn p) { mma_fwd<HD, LSE>(p); }
template <int HD>
__global__ void __launch_bounds__(MMA_THREADS) attn_tc_dq_kernel(const MmaAttn p) { mma_dq<HD>(p); }
template <int HD>
__global__ void __launch_bounds__(MMA_THREADS, dkv_min_ctas<HD>()) attn_tc_dkv_kernel(const MmaAttn p) { mma_dkv<HD>(p); }

// ------------------------------------------------------------------------------------------------ whole problems
// Packed-qkv attention at head dim 64 and N <= WHOLE_MAX_N (Nq == Nk): a CTA owns one (b, h) problem and keeps its
// operands resident in shared memory, so each is read from L2 once and no CTA works on a partial 64-row tile alone.
// Warps own 16-row groups; each group walks the 64-row tiles of the resident operands with the step functions above.
// Operands are SwizzledTile [R][64] bf16, R = N rounded up to 16 (rows >= N zero-filled: the 16-row reads of the last
// group and the k16 chunks past the end see the zeros the tiled kernels stage).
constexpr int WHOLE_MAX_N = 256;
constexpr int WF_THREADS = 256;     // forward: 8 warps, two CTAs per SM
constexpr int WB_THREADS = 192;     // backward: 6 warps, two CTAs per SM (12 warps at <= 168 registers)

// rows [r_begin, r_end) of a strided [N][64] bf16 matrix -> swizzled dst, in flight; rows >= n are zero-filled
template <int THREADS>
__device__ __forceinline__ void stage_whole(__nv_bfloat16* dst, const __nv_bfloat16* src, long long rs, int r_begin, int r_end,
                                            int n) {
  for (int i = r_begin * 8 + threadIdx.x; i < r_end * 8; i += THREADS) {
    const int r = i >> 3, c = i & 7;
    const bool ok = r < n;
    cp_async16(dst + swz(r, c), ok ? src + (long long)r * rs + c * 8 : src, ok);
  }
}

// shared memory: Q, K, V of the problem.  K and V arrive in two groups, the first 64 keys first, so the first key tile's
// MMAs start while the rest lands.  Warp w takes the 16-row groups w, w + 8, ...
template <bool LSE>
__global__ void __launch_bounds__(WF_THREADS, 2) attn_whole_fwd_kernel(const MmaAttn p) {
  constexpr int HD = 64, NW = WF_THREADS / 32;
  extern __shared__ __align__(16) uint8_t mma_smem[];
  const int N = p.Nq, R = (N + 15) & ~15, R0 = min(R, MT);
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(mma_smem);
  __nv_bfloat16* Ks = Qs + R * HD;
  __nv_bfloat16* Vs = Ks + R * HD;
  const int bh = blockIdx.x, b = bh / p.H, h = bh % p.H;
  const int warp = threadIdx.x >> 5;
  const __nv_bfloat16* kb = p.k + b * p.k_bs + h * p.k_hs;
  const __nv_bfloat16* vb = p.v + b * p.v_bs + h * p.v_hs;
  stage_whole<WF_THREADS>(Qs, p.q + b * p.q_bs + h * p.q_hs, p.q_rs, 0, R, N);
  stage_whole<WF_THREADS>(Ks, kb, p.k_rs, 0, R0, N);
  stage_whole<WF_THREADS>(Vs, vb, p.v_rs, 0, R0, N);
  cp_async_commit();
  stage_whole<WF_THREADS>(Ks, kb, p.k_rs, R0, R, N);
  stage_whole<WF_THREADS>(Vs, vb, p.v_rs, R0, R, N);
  cp_async_commit();
  cp_async_wait<1>();
  __syncthreads();
  const float c = p.scale * MMA_LOG2E;
  const int rounds = (R / 16 + NW - 1) / NW;
  for (int round = 0; round < rounds; ++round) {
    const int rb = (round * NW + warp) * 16;
    const bool active = rb < N;                 // warp-uniform
    uint32_t qa[HD / 16][4];
    if (active) load_a(qa, SwizzledTile(smem_addr(Qs), 0), rb);
    FwdAcc<HD> f;
    for (int k0 = 0; k0 < N; k0 += MT) {
      if (round == 0 && k0 == MT) {             // every thread passes here once: keys 64.. landed
        cp_async_wait<0>();
        __syncthreads();
      }
      if (!active) continue;
      fwd_tile<HD>(f, qa, SwizzledTile(smem_addr(Ks), k0), SwizzledTile(smem_addr(Vs), k0), k0, N, c);
    }
    if (active) fwd_store<HD, LSE>(f, p, b, h, rb);
  }
}

// The resident operands of one backward problem (attn_whole_bwd_kernel's shared memory).  Rebuilt from the launch in
// each task rather than carried across tasks, so that the registers go to the accumulators.
struct WholeBwd {
  uint32_t Qs, Ks, Vs, dOs;                     // shared-memory byte addresses of the [R][64] operands
  const float *lse_s, *del_s;                   // per query row, log2 domain / rowsum(dO * O); +inf / 0 past the end
  __device__ __forceinline__ WholeBwd(int N) {
    extern __shared__ __align__(16) uint8_t mma_smem[];
    const int R = (N + 15) & ~15, R64 = (N + MT - 1) & ~(MT - 1);
    Qs = smem_addr(mma_smem); Ks = Qs + R * 128; Vs = Ks + R * 128; dOs = Vs + R * 128;
    lse_s = reinterpret_cast<const float*>(mma_smem + 4 * R * 128);
    del_s = lse_s + R64;
  }
};

// dQ of query rows [rb, rb + 16)
__device__ __forceinline__ void whole_dq_task(const MmaAttn& p, int rb) {
  const int N = p.Nq, g = (threadIdx.x & 31) >> 2;
  const WholeBwd w(N);
  uint32_t qa[4][4], da[4][4];
  load_a(qa, SwizzledTile(w.Qs, 0), rb);
  load_a(da, SwizzledTile(w.dOs, 0), rb);
  const float lse0 = w.lse_s[rb + g], lse1 = w.lse_s[rb + g + 8], del0 = w.del_s[rb + g], del1 = w.del_s[rb + g + 8];
  float dq[8][4];
  zero(dq);
  const float c = p.scale * MMA_LOG2E;
  for (int k0 = 0; k0 < N; k0 += MT)
    dq_tile<64>(dq, qa, da, SwizzledTile(w.Ks, k0), SwizzledTile(w.Vs, k0), k0, N, c, lse0, lse1, del0, del1);
  dq_store<64>(dq, p, blockIdx.x / p.H, blockIdx.x % p.H, rb);
}

// dK and dV of key rows [rb, rb + 16)
__device__ __forceinline__ void whole_dkv_task(const MmaAttn& p, int rb) {
  const int N = p.Nq;
  const WholeBwd w(N);
  float dk[8][4], dv[8][4];
  zero(dk);
  zero(dv);
  const float c = p.scale * MMA_LOG2E;
  for (int q0 = 0; q0 < N; q0 += MT)
    dkv_tile<64>(dk, dv, SwizzledTile(w.Ks, 0), SwizzledTile(w.Vs, 0), rb, SwizzledTile(w.Qs, q0), SwizzledTile(w.dOs, q0), q0, N, c,
                 w.lse_s + q0, w.del_s + q0);
  dkv_store<64>(dk, dv, p, blockIdx.x / p.H, blockIdx.x % p.H, rb, false);   // attn_whole_ok: bf16 outputs only
}

// dQ, dK and dV of one problem in one CTA.  shared memory: Q, K, V, dO of the problem, then lse and delta of its rows
// (R64 = N rounded up to 64 of each; computed once, with row_delta).  The 2 * R / 16 tasks (dK / dV of 16 key rows, about
// 4/3 the work of dQ of 16 query rows) are independent; warps take them from a counter in shared memory, the dK / dV
// tasks first.
__global__ void __launch_bounds__(WB_THREADS, 2) attn_whole_bwd_kernel(const MmaAttn p) {
  constexpr int HD = 64;
  extern __shared__ __align__(16) uint8_t mma_smem[];
  __shared__ int next_task;
  const int N = p.Nq, R = (N + 15) & ~15, R64 = (N + MT - 1) & ~(MT - 1);
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(mma_smem);
  __nv_bfloat16* Ks = Qs + R * HD;
  __nv_bfloat16* Vs = Ks + R * HD;
  __nv_bfloat16* dOs = Vs + R * HD;
  float* lse_s = reinterpret_cast<float*>(dOs + R * HD);
  float* del_s = lse_s + R64;
  const int bh = blockIdx.x, b = bh / p.H, h = bh % p.H;
  const int lane = threadIdx.x & 31;
  stage_whole<WB_THREADS>(Qs, p.q + b * p.q_bs + h * p.q_hs, p.q_rs, 0, R, N);
  stage_whole<WB_THREADS>(Ks, p.k + b * p.k_bs + h * p.k_hs, p.k_rs, 0, R, N);
  stage_whole<WB_THREADS>(Vs, p.v + b * p.v_bs + h * p.v_hs, p.v_rs, 0, R, N);
  stage_whole<WB_THREADS>(dOs, p.dout + b * p.o_bs + h * p.o_hs, p.o_rs, 0, R, N);
  cp_async_commit();
  if (threadIdx.x == 0) next_task = 0;
  cp_async_wait<0>();
  __syncthreads();
  // lse (log2 domain) and delta of every row, two threads per row as in stage_row_stats
  const __nv_bfloat16* ob = p.o + b * p.o_bs + h * p.o_hs;
  const float* lrow = p.lse + (long long)bh * N;
  for (int r0 = 0; r0 < R64; r0 += WB_THREADS / 2) {
    const int r = r0 + (threadIdx.x >> 1), half = threadIdx.x & 1;
    const bool ok = r < N;
    const float d = row_delta<HD>(ok, half, [=](int c) { return ld32(dOs + swz(r, c >> 3) + (c & 7)); }, ob + (long long)r * p.o_rs);
    if (half == 0 && r < R64) {
      del_s[r] = d;
      lse_s[r] = ok ? lrow[r] * MMA_LOG2E : INFINITY;
    }
  }
  __syncthreads();
  for (;;) {
    int task = 0;
    if (lane == 0) task = atomicAdd(&next_task, 1);
    task = __shfl_sync(0xffffffffu, task, 0) * 16;   // tasks [0, R): dK / dV of key rows task..; [R, 2R): dQ
    const int rows = (p.Nq + 15) & ~15;             // R, reread rather than held across the tasks
    if (task >= 2 * rows) break;
    if (task < rows) whole_dkv_task(p, task);
    else whole_dq_task(p, task - rows);
  }
}

// ------------------------------------------------------------------------------------------------ host side
bool mma_layout_ok(const void* ptr, long long bs, long long hs, long long rs, int hd) {
  return ((uintptr_t)ptr & 15) == 0 && bs % 8 == 0 && hs % 8 == 0 && rs % 8 == 0 && (hs == hd || rs == hd);
}

// dynamic shared memory of each kernel: bf16 tiles of MT x (HD + 8), then fp32 rows of MT
template <int HD>
static constexpr int tile_bytes() { return MT * (HD + 8) * 2; }
template <int HD>
static constexpr int fwd_smem() { return 5 * tile_bytes<HD>(); }
template <int HD>
static constexpr int dq_smem() { return 6 * tile_bytes<HD>() + 2 * MT * 4; }
template <int HD>
static constexpr int dkv_smem() { return 8 * tile_bytes<HD>() + 4 * MT * 4; }

// one launch of `Kern`; its shared-memory limit is raised on first use
template <auto Kern>
static int launch(dim3 grid, int smem, const MmaAttn& a, cudaStream_t st, const char* what) {
  static bool done = false;
  if (!done) {
    cudaError_t e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    VT_REQUIRE(e == cudaSuccess, "%s: smem attribute: %s", what, cudaGetErrorString(e));
    done = true;
  }
  Kern<<<grid, MMA_THREADS, smem, st>>>(a);
  return check_launch(what);
}

template <int HD>
static int mma_fwd_launch(const MmaAttn& a, dim3 grid, cudaStream_t st) {
  if constexpr (HD == 64 || HD == 96) {
    const char* what = "attn_mma_fwd_kernel";
    if (a.lse) return launch<attn_mma_fwd_kernel<HD, true>>(grid, fwd_smem<HD>(), a, st, what);
    return launch<attn_mma_fwd_kernel<HD, false>>(grid, fwd_smem<HD>(), a, st, what);
  } else {
    const char* what = "attn_tc_fwd_kernel";
    if (a.lse) return launch<attn_tc_fwd_kernel<HD, true>>(grid, fwd_smem<HD>(), a, st, what);
    return launch<attn_tc_fwd_kernel<HD, false>>(grid, fwd_smem<HD>(), a, st, what);
  }
}

template <int HD>
static int mma_bwd_launch(const MmaAttn& a, dim3 gq, dim3 gk, cudaStream_t st) {
  int rc;
  if constexpr (HD == 64 || HD == 96) {
    if ((rc = launch<attn_mma_dq_kernel<HD>>(gq, dq_smem<HD>(), a, st, "attn_mma_dq_kernel"))) return rc;
    return launch<attn_mma_dkv_kernel<HD>>(gk, dkv_smem<HD>(), a, st, "attn_mma_dkv_kernel");
  } else {
    if ((rc = launch<attn_tc_dq_kernel<HD>>(gq, dq_smem<HD>(), a, st, "attn_tc_dq_kernel"))) return rc;
    return launch<attn_tc_dkv_kernel<HD>>(gk, dkv_smem<HD>(), a, st, "attn_tc_dkv_kernel");
  }
}

int attn_mma_fwd(const MmaAttn& a, int B, int hd, cudaStream_t st) {
  VT_REQUIRE(attn_head_dim_ok(hd), "tensor-core attention: head dim %d unsupported (32, 64, 96 or 128)", hd);
  VT_REQUIRE((long long)B * a.H <= 65535, "tensor-core attention: B*H too large");
  const dim3 grid((a.Nq + MT - 1) / MT, B * a.H);
  return with_head_dim(hd, [&](auto d) { return mma_fwd_launch<d.value>(a, grid, st); });
}

int attn_mma_bwd(const MmaAttn& a, int B, int hd, cudaStream_t st) {
  VT_REQUIRE(attn_head_dim_ok(hd), "tensor-core attention: head dim %d unsupported (32, 64, 96 or 128)", hd);
  VT_REQUIRE((long long)B * a.H <= 65535, "tensor-core attention: B*H too large");
  const dim3 gq((a.Nq + MT - 1) / MT, B * a.H), gk((a.Nk + MT - 1) / MT, B * a.H);
  return with_head_dim(hd, [&](auto d) { return mma_bwd_launch<d.value>(a, gq, gk, st); });
}

bool attn_whole_ok(const MmaAttn& a, int hd) {
  return hd == 64 && a.Nq == a.Nk && a.Nq >= 1 && a.Nq <= WHOLE_MAX_N && !a.dk32 && !a.delta;
}

// [R][64] bf16 operands, R = N rounded up to 16; the backward adds two fp32 rows of N rounded up to 64
static int whole_fwd_smem(int n) { return 3 * ((n + 15) & ~15) * 64 * 2; }
static int whole_bwd_smem(int n) { return 4 * ((n + 15) & ~15) * 64 * 2 + 2 * ((n + MT - 1) & ~(MT - 1)) * 4; }

// one CTA per problem; the shared-memory limit is raised to the largest N's on first use, with the carveout that lets
// two CTAs share an SM
template <auto Kern>
static int launch_whole(int problems, int threads, int smem, int smem_max, const MmaAttn& a, cudaStream_t st, const char* what) {
  static bool done = false;
  if (!done) {
    cudaError_t e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(Kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    VT_REQUIRE(e == cudaSuccess, "%s: smem attribute: %s", what, cudaGetErrorString(e));
    done = true;
  }
  Kern<<<problems, threads, smem, st>>>(a);
  return check_launch(what);
}

int attn_whole_fwd(const MmaAttn& a, int B, cudaStream_t st) {
  VT_REQUIRE(attn_whole_ok(a, 64), "attn_whole_fwd: unsupported operands (N=%d)", a.Nq);
  VT_REQUIRE((long long)B * a.H <= 65535, "tensor-core attention: B*H too large");   // the tiled kernels' limit, kept
  const int smem = whole_fwd_smem(a.Nq), smax = whole_fwd_smem(WHOLE_MAX_N);
  return a.lse ? launch_whole<attn_whole_fwd_kernel<true>>(B * a.H, WF_THREADS, smem, smax, a, st, "attn_whole_fwd_kernel")
               : launch_whole<attn_whole_fwd_kernel<false>>(B * a.H, WF_THREADS, smem, smax, a, st, "attn_whole_fwd_kernel");
}

int attn_whole_bwd(const MmaAttn& a, int B, cudaStream_t st) {
  VT_REQUIRE(attn_whole_ok(a, 64), "attn_whole_bwd: unsupported operands (N=%d)", a.Nq);
  VT_REQUIRE((long long)B * a.H <= 65535, "tensor-core attention: B*H too large");
  return launch_whole<attn_whole_bwd_kernel>(B * a.H, WB_THREADS, whole_bwd_smem(a.Nq), whole_bwd_smem(WHOLE_MAX_N), a, st,
                                             "attn_whole_bwd_kernel");
}

}  // namespace vt
