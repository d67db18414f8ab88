// Tensor-core flash attention for sm_90a (mma.sync.m16n8k16, bf16 operands, fp32 accumulators), head dim 64 or 96.
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
// ldmatrix phase in distinct banks at both head dims, so no swizzle is needed.  MMAs whose operands are all padding are
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
// Each group runs the per-warp arithmetic of the tiled kernels unchanged, so o, lse, dq, dk and dv are the same bits;
// VT_ATTN_WHOLE=0 selects the tiled kernels instead (vt_attention.cu).  vt_xattn_* always takes the tiled kernels.
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

// four 8x8 bf16 matrices; lane l supplies the address of row l % 8 of matrix l / 8
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const __nv_bfloat16* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_addr(p)));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const __nv_bfloat16* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_addr(p)));
}
// Per-lane ldmatrix offsets into a [rows][P] tile (tests/test_attn_fragments_sim.py walks both against the mma layout):
//   lane_a: x4 at (r0, c0) -> A fragment {a0..a3} of rows r0..r0+15, cols c0..c0+15; with .trans at (k0, n0) of a
//           row-major [k][n] tile -> B fragments {b0, b1} of n block n0 and {b0, b1} of n block n0 + 8 (k rows k0..k0+15).
//   lane_b: x4 at (n0, c0) of an [n][k] tile -> {b0, b1} of n block n0, then of n block n0 + 8, k cols c0..c0+15.
template <int P>
__device__ __forceinline__ int lane_a(int lane) { return (lane & 15) * P + (lane >> 4) * 8; }
template <int P>
__device__ __forceinline__ int lane_b(int lane) { return ((lane & 7) + (lane >> 4) * 8) * P + ((lane >> 3) & 1) * 8; }

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
// lse (log2 domain; +inf past the end: p = 0) and delta = rowsum(dO * O) of rows [r0, r0 + MT).  dOs is the staged dO
// tile; orow / o_rs and lrow address O and lse of row r0 (global memory, or a staged tile); delta_out is optional
template <int HD>
__device__ __forceinline__ void stage_row_stats(float* lse_s, float* del_s, const __nv_bfloat16* dOs, const __nv_bfloat16* orow,
                                                long long o_rs, const float* lrow, int r0, int limit, float* delta_out) {
  const int r = threadIdx.x >> 1, half = threadIdx.x & 1;
  const bool ok = r0 + r < limit;
  float d = 0.f;
  if (ok) {
#pragma unroll 4
    for (int c = half * (HD / 2); c < (half + 1) * (HD / 2); c += 2) {
      const float2 g = unpack_bf16x2(ld32(dOs + r * (HD + 8) + c));
      const float2 o = unpack_bf16x2(ld32(orow + r * o_rs + c));
      d = fmaf(g.x, o.x, fmaf(g.y, o.y, d));
    }
  }
  d += __shfl_xor_sync(0xffffffffu, d, 1);
  if (half == 0) {
    del_s[r] = d;
    lse_s[r] = ok ? lrow[r] * MMA_LOG2E : INFINITY;
    if (ok && delta_out) delta_out[r0 + r] = d;
  }
}

// ------------------------------------------------------------------------------------------------ forward
// LSE = false: p.lse is not written (forward-only calls); a template flag, so the saving form's code is unchanged
// shared memory: Q, then a ring of two (K, V) stages
template <int HD, bool LSE>
__global__ void __launch_bounds__(MMA_THREADS) attn_mma_fwd_kernel(const MmaAttn p) {
  constexpr int P = HD + 8, NB = HD / 8, KC = HD / 16, TILE = MT * P;
  extern __shared__ __align__(16) uint8_t mma_smem[];
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(mma_smem);
  __nv_bfloat16* ring = Qs + TILE;
  const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H;
  const int q0 = blockIdx.x * MT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, rb = warp * 16;
  const int la = lane_a<P>(lane), lb = lane_b<P>(lane);
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
  uint32_t qa[KC][4];
#pragma unroll
  for (int kc = 0; kc < KC; ++kc) ldsm_x4(qa[kc], Qs + rb * P + kc * 16 + la);
  float o[NB][4];
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) o[nb][0] = o[nb][1] = o[nb][2] = o[nb][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
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
    const __nv_bfloat16* Vs = Ks + TILE;
    float s[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) s[nb][0] = s[nb][1] = s[nb][2] = s[nb][3] = 0.f;
#pragma unroll
    for (int nb = 0; nb < 8; nb += 2) {
      if (k0 + nb * 8 >= p.Nk) break;           // n8 blocks past the last key stay 0 and are masked below
      const bool hi = k0 + nb * 8 + 8 < p.Nk;
#pragma unroll
      for (int kc = 0; kc < KC; ++kc) {
        uint32_t kf[4];
        ldsm_x4(kf, Ks + nb * 8 * P + kc * 16 + lb);
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
        const float v = key < p.Nk ? s[nb][e] * c : -INFINITY;
        s[nb][e] = v;
        if (e < 2) mx0 = fmaxf(mx0, v); else mx1 = fmaxf(mx1, v);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);      // finite: every tile holds at least one key
    const float corr0 = fast_exp2(m0 - mn0), corr1 = fast_exp2(m1 - mn1);
    l0 *= corr0; l1 *= corr1;
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) { o[nb][0] *= corr0; o[nb][1] *= corr0; o[nb][2] *= corr1; o[nb][3] *= corr1; }
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
      s[nb][0] = fast_exp2(s[nb][0] - mn0); s[nb][1] = fast_exp2(s[nb][1] - mn0);
      s[nb][2] = fast_exp2(s[nb][2] - mn1); s[nb][3] = fast_exp2(s[nb][3] - mn1);
      l0 += s[nb][0] + s[nb][1];
      l1 += s[nb][2] + s[nb][3];
    }
    m0 = mn0; m1 = mn1;
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) {
      if (k0 + kc * 16 >= p.Nk) break;          // P = 0 over the whole chunk
      const uint32_t a0 = pack_bf16x2(s[2 * kc][0], s[2 * kc][1]), a1 = pack_bf16x2(s[2 * kc][2], s[2 * kc][3]);
      const uint32_t a2 = pack_bf16x2(s[2 * kc + 1][0], s[2 * kc + 1][1]), a3 = pack_bf16x2(s[2 * kc + 1][2], s[2 * kc + 1][3]);
#pragma unroll
      for (int nb = 0; nb < NB; nb += 2) {
        uint32_t vf[4];
        ldsm_x4_t(vf, Vs + kc * 16 * P + nb * 8 + la);
        mma16816(o[nb], a0, a1, a2, a3, vf[0], vf[1]);
        mma16816(o[nb + 1], a0, a1, a2, a3, vf[2], vf[3]);
      }
    }
  }
  if (!active) return;
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
  __nv_bfloat16* ob = p.o_out + b * p.o_bs + h * p.o_hs;
  const int r0 = q0 + rb + g, r1 = r0 + 8;
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) {
    if (r0 < p.Nq) *reinterpret_cast<uint32_t*>(ob + (long long)r0 * p.o_rs + nb * 8 + 2 * t) = pack_bf16x2(o[nb][0] * inv0, o[nb][1] * inv0);
    if (r1 < p.Nq) *reinterpret_cast<uint32_t*>(ob + (long long)r1 * p.o_rs + nb * 8 + 2 * t) = pack_bf16x2(o[nb][2] * inv1, o[nb][3] * inv1);
  }
  if (LSE && t == 0) {
    if (r0 < p.Nq) p.lse[(long long)bh * p.Nq + r0] = (m0 + log2f(l0)) * MMA_LN2;
    if (r1 < p.Nq) p.lse[(long long)bh * p.Nq + r1] = (m1 + log2f(l1)) * MMA_LN2;
  }
}

// ------------------------------------------------------------------------------------------------ dQ
// shared memory: Q, dO, a ring of two (K, V) stages, lse and delta of the CTA's rows
template <int HD>
__global__ void __launch_bounds__(MMA_THREADS) attn_mma_dq_kernel(const MmaAttn p) {
  constexpr int P = HD + 8, NB = HD / 8, KC = HD / 16, TILE = MT * P;
  extern __shared__ __align__(16) uint8_t mma_smem[];
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(mma_smem);
  __nv_bfloat16* dOs = Qs + TILE;
  __nv_bfloat16* ring = dOs + TILE;
  float* lse_s = reinterpret_cast<float*>(ring + 4 * TILE);
  float* del_s = lse_s + MT;
  const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H;
  const int q0 = blockIdx.x * MT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, rb = warp * 16;
  const int la = lane_a<P>(lane), lb = lane_b<P>(lane);
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
  uint32_t qa[KC][4], da[KC][4];
#pragma unroll
  for (int kc = 0; kc < KC; ++kc) {
    ldsm_x4(qa[kc], Qs + rb * P + kc * 16 + la);
    ldsm_x4(da[kc], dOs + rb * P + kc * 16 + la);
  }
  __syncthreads();
  const float lse0 = lse_s[rb + g], lse1 = lse_s[rb + g + 8], del0 = del_s[rb + g], del1 = del_s[rb + g + 8];
  float dq[NB][4];
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) dq[nb][0] = dq[nb][1] = dq[nb][2] = dq[nb][3] = 0.f;
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
    const __nv_bfloat16* Vs = Ks + TILE;
    float s[8][4], dpv[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) s[nb][e] = dpv[nb][e] = 0.f;
    }
#pragma unroll
    for (int nb = 0; nb < 8; nb += 2) {
      if (k0 + nb * 8 >= p.Nk) break;
      const bool hi = k0 + nb * 8 + 8 < p.Nk;
#pragma unroll
      for (int kc = 0; kc < KC; ++kc) {
        uint32_t kf[4], vf[4];
        ldsm_x4(kf, Ks + nb * 8 * P + kc * 16 + lb);
        ldsm_x4(vf, Vs + nb * 8 * P + kc * 16 + lb);
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
        const float pr = key < p.Nk ? fast_exp2(s[nb][e] * c - (e < 2 ? lse0 : lse1)) : 0.f;
        s[nb][e] = pr * (dpv[nb][e] - (e < 2 ? del0 : del1));
      }
    }
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) {
      if (k0 + kc * 16 >= p.Nk) break;          // dS = 0 over the whole chunk
      const uint32_t a0 = pack_bf16x2(s[2 * kc][0], s[2 * kc][1]), a1 = pack_bf16x2(s[2 * kc][2], s[2 * kc][3]);
      const uint32_t a2 = pack_bf16x2(s[2 * kc + 1][0], s[2 * kc + 1][1]), a3 = pack_bf16x2(s[2 * kc + 1][2], s[2 * kc + 1][3]);
#pragma unroll
      for (int nb = 0; nb < NB; nb += 2) {
        uint32_t kf[4];
        ldsm_x4_t(kf, Ks + kc * 16 * P + nb * 8 + la);
        mma16816(dq[nb], a0, a1, a2, a3, kf[0], kf[1]);
        mma16816(dq[nb + 1], a0, a1, a2, a3, kf[2], kf[3]);
      }
    }
  }
  if (!active) return;
  __nv_bfloat16* dqb = p.dq + b * p.dq_bs + h * p.dq_hs;
  const int r0 = q0 + rb + g, r1 = r0 + 8;
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) {
    if (r0 < p.Nq)
      *reinterpret_cast<uint32_t*>(dqb + (long long)r0 * p.dq_rs + nb * 8 + 2 * t) = pack_bf16x2(dq[nb][0] * p.scale, dq[nb][1] * p.scale);
    if (r1 < p.Nq)
      *reinterpret_cast<uint32_t*>(dqb + (long long)r1 * p.dq_rs + nb * 8 + 2 * t) = pack_bf16x2(dq[nb][2] * p.scale, dq[nb][3] * p.scale);
  }
}

// ------------------------------------------------------------------------------------------------ dK / dV
// shared memory: K, V, a ring of two (Q, dO, O) stages, the ring's two lse rows, lse and delta of the current query tile.
// At head dim 64 three CTAs fit an SM (162 registers without spills, 75 KB); at 96 the register cap would spill.
template <int HD>
__global__ void __launch_bounds__(MMA_THREADS, HD == 64 ? 3 : 1) attn_mma_dkv_kernel(const MmaAttn p) {
  constexpr int P = HD + 8, NB = HD / 8, KC = HD / 16, TILE = MT * P;
  extern __shared__ __align__(16) uint8_t mma_smem[];
  __nv_bfloat16* Ks = reinterpret_cast<__nv_bfloat16*>(mma_smem);
  __nv_bfloat16* Vs = Ks + TILE;
  __nv_bfloat16* ring = Vs + TILE;
  float* lse_ring = reinterpret_cast<float*>(ring + 6 * TILE);
  float* lse_s = lse_ring + 2 * MT;
  float* del_s = lse_s + MT;
  const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H;
  const int k0 = blockIdx.x * MT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, rb = warp * 16;
  const int la = lane_a<P>(lane), lb = lane_b<P>(lane);
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
  float dk[NB][4], dv[NB][4];
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) {
#pragma unroll
    for (int e = 0; e < 4; ++e) dk[nb][e] = dv[nb][e] = 0.f;
  }
  const float c = p.scale * MMA_LOG2E;
  for (int q0 = 0, it = 0; q0 < p.Nq; q0 += MT, ++it) {
    cp_async_wait<0>();
    __syncthreads();                            // tile `it` landed; stage it + 1, lse_s and del_s are no longer read
    if (q0 + MT < p.Nq) stage_tile((it + 1) & 1, q0 + MT);
    const __nv_bfloat16* Qs = ring + (it & 1) * 3 * TILE;
    const __nv_bfloat16* dOs = Qs + TILE;
    stage_row_stats<HD>(lse_s, del_s, dOs, dOs + TILE, P, lse_ring + (it & 1) * MT, q0, p.Nq, nullptr);
    __syncthreads();
    if (!active) continue;
    float s[8][4], dpv[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) s[nb][e] = dpv[nb][e] = 0.f;
    }
#pragma unroll
    for (int kc = 0; kc < KC; ++kc) {
      uint32_t ka[4], va[4];
      ldsm_x4(ka, Ks + rb * P + kc * 16 + la);
      ldsm_x4(va, Vs + rb * P + kc * 16 + la);
#pragma unroll
      for (int nb = 0; nb < 8; nb += 2) {
        if (q0 + nb * 8 >= p.Nq) break;         // n8 blocks past the last query stay 0: lse_s = +inf there, P = 0
        uint32_t qf[4], df[4];
        ldsm_x4(qf, Qs + nb * 8 * P + kc * 16 + lb);
        ldsm_x4(df, dOs + nb * 8 * P + kc * 16 + lb);
        mma16816(s[nb], ka[0], ka[1], ka[2], ka[3], qf[0], qf[1]);
        mma16816(dpv[nb], va[0], va[1], va[2], va[3], df[0], df[1]);
        if (q0 + nb * 8 + 8 < p.Nq) {
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
        const float pr = fast_exp2(s[nb][e] * c - lse_s[qi]);      // lse_s = +inf past the end: 0
        s[nb][e] = pr;
        dpv[nb][e] = pr * (dpv[nb][e] - del_s[qi]);
      }
    }
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) {
      if (q0 + kc * 16 >= p.Nq) break;          // P = dS = 0 over the whole chunk
      const uint32_t p0 = pack_bf16x2(s[2 * kc][0], s[2 * kc][1]), p1 = pack_bf16x2(s[2 * kc][2], s[2 * kc][3]);
      const uint32_t p2 = pack_bf16x2(s[2 * kc + 1][0], s[2 * kc + 1][1]), p3 = pack_bf16x2(s[2 * kc + 1][2], s[2 * kc + 1][3]);
      const uint32_t d0 = pack_bf16x2(dpv[2 * kc][0], dpv[2 * kc][1]), d1 = pack_bf16x2(dpv[2 * kc][2], dpv[2 * kc][3]);
      const uint32_t d2 = pack_bf16x2(dpv[2 * kc + 1][0], dpv[2 * kc + 1][1]), d3 = pack_bf16x2(dpv[2 * kc + 1][2], dpv[2 * kc + 1][3]);
#pragma unroll
      for (int nb = 0; nb < NB; nb += 2) {
        uint32_t gf[4], qf[4];
        ldsm_x4_t(gf, dOs + kc * 16 * P + nb * 8 + la);
        ldsm_x4_t(qf, Qs + kc * 16 * P + nb * 8 + la);
        mma16816(dv[nb], p0, p1, p2, p3, gf[0], gf[1]);
        mma16816(dv[nb + 1], p0, p1, p2, p3, gf[2], gf[3]);
        mma16816(dk[nb], d0, d1, d2, d3, qf[0], qf[1]);
        mma16816(dk[nb + 1], d0, d1, d2, d3, qf[2], qf[3]);
      }
    }
  }
  if (!active) return;
  const int r0 = k0 + rb + g, r1 = r0 + 8;
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) {
    const int col = nb * 8 + 2 * t;
    if (p.dk32) {
      float* dkb = p.dk32 + (long long)bh * p.Nk * HD;
      float* dvb = p.dv32 + (long long)bh * p.Nk * HD;
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

// ------------------------------------------------------------------------------------------------ whole problems
// Packed-qkv attention at head dim 64 and N <= WHOLE_MAX_N (Nq == Nk): a CTA owns one (b, h) problem and keeps its
// operands resident in shared memory, so each is read from L2 once and no CTA works on a partial 64-row tile alone.
// Warps own 16-row groups; each group runs exactly the per-warp arithmetic of the tiled kernels above (64-row tile
// walk, the same MMAs, the same skipping and the same bf16 roundings), so the results are the same bits.
// Operands are [R][64] bf16, R = N rounded up to 16 (rows >= N zero-filled: the 16-row reads of the last group and the
// k16 chunks past the end see the zeros the tiled kernels stage), with an XOR swizzle instead of a pad: the 16-byte
// chunk c of row r sits at chunk c ^ (r & 7), so the 8 rows of every ldmatrix phase fall in distinct bank groups.
constexpr int WHOLE_MAX_N = 256;
constexpr int WF_THREADS = 256;     // forward: 8 warps, two CTAs per SM
constexpr int WB_THREADS = 192;     // backward: 6 warps, two CTAs per SM (12 warps at <= 168 registers)

__device__ __forceinline__ int swz(int r, int c) { return r * 64 + ((c ^ (r & 7)) << 3); }
// The swizzled lane_a / lane_b: a lane's row offset ar / br and chunk key ak / bk, so that the fragment at (r0, c0),
// r0 % 8 == 0 and c0 % 16 == 0, is read at sw_at(row, key, r0, c0) (c0 / 8 is even: (c0 / 8 + lc) ^ (r & 7) ==
// (c0 / 8) ^ (lc ^ (r & 7)))
__device__ __forceinline__ int sw_at(int row, int key, int r0, int c0) { return row + r0 * 64 + (((c0 >> 3) ^ key) << 3); }
// the same in bytes (row = the lane's row offset in bytes), for ldmatrix on a 32-bit shared address
__device__ __forceinline__ uint32_t sw_at_b(int row, int key, int r0, int c0) { return row + r0 * 128 + (((c0 >> 3) ^ key) << 4); }
__device__ __forceinline__ void ldsm_x4_s(uint32_t (&r)[4], uint32_t a) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_ts(uint32_t (&r)[4], uint32_t a) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}

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
  constexpr int HD = 64, NB = 8, KC = 4, NW = WF_THREADS / 32;
  extern __shared__ __align__(16) uint8_t mma_smem[];
  const int N = p.Nq, R = (N + 15) & ~15, R0 = min(R, MT);
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(mma_smem);
  __nv_bfloat16* Ks = Qs + R * HD;
  __nv_bfloat16* Vs = Ks + R * HD;
  const int bh = blockIdx.x, b = bh / p.H, h = bh % p.H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int ar = (lane & 15) * HD, ak = (lane >> 4) ^ (lane & 7);
  const int br = ((lane & 7) + (lane >> 4) * 8) * HD, bk = ((lane >> 3) & 1) ^ (lane & 7);
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
    uint32_t qa[KC][4];
    if (active) {
#pragma unroll
      for (int kc = 0; kc < KC; ++kc) ldsm_x4(qa[kc], Qs + sw_at(ar, ak, rb, kc * 16));
    }
    float o[NB][4];
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) o[nb][0] = o[nb][1] = o[nb][2] = o[nb][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    for (int k0 = 0; k0 < N; k0 += MT) {
      if (round == 0 && k0 == MT) {             // every thread passes here once: keys 64.. landed
        cp_async_wait<0>();
        __syncthreads();
      }
      if (!active) continue;
      float s[8][4];
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) s[nb][0] = s[nb][1] = s[nb][2] = s[nb][3] = 0.f;
#pragma unroll
      for (int nb = 0; nb < 8; nb += 2) {
        if (k0 + nb * 8 >= N) break;
        const bool hi = k0 + nb * 8 + 8 < N;
#pragma unroll
        for (int kc = 0; kc < KC; ++kc) {
          uint32_t kf[4];
          ldsm_x4(kf, Ks + sw_at(br, bk, k0 + nb * 8, kc * 16));
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
      const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
      const float corr0 = fast_exp2(m0 - mn0), corr1 = fast_exp2(m1 - mn1);
      l0 *= corr0; l1 *= corr1;
#pragma unroll
      for (int nb = 0; nb < NB; ++nb) { o[nb][0] *= corr0; o[nb][1] *= corr0; o[nb][2] *= corr1; o[nb][3] *= corr1; }
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) {
        s[nb][0] = fast_exp2(s[nb][0] - mn0); s[nb][1] = fast_exp2(s[nb][1] - mn0);
        s[nb][2] = fast_exp2(s[nb][2] - mn1); s[nb][3] = fast_exp2(s[nb][3] - mn1);
        l0 += s[nb][0] + s[nb][1];
        l1 += s[nb][2] + s[nb][3];
      }
      m0 = mn0; m1 = mn1;
#pragma unroll
      for (int kc = 0; kc < 4; ++kc) {
        if (k0 + kc * 16 >= N) break;
        const uint32_t a0 = pack_bf16x2(s[2 * kc][0], s[2 * kc][1]), a1 = pack_bf16x2(s[2 * kc][2], s[2 * kc][3]);
        const uint32_t a2 = pack_bf16x2(s[2 * kc + 1][0], s[2 * kc + 1][1]), a3 = pack_bf16x2(s[2 * kc + 1][2], s[2 * kc + 1][3]);
#pragma unroll
        for (int nb = 0; nb < NB; nb += 2) {
          uint32_t vf[4];
          ldsm_x4_t(vf, Vs + sw_at(ar, ak, k0 + kc * 16, nb * 8));
          mma16816(o[nb], a0, a1, a2, a3, vf[0], vf[1]);
          mma16816(o[nb + 1], a0, a1, a2, a3, vf[2], vf[3]);
        }
      }
    }
    if (!active) continue;
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
    __nv_bfloat16* ob = p.o_out + b * p.o_bs + h * p.o_hs;
    const int r0 = rb + g, r1 = r0 + 8;
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) {
      if (r0 < N) *reinterpret_cast<uint32_t*>(ob + (long long)r0 * p.o_rs + nb * 8 + 2 * t) = pack_bf16x2(o[nb][0] * inv0, o[nb][1] * inv0);
      if (r1 < N) *reinterpret_cast<uint32_t*>(ob + (long long)r1 * p.o_rs + nb * 8 + 2 * t) = pack_bf16x2(o[nb][2] * inv1, o[nb][3] * inv1);
    }
    if (LSE && t == 0) {
      if (r0 < N) p.lse[(long long)bh * N + r0] = (m0 + log2f(l0)) * MMA_LN2;
      if (r1 < N) p.lse[(long long)bh * N + r1] = (m1 + log2f(l1)) * MMA_LN2;
    }
  }
}

// The resident operands of one backward problem (attn_whole_bwd_kernel's shared memory) and the lane offsets into them.
// Rebuilt from the launch in each task rather than carried across tasks, so that the registers go to the accumulators.
struct WholeBwd {
  uint32_t Qs, Ks, Vs, dOs;                     // shared-memory byte addresses of the [R][64] operands
  const float *lse_s, *del_s;                   // per query row, log2 domain / rowsum(dO * O); +inf / 0 past the end
  int ar, ak, br, bk;
  __device__ __forceinline__ WholeBwd(int N) {
    extern __shared__ __align__(16) uint8_t mma_smem[];
    const int R = (N + 15) & ~15, R64 = (N + MT - 1) & ~(MT - 1), lane = threadIdx.x & 31;
    Qs = smem_addr(mma_smem); Ks = Qs + R * 128; Vs = Ks + R * 128; dOs = Vs + R * 128;
    lse_s = reinterpret_cast<const float*>(mma_smem + 4 * R * 128);
    del_s = lse_s + R64;
    ar = (lane & 15) * 128; ak = (lane >> 4) ^ (lane & 7);
    br = ((lane & 7) + (lane >> 4) * 8) * 128; bk = ((lane >> 3) & 1) ^ (lane & 7);
  }
};

// dQ of query rows [rb, rb + 16): attn_mma_dq_kernel's warp, with K and V read from the resident copies
__device__ __forceinline__ void whole_dq_task(const MmaAttn& p, int rb) {
  constexpr int NB = 8, KC = 4;
  const int N = p.Nq, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const WholeBwd w(N);
  uint32_t qa[KC][4], da[KC][4];
#pragma unroll
  for (int kc = 0; kc < KC; ++kc) {
    ldsm_x4_s(qa[kc], w.Qs + sw_at_b(w.ar, w.ak, rb, kc * 16));
    ldsm_x4_s(da[kc], w.dOs + sw_at_b(w.ar, w.ak, rb, kc * 16));
  }
  const float lse0 = w.lse_s[rb + g], lse1 = w.lse_s[rb + g + 8], del0 = w.del_s[rb + g], del1 = w.del_s[rb + g + 8];
  float dq[NB][4];
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) dq[nb][0] = dq[nb][1] = dq[nb][2] = dq[nb][3] = 0.f;
  const float c = p.scale * MMA_LOG2E;
  for (int k0 = 0; k0 < N; k0 += MT) {
    float s[8][4], dpv[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) s[nb][e] = dpv[nb][e] = 0.f;
    }
#pragma unroll
    for (int nb = 0; nb < 8; nb += 2) {
      if (k0 + nb * 8 >= N) break;
      const bool hi = k0 + nb * 8 + 8 < N;
#pragma unroll
      for (int kc = 0; kc < KC; ++kc) {
        uint32_t kf[4], vf[4];
        ldsm_x4_s(kf, w.Ks + sw_at_b(w.br, w.bk, k0 + nb * 8, kc * 16));
        ldsm_x4_s(vf, w.Vs + sw_at_b(w.br, w.bk, k0 + nb * 8, kc * 16));
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
      if (k0 + kc * 16 >= N) break;
      const uint32_t a0 = pack_bf16x2(s[2 * kc][0], s[2 * kc][1]), a1 = pack_bf16x2(s[2 * kc][2], s[2 * kc][3]);
      const uint32_t a2 = pack_bf16x2(s[2 * kc + 1][0], s[2 * kc + 1][1]), a3 = pack_bf16x2(s[2 * kc + 1][2], s[2 * kc + 1][3]);
#pragma unroll
      for (int nb = 0; nb < NB; nb += 2) {
        uint32_t kf[4];
        ldsm_x4_ts(kf, w.Ks + sw_at_b(w.ar, w.ak, k0 + kc * 16, nb * 8));
        mma16816(dq[nb], a0, a1, a2, a3, kf[0], kf[1]);
        mma16816(dq[nb + 1], a0, a1, a2, a3, kf[2], kf[3]);
      }
    }
  }
  const int b = blockIdx.x / p.H, h = blockIdx.x % p.H;
  __nv_bfloat16* dqb = p.dq + b * p.dq_bs + h * p.dq_hs;
  const int r0 = rb + g, r1 = r0 + 8;
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) {
    if (r0 < N)
      *reinterpret_cast<uint32_t*>(dqb + (long long)r0 * p.dq_rs + nb * 8 + 2 * t) = pack_bf16x2(dq[nb][0] * p.scale, dq[nb][1] * p.scale);
    if (r1 < N)
      *reinterpret_cast<uint32_t*>(dqb + (long long)r1 * p.dq_rs + nb * 8 + 2 * t) = pack_bf16x2(dq[nb][2] * p.scale, dq[nb][3] * p.scale);
  }
}

// dK and dV of key rows [rb, rb + 16): attn_mma_dkv_kernel's warp, with Q, dO and the row stats read from the
// resident copies; bf16 outputs
__device__ __forceinline__ void whole_dkv_task(const MmaAttn& p, int rb) {
  constexpr int NB = 8, KC = 4;
  const int N = p.Nq, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const WholeBwd w(N);
  float dk[NB][4], dv[NB][4];
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) {
#pragma unroll
    for (int e = 0; e < 4; ++e) dk[nb][e] = dv[nb][e] = 0.f;
  }
  const float c = p.scale * MMA_LOG2E;
  for (int q0 = 0; q0 < N; q0 += MT) {
    float s[8][4], dpv[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) s[nb][e] = dpv[nb][e] = 0.f;
    }
#pragma unroll
    for (int kc = 0; kc < KC; ++kc) {
      uint32_t ka[4], va[4];
      ldsm_x4_s(ka, w.Ks + sw_at_b(w.ar, w.ak, rb, kc * 16));
      ldsm_x4_s(va, w.Vs + sw_at_b(w.ar, w.ak, rb, kc * 16));
#pragma unroll
      for (int nb = 0; nb < 8; nb += 2) {
        if (q0 + nb * 8 >= N) break;
        uint32_t qf[4], df[4];
        ldsm_x4_s(qf, w.Qs + sw_at_b(w.br, w.bk, q0 + nb * 8, kc * 16));
        ldsm_x4_s(df, w.dOs + sw_at_b(w.br, w.bk, q0 + nb * 8, kc * 16));
        mma16816(s[nb], ka[0], ka[1], ka[2], ka[3], qf[0], qf[1]);
        mma16816(dpv[nb], va[0], va[1], va[2], va[3], df[0], df[1]);
        if (q0 + nb * 8 + 8 < N) {
          mma16816(s[nb + 1], ka[0], ka[1], ka[2], ka[3], qf[2], qf[3]);
          mma16816(dpv[nb + 1], va[0], va[1], va[2], va[3], df[2], df[3]);
        }
      }
    }
    const float* lse_t = w.lse_s + q0;
    const float* del_t = w.del_s + q0;
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qi = nb * 8 + 2 * t + (e & 1);
        const float pr = fast_exp2(s[nb][e] * c - lse_t[qi]);
        s[nb][e] = pr;
        dpv[nb][e] = pr * (dpv[nb][e] - del_t[qi]);
      }
    }
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) {
      if (q0 + kc * 16 >= N) break;
      const uint32_t p0 = pack_bf16x2(s[2 * kc][0], s[2 * kc][1]), p1 = pack_bf16x2(s[2 * kc][2], s[2 * kc][3]);
      const uint32_t p2 = pack_bf16x2(s[2 * kc + 1][0], s[2 * kc + 1][1]), p3 = pack_bf16x2(s[2 * kc + 1][2], s[2 * kc + 1][3]);
      const uint32_t d0 = pack_bf16x2(dpv[2 * kc][0], dpv[2 * kc][1]), d1 = pack_bf16x2(dpv[2 * kc][2], dpv[2 * kc][3]);
      const uint32_t d2 = pack_bf16x2(dpv[2 * kc + 1][0], dpv[2 * kc + 1][1]), d3 = pack_bf16x2(dpv[2 * kc + 1][2], dpv[2 * kc + 1][3]);
#pragma unroll
      for (int nb = 0; nb < NB; nb += 2) {
        uint32_t gf[4], qf[4];
        ldsm_x4_ts(gf, w.dOs + sw_at_b(w.ar, w.ak, q0 + kc * 16, nb * 8));
        ldsm_x4_ts(qf, w.Qs + sw_at_b(w.ar, w.ak, q0 + kc * 16, nb * 8));
        mma16816(dv[nb], p0, p1, p2, p3, gf[0], gf[1]);
        mma16816(dv[nb + 1], p0, p1, p2, p3, gf[2], gf[3]);
        mma16816(dk[nb], d0, d1, d2, d3, qf[0], qf[1]);
        mma16816(dk[nb + 1], d0, d1, d2, d3, qf[2], qf[3]);
      }
    }
  }
  const int b = blockIdx.x / p.H, h = blockIdx.x % p.H;
  __nv_bfloat16* dkb = p.dk16 + b * p.dk_bs + h * p.dk_hs;
  __nv_bfloat16* dvb = p.dv16 + b * p.dv_bs + h * p.dv_hs;
  const int r0 = rb + g, r1 = r0 + 8;
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) {
    const int col = nb * 8 + 2 * t;
    if (r0 < N) {
      *reinterpret_cast<uint32_t*>(dkb + (long long)r0 * p.dk_rs + col) = pack_bf16x2(dk[nb][0] * p.scale, dk[nb][1] * p.scale);
      *reinterpret_cast<uint32_t*>(dvb + (long long)r0 * p.dv_rs + col) = pack_bf16x2(dv[nb][0], dv[nb][1]);
    }
    if (r1 < N) {
      *reinterpret_cast<uint32_t*>(dkb + (long long)r1 * p.dk_rs + col) = pack_bf16x2(dk[nb][2] * p.scale, dk[nb][3] * p.scale);
      *reinterpret_cast<uint32_t*>(dvb + (long long)r1 * p.dv_rs + col) = pack_bf16x2(dv[nb][2], dv[nb][3]);
    }
  }
}

// dQ, dK and dV of one problem in one CTA.  shared memory: Q, K, V, dO of the problem, then lse and delta of its rows
// (R64 = N rounded up to 64 of each; computed once, with stage_row_stats' summation order).  The 2 * R / 16 tasks
// (dK / dV of 16 key rows, about 4/3 the work of dQ of 16 query rows) are independent; warps take them from a
// counter in shared memory, the dK / dV tasks first.
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
    float d = 0.f;
    if (ok) {
#pragma unroll 4
      for (int c = half * (HD / 2); c < (half + 1) * (HD / 2); c += 2) {
        const float2 gv = unpack_bf16x2(ld32(dOs + swz(r, c >> 3) + (c & 7)));
        const float2 o = unpack_bf16x2(ld32(ob + (long long)r * p.o_rs + c));
        d = fmaf(gv.x, o.x, fmaf(gv.y, o.y, d));
      }
    }
    d += __shfl_xor_sync(0xffffffffu, d, 1);
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

int attn_mma_fwd(const MmaAttn& a, int B, int hd, cudaStream_t st) {
  VT_REQUIRE(hd == 64 || hd == 96, "tensor-core attention: head dim %d unsupported (64 or 96)", hd);
  VT_REQUIRE((long long)B * a.H <= 65535, "tensor-core attention: B*H too large");
  const dim3 grid((a.Nq + MT - 1) / MT, B * a.H);
  const char* what = "attn_mma_fwd_kernel";
  if (hd == 64)
    return a.lse ? launch<attn_mma_fwd_kernel<64, true>>(grid, fwd_smem<64>(), a, st, what)
                 : launch<attn_mma_fwd_kernel<64, false>>(grid, fwd_smem<64>(), a, st, what);
  return a.lse ? launch<attn_mma_fwd_kernel<96, true>>(grid, fwd_smem<96>(), a, st, what)
               : launch<attn_mma_fwd_kernel<96, false>>(grid, fwd_smem<96>(), a, st, what);
}

int attn_mma_bwd(const MmaAttn& a, int B, int hd, cudaStream_t st) {
  VT_REQUIRE(hd == 64 || hd == 96, "tensor-core attention: head dim %d unsupported (64 or 96)", hd);
  VT_REQUIRE((long long)B * a.H <= 65535, "tensor-core attention: B*H too large");
  int rc;
  const dim3 gq((a.Nq + MT - 1) / MT, B * a.H), gk((a.Nk + MT - 1) / MT, B * a.H);
  if (hd == 64) {
    if ((rc = launch<attn_mma_dq_kernel<64>>(gq, dq_smem<64>(), a, st, "attn_mma_dq_kernel"))) return rc;
    return launch<attn_mma_dkv_kernel<64>>(gk, dkv_smem<64>(), a, st, "attn_mma_dkv_kernel");
  }
  if ((rc = launch<attn_mma_dq_kernel<96>>(gq, dq_smem<96>(), a, st, "attn_mma_dq_kernel"))) return rc;
  return launch<attn_mma_dkv_kernel<96>>(gk, dkv_smem<96>(), a, st, "attn_mma_dkv_kernel");
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
