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

}  // namespace vt
