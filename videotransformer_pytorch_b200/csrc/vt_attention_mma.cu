// Tensor-core flash attention for sm_90a (mma.sync.m16n8k16, bf16 operands, fp32 accumulators), head dim 64 or 96.
// One kernel family serves both entry points: the packed-qkv attention of vt_attn_* (the 197-token spatial pass) and the
// strided pooling / long-sequence attention of vt_xattn_* (Nq != Nk).  Operands are addressed as
// base + b * bs + h * hs + n * rs (bf16 rows, 16-byte aligned), so q / k / v / dq are read and written in place.
//   forward : CTA = 64 query rows (4 warps x 16), key tiles of 64 staged in shared memory (K row-major, V transposed),
//             online softmax in registers, P rounded to bf16 as the A operand of P V.
//   dQ      : CTA = 64 query rows; S = Q K^T and dP = dO V^T per key tile, dS = P (dP - delta), dQ += dS K.
//   dK / dV : CTA = 64 key rows; S^T = K Q^T and dP^T = V dO^T per query tile, dV += P^T dO, dK += dS^T Q.
// delta = rowsum(dO * O) is recomputed where it is needed, so no scratch is required and no atomics are used.
#include "vt_attention_mma.cuh"

namespace vt {

constexpr int MT = 64;          // rows per CTA and per staged tile
constexpr int MMA_THREADS = 128;
constexpr int PT = MT + 8;      // pitch (bf16) of a transposed tile [HD][MT]
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

// rows [r0, r0 + MT) of a strided bf16 matrix -> dst[MT][HD + 8]; rows >= limit are zero
template <int HD>
__device__ __forceinline__ void stage_rows(__nv_bfloat16* dst, const __nv_bfloat16* src, long long rs, int r0, int limit) {
  for (int i = threadIdx.x; i < MT * HD / 8; i += MMA_THREADS) {
    const int r = i / (HD / 8), c = (i % (HD / 8)) * 8;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (r0 + r < limit) v = *reinterpret_cast<const uint4*>(src + (long long)(r0 + r) * rs + c);
    *reinterpret_cast<uint4*>(dst + r * (HD + 8) + c) = v;
  }
}
// same rows, transposed: dst[HD][PT]
template <int HD>
__device__ __forceinline__ void stage_rows_t(__nv_bfloat16* dst, const __nv_bfloat16* src, long long rs, int r0, int limit) {
  for (int i = threadIdx.x; i < MT * HD / 8; i += MMA_THREADS) {
    const int r = i % MT, c = (i / MT) * 8;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (r0 + r < limit) v = *reinterpret_cast<const uint4*>(src + (long long)(r0 + r) * rs + c);
    const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(&v);
#pragma unroll
    for (int j = 0; j < 8; ++j) dst[(c + j) * PT + r] = e[j];
  }
}
// lse (log2 domain; +inf past the end: p = 0) and delta = rowsum(dO * O) of rows [r0, r0 + MT); dOs is the staged dO tile
template <int HD>
__device__ __forceinline__ void stage_row_stats(float* lse_s, float* del_s, const __nv_bfloat16* dOs, const __nv_bfloat16* ob,
                                                long long o_rs, const float* lse, int r0, int limit, float* delta_out) {
  const int r = threadIdx.x >> 1, half = threadIdx.x & 1;
  const bool ok = r0 + r < limit;
  float d = 0.f;
  if (ok) {
#pragma unroll 4
    for (int c = half * (HD / 2); c < (half + 1) * (HD / 2); c += 2) {
      const float2 g = unpack_bf16x2(ld32(dOs + r * (HD + 8) + c));
      const float2 o = unpack_bf16x2(ld32(ob + (long long)(r0 + r) * o_rs + c));
      d = fmaf(g.x, o.x, fmaf(g.y, o.y, d));
    }
  }
  d += __shfl_xor_sync(0xffffffffu, d, 1);
  if (half == 0) {
    del_s[r] = d;
    lse_s[r] = ok ? lse[r0 + r] * MMA_LOG2E : INFINITY;
    if (ok && delta_out) delta_out[r0 + r] = d;
  }
}

// ------------------------------------------------------------------------------------------------ forward
// LSE = false: p.lse is not written (forward-only calls); a template flag, so the saving form's code is unchanged
template <int HD, bool LSE>
__global__ void __launch_bounds__(MMA_THREADS) attn_mma_fwd_kernel(const MmaAttn p) {
  constexpr int P = HD + 8, NB = HD / 8, KC = HD / 16;
  __shared__ __align__(16) __nv_bfloat16 Qs[MT * P];
  __shared__ __align__(16) __nv_bfloat16 Ks[MT * P];
  __shared__ __align__(16) __nv_bfloat16 Vt[HD * PT];
  const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H;
  const int q0 = blockIdx.x * MT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, rb = warp * 16;
  const __nv_bfloat16* qb = p.q + b * p.q_bs + h * p.q_hs;
  const __nv_bfloat16* kb = p.k + b * p.k_bs + h * p.k_hs;
  const __nv_bfloat16* vb = p.v + b * p.v_bs + h * p.v_hs;
  stage_rows<HD>(Qs, qb, p.q_rs, q0, p.Nq);
  __syncthreads();
  uint32_t qa[KC][4];
#pragma unroll
  for (int kc = 0; kc < KC; ++kc) {
    const __nv_bfloat16* r0p = Qs + (rb + g) * P + kc * 16 + 2 * t;
    qa[kc][0] = ld32(r0p); qa[kc][1] = ld32(r0p + 8 * P); qa[kc][2] = ld32(r0p + 8); qa[kc][3] = ld32(r0p + 8 * P + 8);
  }
  float o[NB][4];
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) o[nb][0] = o[nb][1] = o[nb][2] = o[nb][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const float c = p.scale * MMA_LOG2E;
  for (int k0 = 0; k0 < p.Nk; k0 += MT) {
    __syncthreads();
    stage_rows<HD>(Ks, kb, p.k_rs, k0, p.Nk);
    stage_rows_t<HD>(Vt, vb, p.v_rs, k0, p.Nk);
    __syncthreads();
    float s[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
      s[nb][0] = s[nb][1] = s[nb][2] = s[nb][3] = 0.f;
#pragma unroll
      for (int kc = 0; kc < KC; ++kc) {
        const __nv_bfloat16* bp = Ks + (nb * 8 + g) * P + kc * 16 + 2 * t;
        mma16816(s[nb], qa[kc][0], qa[kc][1], qa[kc][2], qa[kc][3], ld32(bp), ld32(bp + 8));
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
      const uint32_t a0 = pack_bf16x2(s[2 * kc][0], s[2 * kc][1]), a1 = pack_bf16x2(s[2 * kc][2], s[2 * kc][3]);
      const uint32_t a2 = pack_bf16x2(s[2 * kc + 1][0], s[2 * kc + 1][1]), a3 = pack_bf16x2(s[2 * kc + 1][2], s[2 * kc + 1][3]);
#pragma unroll
      for (int nb = 0; nb < NB; ++nb) {
        const __nv_bfloat16* bp = Vt + (nb * 8 + g) * PT + kc * 16 + 2 * t;
        mma16816(o[nb], a0, a1, a2, a3, ld32(bp), ld32(bp + 8));
      }
    }
  }
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
template <int HD>
__global__ void __launch_bounds__(MMA_THREADS) attn_mma_dq_kernel(const MmaAttn p) {
  constexpr int P = HD + 8, NB = HD / 8, KC = HD / 16;
  extern __shared__ __align__(16) uint8_t mma_smem[];
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(mma_smem);
  __nv_bfloat16* dOs = Qs + MT * P;
  __nv_bfloat16* Ks = dOs + MT * P;
  __nv_bfloat16* Vs = Ks + MT * P;
  __nv_bfloat16* Kt = Vs + MT * P;
  float* lse_s = reinterpret_cast<float*>(Kt + HD * PT);
  float* del_s = lse_s + MT;
  const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H;
  const int q0 = blockIdx.x * MT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, rb = warp * 16;
  const __nv_bfloat16* kb = p.k + b * p.k_bs + h * p.k_hs;
  const __nv_bfloat16* vb = p.v + b * p.v_bs + h * p.v_hs;
  stage_rows<HD>(Qs, p.q + b * p.q_bs + h * p.q_hs, p.q_rs, q0, p.Nq);
  stage_rows<HD>(dOs, p.dout + b * p.o_bs + h * p.o_hs, p.o_rs, q0, p.Nq);
  __syncthreads();
  stage_row_stats<HD>(lse_s, del_s, dOs, p.o + b * p.o_bs + h * p.o_hs, p.o_rs, p.lse + (long long)bh * p.Nq, q0, p.Nq,
                      p.delta ? p.delta + (long long)bh * p.Nq : nullptr);
  uint32_t qa[KC][4], da[KC][4];
#pragma unroll
  for (int kc = 0; kc < KC; ++kc) {
    const __nv_bfloat16* qp = Qs + (rb + g) * P + kc * 16 + 2 * t;
    const __nv_bfloat16* dp = dOs + (rb + g) * P + kc * 16 + 2 * t;
    qa[kc][0] = ld32(qp); qa[kc][1] = ld32(qp + 8 * P); qa[kc][2] = ld32(qp + 8); qa[kc][3] = ld32(qp + 8 * P + 8);
    da[kc][0] = ld32(dp); da[kc][1] = ld32(dp + 8 * P); da[kc][2] = ld32(dp + 8); da[kc][3] = ld32(dp + 8 * P + 8);
  }
  __syncthreads();
  const float lse0 = lse_s[rb + g], lse1 = lse_s[rb + g + 8], del0 = del_s[rb + g], del1 = del_s[rb + g + 8];
  float dq[NB][4];
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) dq[nb][0] = dq[nb][1] = dq[nb][2] = dq[nb][3] = 0.f;
  const float c = p.scale * MMA_LOG2E;
  for (int k0 = 0; k0 < p.Nk; k0 += MT) {
    __syncthreads();
    stage_rows<HD>(Ks, kb, p.k_rs, k0, p.Nk);
    stage_rows<HD>(Vs, vb, p.v_rs, k0, p.Nk);
    stage_rows_t<HD>(Kt, kb, p.k_rs, k0, p.Nk);
    __syncthreads();
    float s[8][4], dpv[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) s[nb][e] = dpv[nb][e] = 0.f;
#pragma unroll
      for (int kc = 0; kc < KC; ++kc) {
        const __nv_bfloat16* kp = Ks + (nb * 8 + g) * P + kc * 16 + 2 * t;
        const __nv_bfloat16* vp = Vs + (nb * 8 + g) * P + kc * 16 + 2 * t;
        mma16816(s[nb], qa[kc][0], qa[kc][1], qa[kc][2], qa[kc][3], ld32(kp), ld32(kp + 8));
        mma16816(dpv[nb], da[kc][0], da[kc][1], da[kc][2], da[kc][3], ld32(vp), ld32(vp + 8));
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = k0 + nb * 8 + 2 * t + (e & 1);
        const float pr = key < p.Nk ? fast_exp2(s[nb][e] * c - (e < 2 ? lse0 : lse1)) : 0.f;
        s[nb][e] = pr * (dpv[nb][e] - (e < 2 ? del0 : del1));
      }
    }
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) {
      const uint32_t a0 = pack_bf16x2(s[2 * kc][0], s[2 * kc][1]), a1 = pack_bf16x2(s[2 * kc][2], s[2 * kc][3]);
      const uint32_t a2 = pack_bf16x2(s[2 * kc + 1][0], s[2 * kc + 1][1]), a3 = pack_bf16x2(s[2 * kc + 1][2], s[2 * kc + 1][3]);
#pragma unroll
      for (int nb = 0; nb < NB; ++nb) {
        const __nv_bfloat16* bp = Kt + (nb * 8 + g) * PT + kc * 16 + 2 * t;
        mma16816(dq[nb], a0, a1, a2, a3, ld32(bp), ld32(bp + 8));
      }
    }
  }
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
template <int HD>
__global__ void __launch_bounds__(MMA_THREADS) attn_mma_dkv_kernel(const MmaAttn p) {
  constexpr int P = HD + 8, NB = HD / 8, KC = HD / 16;
  extern __shared__ __align__(16) uint8_t mma_smem[];
  __nv_bfloat16* Ks = reinterpret_cast<__nv_bfloat16*>(mma_smem);
  __nv_bfloat16* Vs = Ks + MT * P;
  __nv_bfloat16* Qs = Vs + MT * P;
  __nv_bfloat16* dOs = Qs + MT * P;
  __nv_bfloat16* Qt = dOs + MT * P;
  __nv_bfloat16* dOt = Qt + HD * PT;
  float* lse_s = reinterpret_cast<float*>(dOt + HD * PT);
  float* del_s = lse_s + MT;
  const int bh = blockIdx.y, b = bh / p.H, h = bh % p.H;
  const int k0 = blockIdx.x * MT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, rb = warp * 16;
  const __nv_bfloat16* qb = p.q + b * p.q_bs + h * p.q_hs;
  const __nv_bfloat16* db = p.dout + b * p.o_bs + h * p.o_hs;
  const __nv_bfloat16* ob = p.o + b * p.o_bs + h * p.o_hs;
  const float* lse = p.lse + (long long)bh * p.Nq;
  stage_rows<HD>(Ks, p.k + b * p.k_bs + h * p.k_hs, p.k_rs, k0, p.Nk);
  stage_rows<HD>(Vs, p.v + b * p.v_bs + h * p.v_hs, p.v_rs, k0, p.Nk);
  float dk[NB][4], dv[NB][4];
#pragma unroll
  for (int nb = 0; nb < NB; ++nb) {
#pragma unroll
    for (int e = 0; e < 4; ++e) dk[nb][e] = dv[nb][e] = 0.f;
  }
  const float c = p.scale * MMA_LOG2E;
  for (int q0 = 0; q0 < p.Nq; q0 += MT) {
    __syncthreads();
    stage_rows<HD>(Qs, qb, p.q_rs, q0, p.Nq);
    stage_rows<HD>(dOs, db, p.o_rs, q0, p.Nq);
    stage_rows_t<HD>(Qt, qb, p.q_rs, q0, p.Nq);
    stage_rows_t<HD>(dOt, db, p.o_rs, q0, p.Nq);
    __syncthreads();
    stage_row_stats<HD>(lse_s, del_s, dOs, ob, p.o_rs, lse, q0, p.Nq, nullptr);
    __syncthreads();
    float s[8][4], dpv[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) s[nb][e] = dpv[nb][e] = 0.f;
    }
#pragma unroll
    for (int kc = 0; kc < KC; ++kc) {
      const __nv_bfloat16* kp = Ks + (rb + g) * P + kc * 16 + 2 * t;
      const __nv_bfloat16* vp = Vs + (rb + g) * P + kc * 16 + 2 * t;
      const uint32_t ka0 = ld32(kp), ka1 = ld32(kp + 8 * P), ka2 = ld32(kp + 8), ka3 = ld32(kp + 8 * P + 8);
      const uint32_t va0 = ld32(vp), va1 = ld32(vp + 8 * P), va2 = ld32(vp + 8), va3 = ld32(vp + 8 * P + 8);
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) {
        const __nv_bfloat16* qp = Qs + (nb * 8 + g) * P + kc * 16 + 2 * t;
        const __nv_bfloat16* dp = dOs + (nb * 8 + g) * P + kc * 16 + 2 * t;
        mma16816(s[nb], ka0, ka1, ka2, ka3, ld32(qp), ld32(qp + 8));
        mma16816(dpv[nb], va0, va1, va2, va3, ld32(dp), ld32(dp + 8));
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
      const uint32_t p0 = pack_bf16x2(s[2 * kc][0], s[2 * kc][1]), p1 = pack_bf16x2(s[2 * kc][2], s[2 * kc][3]);
      const uint32_t p2 = pack_bf16x2(s[2 * kc + 1][0], s[2 * kc + 1][1]), p3 = pack_bf16x2(s[2 * kc + 1][2], s[2 * kc + 1][3]);
      const uint32_t d0 = pack_bf16x2(dpv[2 * kc][0], dpv[2 * kc][1]), d1 = pack_bf16x2(dpv[2 * kc][2], dpv[2 * kc][3]);
      const uint32_t d2 = pack_bf16x2(dpv[2 * kc + 1][0], dpv[2 * kc + 1][1]), d3 = pack_bf16x2(dpv[2 * kc + 1][2], dpv[2 * kc + 1][3]);
#pragma unroll
      for (int nb = 0; nb < NB; ++nb) {
        const __nv_bfloat16* gp = dOt + (nb * 8 + g) * PT + kc * 16 + 2 * t;
        const __nv_bfloat16* qp = Qt + (nb * 8 + g) * PT + kc * 16 + 2 * t;
        mma16816(dv[nb], p0, p1, p2, p3, ld32(gp), ld32(gp + 8));
        mma16816(dk[nb], d0, d1, d2, d3, ld32(qp), ld32(qp + 8));
      }
    }
  }
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

template <int HD>
static constexpr int dq_smem() { return 4 * MT * (HD + 8) * 2 + HD * PT * 2 + 2 * MT * 4; }
template <int HD>
static constexpr int dkv_smem() { return 4 * MT * (HD + 8) * 2 + 2 * HD * PT * 2 + 2 * MT * 4; }

template <typename Kern>
static int set_smem(Kern kern, int bytes, bool* done, const char* what) {
  if (*done) return 0;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  VT_REQUIRE(e == cudaSuccess, "%s: smem attribute: %s", what, cudaGetErrorString(e));
  *done = true;
  return 0;
}

int attn_mma_fwd(const MmaAttn& a, int B, int hd, cudaStream_t st) {
  VT_REQUIRE(hd == 64 || hd == 96, "tensor-core attention: head dim %d unsupported (64 or 96)", hd);
  VT_REQUIRE((long long)B * a.H <= 65535, "tensor-core attention: B*H too large");
  const dim3 grid((a.Nq + MT - 1) / MT, B * a.H);
  const bool lse = a.lse != nullptr;
  if (hd == 64) (lse ? attn_mma_fwd_kernel<64, true> : attn_mma_fwd_kernel<64, false>)<<<grid, MMA_THREADS, 0, st>>>(a);
  else (lse ? attn_mma_fwd_kernel<96, true> : attn_mma_fwd_kernel<96, false>)<<<grid, MMA_THREADS, 0, st>>>(a);
  return check_launch("attn_mma_fwd_kernel");
}

int attn_mma_bwd(const MmaAttn& a, int B, int hd, cudaStream_t st) {
  VT_REQUIRE(hd == 64 || hd == 96, "tensor-core attention: head dim %d unsupported (64 or 96)", hd);
  VT_REQUIRE((long long)B * a.H <= 65535, "tensor-core attention: B*H too large");
  static bool s64a = false, s64b = false, s96a = false, s96b = false;
  int rc;
  const dim3 gq((a.Nq + MT - 1) / MT, B * a.H), gk((a.Nk + MT - 1) / MT, B * a.H);
  if (hd == 64) {
    if ((rc = set_smem(attn_mma_dq_kernel<64>, dq_smem<64>(), &s64a, "attn_mma_dq_kernel"))) return rc;
    if ((rc = set_smem(attn_mma_dkv_kernel<64>, dkv_smem<64>(), &s64b, "attn_mma_dkv_kernel"))) return rc;
    attn_mma_dq_kernel<64><<<gq, MMA_THREADS, dq_smem<64>(), st>>>(a);
    if ((rc = check_launch("attn_mma_dq_kernel"))) return rc;
    attn_mma_dkv_kernel<64><<<gk, MMA_THREADS, dkv_smem<64>(), st>>>(a);
  } else {
    if ((rc = set_smem(attn_mma_dq_kernel<96>, dq_smem<96>(), &s96a, "attn_mma_dq_kernel"))) return rc;
    if ((rc = set_smem(attn_mma_dkv_kernel<96>, dkv_smem<96>(), &s96b, "attn_mma_dkv_kernel"))) return rc;
    attn_mma_dq_kernel<96><<<gq, MMA_THREADS, dq_smem<96>(), st>>>(a);
    if ((rc = check_launch("attn_mma_dq_kernel"))) return rc;
    attn_mma_dkv_kernel<96><<<gk, MMA_THREADS, dkv_smem<96>(), st>>>(a);
  }
  return check_launch("attn_mma_dkv_kernel");
}

}  // namespace vt
