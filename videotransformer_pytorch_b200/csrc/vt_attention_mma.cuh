// Tensor-core flash attention (vt_attention_mma.cu): operand description shared by vt_attn_* and vt_xattn_*.
#pragma once
#include "vt_common.cuh"

namespace vt {

struct MmaAttn {
  // element (b, h, n, c) of q at q[b * q_bs + h * q_hs + n * q_rs + c]; same for k, v, o / dout (o strides), dq
  const __nv_bfloat16* q;
  const __nv_bfloat16* k;
  const __nv_bfloat16* v;
  const __nv_bfloat16* o;      // backward: forward output
  const __nv_bfloat16* dout;   // backward: gradient of o
  long long q_bs, q_hs, q_rs, k_bs, k_hs, k_rs, v_bs, v_hs, v_rs, o_bs, o_hs, o_rs;
  __nv_bfloat16* o_out;        // forward output
  float* lse;                  // [B, H, Nq]
  float* delta;                // backward, optional: rowsum(dO * O) [B, H, Nq]
  __nv_bfloat16* dq;
  long long dq_bs, dq_hs, dq_rs;
  // dK / dV: fp32 [B, H, Nk, hd] (dk32 != NULL) or bf16 strided
  float* dk32;
  float* dv32;
  __nv_bfloat16* dk16;
  __nv_bfloat16* dv16;
  long long dk_bs, dk_hs, dk_rs, dv_bs, dv_hs, dv_rs;
  int H, Nq, Nk;
  float scale;
};

// 16-byte aligned rows, strides multiples of 8 elements, and either token-major (heads adjacent in a row: hs == hd) or
// head-major contiguous (rs == hd) rows
bool mma_layout_ok(const void* ptr, long long bs, long long hs, long long rs, int hd);
int attn_mma_fwd(const MmaAttn& a, int B, int hd, cudaStream_t st);
int attn_mma_bwd(const MmaAttn& a, int B, int hd, cudaStream_t st);
// One CTA per (b, h) problem with its operands resident in shared memory: Nq == Nk <= 256 at head dim 64, bf16 dK / dV
// and no delta output.  Same bits as attn_mma_fwd / attn_mma_bwd.
bool attn_whole_ok(const MmaAttn& a, int hd);
int attn_whole_fwd(const MmaAttn& a, int B, cudaStream_t st);
int attn_whole_bwd(const MmaAttn& a, int B, cudaStream_t st);

}  // namespace vt
