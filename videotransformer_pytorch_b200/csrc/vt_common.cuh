// Shared host/device helpers for the vt_b200 kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <type_traits>

#include "../../include/vt_b200.h"

namespace vt {

// ---- per-thread error slot (the ABI never throws) ---------------------------------------------
void set_error(const char* fmt, ...);
int check_launch(const char* what);   // cudaGetLastError -> error code

#define VT_REQUIRE(cond, ...)          \
  do {                                 \
    if (!(cond)) {                     \
      ::vt::set_error(__VA_ARGS__);    \
      return 1;                        \
    }                                  \
  } while (0)

int sm_count();
// Feature switch: environment variable `name` ("0" / "1") overrides the compiled default.  INTEGRATION.md §2 lists the
// switches and their defaults; the tests set them to run both sides of each.
bool feature_on(const char* name, bool dflt);
// narrow-row LayerNorm (D = 32..256 step 32, vt_mvit.cu); vt_layernorm_fwd/bwd dispatch here when D % 128 != 0
int layernorm_fwd_small(const vt_ln_fwd_params* p, void* stream);
int layernorm_bwd_small(const vt_ln_bwd_params* p, void* stream);
int persistent_sm_count();   // sm_count() minus vt_set_reserved_sms(): the SM count the GEMM tile planning assumes

// Head widths of the packed-qkv attention kernels (vt_attn_*).  with_head_dim(hd, f) returns
// f(std::integral_constant<int, hd>{}) for a width attn_head_dim_ok accepts, so each kernel is instantiated per width.
inline bool attn_head_dim_ok(int hd) { return hd == 32 || hd == 64 || hd == 96 || hd == 128; }
template <class F>
int with_head_dim(int hd, F&& f) {
  switch (hd) {
    case 32: return f(std::integral_constant<int, 32>{});
    case 64: return f(std::integral_constant<int, 64>{});
    case 96: return f(std::integral_constant<int, 96>{});
    default: return f(std::integral_constant<int, 128>{});
  }
}

// ---- device helpers ---------------------------------------------------------------------------
// x / d and x % d for x >= 0: a shift and a mask when d is a power of two
template <int D>
__host__ __device__ __forceinline__ int div_pos(int x) {
  if constexpr ((D & (D - 1)) == 0) { int s = 0; while ((1 << s) < D) ++s; return x >> s; }
  else return x / D;
}
template <int D>
__host__ __device__ __forceinline__ int mod_pos(int x) {
  if constexpr ((D & (D - 1)) == 0) return x & (D - 1);
  else return x % D;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(t);
}

// 2^x on the SFU (ex2.approx: 2 ulp; inputs here are <= 0 after max subtraction)
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// exact-erf GELU (nn.GELU default) and its derivative, via a fast erf (Abramowitz-Stegun 7.1.26, |abs err| < 1.5e-7 — far below bf16 resolution of the stored results):
// one exp + one reciprocal + 5 FMA instead of erff's ~40 instructions; used by the GEMM epilogues where four
// erf per thread per 4 columns would otherwise out-cost the tile's MMAs.
__device__ __forceinline__ float erf_fast_pos(float x, float e /* = exp(-x*x) */) {
  const float t = __frcp_rn(fmaf(0.3275911f, x, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  return 1.0f - poly * t * e;
}
__device__ __forceinline__ float gelu_fast(float z) {
  const float x = fabsf(z) * 0.70710678118654752f;
  const float e = __expf(-x * x);
  const float er = copysignf(erf_fast_pos(x, e), z);
  return 0.5f * z * (1.0f + er);
}
__device__ __forceinline__ float dgelu_fast(float z) {
  const float x = fabsf(z) * 0.70710678118654752f;
  const float e = __expf(-x * x);               // = exp(-z^2/2), shared by cdf and pdf
  const float er = copysignf(erf_fast_pos(x, e), z);
  return 0.5f * (1.0f + er) + z * 0.39894228040143268f * e;
}

}  // namespace vt
