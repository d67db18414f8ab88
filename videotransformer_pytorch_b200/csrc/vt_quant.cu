// Row quantiser of the fp8 inference forms (vt_quant_rows_e4m3): bf16 / fp32 rows -> e4m3 rows and one fp32 scale per
// row, a power of two, so that x / scale is exact and the e4m3 cast (round to nearest even, saturating) is the only
// rounding.  One warp per row: amax over the row, then the scaled cast; the second read of the row hits L1 / L2.
#include <cuda_fp8.h>

#include "vt_common.cuh"

namespace vt {

constexpr int QR_WARPS = 8;

// smallest power of two s with amax / s <= 448, i.e. 2^ceil(log2(amax / 448)), clamped to [2^-126, 2^127]; 1 for a zero row
__device__ __forceinline__ int e4m3_scale_exp(float amax) {
  if (!(amax > 0.f)) return 0;
  if (isinf(amax)) return 127;
  int e;
  const float m = frexpf(amax, &e);          // amax = m 2^e, m in [0.5, 1); 448 = 0.875 2^9
  const int k = e - 9 + (m > 0.875f ? 1 : 0);
  return k < -126 ? -126 : (k > 127 ? 127 : k);
}

__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16x2(w[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void load8(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
  v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

template <typename T>
__global__ void __launch_bounds__(QR_WARPS * 32)
quant_rows_e4m3_kernel(const T* __restrict__ x, long long ldx, uint8_t* __restrict__ q, long long ldq,
                       float* __restrict__ scale, int M, int K) {
  const int row = blockIdx.x * QR_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const T* xr = x + (long long)row * ldx;
  const int groups = K / 8;
  float amax = 0.f;
  for (int g = lane; g < groups; g += 32) {
    float v[8];
    load8(xr + 8 * g, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(v[i]));
  }
  amax = warp_max(amax);
  const int k = e4m3_scale_exp(amax);
  const float inv = ldexpf(1.0f, -k);        // exact: x * 2^-k only shifts the exponent (results <= 448)
  uint8_t* qr = q + (long long)row * ldq;
  for (int g = lane; g < groups; g += 32) {
    float v[8];
    load8(xr + 8 * g, v);
    uint32_t w[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(v[4 * i] * inv, v[4 * i + 1] * inv), __NV_SATFINITE, __NV_E4M3);
      const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(v[4 * i + 2] * inv, v[4 * i + 3] * inv), __NV_SATFINITE, __NV_E4M3);
      w[i] = lo | (hi << 16);
    }
    *reinterpret_cast<uint2*>(qr + 8 * g) = make_uint2(w[0], w[1]);
  }
  if (lane == 0) scale[row] = ldexpf(1.0f, k);
}

}  // namespace vt

extern "C" int vt_quant_rows_e4m3(const vt_quant_rows_params* p, void* stream) {
  using namespace vt;
  VT_REQUIRE(p && p->x && p->q && p->scale, "vt_quant_rows_e4m3: null argument");
  VT_REQUIRE(p->M > 0 && p->K > 0 && p->K % 16 == 0, "vt_quant_rows_e4m3: bad shape M=%d K=%d (K must be a multiple of 16)",
             p->M, p->K);
  const int esz = p->x_fp32 ? 4 : 2;
  VT_REQUIRE((reinterpret_cast<uintptr_t>(p->x) & 15) == 0 && (p->ldx * esz) % 16 == 0 && p->ldx >= p->K,
             "vt_quant_rows_e4m3: x rows must be 16-byte aligned (ldx=%lld)", (long long)p->ldx);
  VT_REQUIRE((reinterpret_cast<uintptr_t>(p->q) & 15) == 0 && p->ldq % 16 == 0 && p->ldq >= p->K,
             "vt_quant_rows_e4m3: q rows must be 16-byte aligned (ldq=%lld)", (long long)p->ldq);
  const int grid = (p->M + QR_WARPS - 1) / QR_WARPS;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (p->x_fp32)
    quant_rows_e4m3_kernel<float><<<grid, QR_WARPS * 32, 0, st>>>(static_cast<const float*>(p->x), p->ldx,
                                                                  static_cast<uint8_t*>(p->q), p->ldq, p->scale, p->M, p->K);
  else
    quant_rows_e4m3_kernel<__nv_bfloat16><<<grid, QR_WARPS * 32, 0, st>>>(static_cast<const __nv_bfloat16*>(p->x), p->ldx,
                                                                          static_cast<uint8_t*>(p->q), p->ldq, p->scale, p->M, p->K);
  return check_launch("quant_rows_e4m3_kernel");
}
