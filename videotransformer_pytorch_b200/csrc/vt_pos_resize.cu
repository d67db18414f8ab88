// Bicubic resize of the patch rows of a positional-embedding table (reference video_transformer.py:171-191,
// TimeSformer.interpolate_pos_encoding -> F.interpolate(mode='bicubic', align_corners=False, scale_factor=...)).
// Token-major fp32 rows [cells, D], D contiguous, read and written in place: no permute copies.
//
// Coordinates follow PyTorch's scale-factor form (not in/out sizes): src = (dst + 0.5) / scale - 0.5, computed in fp64.
// Cubic convolution with A = -0.75, four taps per axis at floor(src) - 1 .. floor(src) + 2, each clamped to
// [0, n - 1] (so an edge cell can take several taps of one output).  Separable: rows of taps along x first, then y.
//
// Forward: one CTA per output cell, threads stride over D, 16 taps, fp32 accumulation.
// Backward: the exact adjoint as a gather.  One CTA per input cell builds, in shared memory, the weight this input row
// carries in every output row (and column), summed over the clamped taps that land on it, then sums the output
// gradient over the (row, column) pairs with non-zero weight in a fixed order: no atomics, deterministic.
#include "vt_common.cuh"

namespace vt {

__device__ __forceinline__ double cubic_near(double x) { return ((1.25 * x - 2.25) * x) * x + 1.0; }          // |x| <= 1
__device__ __forceinline__ double cubic_far(double x) { return ((-0.75 * x + 3.75) * x - 6.0) * x + 3.0; }     // 1 < |x| < 2

// the 4 tap indices (clamped) and weights of output position o along an axis of n input cells
__device__ __forceinline__ void cubic_taps(int o, double scale, int n, int idx[4], float w[4]) {
  const double src = (o + 0.5) * (1.0 / scale) - 0.5;
  const double f = floor(src);
  const double t = src - f;
  const int i0 = (int)f;
  w[0] = (float)cubic_far(t + 1.0);
  w[1] = (float)cubic_near(t);
  w[2] = (float)cubic_near(1.0 - t);
  w[3] = (float)cubic_far(2.0 - t);
#pragma unroll
  for (int a = 0; a < 4; ++a) idx[a] = min(max(i0 - 1 + a, 0), n - 1);
}

__global__ void __launch_bounds__(256)
pos_resize_fwd_kernel(const float* __restrict__ src, int64_t lds, float* __restrict__ dst, int64_t ldd,
                      int gh, int gw, int ow, int D, double scale_h, double scale_w) {
  const int oy = blockIdx.x / ow, ox = blockIdx.x % ow;
  int iy[4], ix[4];
  float wy[4], wx[4];
  cubic_taps(oy, scale_h, gh, iy, wy);
  cubic_taps(ox, scale_w, gw, ix, wx);
  float* out = dst + (int64_t)blockIdx.x * ldd;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float acc = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const float* row = src + (int64_t)iy[a] * gw * lds + d;
      float r = 0.f;
#pragma unroll
      for (int b = 0; b < 4; ++b) r = fmaf(wx[b], __ldg(row + (int64_t)ix[b] * lds), r);
      acc = fmaf(wy[a], r, acc);
    }
    out[d] = acc;
  }
}

__global__ void __launch_bounds__(256)
pos_resize_bwd_kernel(const float* __restrict__ dy, int64_t lddy, float* __restrict__ dsrc, int64_t ldds,
                      int gh, int gw, int oh, int ow, int D, double scale_h, double scale_w) {
  extern __shared__ float wsh[];          // [oh] weights of input row iy, then [ow] weights of input column ix
  float* wrow = wsh;
  float* wcol = wsh + oh;
  const int iy = blockIdx.x / gw, ix = blockIdx.x % gw;
  for (int o = threadIdx.x; o < oh + ow; o += blockDim.x) {
    const bool is_row = o < oh;
    const int j = is_row ? o : o - oh;
    int idx[4];
    float w[4];
    cubic_taps(j, is_row ? scale_h : scale_w, is_row ? gh : gw, idx, w);
    const int me = is_row ? iy : ix;
    float s = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) s += idx[a] == me ? w[a] : 0.f;
    wsh[o] = s;
  }
  __syncthreads();
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float acc = 0.f;
    for (int oy = 0; oy < oh; ++oy) {
      const float wy = wrow[oy];
      if (wy == 0.f) continue;
      const float* row = dy + (int64_t)oy * ow * lddy + d;
      float r = 0.f;
      for (int ox = 0; ox < ow; ++ox) {
        const float wx = wcol[ox];
        if (wx != 0.f) r = fmaf(wx, row[(int64_t)ox * lddy], r);
      }
      acc = fmaf(wy, r, acc);
    }
    dsrc[(int64_t)blockIdx.x * ldds + d] = acc;
  }
}

static int pos_resize_check(const vt_pos_resize_params* p, const char* fn) {
  VT_REQUIRE(p && p->src && p->dst, "%s: null pointer", fn);
  VT_REQUIRE(p->gh > 0 && p->gw > 0 && p->oh > 0 && p->ow > 0 && p->D > 0, "%s: bad geometry %dx%d -> %dx%d, D=%d", fn,
             p->gh, p->gw, p->oh, p->ow, p->D);
  VT_REQUIRE(p->oh + p->ow <= 8192 && (int64_t)p->oh * p->ow < (1ll << 31) && (int64_t)p->gh * p->gw < (1ll << 31),
             "%s: grid too large", fn);
  VT_REQUIRE(p->scale_h > 0.0 && p->scale_w > 0.0, "%s: scale factors must be positive", fn);
  VT_REQUIRE(p->lds >= p->D && p->ldd >= p->D, "%s: row strides must be >= D", fn);
  return 0;
}

}  // namespace vt

extern "C" int vt_pos_resize_fwd(const vt_pos_resize_params* p, void* stream) {
  using namespace vt;
  if (pos_resize_check(p, "vt_pos_resize_fwd")) return 1;
  const int threads = p->D >= 256 ? 256 : ((p->D + 31) / 32) * 32;
  pos_resize_fwd_kernel<<<p->oh * p->ow, threads, 0, static_cast<cudaStream_t>(stream)>>>(
      p->src, p->lds, p->dst, p->ldd, p->gh, p->gw, p->ow, p->D, p->scale_h, p->scale_w);
  return check_launch("pos_resize_fwd_kernel");
}

/* p->src = gradient of the resized table [oh*ow rows], p->dst = gradient of the source grid [gh*gw rows] */
extern "C" int vt_pos_resize_bwd(const vt_pos_resize_params* p, void* stream) {
  using namespace vt;
  if (pos_resize_check(p, "vt_pos_resize_bwd")) return 1;
  const int threads = p->D >= 256 ? 256 : ((p->D + 31) / 32) * 32;
  const size_t smem = (size_t)(p->oh + p->ow) * sizeof(float);
  pos_resize_bwd_kernel<<<p->gh * p->gw, threads, smem, static_cast<cudaStream_t>(stream)>>>(
      p->src, p->lds, p->dst, p->ldd, p->gh, p->gw, p->oh, p->ow, p->D, p->scale_h, p->scale_w);
  return check_launch("pos_resize_bwd_kernel");
}
