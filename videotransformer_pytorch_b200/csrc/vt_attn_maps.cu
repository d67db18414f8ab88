// Threshold masks of attention maps: show_attn's "keep a certain percentage of the mass" (reference
// visualize_attention.py:73-82) per row of patch probabilities, one CTA of 1024 threads per row with the row in shared
// memory.
//
// For a row x[0, n) (probabilities: finite, >= +0) and a threshold thresh (fp32; show_attn's `1 - threshold` rounded to
// fp32, which is what torch compares an fp32 tensor against):
//   1. sort: keys (order bits of x[i]) << 32 | i, bitonic sort of np = max(1024, 2^ceil(log2 n)) keys (padding ~0):
//      ascending values, ties by patch index (a stable sort);
//   2. s = fp32(sum of the sorted x in fp64): thread t adds its np / 1024 consecutive sorted positions in order, then
//      xor-butterflies add the 32 lanes of each warp and the 32 warp sums;
//   3. v_k = x_(k) / s, one fp32 division rounded to nearest;
//   4. c_k = fp32(prefix sum of v_0 .. v_k in fp64): thread t's positions in order, from an exclusive offset built by
//      Hillis-Steele warp scans (lane sums, then warp sums);
//   5. mask[index of position k] = c_k > thresh ? 1 : 0  (the scatter back to patch order).
//
// show_attn computes the same thing with torch on the host: s' = torch.sum of fp32 (a cascade whose tree depends on the
// host's SIMD width), v'_k = x_(k) / s' in fp32, c'_k = torch.cumsum (fp64 accumulation, fp32 results), and a sort that
// leaves ties in no promised order.  Bound on |c_k - c'_k|, with u = 2^-24, S the exact row sum, C_k <= 1 the exact
// normalised prefix mass:
//   - any fp32 summation tree of n nonnegative terms: |s' - S| <= g S with g = (n-1) u / (1 - (n-1) u), so
//     S / s' = 1 + a', |a'| <= g / (1 - g);
//   - the kernel's s: fp64 sums (relative error < n 2^-52) rounded once to fp32: S / s = 1 + a, |a| <= 1.0001 u;
//   - each division adds a relative u, each fp64 prefix sum of nonnegative terms < n 2^-52 and its fp32 rounding u:
//     c_k = C_k (1 + a)(1 + e), c'_k = C_k (1 + a')(1 + e'), |e|, |e'| <= 2.0001 u.
//   So |c_k - c'_k| <= |a| + |a'| + (|e| + |e'|)(1 + |a'|) + second-order terms <= (n - 1) u (1 + 2.1 n u) + 5.01 u,
//   and for n <= 16384 (n u <= 2^-10):
//       |c_k - c'_k| <= beta(n) = 1.01 (n + 5) 2^-24          (1.2e-5 at n = 196, 7.6e-4 at n = 12544)
// Contract: the mask equals show_attn's at every patch whose cumulative mass c'_k is farther than beta(n) from thresh
// (both sides of the comparison then agree), except that within a run of equal probabilities show_attn's sort may hand
// the run's cumulative values to its members in another order: the number kept in the run is the same, which members
// may differ.  tests/emu_attention_maps.py restates steps 1-5 operation for operation.
#include "vt_common.cuh"
#include "../../include/vt_attn_maps.h"

namespace vt {

constexpr int MM_THREADS = 1024;
constexpr int MM_MAX_N = 16384;    // the longest row: its np keys (128 KB) fill the CTA's shared memory

// order-preserving map of a float to uint32 (negative values flipped, positive ones offset), and its inverse
__device__ __forceinline__ uint32_t order_bits(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float from_order_bits(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__global__ void __launch_bounds__(MM_THREADS)
mass_mask_kernel(const float* __restrict__ probs, long long ld, float* __restrict__ mask, long long ldm, int n, int np,
                 float thresh) {
  extern __shared__ unsigned long long keys[];     // [np]
  __shared__ double wsum[32];
  __shared__ float s_row;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const float* x = probs + (long long)blockIdx.x * ld;
  float* m = mask + (long long)blockIdx.x * ldm;
  for (int i = t; i < np; i += MM_THREADS)
    keys[i] = i < n ? ((unsigned long long)order_bits(x[i]) << 32) | (unsigned)i : ~0ull;
  // bitonic sort: pair p of a (k, j) step compares positions i = p with a zero inserted at bit log2(j), and i + j
  for (int k = 2; k <= np; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      __syncthreads();
      for (int p = t; p < np / 2; p += MM_THREADS) {
        const int i = ((p & ~(j - 1)) << 1) | (p & (j - 1));
        const unsigned long long a = keys[i], b = keys[i + j];
        if ((a > b) == ((i & k) == 0)) { keys[i] = b; keys[i + j] = a; }
      }
    }
  }
  __syncthreads();
  const int chunk = np / MM_THREADS, k0 = t * chunk;
  // 2. the row sum
  double part = 0.0;
  for (int e = 0; e < chunk; ++e)
    if (k0 + e < n) part += (double)from_order_bits((uint32_t)(keys[k0 + e] >> 32));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if (lane == 0) wsum[warp] = part;
  __syncthreads();
  if (warp == 0) {
    double w = wsum[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) w += __shfl_xor_sync(0xffffffffu, w, o);
    if (lane == 0) s_row = (float)w;
  }
  __syncthreads();
  const float s = s_row;
  // 4. offsets of each thread's positions in the prefix sum
  double tot = 0.0;
  for (int e = 0; e < chunk; ++e)
    if (k0 + e < n) tot += (double)(from_order_bits((uint32_t)(keys[k0 + e] >> 32)) / s);
  double inc = tot;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double up = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += up;
  }
  const double prev = __shfl_up_sync(0xffffffffu, inc, 1);
  __syncthreads();                        // wsum is reused
  if (lane == 31) wsum[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    double w = wsum[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double up = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += up;
    }
    wsum[lane] = w;
  }
  __syncthreads();
  double run = (warp > 0 ? wsum[warp - 1] : 0.0) + (lane > 0 ? prev : 0.0);
  // 3-5. normalise, accumulate, compare, scatter back to patch order
  for (int e = 0; e < chunk; ++e) {
    if (k0 + e >= n) break;
    const unsigned long long key = keys[k0 + e];
    run += (double)(from_order_bits((uint32_t)(key >> 32)) / s);
    m[(uint32_t)key] = (float)run > thresh ? 1.f : 0.f;
  }
}

}  // namespace vt

using namespace vt;

extern "C" int vt_attn_mass_mask(const vt_attn_mass_mask_params* p, void* stream) {
  VT_REQUIRE(p && p->probs && p->mask, "vt_attn_mass_mask: null pointer");
  VT_REQUIRE(p->rows > 0, "vt_attn_mass_mask: rows=%d unsupported", p->rows);
  VT_REQUIRE(p->n >= 1 && p->n <= MM_MAX_N, "vt_attn_mass_mask: n=%d unsupported (1..%d)", p->n, MM_MAX_N);
  VT_REQUIRE(p->ld >= p->n && p->ldm >= p->n, "vt_attn_mass_mask: row strides ld=%lld / ldm=%lld shorter than n=%d",
             (long long)p->ld, (long long)p->ldm, p->n);
  int np = MM_THREADS;
  while (np < p->n) np <<= 1;
  const int smem = np * (int)sizeof(unsigned long long);
  static int max_set = 48 * 1024;
  if (smem > max_set) {
    const int lim = MM_MAX_N * (int)sizeof(unsigned long long);
    cudaError_t e = cudaFuncSetAttribute(mass_mask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, lim);
    VT_REQUIRE(e == cudaSuccess, "vt_attn_mass_mask: smem attribute: %s", cudaGetErrorString(e));
    max_set = lim;
  }
  mass_mask_kernel<<<p->rows, MM_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(p->probs, p->ld, p->mask, p->ldm, p->n,
                                                                                       np, p->thresh);
  return check_launch("mass_mask_kernel");
}
