// Bandwidth-bound warp-primitive kernels: LayerNorm fwd/bwd (fused with the token regroupings),
// fp32->bf16 casts (+row gather, +DropPath scale), bias-gradient column sums, im2col / col2im for the
// non-overlapping patch / tubelet embedding.  All loads/stores are 16-byte vectors on contiguous rows.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "vt_common.cuh"

namespace vt {

// ------------------------------------------------------------------------------------------------
// error slot + device info
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = {0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static unsigned long long g_launches = 0;

bool feature_on(const char* name, bool dflt) {
  const char* v = getenv(name);
  if (!v || !*v) return dflt;
  return v[0] != '0';
}

int check_launch(const char* what) {
  __atomic_add_fetch(&g_launches, 1ull, __ATOMIC_RELAXED);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
    return 2;
  }
  return 0;
}

// SMs left free by the persistent kernels (GEMMs) so that concurrently running communication kernels (NCCL
// all-reduce of the gradient buckets, overlapped with backward) find an SM to run on.  0 by default.
static int g_reserved_sms = 0;

int persistent_sm_count() {
  const int n = sm_count() - g_reserved_sms;
  return n < 2 ? 2 : n;
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

// ------------------------------------------------------------------------------------------------
// LayerNorm forward: one warp per row, D = 128*V floats, row held in registers (V float4 per lane).
// ------------------------------------------------------------------------------------------------
constexpr int LN_WARPS = 8;

template <int V>
__global__ void __launch_bounds__(LN_WARPS * 32)
ln_fwd_kernel(const float* __restrict__ x, long long ldx, const int* __restrict__ in_row,
              const float* __restrict__ gamma, const float* __restrict__ beta, void* __restrict__ y,
              float* __restrict__ mean, float* __restrict__ rstd, int rows, float eps, int y_fp32) {
  constexpr int D = V * 128;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4 g[V], b[V];
#pragma unroll
  for (int i = 0; i < V; ++i) {
    g[i] = __ldg(reinterpret_cast<const float4*>(gamma) + lane + 32 * i);
    b[i] = __ldg(reinterpret_cast<const float4*>(beta) + lane + 32 * i);
  }
  for (int m = blockIdx.x * LN_WARPS + warp; m < rows; m += gridDim.x * LN_WARPS) {
    const int src = in_row ? in_row[m] : m;
    const float4* xr = reinterpret_cast<const float4*>(x + (long long)src * ldx);
    float4 v[V];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      v[i] = xr[lane + 32 * i];
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    const float mu = warp_sum(s) * (1.0f / D);
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      const float a = v[i].x - mu, bb = v[i].y - mu, c = v[i].z - mu, d = v[i].w - mu;
      ss += (a * a + bb * bb) + (c * c + d * d);
    }
    const float rs = rsqrtf(warp_sum(ss) * (1.0f / D) + eps);
    if (lane == 0 && mean) {   // mean / rstd NULL: not written
      mean[m] = mu;
      rstd[m] = rs;
    }
#pragma unroll
    for (int i = 0; i < V; ++i) {
      const float o0 = (v[i].x - mu) * rs * g[i].x + b[i].x;
      const float o1 = (v[i].y - mu) * rs * g[i].y + b[i].y;
      const float o2 = (v[i].z - mu) * rs * g[i].z + b[i].z;
      const float o3 = (v[i].w - mu) * rs * g[i].w + b[i].w;
      if (y_fp32) {
        reinterpret_cast<float4*>(static_cast<float*>(y) + (long long)m * D)[lane + 32 * i] = make_float4(o0, o1, o2, o3);
      } else {
        uint2 o;
        o.x = pack_bf16x2(o0, o1);
        o.y = pack_bf16x2(o2, o3);
        reinterpret_cast<uint2*>(static_cast<__nv_bfloat16*>(y) + (long long)m * D)[lane + 32 * i] = o;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm backward: one warp per row; per-lane dgamma/dbeta partial sums kept in registers across
// the CTA's rows, reduced across warps through shared memory, one partial row per CTA.
// ------------------------------------------------------------------------------------------------
template <int V>
__global__ void __launch_bounds__(LN_WARPS * 32)
ln_bwd_kernel(const void* __restrict__ dy, int dy_fp32, const float* __restrict__ x, long long ldx,
              const int* __restrict__ in_row, const float* __restrict__ mean, const float* __restrict__ rstd,
              const float* __restrict__ gamma, const float* __restrict__ dres, float* __restrict__ dx, long long lddx,
              float* __restrict__ dx_aux, const int* __restrict__ out_row, float* __restrict__ partials, int rows) {
  constexpr int D = V * 128;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4 g[V], dg[V], db[V];
#pragma unroll
  for (int i = 0; i < V; ++i) {
    g[i] = __ldg(reinterpret_cast<const float4*>(gamma) + lane + 32 * i);
    dg[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    db[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int m = blockIdx.x * LN_WARPS + warp; m < rows; m += gridDim.x * LN_WARPS) {
    const int src = in_row ? in_row[m] : m;
    const float4* xr = reinterpret_cast<const float4*>(x + (long long)src * ldx);
    const float mu = mean[m], rs = rstd[m];
    float4 xh[V], gy[V];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      float4 d;
      if (dy_fp32) {
        d = reinterpret_cast<const float4*>(static_cast<const float*>(dy) + (long long)m * D)[lane + 32 * i];
      } else {
        const uint2 u = reinterpret_cast<const uint2*>(static_cast<const __nv_bfloat16*>(dy) + (long long)m * D)[lane + 32 * i];
        const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
        d = make_float4(a.x, a.y, b.x, b.y);
      }
      const float4 xv = xr[lane + 32 * i];
      xh[i] = make_float4((xv.x - mu) * rs, (xv.y - mu) * rs, (xv.z - mu) * rs, (xv.w - mu) * rs);
      dg[i].x += d.x * xh[i].x; dg[i].y += d.y * xh[i].y; dg[i].z += d.z * xh[i].z; dg[i].w += d.w * xh[i].w;
      db[i].x += d.x; db[i].y += d.y; db[i].z += d.z; db[i].w += d.w;
      gy[i] = make_float4(d.x * g[i].x, d.y * g[i].y, d.z * g[i].z, d.w * g[i].w);
      s1 += (gy[i].x + gy[i].y) + (gy[i].z + gy[i].w);
      s2 += (gy[i].x * xh[i].x + gy[i].y * xh[i].y) + (gy[i].z * xh[i].z + gy[i].w * xh[i].w);
    }
    const float m1 = warp_sum(s1) * (1.0f / D);
    const float m2 = warp_sum(s2) * (1.0f / D);
    const int t = out_row ? out_row[m] : m;
    float* dst;
    const float* res = nullptr;
    if (t >= 0) {
      dst = dx + (long long)t * lddx;
      if (dres) res = dres + (long long)t * lddx;
    } else {
      dst = dx_aux + (long long)(-t - 1) * D;
    }
#pragma unroll
    for (int i = 0; i < V; ++i) {
      float4 o;
      o.x = rs * (gy[i].x - m1 - xh[i].x * m2);
      o.y = rs * (gy[i].y - m1 - xh[i].y * m2);
      o.z = rs * (gy[i].z - m1 - xh[i].z * m2);
      o.w = rs * (gy[i].w - m1 - xh[i].w * m2);
      if (res) {
        const float4 r = reinterpret_cast<const float4*>(res)[lane + 32 * i];
        o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
      }
      reinterpret_cast<float4*>(dst)[lane + 32 * i] = o;
    }
  }
  // cross-warp reduction of dgamma / dbeta
  __shared__ float4 sh[LN_WARPS][32];
  float* pg = partials + (long long)blockIdx.x * 2 * D;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    for (int pass = 0; pass < 2; ++pass) {
      __syncthreads();
      sh[warp][lane] = pass == 0 ? dg[i] : db[i];
      __syncthreads();
      if (warp == 0) {
        float4 a = sh[0][lane];
        for (int w = 1; w < LN_WARPS; ++w) {
          const float4 c = sh[w][lane];
          a.x += c.x; a.y += c.y; a.z += c.z; a.w += c.w;
        }
        reinterpret_cast<float4*>(pg + pass * D)[lane + 32 * i] = a;
      }
    }
  }
}

// Second version (VT_LN_BWD_V2=1): two CTAs per SM.
template <int V>
__global__ void __launch_bounds__(LN_WARPS * 32, (V <= 6 ? 2 : 1))
ln_bwd2_kernel(const void* __restrict__ dy, int dy_fp32, const float* __restrict__ x, long long ldx,
              const int* __restrict__ in_row, const float* __restrict__ mean, const float* __restrict__ rstd,
              const float* __restrict__ gamma, const float* __restrict__ dres, float* __restrict__ dx, long long lddx,
              float* __restrict__ dx_aux, const int* __restrict__ out_row, float* __restrict__ partials, int rows) {
  constexpr int D = V * 128;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // Register budget: two CTAs (16 warps) per SM need <= 128 registers per thread.  Only the dgamma / dbeta partial sums
  // live across rows; gamma is re-read per row (3 KiB, L1-resident) and dy*gamma is recomputed in the second pass
  // instead of being held (the first version kept gamma, xhat and dy*gamma: 162 registers, one CTA per SM, ~0.6 of HBM).
  float4 dg[V], db[V];
#pragma unroll
  for (int i = 0; i < V; ++i) {
    dg[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    db[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  for (int m = blockIdx.x * LN_WARPS + warp; m < rows; m += gridDim.x * LN_WARPS) {
    const int src = in_row ? in_row[m] : m;
    const float4* xr = reinterpret_cast<const float4*>(x + (long long)src * ldx);
    const float mu = mean[m], rs = rstd[m];
    float4 xh[V];
    float s1 = 0.f, s2 = 0.f;
    auto load_dy = [&](int i) {
      if (dy_fp32) return reinterpret_cast<const float4*>(static_cast<const float*>(dy) + (long long)m * D)[lane + 32 * i];
      const uint2 u = reinterpret_cast<const uint2*>(static_cast<const __nv_bfloat16*>(dy) + (long long)m * D)[lane + 32 * i];
      const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
      return make_float4(a.x, a.y, b.x, b.y);
    };
#pragma unroll
    for (int i = 0; i < V; ++i) {
      const float4 d = load_dy(i);
      const float4 xv = xr[lane + 32 * i];
      const float4 g = __ldg(g4 + lane + 32 * i);
      xh[i] = make_float4((xv.x - mu) * rs, (xv.y - mu) * rs, (xv.z - mu) * rs, (xv.w - mu) * rs);
      dg[i].x += d.x * xh[i].x; dg[i].y += d.y * xh[i].y; dg[i].z += d.z * xh[i].z; dg[i].w += d.w * xh[i].w;
      db[i].x += d.x; db[i].y += d.y; db[i].z += d.z; db[i].w += d.w;
      const float4 gy = make_float4(d.x * g.x, d.y * g.y, d.z * g.z, d.w * g.w);
      s1 += (gy.x + gy.y) + (gy.z + gy.w);
      s2 += (gy.x * xh[i].x + gy.y * xh[i].y) + (gy.z * xh[i].z + gy.w * xh[i].w);
    }
    const float m1 = warp_sum(s1) * (1.0f / D);
    const float m2 = warp_sum(s2) * (1.0f / D);
    const int t = out_row ? out_row[m] : m;
    float* dst;
    const float* res = nullptr;
    if (t >= 0) {
      dst = dx + (long long)t * lddx;
      if (dres) res = dres + (long long)t * lddx;
    } else {
      dst = dx_aux + (long long)(-t - 1) * D;
    }
#pragma unroll
    for (int i = 0; i < V; ++i) {
      const float4 g = __ldg(g4 + lane + 32 * i);
      const float4 d = load_dy(i);          // second read of the row's dy: an L1 hit (1.5 - 3 KiB per warp)
      float4 o;
      o.x = rs * (d.x * g.x - m1 - xh[i].x * m2);
      o.y = rs * (d.y * g.y - m1 - xh[i].y * m2);
      o.z = rs * (d.z * g.z - m1 - xh[i].z * m2);
      o.w = rs * (d.w * g.w - m1 - xh[i].w * m2);
      if (res) {
        const float4 r = reinterpret_cast<const float4*>(res)[lane + 32 * i];
        o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
      }
      reinterpret_cast<float4*>(dst)[lane + 32 * i] = o;
    }
  }
  // cross-warp reduction of dgamma / dbeta
  __shared__ float4 sh[LN_WARPS][32];
  float* pg = partials + (long long)blockIdx.x * 2 * D;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    for (int pass = 0; pass < 2; ++pass) {
      __syncthreads();
      sh[warp][lane] = pass == 0 ? dg[i] : db[i];
      __syncthreads();
      if (warp == 0) {
        float4 a = sh[0][lane];
        for (int w = 1; w < LN_WARPS; ++w) {
          const float4 c = sh[w][lane];
          a.x += c.x; a.y += c.y; a.z += c.z; a.w += c.w;
        }
        reinterpret_cast<float4*>(pg + pass * D)[lane + 32 * i] = a;
      }
    }
  }
}

// the entry points refuse pointers the kernels' 16-byte vector accesses cannot take (NULL passes: optional operands)
static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static int ln_blocks(int rows) {
  int blocks = (rows + LN_WARPS - 1) / LN_WARPS;
  const int cap = sm_count() * 4;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return blocks;
}

// ------------------------------------------------------------------------------------------------
// casts
// ------------------------------------------------------------------------------------------------
__global__ void cast_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n8) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const float4 a = reinterpret_cast<const float4*>(src)[2 * i];
    const float4 b = reinterpret_cast<const float4*>(src)[2 * i + 1];
    uint4 o;
    o.x = pack_bf16x2(a.x, a.y); o.y = pack_bf16x2(a.z, a.w);
    o.z = pack_bf16x2(b.x, b.y); o.w = pack_bf16x2(b.z, b.w);
    reinterpret_cast<uint4*>(dst)[i] = o;
  }
}
__global__ void cast_tail_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long start, long long n) {
  const long long i = start + blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) dst[i] = __float2bfloat16_rn(src[i]);
}

__global__ void gather_cast_kernel(const float* __restrict__ src, long long lds, const int* __restrict__ in_row,
                                   const float* __restrict__ row_scale, __nv_bfloat16* __restrict__ dst, int rows, int D8) {
  // one warp per row, 8 elements (32 B in, 16 B out) per lane per step
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int m = warp; m < rows; m += nwarps) {
    const int s = in_row ? in_row[m] : m;
    const float sc = row_scale ? row_scale[m] : 1.0f;
    uint4* o = reinterpret_cast<uint4*>(dst + (long long)m * D8 * 8);
    if (s < 0) {
      for (int i = lane; i < D8; i += 32) o[i] = make_uint4(0, 0, 0, 0);
      continue;
    }
    const float4* r = reinterpret_cast<const float4*>(src + (long long)s * lds);
    for (int i = lane; i < D8; i += 32) {
      const float4 a = r[2 * i], b = r[2 * i + 1];
      uint4 v;
      v.x = pack_bf16x2(sc * a.x, sc * a.y); v.y = pack_bf16x2(sc * a.z, sc * a.w);
      v.z = pack_bf16x2(sc * b.x, sc * b.y); v.w = pack_bf16x2(sc * b.z, sc * b.w);
      o[i] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Producer kernels that also emit the column sums of what they write (the bias gradient of the layer whose dY they
// produce): the separate column-sum pass re-read 19 - 77 MB per launch at ~1.2 - 3.7 TB/s (profiles/r2_*), 4 of the 7 per
// block disappear this way.  Sums are taken over the bf16-rounded values, as the separate pass does.  Per-CTA partial rows,
// summed by reduce_rows in CTA order (deterministic) — a last-CTA-finishes pass inside the kernel pulled the 1 - 7 MB of
// partials through ONE SM (171 us for the dGELU case).
// ------------------------------------------------------------------------------------------------
constexpr int GCC_CH = 4;         // 8-column pieces per lane: D <= 1024

// DUAL: a second set of sums over the rows *before* the row scale (bf16-rounded as well) — the bias gradient of a layer
// that sits behind DropPath when the scaled rows feed the layer in front of it (merged proj + temporal_fc)
template <bool DUAL>
__global__ void __launch_bounds__(256)
gather_cast_colsum_kernel(const float* __restrict__ src, long long lds, const int* __restrict__ in_row,
                          const float* __restrict__ row_scale, __nv_bfloat16* __restrict__ dst, int rows, int D8,
                          float* __restrict__ ws) {
  extern __shared__ float sh_gcc[];            // [8 warps][D]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int D = D8 * 8;
  float acc[GCC_CH][8], acc2[DUAL ? GCC_CH : 1][8];
#pragma unroll
  for (int c = 0; c < GCC_CH; ++c)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      acc[c][j] = 0.f;
      if (DUAL) acc2[c][j] = 0.f;
    }
  for (int m = blockIdx.x * 8 + warp; m < rows; m += gridDim.x * 8) {
    const int s = in_row ? in_row[m] : m;
    const float sc = row_scale ? row_scale[m] : 1.0f;
    uint4* o = reinterpret_cast<uint4*>(dst + (long long)m * D);
    if (s < 0) {
      for (int i = lane; i < D8; i += 32) o[i] = make_uint4(0, 0, 0, 0);
      continue;
    }
    const float4* r = reinterpret_cast<const float4*>(src + (long long)s * lds);
    float4 a[GCC_CH], b[GCC_CH];
#pragma unroll
    for (int c = 0; c < GCC_CH; ++c) {
      const int i = lane + 32 * c;
      if (i < D8) { a[c] = r[2 * i]; b[c] = r[2 * i + 1]; }
    }
#pragma unroll
    for (int c = 0; c < GCC_CH; ++c) {
      const int i = lane + 32 * c;
      if (i < D8) {
        uint4 v;
        v.x = pack_bf16x2(sc * a[c].x, sc * a[c].y); v.y = pack_bf16x2(sc * a[c].z, sc * a[c].w);
        v.z = pack_bf16x2(sc * b[c].x, sc * b[c].y); v.w = pack_bf16x2(sc * b[c].z, sc * b[c].w);
        o[i] = v;
        const float2 p0 = unpack_bf16x2(v.x), p1 = unpack_bf16x2(v.y), p2 = unpack_bf16x2(v.z), p3 = unpack_bf16x2(v.w);
        acc[c][0] += p0.x; acc[c][1] += p0.y; acc[c][2] += p1.x; acc[c][3] += p1.y;
        acc[c][4] += p2.x; acc[c][5] += p2.y; acc[c][6] += p3.x; acc[c][7] += p3.y;
        if (DUAL) {
          const float2 q0 = unpack_bf16x2(pack_bf16x2(a[c].x, a[c].y)), q1 = unpack_bf16x2(pack_bf16x2(a[c].z, a[c].w));
          const float2 q2 = unpack_bf16x2(pack_bf16x2(b[c].x, b[c].y)), q3 = unpack_bf16x2(pack_bf16x2(b[c].z, b[c].w));
          acc2[c][0] += q0.x; acc2[c][1] += q0.y; acc2[c][2] += q1.x; acc2[c][3] += q1.y;
          acc2[c][4] += q2.x; acc2[c][5] += q2.y; acc2[c][6] += q3.x; acc2[c][7] += q3.y;
        }
      }
    }
  }
  const int W = DUAL ? 2 * D : D;              // columns of a partial row
#pragma unroll 1
  for (int pass = 0; pass < (DUAL ? 2 : 1); ++pass) {
    __syncthreads();
#pragma unroll
    for (int c = 0; c < GCC_CH; ++c) {
      const int i = lane + 32 * c;
      if (i < D8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) sh_gcc[warp * D + i * 8 + j] = pass == 0 ? acc[c][j] : acc2[c][j];
      }
    }
    __syncthreads();
    for (int col = threadIdx.x; col < D; col += 256) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += sh_gcc[w * D + col];
      ws[(long long)blockIdx.x * W + pass * D + col] = t;
    }
  }
}

// dz = dh * gelu'(z) with the column sums of dz: blockDim = N / 8 (thread = 8 columns of every row the CTA walks)
constexpr int GBC_UNROLL = 2;
__global__ void __launch_bounds__(1024)
gelu_bwd_colsum_kernel(const uint4* __restrict__ dh, const uint4* __restrict__ z, uint4* __restrict__ dz, int M, int N8,
                       float* __restrict__ ws) {
  const int c8 = threadIdx.x;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int r0 = blockIdx.x * GBC_UNROLL; r0 < M; r0 += gridDim.x * GBC_UNROLL) {
    uint4 g[GBC_UNROLL], v[GBC_UNROLL];
#pragma unroll
    for (int u = 0; u < GBC_UNROLL; ++u) {
      const int r = min(r0 + u, M - 1);
      g[u] = dh[(long long)r * N8 + c8];
      v[u] = z[(long long)r * N8 + c8];
    }
#pragma unroll
    for (int u = 0; u < GBC_UNROLL; ++u) {
      if (r0 + u >= M) break;
      const uint32_t gw[4] = {g[u].x, g[u].y, g[u].z, g[u].w}, zw[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
      uint32_t o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 a = unpack_bf16x2(gw[k]), f = unpack_bf16x2(zw[k]);
        o[k] = pack_bf16x2(a.x * dgelu_fast(f.x), a.y * dgelu_fast(f.y));
        const float2 q = unpack_bf16x2(o[k]);
        acc[2 * k] += q.x; acc[2 * k + 1] += q.y;
      }
      dz[(long long)(r0 + u) * N8 + c8] = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
  float4* wrow = reinterpret_cast<float4*>(ws + (long long)blockIdx.x * N8 * 8) + 2 * c8;
  wrow[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
  wrow[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// ------------------------------------------------------------------------------------------------
// column sums of a bf16 matrix: CTA = 64 columns x one row chunk; 256 threads = 8 row lanes x 32 column pairs
// ------------------------------------------------------------------------------------------------
constexpr int COLSUM_ROWS = 512;  // rows per chunk

__global__ void __launch_bounds__(256)
colsum_kernel(const __nv_bfloat16* __restrict__ in, long long ld, int M, int N, float* __restrict__ ws, float* __restrict__ out,
              int* __restrict__ counters) {
  const int cp = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int col = blockIdx.x * 64 + cp * 2;
  const int r0 = blockIdx.y * COLSUM_ROWS;
  const int r1 = min(M, r0 + COLSUM_ROWS);
  float a0 = 0.f, a1 = 0.f;
  if (col < N) {
    for (int r = r0 + rl; r < r1; r += 8) {
      const uint32_t u = *reinterpret_cast<const uint32_t*>(in + (long long)r * ld + col);
      const float2 f = unpack_bf16x2(u);
      a0 += f.x;
      a1 += f.y;
    }
  }
  __shared__ float2 sh[8][32];
  sh[rl][cp] = make_float2(a0, a1);
  __syncthreads();
  if (rl == 0 && col < N) {
    float2 s = sh[0][cp];
    for (int w = 1; w < 8; ++w) { s.x += sh[w][cp].x; s.y += sh[w][cp].y; }
    *reinterpret_cast<float2*>(ws + (long long)blockIdx.y * N + col) = s;
  }
  if (counters == nullptr) return;   // two-launch form: the caller reduces the partials
  // single-launch form: the last row-chunk CTA of this column block sums the partials (fixed order => deterministic)
  __shared__ int is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int done = atomicAdd(&counters[blockIdx.x], 1);
    is_last = (done == (int)gridDim.y - 1);
    if (is_last) counters[blockIdx.x] = 0;   // self-cleaning for the next call
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (rl == 0 && col < N) {
    float2 t = make_float2(0.f, 0.f);
    for (int c = 0; c < (int)gridDim.y; ++c) {
      const float2 v = __ldcg(reinterpret_cast<const float2*>(ws + (long long)c * N + col));
      t.x += v.x; t.y += v.y;
    }
    *reinterpret_cast<float2*>(out + col) = t;
  }
}

// ------------------------------------------------------------------------------------------------
// im2col for non-overlapping patches / tubelets, and its adjoint
//   cols[(b,t',hp,wp), ((c*tube+dt)*ph+i)*pw+j] = x[b, t'*tube+dt, c, hp*ph+i, wp*pw+j]
// one thread = 8 consecutive j (pw % 8 == 0)
// ------------------------------------------------------------------------------------------------
__global__ void im2col_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ cols, int B, int T, int C, int H,
                              int W, int tube, int ph, int pw, long long total8) {
  const int Kc = C * tube * ph * pw;
  const int Hp = H / ph, Wp = W / pw, Tp = T / tube;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total8; idx += (long long)gridDim.x * blockDim.x) {
    const long long e = idx * 8;
    const long long row = e / Kc;
    int k = (int)(e - row * Kc);
    const int j = k % pw; k /= pw;
    const int i = k % ph; k /= ph;
    const int dt = k % tube; const int c = k / tube;
    long long rr = row;
    const int wp = (int)(rr % Wp); rr /= Wp;
    const int hp = (int)(rr % Hp); rr /= Hp;
    const int tp = (int)(rr % Tp); const int b = (int)(rr / Tp);
    const float* src = x + ((((long long)b * T + (tp * tube + dt)) * C + c) * H + (hp * ph + i)) * W + wp * pw + j;
    const float4 a = *reinterpret_cast<const float4*>(src);
    const float4 bq = *reinterpret_cast<const float4*>(src + 4);
    uint4 o;
    o.x = pack_bf16x2(a.x, a.y); o.y = pack_bf16x2(a.z, a.w);
    o.z = pack_bf16x2(bq.x, bq.y); o.w = pack_bf16x2(bq.z, bq.w);
    *reinterpret_cast<uint4*>(cols + e) = o;
  }
}

// uint8 clip straight from the decoder ([B, T, H, W, C], channels last) -> normalised bf16 patch rows: fuses ToTensor
// (/255), Normalize(mean, std) and the patch regrouping, so the clip crosses PCIe and HBM as bytes.
// one thread = 8 consecutive j of one (row, c, dt, i)
__global__ void im2col_u8_kernel(const uint8_t* __restrict__ x, const float* __restrict__ scale, const float* __restrict__ shift,
                                 __nv_bfloat16* __restrict__ cols, int B, int T, int C, int H, int W, int tube, int ph,
                                 int pw, long long total8) {
  const int Kc = C * tube * ph * pw;
  const int Hp = H / ph, Wp = W / pw, Tp = T / tube;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total8; idx += (long long)gridDim.x * blockDim.x) {
    const long long e = idx * 8;
    const long long row = e / Kc;
    int k = (int)(e - row * Kc);
    const int j = k % pw; k /= pw;
    const int i = k % ph; k /= ph;
    const int dt = k % tube; const int c = k / tube;
    long long rr = row;
    const int wp = (int)(rr % Wp); rr /= Wp;
    const int hp = (int)(rr % Hp); rr /= Hp;
    const int tp = (int)(rr % Tp); const int b = (int)(rr / Tp);
    const uint8_t* src = x + ((((long long)b * T + (tp * tube + dt)) * H + (hp * ph + i)) * W + wp * pw + j) * C + c;
    const float sc = scale[c], sh = shift[c];
    float v[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) v[q] = fmaf((float)src[(long long)q * C], sc, sh);
    uint4 o;
    o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]);
    o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(cols + e) = o;
  }
}

__global__ void col2im_kernel(const float* __restrict__ cols, float* __restrict__ dx, int B, int T, int C, int H, int W,
                              int tube, int ph, int pw, long long total4) {
  const int Kc = C * tube * ph * pw;
  const int Hp = H / ph, Wp = W / pw, Tp = T / tube;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total4; idx += (long long)gridDim.x * blockDim.x) {
    const long long e = idx * 4;
    const long long row = e / Kc;
    int k = (int)(e - row * Kc);
    const int j = k % pw; k /= pw;
    const int i = k % ph; k /= ph;
    const int dt = k % tube; const int c = k / tube;
    long long rr = row;
    const int wp = (int)(rr % Wp); rr /= Wp;
    const int hp = (int)(rr % Hp); rr /= Hp;
    const int tp = (int)(rr % Tp); const int b = (int)(rr / Tp);
    float* dst = dx + ((((long long)b * T + (tp * tube + dt)) * C + c) * H + (hp * ph + i)) * W + wp * pw + j;
    *reinterpret_cast<float4*>(dst) = *reinterpret_cast<const float4*>(cols + e);
  }
}

// ------------------------------------------------------------------------------------------------
// exact-erf GELU on bf16 rows, forward (h = gelu(z)) and backward (dz = dh * gelu'(z)); 8 elements per thread
// ------------------------------------------------------------------------------------------------
__global__ void gelu_fwd_kernel(const uint4* __restrict__ z, uint4* __restrict__ h, long long n8) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = z[i];
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16x2(w[k]);
      o[k] = pack_bf16x2(gelu_fast(f.x), gelu_fast(f.y));
    }
    h[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}
__global__ void gelu_bwd_kernel(const uint4* __restrict__ dh, const uint4* __restrict__ z, uint4* __restrict__ dz, long long n8) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const uint4 g = dh[i], v = z[i];
    const uint32_t gw[4] = {g.x, g.y, g.z, g.w}, zw[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 a = unpack_bf16x2(gw[k]), f = unpack_bf16x2(zw[k]);
      o[k] = pack_bf16x2(a.x * dgelu_fast(f.x), a.y * dgelu_fast(f.y));
    }
    dz[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

static int grid_for(long long work, int threads) {
  long long b = (work + threads - 1) / threads;
  const long long cap = (long long)sm_count() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace vt

// ================================================================================================
// C ABI
// ================================================================================================
using namespace vt;

extern "C" int vt_version(void) { return VT_ABI_VERSION; }

extern "C" int vt_last_error(char* buf, size_t n) {
  if (!buf || n == 0) return 0;
  strncpy(buf, g_err, n - 1);
  buf[n - 1] = 0;
  return (int)strlen(buf);
}

extern "C" int vt_sm_count(void) { return sm_count(); }

extern "C" int vt_set_reserved_sms(int n) {
  if (n < 0 || n > 64) { set_error("vt_set_reserved_sms: %d out of range [0, 64]", n); return 1; }
  g_reserved_sms = n;
  return 0;
}

extern "C" int vt_launch_count(void) { return (int)(__atomic_load_n(&g_launches, __ATOMIC_RELAXED) & 0x7fffffffull); }

extern "C" int vt_layernorm_fwd(const vt_ln_fwd_params* p, void* stream) {
  VT_REQUIRE(p && p->x && p->gamma && p->beta && p->y, "vt_layernorm_fwd: null pointer");
  VT_REQUIRE((p->mean == nullptr) == (p->rstd == nullptr), "vt_layernorm_fwd: mean and rstd are both given or both NULL");
  VT_REQUIRE(p->rows > 0, "vt_layernorm_fwd: rows=%d", p->rows);
  if (p->D % 128 != 0) return layernorm_fwd_small(p, stream);
  VT_REQUIRE(p->D % 128 == 0 && p->D >= 128 && p->D <= 1024, "vt_layernorm_fwd: D=%d unsupported (multiple of 128, <=1024)", p->D);
  VT_REQUIRE(p->ldx % 4 == 0, "vt_layernorm_fwd: ldx must be a multiple of 4");
  VT_REQUIRE(aligned16(p->x) && aligned16(p->gamma) && aligned16(p->beta) && aligned16(p->y),
             "vt_layernorm_fwd: x, gamma, beta and y must be 16-byte aligned (D=%d)", p->D);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int blocks = ln_blocks(p->rows);
#define VT_LN_FWD(V)                                                                                                    \
  case V:                                                                                                               \
    ln_fwd_kernel<V><<<blocks, LN_WARPS * 32, 0, st>>>(p->x, p->ldx, p->in_row, p->gamma, p->beta, p->y, p->mean,       \
                                                       p->rstd, p->rows, p->eps, p->y_fp32);                           \
    break;
  switch (p->D / 128) {
    VT_LN_FWD(1) VT_LN_FWD(2) VT_LN_FWD(3) VT_LN_FWD(4) VT_LN_FWD(5) VT_LN_FWD(6) VT_LN_FWD(7) VT_LN_FWD(8)
  }
#undef VT_LN_FWD
  return check_launch("ln_fwd_kernel");
}

extern "C" int vt_ln_bwd_blocks(int32_t rows) { return ln_blocks(rows); }

extern "C" int vt_layernorm_bwd(const vt_ln_bwd_params* p, void* stream) {
  VT_REQUIRE(p && p->dy && p->x && p->mean && p->rstd && p->gamma && p->dx && p->partials, "vt_layernorm_bwd: null pointer");
  VT_REQUIRE(p->rows > 0, "vt_layernorm_bwd: rows=%d", p->rows);
  if (p->D % 128 != 0) return layernorm_bwd_small(p, stream);
  VT_REQUIRE(p->D % 128 == 0 && p->D >= 128 && p->D <= 1024, "vt_layernorm_bwd: D=%d unsupported", p->D);
  VT_REQUIRE(p->ldx % 4 == 0 && p->lddx % 4 == 0, "vt_layernorm_bwd: ldx and lddx must be multiples of 4");
  // dy is read as uint2 (bf16) or float4 (fp32) vectors, everything else as float4
  VT_REQUIRE((reinterpret_cast<uintptr_t>(p->dy) & (p->dy_fp32 ? 15 : 7)) == 0 && aligned16(p->x) && aligned16(p->gamma) &&
                 aligned16(p->dx) && aligned16(p->dres) && aligned16(p->dx_aux) && aligned16(p->partials),
             "vt_layernorm_bwd: dy, x, gamma, dx, dres, dx_aux and partials must be 16-byte aligned (bf16 dy: 8-byte)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int blocks = ln_blocks(p->rows);
  const bool v2 = feature_on("VT_LN_BWD_V2", false);
#define VT_LN_BWD(V)                                                                                                    \
  case V:                                                                                                               \
    if (v2)                                                                                                             \
      ln_bwd2_kernel<V><<<blocks, LN_WARPS * 32, 0, st>>>(p->dy, p->dy_fp32, p->x, p->ldx, p->in_row, p->mean, p->rstd, \
                                                          p->gamma, p->dres, p->dx, p->lddx, p->dx_aux, p->out_row,     \
                                                          p->partials, p->rows);                                        \
    else                                                                                                                \
      ln_bwd_kernel<V><<<blocks, LN_WARPS * 32, 0, st>>>(p->dy, p->dy_fp32, p->x, p->ldx, p->in_row, p->mean, p->rstd,  \
                                                         p->gamma, p->dres, p->dx, p->lddx, p->dx_aux, p->out_row,      \
                                                         p->partials, p->rows);                                         \
    break;
  switch (p->D / 128) {
    VT_LN_BWD(1) VT_LN_BWD(2) VT_LN_BWD(3) VT_LN_BWD(4) VT_LN_BWD(5) VT_LN_BWD(6) VT_LN_BWD(7) VT_LN_BWD(8)
  }
#undef VT_LN_BWD
  return check_launch("ln_bwd_kernel");
}

extern "C" int vt_cast_f32_bf16(const vt_cast_params* p, void* stream) {
  VT_REQUIRE(p && p->src && p->dst && p->n > 0, "vt_cast_f32_bf16: bad params");
  VT_REQUIRE(p->n < 8 || (aligned16(p->src) && aligned16(p->dst)), "vt_cast_f32_bf16: src and dst must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long n8 = p->n / 8;
  if (n8 > 0) cast_kernel<<<grid_for(n8, 256), 256, 0, st>>>(p->src, static_cast<__nv_bfloat16*>(p->dst), n8);
  if (p->n % 8) cast_tail_kernel<<<1, 32, 0, st>>>(p->src, static_cast<__nv_bfloat16*>(p->dst), n8 * 8, p->n);
  return check_launch("cast_kernel");
}

extern "C" int vt_gather_cast_bf16(const vt_gather_cast_params* p, void* stream) {
  VT_REQUIRE(p && p->src && p->dst && p->rows > 0, "vt_gather_cast_bf16: bad params");
  VT_REQUIRE(p->D % 8 == 0 && p->lds % 4 == 0, "vt_gather_cast_bf16: D %% 8 and lds %% 4 required");
  VT_REQUIRE(aligned16(p->src) && aligned16(p->dst), "vt_gather_cast_bf16: src and dst must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int blocks = grid_for((long long)p->rows * 32, 256);
  gather_cast_kernel<<<blocks, 256, 0, st>>>(p->src, p->lds, p->in_row, p->row_scale, static_cast<__nv_bfloat16*>(p->dst),
                                             p->rows, p->D / 8);
  return check_launch("gather_cast_kernel");
}

namespace vt { int launch_reduce_rows(const float*, float*, long long, int, long long, int, float, cudaStream_t); }

extern "C" int vt_colsum_chunks(int32_t M) { return (M + COLSUM_ROWS - 1) / COLSUM_ROWS; }   // rows of the partial-sum workspace

extern "C" int vt_colsum_bf16(const vt_colsum_params* p, void* stream) {
  VT_REQUIRE(p && p->in && p->out && p->workspace && p->M > 0 && p->N > 0, "vt_colsum_bf16: bad params");
  VT_REQUIRE(p->N % 4 == 0 && p->ld % 2 == 0, "vt_colsum_bf16: N %% 4 and ld %% 2 required");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int chunks = vt_colsum_chunks(p->M);
  dim3 grid((p->N + 63) / 64, chunks);
  colsum_kernel<<<grid, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(p->in), p->ld, p->M, p->N, p->workspace, p->out,
                                      p->counters);
  int rc = check_launch("colsum_kernel");
  if (rc || p->counters) return rc;
  return launch_reduce_rows(p->workspace, p->out, p->N, chunks, p->N, 0, 1.0f, st);
}

extern "C" int vt_im2col_bf16(const vt_im2col_params* p, void* stream) {
  VT_REQUIRE(p && p->x && p->cols, "vt_im2col_bf16: null pointer");
  VT_REQUIRE(p->pw % 8 == 0 && p->W % p->pw == 0 && p->H % p->ph == 0 && p->T % p->tube == 0 && p->W % 4 == 0,
             "vt_im2col_bf16: unsupported geometry");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long total8 = (long long)p->B * p->T * p->C * p->H * p->W / 8;
  im2col_kernel<<<grid_for(total8, 256), 256, 0, st>>>(p->x, static_cast<__nv_bfloat16*>(p->cols), p->B, p->T, p->C, p->H,
                                                       p->W, p->tube, p->ph, p->pw, total8);
  return check_launch("im2col_kernel");
}

extern "C" int vt_im2col_u8_bf16(const vt_im2col_u8_params* p, void* stream) {
  VT_REQUIRE(p && p->x && p->scale && p->shift && p->cols, "vt_im2col_u8_bf16: null pointer");
  VT_REQUIRE(p->pw % 8 == 0 && p->W % p->pw == 0 && p->H % p->ph == 0 && p->T % p->tube == 0, "vt_im2col_u8_bf16: unsupported geometry");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long total8 = (long long)p->B * p->T * p->C * p->H * p->W / 8;
  im2col_u8_kernel<<<grid_for(total8, 256), 256, 0, st>>>(p->x, p->scale, p->shift, static_cast<__nv_bfloat16*>(p->cols), p->B,
                                                          p->T, p->C, p->H, p->W, p->tube, p->ph, p->pw, total8);
  return check_launch("im2col_u8_kernel");
}

extern "C" int vt_col2im_f32(const vt_col2im_params* p, void* stream) {
  VT_REQUIRE(p && p->cols && p->dx, "vt_col2im_f32: null pointer");
  VT_REQUIRE(p->pw % 4 == 0 && p->W % p->pw == 0 && p->H % p->ph == 0 && p->T % p->tube == 0, "vt_col2im_f32: unsupported geometry");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long total4 = (long long)p->B * p->T * p->C * p->H * p->W / 4;
  col2im_kernel<<<grid_for(total4, 256), 256, 0, st>>>(p->cols, p->dx, p->B, p->T, p->C, p->H, p->W, p->tube, p->ph, p->pw,
                                                       total4);
  return check_launch("col2im_kernel");
}

extern "C" int vt_gelu_fwd_bf16(const vt_gelu_params* p, void* stream) {
  VT_REQUIRE(p && p->z && p->out && p->n > 0 && p->n % 8 == 0, "vt_gelu_fwd_bf16: bad params (n %% 8 == 0 required)");
  const long long n8 = p->n / 8;
  gelu_fwd_kernel<<<grid_for(n8, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const uint4*>(p->z),
                                                                                   static_cast<uint4*>(p->out), n8);
  return check_launch("gelu_fwd_kernel");
}

extern "C" int vt_gelu_bwd_bf16(const vt_gelu_params* p, void* stream) {
  VT_REQUIRE(p && p->z && p->dh && p->out && p->n > 0 && p->n % 8 == 0, "vt_gelu_bwd_bf16: bad params");
  const long long n8 = p->n / 8;
  gelu_bwd_kernel<<<grid_for(n8, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(p->dh), static_cast<const uint4*>(p->z), static_cast<uint4*>(p->out), n8);
  return check_launch("gelu_bwd_kernel");
}

// partial rows of the fused producer + column-sum kernels (one per CTA)
static int fused_colsum_blocks(int rows_per_step, int rows, int per_sm) {
  long long b = ((long long)rows + rows_per_step - 1) / rows_per_step;
  const long long cap = (long long)sm_count() * per_sm;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}
extern "C" int vt_gather_cast_colsum_blocks(int32_t rows) { return fused_colsum_blocks(8, rows, 2); }
extern "C" int vt_gelu_bwd_colsum_blocks(int32_t M) { return fused_colsum_blocks(GBC_UNROLL, M, 4); }

extern "C" int vt_gather_cast_colsum_bf16(const vt_gather_cast_colsum_params* p, void* stream) {
  VT_REQUIRE(p && p->src && p->dst && p->colsum && p->workspace && p->rows > 0, "vt_gather_cast_colsum_bf16: bad params");
  VT_REQUIRE(p->D % 8 == 0 && p->lds % 4 == 0 && p->D <= GCC_CH * 256, "vt_gather_cast_colsum_bf16: D %% 8, lds %% 4 and D <= %d required", GCC_CH * 256);
  VT_REQUIRE(aligned16(p->src) && aligned16(p->dst), "vt_gather_cast_colsum_bf16: src and dst must be 16-byte aligned");
  const int blocks = vt_gather_cast_colsum_blocks(p->rows);
  VT_REQUIRE(p->workspace_rows >= blocks, "vt_gather_cast_colsum_bf16: workspace holds %d partial rows, %d needed", p->workspace_rows, blocks);
  const int W = p->unscaled_sums ? 2 * p->D : p->D;     // colsum then holds [scaled sums | sums before the row scale]
  if (p->unscaled_sums)
    gather_cast_colsum_kernel<true><<<blocks, 256, 8 * p->D * sizeof(float), static_cast<cudaStream_t>(stream)>>>(
        p->src, p->lds, p->in_row, p->row_scale, static_cast<__nv_bfloat16*>(p->dst), p->rows, p->D / 8, p->workspace);
  else
    gather_cast_colsum_kernel<false><<<blocks, 256, 8 * p->D * sizeof(float), static_cast<cudaStream_t>(stream)>>>(
        p->src, p->lds, p->in_row, p->row_scale, static_cast<__nv_bfloat16*>(p->dst), p->rows, p->D / 8, p->workspace);
  const int rc = check_launch("gather_cast_colsum_kernel");
  if (rc) return rc;
  return launch_reduce_rows(p->workspace, p->colsum, W, blocks, W, 0, 1.0f, static_cast<cudaStream_t>(stream));
}

extern "C" int vt_gelu_bwd_colsum_bf16(const vt_gelu_bwd_colsum_params* p, void* stream) {
  VT_REQUIRE(p && p->z && p->dh && p->out && p->colsum && p->workspace && p->M > 0 && p->N > 0, "vt_gelu_bwd_colsum_bf16: bad params");
  VT_REQUIRE(p->N % 256 == 0 && p->N <= 8192, "vt_gelu_bwd_colsum_bf16: N must be a multiple of 256, at most 8192 (got %d)", p->N);
  const int blocks = vt_gelu_bwd_colsum_blocks(p->M);
  VT_REQUIRE(p->workspace_rows >= blocks, "vt_gelu_bwd_colsum_bf16: workspace holds %d partial rows, %d needed", p->workspace_rows, blocks);
  gelu_bwd_colsum_kernel<<<blocks, p->N / 8, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(p->dh), static_cast<const uint4*>(p->z), static_cast<uint4*>(p->out), p->M, p->N / 8, p->workspace);
  const int rc = check_launch("gelu_bwd_colsum_kernel");
  if (rc) return rc;
  return launch_reduce_rows(p->workspace, p->colsum, p->N, blocks, p->N, 0, 1.0f, static_cast<cudaStream_t>(stream));
}
