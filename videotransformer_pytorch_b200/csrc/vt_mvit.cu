// MaskFeat / MViT kernels (SURVEY §8 a13-a15): depthwise-conv pooling + LayerNorm of q/k/v, strided pooling attention
// (head dim 96), skip-path max pooling, overlapping Conv3d im2col, token preparation and the masked-MSE loss.
// Block arithmetic follows pytorchvideo's MultiScaleBlock as configured by video_transformer.py:764-785; the CPU
// restatement is oracle/mvit_oracle.py.
#include <math.h>
#include <string.h>

#include "vt_attention_mma.cuh"

namespace vt {

constexpr int ROW_WARPS = 8;   // warp-per-row kernels: 8 rows per CTA step

static int row_blocks(long long rows, int per_sm) {
  long long blocks = (rows + ROW_WARPS - 1) / ROW_WARPS;
  const long long cap = (long long)sm_count() * per_sm;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}
static int flat_blocks(long long n, int threads) {
  long long blocks = (n + threads - 1) / threads;
  const long long cap = (long long)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

__device__ __forceinline__ float bf2f(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// ================================================================================================
// LayerNorm for narrow rows: D = 32*E, one warp per row, lane owns columns lane + 32*i (coalesced 128-B segments).
// Same contract as ln_fwd_kernel / ln_bwd_kernel of vt_elementwise.cu without row maps.
// ================================================================================================
// STATS = false: mean / rstd are not written (forward-only calls); a template flag, so the saving form's code is unchanged
template <int E, bool STATS>
__global__ void __launch_bounds__(ROW_WARPS * 32)
ln_small_fwd_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ gamma,
                    const float* __restrict__ beta, void* __restrict__ y, float* __restrict__ mean,
                    float* __restrict__ rstd, int rows, float eps, int y_fp32) {
  constexpr int D = 32 * E;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float g[E], b[E];
#pragma unroll
  for (int i = 0; i < E; ++i) {
    g[i] = __ldg(gamma + lane + 32 * i);
    b[i] = __ldg(beta + lane + 32 * i);
  }
  for (int m = blockIdx.x * ROW_WARPS + warp; m < rows; m += gridDim.x * ROW_WARPS) {
    const float* xr = x + (long long)m * ldx;
    float v[E];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < E; ++i) {
      v[i] = xr[lane + 32 * i];
      s += v[i];
    }
    // rounded before use (never contracted into the subtractions below), so both STATS forms give the same bits
    const float mu = __fmul_rn(warp_sum(s), 1.0f / D);
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < E; ++i) {
      const float d = v[i] - mu;
      ss += d * d;
    }
    const float rs = rsqrtf(warp_sum(ss) * (1.0f / D) + eps);
    if (STATS && lane == 0) {
      mean[m] = mu;
      rstd[m] = rs;
    }
#pragma unroll
    for (int i = 0; i < E; ++i) {
      const float o = (v[i] - mu) * rs * g[i] + b[i];
      if (y_fp32) static_cast<float*>(y)[(long long)m * D + lane + 32 * i] = o;
      else static_cast<__nv_bfloat16*>(y)[(long long)m * D + lane + 32 * i] = __float2bfloat16_rn(o);
    }
  }
}

// partials: [gridDim.x][2][D] (dgamma row, dbeta row) like ln_bwd_kernel
template <int E>
__global__ void __launch_bounds__(ROW_WARPS * 32)
ln_small_bwd_kernel(const void* __restrict__ dy, int dy_fp32, const float* __restrict__ x, long long ldx,
                    const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
                    const float* __restrict__ dres, float* __restrict__ dx, long long lddx,
                    float* __restrict__ partials, int rows) {
  constexpr int D = 32 * E;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float g[E], dg[E], db[E];
#pragma unroll
  for (int i = 0; i < E; ++i) {
    g[i] = __ldg(gamma + lane + 32 * i);
    dg[i] = 0.f;
    db[i] = 0.f;
  }
  for (int m = blockIdx.x * ROW_WARPS + warp; m < rows; m += gridDim.x * ROW_WARPS) {
    const float* xr = x + (long long)m * ldx;
    const float mu = mean[m], rs = rstd[m];
    float xh[E], gy[E];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < E; ++i) {
      const long long at = (long long)m * D + lane + 32 * i;
      const float d = dy_fp32 ? static_cast<const float*>(dy)[at] : __bfloat162float(static_cast<const __nv_bfloat16*>(dy)[at]);
      xh[i] = (xr[lane + 32 * i] - mu) * rs;
      dg[i] += d * xh[i];
      db[i] += d;
      gy[i] = d * g[i];
      s1 += gy[i];
      s2 += gy[i] * xh[i];
    }
    const float m1 = warp_sum(s1) * (1.0f / D);
    const float m2 = warp_sum(s2) * (1.0f / D);
#pragma unroll
    for (int i = 0; i < E; ++i) {
      float o = rs * (gy[i] - m1 - xh[i] * m2);
      if (dres) o += dres[(long long)m * lddx + lane + 32 * i];
      dx[(long long)m * lddx + lane + 32 * i] = o;
    }
  }
  __shared__ float sh[ROW_WARPS][32];
  float* pg = partials + (long long)blockIdx.x * 2 * D;
#pragma unroll
  for (int i = 0; i < E; ++i) {
    for (int pass = 0; pass < 2; ++pass) {
      __syncthreads();
      sh[warp][lane] = pass == 0 ? dg[i] : db[i];
      __syncthreads();
      if (warp == 0) {
        float a = sh[0][lane];
        for (int w = 1; w < ROW_WARPS; ++w) a += sh[w][lane];
        pg[pass * D + lane + 32 * i] = a;
      }
    }
  }
}

// ================================================================================================
// q/k/v pooling: depthwise 3x3x3 Conv3d (padding 1) over the (T,H,W) token grid + LayerNorm(hd), one warp per output
// row (b, h, l).  Filter taps sit in shared memory as [tap][hd] so a lane reads its own channels conflict-free.
// ================================================================================================
struct PoolDims {
  int B, H, T, Hin, Win, st, sh, sw, To, Ho, Wo;
};

// STATS = false: pooled / mean / rstd are not written (forward-only calls)
template <int E, bool STATS>
__global__ void __launch_bounds__(ROW_WARPS * 32)
pool_ln_fwd_kernel(const __nv_bfloat16* __restrict__ in, long long in_bs, long long in_rs,
                   const float* __restrict__ w, const float* __restrict__ gamma, const float* __restrict__ beta,
                   float* __restrict__ pooled, __nv_bfloat16* __restrict__ out, float* __restrict__ mean,
                   float* __restrict__ rstd, PoolDims d, float eps) {
  constexpr int HD = 32 * E;
  __shared__ float sw[27 * HD];
  for (int i = threadIdx.x; i < 27 * HD; i += blockDim.x) {
    const int tap = i / HD, c = i % HD;
    sw[i] = w[c * 27 + tap];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float g[E], bt[E];
#pragma unroll
  for (int i = 0; i < E; ++i) {
    g[i] = __ldg(gamma + lane + 32 * i);
    bt[i] = __ldg(beta + lane + 32 * i);
  }
  const int Lo1 = 1 + d.To * d.Ho * d.Wo;
  const int rows = d.B * d.H * Lo1;                             // < 2^31, checked by the launcher
  for (int r = blockIdx.x * ROW_WARPS + warp; r < rows; r += gridDim.x * ROW_WARPS) {
    const int bh = r / Lo1, l = r - bh * Lo1;
    const int b = bh / d.H, h = bh - b * d.H;
    const __nv_bfloat16* base = in + (long long)b * in_bs + (long long)h * HD;
    float acc[E];
#pragma unroll
    for (int i = 0; i < E; ++i) acc[i] = 0.f;
    if (l == 0) {
#pragma unroll
      for (int i = 0; i < E; ++i) acc[i] = bf2f(base + lane + 32 * i);
    } else {
      const int o = l - 1;
      const int o2 = o / d.Wo;
      const int ow = o - o2 * d.Wo, ot = o2 / d.Ho, oh = o2 - ot * d.Ho;
      // the nine (dh, dw) taps of a dt plane are loaded unconditionally from clamped coordinates (out-of-range taps are
      // zeroed after the load) so that all of them are in flight together; dt planes outside the clip are skipped
      int hrow[3], wcol[3];
      bool hok[3], wok[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int hi = oh * d.sh - 1 + k, wi = ow * d.sw - 1 + k;
        hok[k] = hi >= 0 && hi < d.Hin;
        wok[k] = wi >= 0 && wi < d.Win;
        hrow[k] = min(max(hi, 0), d.Hin - 1);
        wcol[k] = min(max(wi, 0), d.Win - 1);
      }
      for (int dt = 0; dt < 3; ++dt) {
        const int ti = ot * d.st - 1 + dt;
        if (ti < 0 || ti >= d.T) continue;
        float x[9][E];
#pragma unroll
        for (int dh = 0; dh < 3; ++dh)
#pragma unroll
          for (int dw = 0; dw < 3; ++dw) {
            const __nv_bfloat16* src = base + (1 + ((long long)ti * d.Hin + hrow[dh]) * d.Win + wcol[dw]) * in_rs;
#pragma unroll
            for (int i = 0; i < E; ++i) x[dh * 3 + dw][i] = bf2f(src + lane + 32 * i);
          }
#pragma unroll
        for (int dh = 0; dh < 3; ++dh)
#pragma unroll
          for (int dw = 0; dw < 3; ++dw) {
            const float* f = sw + ((dt * 3 + dh) * 3 + dw) * HD;
            const bool ok = hok[dh] && wok[dw];
#pragma unroll
            for (int i = 0; i < E; ++i) acc[i] = fmaf(ok ? x[dh * 3 + dw][i] : 0.f, f[lane + 32 * i], acc[i]);
          }
      }
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < E; ++i) s += acc[i];
    const float mu = __fmul_rn(warp_sum(s), 1.0f / HD);   // rounded before use, as in ln_small_fwd_kernel
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < E; ++i) {
      const float c = acc[i] - mu;
      ss += c * c;
    }
    const float rs = rsqrtf(warp_sum(ss) * (1.0f / HD) + eps);
    if (STATS && lane == 0) {
      mean[r] = mu;
      rstd[r] = rs;
    }
#pragma unroll
    for (int i = 0; i < E; ++i) {
      if (STATS) pooled[(long long)r * HD + lane + 32 * i] = acc[i];
      out[(long long)r * HD + lane + 32 * i] = __float2bfloat16_rn((acc[i] - mu) * rs * g[i] + bt[i]);
    }
  }
}

// gradient w.r.t. the pooling input: one warp per input token (b, n), looping over the heads; gathers the outputs whose
// window covers the token.  Which output (if any) is reached through tap k along an axis is a pure function of the
// coordinate, so it is tabulated once per CTA — the row loop itself is free of div/mod chains (they dominated the
// first version of this kernel).
constexpr int POOL_MAX_DIM = 64;

template <int E>
__global__ void __launch_bounds__(ROW_WARPS * 32)
pool_din_kernel(const float* __restrict__ dpooled, const float* __restrict__ w, __nv_bfloat16* __restrict__ din,
                long long din_bs, long long din_rs, PoolDims d) {
  constexpr int HD = 32 * E;
  __shared__ float sw[27 * HD];
  __shared__ short tab[3][3][POOL_MAX_DIM];     // [axis t/h/w][tap][input coordinate] -> output coordinate, -1 = none
  for (int i = threadIdx.x; i < 27 * HD; i += blockDim.x) {
    const int tap = i / HD, c = i % HD;
    sw[i] = w[c * 27 + tap];
  }
  for (int i = threadIdx.x; i < 9 * POOL_MAX_DIM; i += blockDim.x) {
    const int axis = i / (3 * POOL_MAX_DIM), k = (i / POOL_MAX_DIM) % 3, c = i % POOL_MAX_DIM;
    const int n_in = axis == 0 ? d.T : axis == 1 ? d.Hin : d.Win;
    const int s = axis == 0 ? d.st : axis == 1 ? d.sh : d.sw;
    const int n_out = axis == 0 ? d.To : axis == 1 ? d.Ho : d.Wo;
    int v = -1;
    if (c < n_in) {
      const int nn = c + 1 - k;                   // o * s - 1 + k == c
      if (nn >= 0 && nn % s == 0 && nn / s < n_out) v = nn / s;
    }
    tab[axis][k][c] = (short)v;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int L1 = 1 + d.T * d.Hin * d.Win;
  const int Lo1 = 1 + d.To * d.Ho * d.Wo;
  const int tokens = d.B * L1;
  for (int tok = blockIdx.x * ROW_WARPS + warp; tok < tokens; tok += gridDim.x * ROW_WARPS) {
    const int b = tok / L1, n = tok - b * L1;
    __nv_bfloat16* dst = din + (long long)b * din_bs + (long long)n * din_rs;
    int ot3[3], oh3[3], ow3[3];
    if (n > 0) {
      const int idx = n - 1;
      const int t2 = idx / d.Win;
      const int wi = idx - t2 * d.Win, ti = t2 / d.Hin, hi = t2 - ti * d.Hin;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        ot3[k] = tab[0][k][ti];
        oh3[k] = tab[1][k][hi];
        ow3[k] = tab[2][k][wi];
      }
    }
    for (int h = 0; h < d.H; ++h) {
      const float* dp = dpooled + ((long long)b * d.H + h) * Lo1 * HD;
      float acc[E];
#pragma unroll
      for (int i = 0; i < E; ++i) acc[i] = 0.f;
      if (n == 0) {
#pragma unroll
        for (int i = 0; i < E; ++i) acc[i] = dp[lane + 32 * i];
      } else {
#pragma unroll
        for (int dt = 0; dt < 3; ++dt) {
          if (ot3[dt] < 0) continue;
#pragma unroll
          for (int dh = 0; dh < 3; ++dh) {
            if (oh3[dh] < 0) continue;
#pragma unroll
            for (int dw = 0; dw < 3; ++dw) {
              if (ow3[dw] < 0) continue;
              const float* src = dp + (1 + (ot3[dt] * d.Ho + oh3[dh]) * d.Wo + ow3[dw]) * HD;
              const float* f = sw + ((dt * 3 + dh) * 3 + dw) * HD;
#pragma unroll
              for (int i = 0; i < E; ++i) acc[i] = fmaf(src[lane + 32 * i], f[lane + 32 * i], acc[i]);
            }
          }
        }
      }
#pragma unroll
      for (int i = 0; i < E; ++i) dst[h * HD + lane + 32 * i] = __float2bfloat16_rn(acc[i]);
    }
  }
}

// filter gradient: dw[c][tap] = sum over output rows of dpooled[row][c] * in[window tap][c].
// CTA = 27 warps, warp = filter tap, lane = channels (c = lane + 32 i): every (tap, channel) sum is owned by one thread, so
// there is no cross-warp reduction; rows are walked four at a time with all loads issued before the FMAs.
// Per-CTA partial rows [hd*27] are summed by reduce_rows.
constexpr int DW_ROWS_UNROLL = 4;

template <int E>
__global__ void __launch_bounds__(27 * 32)
pool_dw_kernel(const float* __restrict__ dpooled, const __nv_bfloat16* __restrict__ in, long long in_bs, long long in_rs,
               float* __restrict__ partials, PoolDims d, int rows_per_cta) {
  constexpr int HD = 32 * E;
  const int tap = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int dt = tap / 9, dh = (tap / 3) % 3, dw = tap % 3;
  const int Lo = d.To * d.Ho * d.Wo;
  const long long rows = (long long)d.B * d.H * Lo;
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const long long r1 = min(rows, r0 + rows_per_cta);
  float acc[E];
#pragma unroll
  for (int i = 0; i < E; ++i) acc[i] = 0.f;
  // (b, h, ot, oh, ow) of the current row: decoded once, then advanced like an odometer (rows of a CTA are consecutive)
  int ow, oh, ot, h, b;
  {
    const long long rs = min(r0, rows - 1);
    const int o = (int)(rs % Lo);
    const int bh = (int)(rs / Lo);
    h = bh % d.H;
    b = bh / d.H;
    ow = o % d.Wo;
    oh = (o / d.Wo) % d.Ho;
    ot = o / (d.Wo * d.Ho);
  }
  for (long long rb = r0; rb < r1; rb += DW_ROWS_UNROLL) {
    float g[DW_ROWS_UNROLL][E], x[DW_ROWS_UNROLL][E];
    bool ok[DW_ROWS_UNROLL];
#pragma unroll
    for (int u = 0; u < DW_ROWS_UNROLL; ++u) {
      const bool live = rb + u < r1;                             // past the end: re-read the last row, masked
      const int ti = ot * d.st - 1 + dt, hi = oh * d.sh - 1 + dh, wi = ow * d.sw - 1 + dw;
      ok[u] = live && ti >= 0 && ti < d.T && hi >= 0 && hi < d.Hin && wi >= 0 && wi < d.Win;
      const int tc = min(max(ti, 0), d.T - 1), hc = min(max(hi, 0), d.Hin - 1), wc = min(max(wi, 0), d.Win - 1);
      const int o = (ot * d.Ho + oh) * d.Wo + ow;
      const float* dp = dpooled + (((long long)b * d.H + h) * (Lo + 1) + 1 + o) * HD;
      const __nv_bfloat16* src = in + (long long)b * in_bs + (long long)h * HD + (1 + ((long long)tc * d.Hin + hc) * d.Win + wc) * in_rs;
#pragma unroll
      for (int i = 0; i < E; ++i) {
        g[u][i] = dp[lane + 32 * i];
        x[u][i] = bf2f(src + lane + 32 * i);
      }
      if (rb + u + 1 < r1) {
        if (++ow == d.Wo) {
          ow = 0;
          if (++oh == d.Ho) {
            oh = 0;
            if (++ot == d.To) {
              ot = 0;
              if (++h == d.H) {
                h = 0;
                ++b;
              }
            }
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < DW_ROWS_UNROLL; ++u)
#pragma unroll
      for (int i = 0; i < E; ++i) acc[i] = fmaf(ok[u] ? g[u][i] : 0.f, x[u][i], acc[i]);
  }
  float* pg = partials + (long long)blockIdx.x * 27 * HD;
#pragma unroll
  for (int i = 0; i < E; ++i) pg[(lane + 32 * i) * 27 + tap] = acc[i];
}

// ================================================================================================
// Second generation of the three pooling kernels (head dim 96): lane l < 24 owns the four consecutive channels
// [4l, 4l+4) of a head, so one token row of a head is ONE 8-byte load per lane (bf16) or one 16-byte load (fp32) instead
// of three 2-byte / 4-byte ones, filter taps sit in shared memory as float4 [tap][lane], and every tap of a window is
// in flight before the first FMA.  Lanes 24..31 carry zeros through the warp reductions.
//   d(input): CTA = one (b, t) plane of the input grid and one head, warp = token; the covering outputs come from the
//             per-axis tables, the nine taps of a time plane are in flight together, tokens without any store zeros
//   (the forward kernel keeps the first-generation mapping: a 27 x 8-byte-load version measured slower, 1.35 vs 1.08 ms)
//   d(filter): warp = (pooled row, time tap): 9 taps x 4 channels of accumulators per lane, CTA = 4 row slots x 3 time
//             taps; the four slots are summed in shared memory in a fixed order (deterministic), one partial row per CTA
// Needs 8-byte aligned token rows (row / batch strides multiples of 4 elements) — the launchers check.
// ================================================================================================
constexpr int PV_LANES = 24;
constexpr int PV_HD = 96;

__device__ __forceinline__ void bf16x4_to_f(uint2 raw, float (&f)[4]) {
  f[0] = __uint_as_float(raw.x << 16);
  f[1] = __uint_as_float(raw.x & 0xffff0000u);
  f[2] = __uint_as_float(raw.y << 16);
  f[3] = __uint_as_float(raw.y & 0xffff0000u);
}
__device__ __forceinline__ uint2 f_to_bf16x4(const float (&f)[4]) {
  const __nv_bfloat162 a = __floats2bfloat162_rn(f[0], f[1]), b = __floats2bfloat162_rn(f[2], f[3]);
  uint2 r;
  r.x = *reinterpret_cast<const unsigned*>(&a);
  r.y = *reinterpret_cast<const unsigned*>(&b);
  return r;
}
// filter taps as float4 [tap][lane]: element j of entry (tap, l) is w[(4l + j) * 27 + tap]
__device__ __forceinline__ void stage_taps(float4* sw4, const float* __restrict__ w) {
  for (int i = threadIdx.x; i < 27 * PV_LANES; i += blockDim.x) {
    const int tap = i / PV_LANES, l = i - tap * PV_LANES;
    sw4[i] = make_float4(w[(4 * l + 0) * 27 + tap], w[(4 * l + 1) * 27 + tap], w[(4 * l + 2) * 27 + tap], w[(4 * l + 3) * 27 + tap]);
  }
}

// blockIdx.y = (b, ti) plane of the input grid (one extra y for the B cls tokens): the time taps are decoded once per CTA,
// a token costs one division, and tokens no output window covers (most of them at strides 4 and 8) leave through a
// zero store without touching the gradient
__global__ void __launch_bounds__(ROW_WARPS * 32)
pool_din_v2_kernel(const float* __restrict__ dpooled, const float* __restrict__ w, __nv_bfloat16* __restrict__ din,
                   long long din_bs, long long din_rs, PoolDims d) {
  __shared__ float4 sw4[27 * PV_LANES];
  __shared__ short tab[3][3][POOL_MAX_DIM];     // [axis t/h/w][tap][input coordinate] -> output coordinate, -1 = none
  stage_taps(sw4, w);
  for (int i = threadIdx.x; i < 9 * POOL_MAX_DIM; i += blockDim.x) {
    const int axis = i / (3 * POOL_MAX_DIM), k = (i / POOL_MAX_DIM) % 3, c = i % POOL_MAX_DIM;
    const int n_in = axis == 0 ? d.T : axis == 1 ? d.Hin : d.Win;
    const int s = axis == 0 ? d.st : axis == 1 ? d.sh : d.sw;
    const int n_out = axis == 0 ? d.To : axis == 1 ? d.Ho : d.Wo;
    int v = -1;
    if (c < n_in) {
      const int nn = c + 1 - k;                   // o * s - 1 + k == c
      if (nn >= 0 && nn % s == 0 && nn / s < n_out) v = nn / s;
    }
    tab[axis][k][c] = (short)v;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool act = lane < PV_LANES;
  const int cl = act ? lane : 0;
  const int Lo1 = 1 + d.To * d.Ho * d.Wo;
  const int planes = d.B * d.T;
  const int h = blockIdx.z;                        // one head per CTA: 4 - 8x more warps in flight than looping over the heads
  if ((int)blockIdx.y == planes) {                 // cls tokens: straight copy of the pooled cls gradient
    for (int b = blockIdx.x * ROW_WARPS + warp; b < d.B; b += gridDim.x * ROW_WARPS) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(dpooled + ((long long)b * d.H + h) * Lo1 * PV_HD + 4 * cl));
      const float v[4] = {g.x, g.y, g.z, g.w};
      if (act) *reinterpret_cast<uint2*>(din + (long long)b * din_bs + h * PV_HD + 4 * lane) = f_to_bf16x4(v);
    }
    return;
  }
  const int b = blockIdx.y / d.T, ti = blockIdx.y - b * d.T;
  int ot3[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) ot3[k] = tab[0][k][ti];
  const bool t_any = ot3[0] >= 0 || ot3[1] >= 0 || ot3[2] >= 0;
  const int HW = d.Hin * d.Win;
  const float* dp = dpooled + (((long long)b * d.H + h) * Lo1 + 1) * PV_HD + 4 * cl;
  for (int idx = blockIdx.x * ROW_WARPS + warp; idx < HW; idx += gridDim.x * ROW_WARPS) {
    const int hi = idx / d.Win, wi = idx - hi * d.Win;
    __nv_bfloat16* dst = din + (long long)b * din_bs + (1 + (long long)ti * HW + idx) * din_rs + h * PV_HD + 4 * lane;
    int rowoff[9];                                 // (oh * Wo + ow) of the output reached through (dh, dw), -1 = none
    bool any = false;
#pragma unroll
    for (int dh = 0; dh < 3; ++dh)
#pragma unroll
      for (int dw = 0; dw < 3; ++dw) {
        const int oh = tab[1][dh][hi], ow = tab[2][dw][wi];
        rowoff[dh * 3 + dw] = oh >= 0 && ow >= 0 ? oh * d.Wo + ow : -1;
        any = any || (oh >= 0 && ow >= 0);
      }
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (any && t_any) {                            // warp-uniform
#pragma unroll
      for (int dt = 0; dt < 3; ++dt) {
        if (ot3[dt] < 0) continue;                 // warp-uniform
        const float* plane = dp + (long long)ot3[dt] * d.Ho * d.Wo * PV_HD;
        float4 g[9];                               // the nine taps of the plane in flight together; absent ones predicated off
#pragma unroll
        for (int k = 0; k < 9; ++k)
          g[k] = rowoff[k] >= 0 ? __ldg(reinterpret_cast<const float4*>(plane + (long long)rowoff[k] * PV_HD)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          if (rowoff[k] < 0) continue;             // warp-uniform
          const float4 f = sw4[(dt * 9 + k) * PV_LANES + cl];
          acc[0] = fmaf(g[k].x, f.x, acc[0]);
          acc[1] = fmaf(g[k].y, f.y, acc[1]);
          acc[2] = fmaf(g[k].z, f.z, acc[2]);
          acc[3] = fmaf(g[k].w, f.w, acc[3]);
        }
      }
    }
    if (act) *reinterpret_cast<uint2*>(dst) = f_to_bf16x4(acc);        // zeros when no output window covers the token
  }
}

constexpr int DW2_SLOTS = 4;                      // pooled rows in flight per CTA (x 3 time taps = 12 warps)
constexpr int DW2_MIN_ROWS_PER_CTA = 8;

__global__ void __launch_bounds__(DW2_SLOTS * 3 * 32)
pool_dw_v2_kernel(const float* __restrict__ dpooled, const __nv_bfloat16* __restrict__ in, long long in_bs, long long in_rs,
                  float* __restrict__ partials, PoolDims d, int rows_per_cta) {
  __shared__ float red[DW2_SLOTS][27 * PV_HD];     // 41 KB
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int slot = warp / 3, dt = warp - slot * 3;
  const bool act = lane < PV_LANES;
  const int cl = act ? lane : 0;
  const int Lo = d.To * d.Ho * d.Wo;
  const long long rows = (long long)d.B * d.H * Lo;
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const long long r1 = min(rows, r0 + rows_per_cta);
  float acc[9][4];
#pragma unroll
  for (int k = 0; k < 9; ++k) acc[k][0] = acc[k][1] = acc[k][2] = acc[k][3] = 0.f;
  for (long long r = r0 + slot; r < r1; r += DW2_SLOTS) {
    const int bh = (int)(r / Lo), o = (int)(r - (long long)bh * Lo);
    const int b = bh / d.H, h = bh - b * d.H;
    const int o2 = o / d.Wo;
    const int ow = o - o2 * d.Wo, ot = o2 / d.Ho, oh = o2 - ot * d.Ho;
    const int ti = ot * d.st - 1 + dt;
    if (ti < 0 || ti >= d.T) continue;             // warp-uniform: this time tap falls outside the clip
    const float4 g = __ldg(reinterpret_cast<const float4*>(dpooled + ((long long)bh * (Lo + 1) + 1 + o) * PV_HD + 4 * cl));
    const __nv_bfloat16* plane = in + (long long)b * in_bs + (long long)h * PV_HD + 4 * cl + (1 + (long long)ti * d.Hin * d.Win) * in_rs;
    uint2 x[9];
    bool ok[9];
#pragma unroll
    for (int dh = 0; dh < 3; ++dh)
#pragma unroll
      for (int dw = 0; dw < 3; ++dw) {
        const int hi = oh * d.sh - 1 + dh, wi = ow * d.sw - 1 + dw;
        ok[dh * 3 + dw] = hi >= 0 && hi < d.Hin && wi >= 0 && wi < d.Win;
        x[dh * 3 + dw] = __ldg(reinterpret_cast<const uint2*>(plane + ((long long)min(max(hi, 0), d.Hin - 1) * d.Win + min(max(wi, 0), d.Win - 1)) * in_rs));
      }
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      float xv[4];
      bf16x4_to_f(x[k], xv);
      const float m = ok[k] ? 1.f : 0.f;
      acc[k][0] = fmaf(g.x * m, xv[0], acc[k][0]);
      acc[k][1] = fmaf(g.y * m, xv[1], acc[k][1]);
      acc[k][2] = fmaf(g.z * m, xv[2], acc[k][2]);
      acc[k][3] = fmaf(g.w * m, xv[3], acc[k][3]);
    }
  }
  if (act) {
#pragma unroll
    for (int k = 0; k < 9; ++k)
#pragma unroll
      for (int j = 0; j < 4; ++j) red[slot][(4 * lane + j) * 27 + dt * 9 + k] = acc[k][j];
  }
  __syncthreads();
  float* pg = partials + (long long)blockIdx.x * 27 * PV_HD;
  for (int i = threadIdx.x; i < 27 * PV_HD; i += blockDim.x) {
    float a = red[0][i];
#pragma unroll
    for (int s2 = 1; s2 < DW2_SLOTS; ++s2) a += red[s2][i];
    pg[i] = a;
  }
}

// ================================================================================================
// Pooling attention, head dim HD (96): CUDA-core flash kernels.
//   forward / dQ: two threads per query row (each owns HD/2 dims), 64 queries per CTA, K/V tiles of 16 keys in smem
//   dK/dV: four threads per key row (each owns HD/4 dims), 32 keys per CTA, Q/dO tiles of 16 queries in smem,
//          query range split over blockIdx.y, fp32 atomics into dk/dv.
// Scores are kept in the log2 domain (q pre-multiplied by scale*log2(e)) so softmax uses ex2.approx.
// ================================================================================================
constexpr int XA_KT = 16;        // keys per shared-memory tile (fwd / dQ)
constexpr int XA_QPB = 64;       // queries per CTA (fwd / dQ)
constexpr int XA_QT = 16;        // queries per shared-memory tile (dK/dV)
constexpr int XA_KPB = 32;       // keys per CTA (dK/dV)
constexpr int XA_QCHUNK = 512;   // queries per CTA along blockIdx.y (dK/dV)
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

struct XaStrides {
  long long q_bs, q_hs, q_rs, k_bs, k_hs, k_rs, v_bs, v_hs, v_rs, o_bs, o_hs, o_rs, dq_bs, dq_hs, dq_rs;
};

// stage `rows` rows of HD bf16 (row r at src + (r0 + r) * rs) as fp32 into dst[r][HD]; rows past `limit` are zero
template <int HD, int ROWS, int THREADS>
__device__ __forceinline__ void stage_rows(float* __restrict__ dst, const __nv_bfloat16* __restrict__ src, long long rs,
                                           int r0, int limit) {
  constexpr int PAIRS = ROWS * HD / 2;
  for (int i = threadIdx.x; i < PAIRS; i += THREADS) {
    const int r = i / (HD / 2), c2 = i % (HD / 2);
    float2 v = make_float2(0.f, 0.f);
    if (r0 + r < limit) {
      const uint32_t u = *reinterpret_cast<const uint32_t*>(src + (long long)(r0 + r) * rs + 2 * c2);
      v = unpack_bf16x2(u);
    }
    dst[r * HD + 2 * c2] = v.x;
    dst[r * HD + 2 * c2 + 1] = v.y;
  }
}

template <int HD, bool LSE>   // LSE = false: lse is not written (forward-only calls)
__global__ void __launch_bounds__(2 * XA_QPB)
xattn_fwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                 const __nv_bfloat16* __restrict__ v, __nv_bfloat16* __restrict__ o, float* __restrict__ lse,
                 XaStrides s, int H, int Nq, int Nk, float scale) {
  constexpr int HALF = HD / 2;
  __shared__ __align__(16) float Ks[XA_KT * HD];
  __shared__ __align__(16) float Vs[XA_KT * HD];
  const int bh = blockIdx.y, b = bh / H, h = bh % H;
  const int pair = threadIdx.x >> 1, half = threadIdx.x & 1;
  const int qi = blockIdx.x * XA_QPB + pair;
  const bool valid = qi < Nq;
  const __nv_bfloat16* kb = k + (long long)b * s.k_bs + (long long)h * s.k_hs;
  const __nv_bfloat16* vb = v + (long long)b * s.v_bs + (long long)h * s.v_hs;
  float qr[HALF], acc[HALF];
  {
    const __nv_bfloat16* qp = q + (long long)b * s.q_bs + (long long)h * s.q_hs + (long long)(valid ? qi : 0) * s.q_rs + half * HALF;
    const float c = scale * LOG2E;
#pragma unroll
    for (int d2 = 0; d2 < HALF / 2; ++d2) {
      const float2 t = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(qp + 2 * d2));
      qr[2 * d2] = t.x * c;
      qr[2 * d2 + 1] = t.y * c;
    }
#pragma unroll
    for (int d = 0; d < HALF; ++d) acc[d] = 0.f;
  }
  float m = -INFINITY, l = 0.f;
  for (int k0 = 0; k0 < Nk; k0 += XA_KT) {
    __syncthreads();
    stage_rows<HD, XA_KT, 2 * XA_QPB>(Ks, kb, s.k_rs, k0, Nk);
    stage_rows<HD, XA_KT, 2 * XA_QPB>(Vs, vb, s.v_rs, k0, Nk);
    __syncthreads();
    const int nk = min(XA_KT, Nk - k0);
    float sc[XA_KT];
    float mt = -INFINITY;
#pragma unroll
    for (int j = 0; j < XA_KT; ++j) {
      const float4* kr = reinterpret_cast<const float4*>(Ks + j * HD + half * HALF);
      float p = 0.f;
#pragma unroll
      for (int d4 = 0; d4 < HALF / 4; ++d4) {
        const float4 kv = kr[d4];
        p = fmaf(qr[4 * d4], kv.x, p);
        p = fmaf(qr[4 * d4 + 1], kv.y, p);
        p = fmaf(qr[4 * d4 + 2], kv.z, p);
        p = fmaf(qr[4 * d4 + 3], kv.w, p);
      }
      p += __shfl_xor_sync(0xffffffffu, p, 1);
      sc[j] = j < nk ? p : -INFINITY;
      mt = fmaxf(mt, sc[j]);
    }
    const float mn = fmaxf(m, mt);            // finite: every tile holds at least one key
    const float corr = fast_exp2(m - mn);     // m = -inf on the first tile -> 0
    l *= corr;
#pragma unroll
    for (int d = 0; d < HALF; ++d) acc[d] *= corr;
#pragma unroll
    for (int j = 0; j < XA_KT; ++j) {
      const float pj = fast_exp2(sc[j] - mn);
      l += pj;
      const float4* vr = reinterpret_cast<const float4*>(Vs + j * HD + half * HALF);
#pragma unroll
      for (int d4 = 0; d4 < HALF / 4; ++d4) {
        const float4 vv = vr[d4];
        acc[4 * d4] = fmaf(pj, vv.x, acc[4 * d4]);
        acc[4 * d4 + 1] = fmaf(pj, vv.y, acc[4 * d4 + 1]);
        acc[4 * d4 + 2] = fmaf(pj, vv.z, acc[4 * d4 + 2]);
        acc[4 * d4 + 3] = fmaf(pj, vv.w, acc[4 * d4 + 3]);
      }
    }
    m = mn;
  }
  if (valid) {
    const float inv = 1.0f / l;
    __nv_bfloat16* op = o + (long long)b * s.o_bs + (long long)h * s.o_hs + (long long)qi * s.o_rs + half * HALF;
#pragma unroll
    for (int d2 = 0; d2 < HALF / 2; ++d2)
      *reinterpret_cast<uint32_t*>(op + 2 * d2) = pack_bf16x2(acc[2 * d2] * inv, acc[2 * d2 + 1] * inv);
    if (LSE && half == 0) lse[(long long)bh * Nq + qi] = (m + log2f(l)) * LN2;
  }
}

template <int HD>
__global__ void __launch_bounds__(2 * XA_QPB)
xattn_dq_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ o,
                const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse, float* __restrict__ delta,
                __nv_bfloat16* __restrict__ dq, XaStrides s, int H, int Nq, int Nk, float scale) {
  constexpr int HALF = HD / 2;
  __shared__ __align__(16) float Ks[XA_KT * HD];
  __shared__ __align__(16) float Vs[XA_KT * HD];
  const int bh = blockIdx.y, b = bh / H, h = bh % H;
  const int pair = threadIdx.x >> 1, half = threadIdx.x & 1;
  const int qi = blockIdx.x * XA_QPB + pair;
  const bool valid = qi < Nq;
  const int qrow = valid ? qi : 0;
  const __nv_bfloat16* kb = k + (long long)b * s.k_bs + (long long)h * s.k_hs;
  const __nv_bfloat16* vb = v + (long long)b * s.v_bs + (long long)h * s.v_hs;
  float qr[HALF], dor[HALF], dqr[HALF];
  float dl = 0.f;
  {
    const __nv_bfloat16* qp = q + (long long)b * s.q_bs + (long long)h * s.q_hs + (long long)qrow * s.q_rs + half * HALF;
    const __nv_bfloat16* op = o + (long long)b * s.o_bs + (long long)h * s.o_hs + (long long)qrow * s.o_rs + half * HALF;
    const __nv_bfloat16* dp = dout + (long long)b * s.o_bs + (long long)h * s.o_hs + (long long)qrow * s.o_rs + half * HALF;
    const float c = scale * LOG2E;
#pragma unroll
    for (int d2 = 0; d2 < HALF / 2; ++d2) {
      const float2 tq = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(qp + 2 * d2));
      const float2 to = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(op + 2 * d2));
      const float2 td = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dp + 2 * d2));
      qr[2 * d2] = tq.x * c;
      qr[2 * d2 + 1] = tq.y * c;
      dor[2 * d2] = td.x;
      dor[2 * d2 + 1] = td.y;
      dl = fmaf(td.x, to.x, dl);
      dl = fmaf(td.y, to.y, dl);
      dqr[2 * d2] = 0.f;
      dqr[2 * d2 + 1] = 0.f;
    }
  }
  dl += __shfl_xor_sync(0xffffffffu, dl, 1);
  const float lse2 = valid ? lse[(long long)bh * Nq + qi] * LOG2E : INFINITY;   // invalid rows: p = 0
  for (int k0 = 0; k0 < Nk; k0 += XA_KT) {
    __syncthreads();
    stage_rows<HD, XA_KT, 2 * XA_QPB>(Ks, kb, s.k_rs, k0, Nk);
    stage_rows<HD, XA_KT, 2 * XA_QPB>(Vs, vb, s.v_rs, k0, Nk);
    __syncthreads();
    const int nk = min(XA_KT, Nk - k0);
#pragma unroll 4
    for (int j = 0; j < XA_KT; ++j) {
      const float4* kr = reinterpret_cast<const float4*>(Ks + j * HD + half * HALF);
      const float4* vr = reinterpret_cast<const float4*>(Vs + j * HD + half * HALF);
      float p1 = 0.f, p2 = 0.f;
#pragma unroll
      for (int d4 = 0; d4 < HALF / 4; ++d4) {
        const float4 kv = kr[d4], vv = vr[d4];
        p1 = fmaf(qr[4 * d4], kv.x, p1);
        p1 = fmaf(qr[4 * d4 + 1], kv.y, p1);
        p1 = fmaf(qr[4 * d4 + 2], kv.z, p1);
        p1 = fmaf(qr[4 * d4 + 3], kv.w, p1);
        p2 = fmaf(dor[4 * d4], vv.x, p2);
        p2 = fmaf(dor[4 * d4 + 1], vv.y, p2);
        p2 = fmaf(dor[4 * d4 + 2], vv.z, p2);
        p2 = fmaf(dor[4 * d4 + 3], vv.w, p2);
      }
      p1 += __shfl_xor_sync(0xffffffffu, p1, 1);
      p2 += __shfl_xor_sync(0xffffffffu, p2, 1);
      const float pj = j < nk ? fast_exp2(p1 - lse2) : 0.f;
      const float ds = pj * (p2 - dl);
#pragma unroll
      for (int d4 = 0; d4 < HALF / 4; ++d4) {
        const float4 kv = kr[d4];
        dqr[4 * d4] = fmaf(ds, kv.x, dqr[4 * d4]);
        dqr[4 * d4 + 1] = fmaf(ds, kv.y, dqr[4 * d4 + 1]);
        dqr[4 * d4 + 2] = fmaf(ds, kv.z, dqr[4 * d4 + 2]);
        dqr[4 * d4 + 3] = fmaf(ds, kv.w, dqr[4 * d4 + 3]);
      }
    }
  }
  if (valid) {
    __nv_bfloat16* dst = dq + (long long)b * s.dq_bs + (long long)h * s.dq_hs + (long long)qi * s.dq_rs + half * HALF;
#pragma unroll
    for (int d2 = 0; d2 < HALF / 2; ++d2)
      *reinterpret_cast<uint32_t*>(dst + 2 * d2) = pack_bf16x2(dqr[2 * d2] * scale, dqr[2 * d2 + 1] * scale);
    if (half == 0) delta[(long long)bh * Nq + qi] = dl;
  }
}

template <int HD>
__global__ void __launch_bounds__(4 * XA_KPB)
xattn_dkv_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                 const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ dout,
                 const float* __restrict__ lse, const float* __restrict__ delta, float* __restrict__ dk,
                 float* __restrict__ dv, XaStrides s, int H, int Nq, int Nk, float scale) {
  constexpr int QUART = HD / 4;
  __shared__ __align__(16) float Qs[XA_QT * HD];
  __shared__ __align__(16) float Ds[XA_QT * HD];
  __shared__ float Ls[XA_QT], Dl[XA_QT];
  const int bh = blockIdx.z, b = bh / H, h = bh % H;
  const int kl = threadIdx.x >> 2, quart = threadIdx.x & 3;
  const int kj = blockIdx.x * XA_KPB + kl;
  const bool valid = kj < Nk;
  const __nv_bfloat16* qb = q + (long long)b * s.q_bs + (long long)h * s.q_hs;
  const __nv_bfloat16* db = dout + (long long)b * s.o_bs + (long long)h * s.o_hs;
  float kr[QUART], vr[QUART], dkr[QUART], dvr[QUART];
  {
    const __nv_bfloat16* kp = k + (long long)b * s.k_bs + (long long)h * s.k_hs + (long long)(valid ? kj : 0) * s.k_rs + quart * QUART;
    const __nv_bfloat16* vp = v + (long long)b * s.v_bs + (long long)h * s.v_hs + (long long)(valid ? kj : 0) * s.v_rs + quart * QUART;
    const float c = scale * LOG2E;
#pragma unroll
    for (int d2 = 0; d2 < QUART / 2; ++d2) {
      const float2 tk = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(kp + 2 * d2));
      const float2 tv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(vp + 2 * d2));
      kr[2 * d2] = valid ? tk.x * c : 0.f;
      kr[2 * d2 + 1] = valid ? tk.y * c : 0.f;
      vr[2 * d2] = valid ? tv.x : 0.f;
      vr[2 * d2 + 1] = valid ? tv.y : 0.f;
      dkr[2 * d2] = dkr[2 * d2 + 1] = 0.f;
      dvr[2 * d2] = dvr[2 * d2 + 1] = 0.f;
    }
  }
  const int q_begin = blockIdx.y * XA_QCHUNK;
  const int q_end = min(Nq, q_begin + XA_QCHUNK);
  for (int q0 = q_begin; q0 < q_end; q0 += XA_QT) {
    __syncthreads();
    stage_rows<HD, XA_QT, 4 * XA_KPB>(Qs, qb, s.q_rs, q0, q_end);
    stage_rows<HD, XA_QT, 4 * XA_KPB>(Ds, db, s.o_rs, q0, q_end);
    if (threadIdx.x < XA_QT) {
      const int qi = q0 + threadIdx.x;
      Ls[threadIdx.x] = qi < q_end ? lse[(long long)bh * Nq + qi] * LOG2E : INFINITY;   // past the end: p = 0
      Dl[threadIdx.x] = qi < q_end ? delta[(long long)bh * Nq + qi] : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int i = 0; i < XA_QT; ++i) {
      const float4* qv = reinterpret_cast<const float4*>(Qs + i * HD + quart * QUART);
      const float4* dv4 = reinterpret_cast<const float4*>(Ds + i * HD + quart * QUART);
      float p1 = 0.f, p2 = 0.f;
#pragma unroll
      for (int d4 = 0; d4 < QUART / 4; ++d4) {
        const float4 a = qv[d4], g = dv4[d4];
        p1 = fmaf(kr[4 * d4], a.x, p1);
        p1 = fmaf(kr[4 * d4 + 1], a.y, p1);
        p1 = fmaf(kr[4 * d4 + 2], a.z, p1);
        p1 = fmaf(kr[4 * d4 + 3], a.w, p1);
        p2 = fmaf(vr[4 * d4], g.x, p2);
        p2 = fmaf(vr[4 * d4 + 1], g.y, p2);
        p2 = fmaf(vr[4 * d4 + 2], g.z, p2);
        p2 = fmaf(vr[4 * d4 + 3], g.w, p2);
      }
      p1 += __shfl_xor_sync(0xffffffffu, p1, 1);
      p1 += __shfl_xor_sync(0xffffffffu, p1, 2);
      p2 += __shfl_xor_sync(0xffffffffu, p2, 1);
      p2 += __shfl_xor_sync(0xffffffffu, p2, 2);
      const float pj = fast_exp2(p1 - Ls[i]);
      const float ds = pj * (p2 - Dl[i]);
#pragma unroll
      for (int d4 = 0; d4 < QUART / 4; ++d4) {
        const float4 a = qv[d4], g = dv4[d4];
        dvr[4 * d4] = fmaf(pj, g.x, dvr[4 * d4]);
        dvr[4 * d4 + 1] = fmaf(pj, g.y, dvr[4 * d4 + 1]);
        dvr[4 * d4 + 2] = fmaf(pj, g.z, dvr[4 * d4 + 2]);
        dvr[4 * d4 + 3] = fmaf(pj, g.w, dvr[4 * d4 + 3]);
        dkr[4 * d4] = fmaf(ds, a.x, dkr[4 * d4]);
        dkr[4 * d4 + 1] = fmaf(ds, a.y, dkr[4 * d4 + 1]);
        dkr[4 * d4 + 2] = fmaf(ds, a.z, dkr[4 * d4 + 2]);
        dkr[4 * d4 + 3] = fmaf(ds, a.w, dkr[4 * d4 + 3]);
      }
    }
  }
  if (valid) {
    float* dkp = dk + ((long long)bh * Nk + kj) * HD + quart * QUART;
    float* dvp = dv + ((long long)bh * Nk + kj) * HD + quart * QUART;
#pragma unroll
    for (int d = 0; d < QUART; ++d) {
      atomicAdd(dkp + d, dkr[d] * scale);
      atomicAdd(dvp + d, dvr[d]);
    }
  }
}

// ================================================================================================
// skip-path max pooling on the fp32 stream (cls row copied)
// ================================================================================================
struct MpDims {
  int B, D, T, H, W, kt, kh, kw, st, sh, sw, To, Ho, Wo;
};

// four channels per thread: the window walk (divisions, bounds) is shared by a float4 of channels
template <bool IDX>   // IDX = false: the winners are not recorded (forward-only calls)
__global__ void maxpool_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, uint8_t* __restrict__ idx, MpDims d) {
  const int Lo1 = 1 + d.To * d.Ho * d.Wo, L1 = 1 + d.T * d.H * d.W;
  const int D4 = d.D / 4;
  const long long n = (long long)d.B * Lo1 * D4;
  const int pt = d.kt / 2, ph = d.kh / 2, pw = d.kw / 2;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(e % D4);
    const int l = (int)((e / D4) % Lo1);
    const int b = (int)(e / ((long long)D4 * Lo1));
    const float4* xb = reinterpret_cast<const float4*>(x + (long long)b * L1 * d.D) + c4;
    float4* yo = reinterpret_cast<float4*>(y) + e;
    uchar4* io = reinterpret_cast<uchar4*>(idx) + e;
    if (l == 0) {
      *yo = xb[0];
      if (IDX) *io = make_uchar4(0, 0, 0, 0);
      continue;
    }
    const int o = l - 1;
    const int ow = o % d.Wo, oh = (o / d.Wo) % d.Ho, ot = o / (d.Wo * d.Ho);
    float4 best = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    int ax = 255, ay = 255, az = 255, aw = 255;
    for (int dt = 0; dt < d.kt; ++dt) {
      const int ti = ot * d.st - pt + dt;
      if (ti < 0 || ti >= d.T) continue;
      for (int dh = 0; dh < d.kh; ++dh) {
        const int hi = oh * d.sh - ph + dh;
        if (hi < 0 || hi >= d.H) continue;
        for (int dw = 0; dw < d.kw; ++dw) {
          const int wi = ow * d.sw - pw + dw;
          if (wi < 0 || wi >= d.W) continue;
          const float4 v = xb[(1 + ((long long)ti * d.H + hi) * d.W + wi) * D4];
          const int tap = (dt * d.kh + dh) * d.kw + dw;
          if (v.x > best.x || ax == 255) { best.x = v.x; ax = tap; }     // first maximum in scan order
          if (v.y > best.y || ay == 255) { best.y = v.y; ay = tap; }
          if (v.z > best.z || az == 255) { best.z = v.z; az = tap; }
          if (v.w > best.w || aw == 255) { best.w = v.w; aw = tap; }
        }
      }
    }
    *yo = best;
    if (IDX) *io = make_uchar4((unsigned char)ax, (unsigned char)ay, (unsigned char)az, (unsigned char)aw);
  }
}

__global__ void maxpool_bwd_kernel(const float* __restrict__ dy, const uint8_t* __restrict__ idx, float* __restrict__ dx, MpDims d) {
  const int Lo1 = 1 + d.To * d.Ho * d.Wo, L1 = 1 + d.T * d.H * d.W;
  const int D4 = d.D / 4;
  const long long n = (long long)d.B * L1 * D4;
  const int pt = d.kt / 2, ph = d.kh / 2, pw = d.kw / 2;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(e % D4);
    const int l = (int)((e / D4) % L1);
    const int b = (int)(e / ((long long)D4 * L1));
    const float4* gb = reinterpret_cast<const float4*>(dy + (long long)b * Lo1 * d.D) + c4;
    const uchar4* ib = reinterpret_cast<const uchar4*>(idx + (long long)b * Lo1 * d.D) + c4;
    float4* out = reinterpret_cast<float4*>(dx) + e;
    if (l == 0) {
      *out = gb[0];
      continue;
    }
    const int i = l - 1;
    const int wi = i % d.W, hi = (i / d.W) % d.H, ti = i / (d.W * d.H);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int dt = 0; dt < d.kt; ++dt) {
      const int nt = ti + pt - dt;
      if (nt < 0 || nt % d.st != 0) continue;
      const int ot = nt / d.st;
      if (ot >= d.To) continue;
      for (int dh = 0; dh < d.kh; ++dh) {
        const int nh = hi + ph - dh;
        if (nh < 0 || nh % d.sh != 0) continue;
        const int oh = nh / d.sh;
        if (oh >= d.Ho) continue;
        for (int dw = 0; dw < d.kw; ++dw) {
          const int nw = wi + pw - dw;
          if (nw < 0 || nw % d.sw != 0) continue;
          const int ow = nw / d.sw;
          if (ow >= d.Wo) continue;
          const long long at = (1 + ((long long)ot * d.Ho + oh) * d.Wo + ow) * D4;
          const uchar4 w = ib[at];
          const float4 g = gb[at];
          const int tap = (dt * d.kh + dh) * d.kw + dw;
          if (w.x == tap) acc.x += g.x;
          if (w.y == tap) acc.y += g.y;
          if (w.z == tap) acc.z += g.z;
          if (w.w == tap) acc.w += g.w;
        }
      }
    }
    *out = acc;
  }
}

// ================================================================================================
// overlapping Conv3d im2col
// ================================================================================================
struct I3Dims {
  int B, T, C, H, W, kt, kh, kw, st, sh, sw, pt, ph, pw, To, Ho, Wo, Kpad;
};

// one thread per (output row, kw-wide group of columns): the kw taps of a (c, dt, dh) filter row are contiguous both in
// the clip and in the column layout, so the coordinate arithmetic is shared by kw elements
__global__ void im2col3d_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ cols, I3Dims d) {
  const long long rows = (long long)d.B * d.To * d.Ho * d.Wo;
  const int groups = (d.Kpad + d.kw - 1) / d.kw;
  const int Kreal = d.C * d.kt * d.kh * d.kw;
  const long long n = rows * groups;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int grp = (int)(e % groups);
    const long long row = e / groups;
    const int col0 = grp * d.kw;
    __nv_bfloat16* dst = cols + row * d.Kpad + col0;
    const int ncol = min(d.kw, d.Kpad - col0);
    const __nv_bfloat16 zero = __float2bfloat16_rn(0.f);
    if (col0 >= Kreal) {
      for (int j = 0; j < ncol; ++j) dst[j] = zero;
      continue;
    }
    const int dh = grp % d.kh, dt = (grp / d.kh) % d.kt, c = grp / (d.kh * d.kt);
    const int ow = (int)(row % d.Wo), oh = (int)((row / d.Wo) % d.Ho), ot = (int)((row / ((long long)d.Wo * d.Ho)) % d.To);
    const int b = (int)(row / ((long long)d.Wo * d.Ho * d.To));
    const int ti = ot * d.st - d.pt + dt, hi = oh * d.sh - d.ph + dh, w0 = ow * d.sw - d.pw;
    const bool line_ok = ti >= 0 && ti < d.T && hi >= 0 && hi < d.H;
    const float* src = x + ((((long long)b * d.T + (line_ok ? ti : 0)) * d.C + c) * d.H + (line_ok ? hi : 0)) * d.W;
    for (int j = 0; j < ncol; ++j) {
      const int wi = w0 + j;
      const float v = (line_ok && wi >= 0 && wi < d.W) ? src[wi] : 0.f;
      dst[j] = __float2bfloat16_rn(v);
    }
  }
}

// The same operand from the decoder's uint8 clip [B, T, H, W, C].  One CTA owns the output rows (b, ot, oh0..oh0+ohb-1):
//   1. it stages the C x kt x R source lines those rows read (R = (ohb-1)*sh + kh) in shared memory as bf16
//      [c][dt][r][Wp], Wp = W + 2*pw: normalised, mixed and rounded once per CTA, each line widened by pw zeros per side
//      and lines outside the clip all zeros, so the gather below has no bounds tests;
//   2. its rows of cols are one contiguous span (rows are ow-, then oh-major), written with 16-byte stores, consecutive
//      threads on consecutive chunks; a column -> window offset table (-1 = pad column) replaces the per-element
//      (c, dt, dh, dw) decode.
struct I3U8Dims {
  I3Dims g;
  int ohb, R, Wp, Kreal;
};

// ToTensor + Normalize as the reference runs them in fp32 (pic.float().div(255), then sub_(mean).div_(std)): no
// contraction, no reciprocal, so the value is bit for bit the reference's float clip
__device__ __forceinline__ float u8_normalize(uint8_t u, float mean, float std) {
  return __fdiv_rn(__fsub_rn(__fdiv_rn((float)u, 255.f), mean), std);
}

__global__ void __launch_bounds__(256) im2col3d_u8_kernel(const uint8_t* __restrict__ x, const float* __restrict__ mean,
                                                          const float* __restrict__ stdv, const float* __restrict__ plan,
                                                          __nv_bfloat16* __restrict__ cols, I3U8Dims u) {
  extern __shared__ __align__(16) unsigned char i3u8_smem[];
  const I3Dims& d = u.g;
  int* tab = reinterpret_cast<int*>(i3u8_smem);                          // [Kpad]
  __nv_bfloat16* win = reinterpret_cast<__nv_bfloat16*>(tab + d.Kpad);  // [C][kt][R][Wp]
  const int hblocks = (d.Ho + u.ohb - 1) / u.ohb;
  const int hb = blockIdx.x % hblocks;
  const int ot = (blockIdx.x / hblocks) % d.To;
  const int b = blockIdx.x / (hblocks * d.To);
  const int oh0 = hb * u.ohb;
  const int noh = min(u.ohb, d.Ho - oh0);
  int mode = 0, yl = 0, yh = 0, xl = 0, xh = 0;
  float lam = 1.f;
  if (plan) {
    mode = (int)plan[0];
    lam = plan[1];
    yl = (int)plan[2], yh = (int)plan[3], xl = (int)plan[4], xh = (int)plan[5];
  }
  const float lam_o = __fsub_rn(1.0f, lam);

  for (int k = threadIdx.x; k < d.Kpad; k += blockDim.x) {
    int off = -1;
    if (k < u.Kreal) {
      const int dw = k % d.kw, dh = (k / d.kw) % d.kh, dt = (k / (d.kw * d.kh)) % d.kt, c = k / (d.kw * d.kh * d.kt);
      off = ((c * d.kt + dt) * u.R + dh) * u.Wp + dw;
    }
    tab[k] = off;
  }
  const long long clip = (long long)d.T * d.H * d.W * d.C;
  const uint8_t* xs = x + b * clip;
  const uint8_t* xf = x + (d.B - 1 - b) * clip;                          // x.flip(0)[b]
  const int staged = d.C * d.kt * u.R * u.Wp;
  for (int e = threadIdx.x; e < staged; e += blockDim.x) {
    const int xw = e % u.Wp, line = e / u.Wp;
    const int r = line % u.R, dt = (line / u.R) % d.kt, c = line / (u.R * d.kt);
    const int ti = ot * d.st - d.pt + dt, hi = oh0 * d.sh - d.ph + r, wi = xw - d.pw;
    float v = 0.f;                                                       // Conv3d padding: 0 after Normalize
    if (ti >= 0 && ti < d.T && hi >= 0 && hi < d.H && wi >= 0 && wi < d.W) {
      const long long o = (((long long)ti * d.H + hi) * d.W + wi) * d.C + c;
      const float m = mean[c], s = stdv[c];
      v = u8_normalize(xs[o], m, s);
      if (mode == 1) {
        v = __fadd_rn(__fmul_rn(v, lam), __fmul_rn(u8_normalize(xf[o], m, s), lam_o));   // x*lam + x.flip(0)*(1-lam)
      } else if (mode == 2 && hi >= yl && hi < yh && wi >= xl && wi < xh) {
        v = u8_normalize(xf[o], m, s);                                   // x[..., yl:yh, xl:xh] = x.flip(0)[...]
      }
    }
    win[e] = __float2bfloat16_rn(v);
  }
  __syncthreads();

  const int cpr = d.Kpad / 8;                                            // 16-byte chunks per row
  const long long row0 = (((long long)b * d.To + ot) * d.Ho + oh0) * d.Wo;
  uint4* dst = reinterpret_cast<uint4*>(cols + row0 * d.Kpad);
  const int chunks = noh * d.Wo * cpr;
  const __nv_bfloat16 zero = __float2bfloat16_rn(0.f);
  for (int q = threadIdx.x; q < chunks; q += blockDim.x) {
    const int rl = q / cpr, k0 = (q - rl * cpr) * 8;
    const int ohl = rl / d.Wo, ow = rl - ohl * d.Wo;
    const __nv_bfloat16* src = win + ohl * d.sh * u.Wp + ow * d.sw;
    __align__(16) __nv_bfloat16 h[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int off = tab[k0 + j];
      h[j] = off >= 0 ? src[off] : zero;
    }
    dst[q] = *reinterpret_cast<const uint4*>(h);
  }
}

// ================================================================================================
// token preparation
// ================================================================================================
__global__ void mvit_tokens_fwd_kernel(const float* __restrict__ t, const float* __restrict__ wmask,
                                       const float* __restrict__ mask_token, const float* __restrict__ cls_token,
                                       const float* __restrict__ pos_s, const float* __restrict__ pos_t,
                                       const float* __restrict__ pos_cls, float* __restrict__ x, int B, int T, int HW, int C) {
  const int L = T * HW;
  const long long n = (long long)B * (L + 1) * C;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % C);
    const int l1 = (int)((e / C) % (L + 1));
    const int b = (int)(e / ((long long)C * (L + 1)));
    float val;
    if (l1 == 0) {
      val = cls_token[c] + pos_cls[c];
    } else {
      const int l = l1 - 1;
      const float w = wmask ? wmask[(long long)b * L + l] : 0.f;
      val = t[((long long)b * L + l) * C + c] * (1.0f - w) + mask_token[c] * w + pos_s[(long long)(l % HW) * C + c] +
            pos_t[(long long)(l / HW) * C + c];
    }
    x[e] = val;
  }
}

__global__ void mvit_tokens_bwd_kernel(const float* __restrict__ dx, const float* __restrict__ wmask,
                                       __nv_bfloat16* __restrict__ dt, int B, int L, int C) {
  const long long n = (long long)B * L * C;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % C);
    const long long bl = e / C;
    const int l = (int)(bl % L);
    const int b = (int)(bl / L);
    const float w = wmask ? wmask[bl] : 0.f;
    dt[e] = __float2bfloat16_rn(dx[((long long)b * (L + 1) + 1 + l) * C + c] * (1.0f - w));
  }
}

// ================================================================================================
// masked MSE (one warp per (b, frame, h, w) cell)
// ================================================================================================
struct MseDims {
  int B, t, dt, h, w, dc;
};

// fp64 variant: targets, differences and sums in double (reference semantics with fp64 numpy targets)
__global__ void __launch_bounds__(ROW_WARPS * 32)
mse_fwd64_kernel(const float* __restrict__ pred, const double* __restrict__ target, const float* __restrict__ mask,
                 double* __restrict__ partials, MseDims d) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int F = d.t * d.dt, hw = d.h * d.w;
  const long long cells = (long long)d.B * F * hw;
  const int L1 = 1 + d.t * hw, PD = d.dt * d.dc;
  double acc = 0.0;
  for (long long cell = (long long)blockIdx.x * ROW_WARPS + warp; cell < cells; cell += (long long)gridDim.x * ROW_WARPS) {
    const float m = mask[cell];
    if (m == 0.f) continue;
    const int p = (int)(cell % hw);
    const int f = (int)((cell / hw) % F);
    const int b = (int)(cell / ((long long)hw * F));
    const float* pr = pred + ((long long)b * L1 + 1 + (long long)(f / d.dt) * hw + p) * PD + (f % d.dt) * d.dc;
    const double* tg = target + cell * d.dc;
    double s = 0.0;
    for (int c = lane; c < d.dc; c += 32) {
      const double e = (double)pr[c] - tg[c];
      s = fma(e, e, s);
    }
    acc += (double)m * s / (double)d.dc;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ double sh[ROW_WARPS];
  if (lane == 0) sh[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    for (int i = 0; i < ROW_WARPS; ++i) a += sh[i];
    partials[blockIdx.x] = a;
  }
}
__global__ void mse_sum64_kernel(const double* __restrict__ partials, int n, double* __restrict__ out) {
  // single warp, fixed order: deterministic
  double a = 0.0;
  for (int i = threadIdx.x; i < n; i += 32) a += partials[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (threadIdx.x == 0) out[0] = a;
}

__global__ void __launch_bounds__(ROW_WARPS * 32)
mse_fwd_kernel(const float* __restrict__ pred, const float* __restrict__ target, const float* __restrict__ mask,
               float* __restrict__ partials, MseDims d) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int F = d.t * d.dt, hw = d.h * d.w;
  const long long cells = (long long)d.B * F * hw;
  const int L1 = 1 + d.t * hw, PD = d.dt * d.dc;
  float acc = 0.f;
  for (long long cell = (long long)blockIdx.x * ROW_WARPS + warp; cell < cells; cell += (long long)gridDim.x * ROW_WARPS) {
    const float m = mask[cell];
    if (m == 0.f) continue;
    const int p = (int)(cell % hw);
    const int f = (int)((cell / hw) % F);
    const int b = (int)(cell / ((long long)hw * F));
    const float* pr = pred + ((long long)b * L1 + 1 + (long long)(f / d.dt) * hw + p) * PD + (f % d.dt) * d.dc;
    const float* tg = target + cell * d.dc;
    float s = 0.f;
    for (int c = lane; c < d.dc; c += 32) {
      const float e = pr[c] - tg[c];
      s = fmaf(e, e, s);
    }
    acc += m * s / (float)d.dc;
  }
  acc = warp_sum(acc);
  __shared__ float sh[ROW_WARPS];
  if (lane == 0) sh[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f;
    for (int i = 0; i < ROW_WARPS; ++i) a += sh[i];
    float4* o = reinterpret_cast<float4*>(partials) + blockIdx.x;
    *o = make_float4(a, 0.f, 0.f, 0.f);
  }
}

__global__ void mse_bwd_kernel(const float* __restrict__ pred, const float* __restrict__ target,
                               const double* __restrict__ target64, const float* __restrict__ mask,
                               const float* __restrict__ coef, __nv_bfloat16* __restrict__ dpred, MseDims d) {
  const int hw = d.h * d.w, F = d.t * d.dt;
  const int L1 = 1 + d.t * hw, PD = d.dt * d.dc;
  const long long n = (long long)d.B * L1 * PD;
  const float cf = coef[0];
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(e % PD);
    const int l1 = (int)((e / PD) % L1);
    const int b = (int)(e / ((long long)PD * L1));
    float g = 0.f;
    if (l1 > 0) {
      const int l = l1 - 1;
      const int tt = l / hw, p = l % hw;
      const int f = tt * d.dt + j / d.dc, c = j % d.dc;
      const long long cell = ((long long)b * F + f) * hw + p;
      const float m = mask[cell];
      if (m != 0.f) {
        const float tv = target64 ? (float)((double)pred[e] - target64[cell * d.dc + c]) : pred[e] - target[cell * d.dc + c];
        g = cf * m * tv;
      }
    }
    dpred[e] = __float2bfloat16_rn(g);
  }
}

}  // namespace vt

// ================================================================================================
// C ABI
// ================================================================================================
using namespace vt;

int vt::layernorm_fwd_small(const vt_ln_fwd_params* p, void* stream) {
  VT_REQUIRE(p->D % 32 == 0 && p->D >= 32 && p->D <= 256, "vt_layernorm_fwd: D=%d unsupported", p->D);
  VT_REQUIRE(p->in_row == nullptr, "vt_layernorm_fwd: row maps need D %% 128 == 0 (D=%d)", p->D);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int blocks = row_blocks(p->rows, 4);
#define VT_CASE(E)                                                                                                    \
  case E:                                                                                                             \
    (p->mean ? ln_small_fwd_kernel<E, true> : ln_small_fwd_kernel<E, false>)<<<blocks, ROW_WARPS * 32, 0, st>>>(          \
        p->x, p->ldx, p->gamma, p->beta, p->y, p->mean, p->rstd, p->rows, p->eps, p->y_fp32);                          \
    break;
  switch (p->D / 32) { VT_CASE(1) VT_CASE(2) VT_CASE(3) VT_CASE(4) VT_CASE(5) VT_CASE(6) VT_CASE(7) VT_CASE(8) }
#undef VT_CASE
  return check_launch("ln_small_fwd_kernel");
}

int vt::layernorm_bwd_small(const vt_ln_bwd_params* p, void* stream) {
  VT_REQUIRE(p->D % 32 == 0 && p->D >= 32 && p->D <= 256, "vt_layernorm_bwd: D=%d unsupported", p->D);
  VT_REQUIRE(p->in_row == nullptr && p->out_row == nullptr && p->dx_aux == nullptr,
             "vt_layernorm_bwd: row maps need D %% 128 == 0 (D=%d)", p->D);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int blocks = vt_ln_bwd_blocks(p->rows);   // the caller sized `partials` with this
#define VT_CASE(E)                                                                                                     \
  case E:                                                                                                              \
    ln_small_bwd_kernel<E><<<blocks, ROW_WARPS * 32, 0, st>>>(p->dy, p->dy_fp32, p->x, p->ldx, p->mean, p->rstd,       \
                                                              p->gamma, p->dres, p->dx, p->lddx, p->partials, p->rows); \
    break;
  switch (p->D / 32) { VT_CASE(1) VT_CASE(2) VT_CASE(3) VT_CASE(4) VT_CASE(5) VT_CASE(6) VT_CASE(7) VT_CASE(8) }
#undef VT_CASE
  return check_launch("ln_small_bwd_kernel");
}

// the 4-channels-per-lane kernels (second generation) need 8-byte aligned token rows; other views take the first
static bool pool_v2(const void* ptr, long long bs, long long rs) {
  return ((uintptr_t)ptr & 7) == 0 && bs % 4 == 0 && rs % 4 == 0;
}

static int pool_dims_ok(int T, int Hin, int Win, int st, int sh, int sw, int To, int Ho, int Wo) {
  return st >= 1 && sh >= 1 && sw >= 1 && To == (T + 2 - 3) / st + 1 && Ho == (Hin + 2 - 3) / sh + 1 && Wo == (Win + 2 - 3) / sw + 1;
}

extern "C" int vt_pool_fwd(const vt_pool_fwd_params* p, void* stream) {
  VT_REQUIRE(p && p->in && p->w && p->gamma && p->beta && p->out, "vt_pool_fwd: null pointer");
  VT_REQUIRE((p->pooled == nullptr) == (p->mean == nullptr) && (p->mean == nullptr) == (p->rstd == nullptr),
             "vt_pool_fwd: pooled, mean and rstd are all given or all NULL");
  VT_REQUIRE(p->hd == 96, "vt_pool_fwd: head dim %d unsupported (96 only)", p->hd);
  VT_REQUIRE(p->B > 0 && p->H > 0 && p->T > 0 && p->Hin > 0 && p->Win > 0, "vt_pool_fwd: bad dims");
  VT_REQUIRE(pool_dims_ok(p->T, p->Hin, p->Win, p->st, p->sh, p->sw, p->To, p->Ho, p->Wo), "vt_pool_fwd: output dims inconsistent");
  const PoolDims d{p->B, p->H, p->T, p->Hin, p->Win, p->st, p->sh, p->sw, p->To, p->Ho, p->Wo};
  const long long rows = (long long)p->B * p->H * (1 + (long long)p->To * p->Ho * p->Wo);
  VT_REQUIRE(rows < 0x7fffffffll, "vt_pool_fwd: too many rows");
  (p->pooled ? pool_ln_fwd_kernel<3, true> : pool_ln_fwd_kernel<3, false>)<<<row_blocks(rows, 8), ROW_WARPS * 32, 0,
                                                                             static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(p->in), p->in_bs, p->in_rs, p->w, p->gamma, p->beta, p->pooled,
      static_cast<__nv_bfloat16*>(p->out), p->mean, p->rstd, d, p->eps);
  return check_launch("pool_ln_fwd_kernel");
}

constexpr int DW_MIN_ROWS_PER_CTA = 64;
static int pool_dw_blocks(long long rows) {                        // sized for the finer-grained second generation
  long long blocks = (rows + DW2_MIN_ROWS_PER_CTA - 1) / DW2_MIN_ROWS_PER_CTA;
  const long long cap = (long long)sm_count() * 2;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

extern "C" int vt_pool_bwd_scratch(int32_t rows_out, int32_t hd) {
  // dpooled [rows_out, hd] + LN partials [blocks, 2, hd] + filter partials [blocks, 27*hd]
  const long long f = (long long)rows_out * hd + (long long)vt_ln_bwd_blocks(rows_out) * 2 * hd +
                      (long long)pool_dw_blocks(rows_out) * 27 * hd;
  return f > 0x7fffffffll ? -1 : (int)f;
}

extern "C" int vt_pool_bwd(const vt_pool_bwd_params* p, void* stream) {
  VT_REQUIRE(p && p->dout && p->pooled && p->mean && p->rstd && p->gamma && p->in && p->w && p->din && p->dw && p->dgamma &&
                 p->dbeta && p->scratch, "vt_pool_bwd: null pointer");
  VT_REQUIRE(p->hd == 96, "vt_pool_bwd: head dim %d unsupported (96 only)", p->hd);
  VT_REQUIRE(pool_dims_ok(p->T, p->Hin, p->Win, p->st, p->sh, p->sw, p->To, p->Ho, p->Wo), "vt_pool_bwd: output dims inconsistent");
  const long long Lo = (long long)p->To * p->Ho * p->Wo;
  const long long rows_out = (long long)p->B * p->H * (1 + Lo);
  VT_REQUIRE(rows_out < 0x7fffffffll, "vt_pool_bwd: too many rows");
  // the d(input) kernels tabulate each axis in shared memory; checked before the first launch, so a refused call leaves
  // every output untouched
  VT_REQUIRE(p->T <= POOL_MAX_DIM && p->Hin <= POOL_MAX_DIM && p->Win <= POOL_MAX_DIM, "vt_pool_bwd: token grid %dx%dx%d exceeds %d per axis",
             p->T, p->Hin, p->Win, POOL_MAX_DIM);
  const long long tokens_in = (long long)p->B * (1 + (long long)p->T * p->Hin * p->Win);
  VT_REQUIRE(tokens_in < 0x7fffffffll, "vt_pool_bwd: too many tokens");
  const int need = vt_pool_bwd_scratch((int)rows_out, p->hd);
  VT_REQUIRE(need > 0 && p->scratch_floats >= need, "vt_pool_bwd: scratch too small (%lld < %d floats)", (long long)p->scratch_floats, need);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int hd = p->hd;
  float* dpooled = p->scratch;
  float* ln_part = dpooled + rows_out * hd;
  const int ln_blocks_n = vt_ln_bwd_blocks((int)rows_out);
  float* dw_part = ln_part + (long long)ln_blocks_n * 2 * hd;
  const PoolDims d{p->B, p->H, p->T, p->Hin, p->Win, p->st, p->sh, p->sw, p->To, p->Ho, p->Wo};
  // 1. LayerNorm backward over every pooled row (cls included) -> dpooled, dgamma/dbeta partials
  ln_small_bwd_kernel<3><<<ln_blocks_n, ROW_WARPS * 32, 0, st>>>(p->dout, p->dout_fp32, p->pooled, hd, p->mean, p->rstd, p->gamma,
                                                                 nullptr, dpooled, hd, ln_part, (int)rows_out);
  int rc = check_launch("ln_small_bwd_kernel(pool)");
  if (rc) return rc;
  {
    if (p->dbeta == p->dgamma + hd) {        // adjacent outputs ([2, hd], what the Python wrapper allocates): one launch
      vt_reduce_params r{ln_part, p->dgamma, 2ll * hd, ln_blocks_n, 2ll * hd, 0, 1.0f};
      rc = vt_reduce_rows(&r, stream);
      if (rc) return rc;
    } else {                                 // separate buffers: reduce each half of the [blocks, 2, hd] partials
      vt_reduce_params r{ln_part, p->dgamma, 2ll * hd, ln_blocks_n, hd, 0, 1.0f};
      rc = vt_reduce_rows(&r, stream);
      if (rc) return rc;
      vt_reduce_params r2{ln_part + hd, p->dbeta, 2ll * hd, ln_blocks_n, hd, 0, 1.0f};
      rc = vt_reduce_rows(&r2, stream);
      if (rc) return rc;
    }
  }
  // 2. gradient w.r.t. the input tokens
  const bool v2 = pool_v2(p->in, p->in_bs, p->in_rs) && pool_v2(p->din, p->din_bs, p->din_rs);
  if (v2) {
    const int hw = p->Hin * p->Win;
    const dim3 dgrid((hw + ROW_WARPS * 4 - 1) / (ROW_WARPS * 4), p->B * p->T + 1, p->H);   // ~4 tokens per warp; y + 1: the cls tokens
    pool_din_v2_kernel<<<dgrid, ROW_WARPS * 32, 0, st>>>(dpooled, p->w, static_cast<__nv_bfloat16*>(p->din), p->din_bs, p->din_rs, d);
    rc = check_launch("pool_din_v2_kernel");
  } else {
    pool_din_kernel<3><<<row_blocks(tokens_in, 8), ROW_WARPS * 32, 0, st>>>(dpooled, p->w, static_cast<__nv_bfloat16*>(p->din),
                                                                          p->din_bs, p->din_rs, d);
    rc = check_launch("pool_din_kernel");
  }
  if (rc) return rc;
  // 3. filter gradient
  const long long rows_conv = (long long)p->B * p->H * Lo;         // pooled rows without the cls rows
  int dwb = pool_dw_blocks(rows_conv);
  if (!v2 && dwb > (rows_conv + DW_MIN_ROWS_PER_CTA - 1) / DW_MIN_ROWS_PER_CTA)
    dwb = (int)((rows_conv + DW_MIN_ROWS_PER_CTA - 1) / DW_MIN_ROWS_PER_CTA);
  const int rows_per_cta = (int)((rows_conv + dwb - 1) / dwb);
  dwb = (int)((rows_conv + rows_per_cta - 1) / rows_per_cta);      // no empty CTAs: every partial row is written
  if (v2) {
    pool_dw_v2_kernel<<<dwb, DW2_SLOTS * 3 * 32, 0, st>>>(dpooled, static_cast<const __nv_bfloat16*>(p->in), p->in_bs, p->in_rs, dw_part,
                                                          d, rows_per_cta);
    rc = check_launch("pool_dw_v2_kernel");
  } else {
    pool_dw_kernel<3><<<dwb, 27 * 32, 0, st>>>(dpooled, static_cast<const __nv_bfloat16*>(p->in), p->in_bs, p->in_rs, dw_part, d,
                                               rows_per_cta);
    rc = check_launch("pool_dw_kernel");
  }
  if (rc) return rc;
  vt_reduce_params r3{dw_part, p->dw, 27ll * hd, dwb, 27ll * hd, 0, 1.0f};
  return vt_reduce_rows(&r3, stream);
}

// q / k / v / o of either pooling-attention entry point as operands of the tensor-core kernels
template <typename Params>
static MmaAttn xattn_operands(const Params* p) {
  MmaAttn a{};
  a.q = static_cast<const __nv_bfloat16*>(p->q); a.k = static_cast<const __nv_bfloat16*>(p->k);
  a.v = static_cast<const __nv_bfloat16*>(p->v); a.o = static_cast<const __nv_bfloat16*>(p->o);
  a.o_out = static_cast<__nv_bfloat16*>(const_cast<void*>(static_cast<const void*>(p->o)));
  a.q_bs = p->q_bs; a.q_hs = p->q_hs; a.q_rs = p->q_rs; a.k_bs = p->k_bs; a.k_hs = p->k_hs; a.k_rs = p->k_rs;
  a.v_bs = p->v_bs; a.v_hs = p->v_hs; a.v_rs = p->v_rs; a.o_bs = p->o_bs; a.o_hs = p->o_hs; a.o_rs = p->o_rs;
  a.lse = const_cast<float*>(p->lse);
  a.H = p->H; a.Nq = p->Nq; a.Nk = p->Nk; a.scale = p->scale;
  return a;
}

static int xa_strides_ok(const long long* s, int n) {
  for (int i = 0; i < n; ++i)
    if (s[i] % 2 != 0) return 0;
  return 1;
}

extern "C" int vt_xattn_fwd(const vt_xattn_fwd_params* p, void* stream) {
  VT_REQUIRE(p && p->q && p->k && p->v && p->o, "vt_xattn_fwd: null pointer");   // lse may be NULL (not written)
  VT_REQUIRE(p->hd == 96 || p->hd == 64, "vt_xattn_fwd: head dim %d unsupported (64 or 96)", p->hd);
  VT_REQUIRE(p->B > 0 && p->H > 0 && p->Nq > 0 && p->Nk > 0 && (long long)p->B * p->H <= 65535, "vt_xattn_fwd: bad dims");
  VT_REQUIRE(p->impl >= VT_XATTN_AUTO && p->impl <= VT_XATTN_TCGEN05, "vt_xattn_fwd: bad impl %d", p->impl);
  const bool tc_ok = mma_layout_ok(p->q, p->q_bs, p->q_hs, p->q_rs, p->hd) && mma_layout_ok(p->k, p->k_bs, p->k_hs, p->k_rs, p->hd) &&
                     mma_layout_ok(p->v, p->v_bs, p->v_hs, p->v_rs, p->hd) && mma_layout_ok(p->o, p->o_bs, p->o_hs, p->o_rs, p->hd);
  if (p->impl == VT_XATTN_TCGEN05 || (p->impl == VT_XATTN_AUTO && tc_ok)) {
    VT_REQUIRE(mma_layout_ok(p->q, p->q_bs, p->q_hs, p->q_rs, p->hd), "vt_xattn_fwd: unsupported q layout for the tensor-core kernel");
    VT_REQUIRE(tc_ok, "vt_xattn_fwd: unsupported k / v / o layout for the tensor-core kernel");
    return attn_mma_fwd(xattn_operands(p), p->B, p->hd, static_cast<cudaStream_t>(stream));
  }
  const long long ss[12] = {p->q_bs, p->q_hs, p->q_rs, p->k_bs, p->k_hs, p->k_rs, p->v_bs, p->v_hs, p->v_rs, p->o_bs, p->o_hs, p->o_rs};
  VT_REQUIRE(xa_strides_ok(ss, 12), "vt_xattn_fwd: strides must be even (4-byte aligned bf16 pairs)");
  VT_REQUIRE(((uintptr_t)p->q | (uintptr_t)p->k | (uintptr_t)p->v | (uintptr_t)p->o) % 4 == 0, "vt_xattn_fwd: pointers must be 4-byte aligned");
  const XaStrides s{p->q_bs, p->q_hs, p->q_rs, p->k_bs, p->k_hs, p->k_rs, p->v_bs, p->v_hs, p->v_rs, p->o_bs, p->o_hs, p->o_rs, 0, 0, 0};
  dim3 grid((p->Nq + XA_QPB - 1) / XA_QPB, p->B * p->H);
  auto kern = p->hd == 96 ? (p->lse ? xattn_fwd_kernel<96, true> : xattn_fwd_kernel<96, false>)
                          : (p->lse ? xattn_fwd_kernel<64, true> : xattn_fwd_kernel<64, false>);
  kern<<<grid, 2 * XA_QPB, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(p->q), static_cast<const __nv_bfloat16*>(p->k), static_cast<const __nv_bfloat16*>(p->v),
      static_cast<__nv_bfloat16*>(p->o), p->lse, s, p->H, p->Nq, p->Nk, p->scale);
  return check_launch("xattn_fwd_kernel");
}

extern "C" int vt_xattn_bwd(const vt_xattn_bwd_params* p, void* stream) {
  VT_REQUIRE(p && p->q && p->k && p->v && p->o && p->dout && p->lse && p->delta && p->dq && p->dk && p->dv, "vt_xattn_bwd: null pointer");
  VT_REQUIRE(p->hd == 96 || p->hd == 64, "vt_xattn_bwd: head dim %d unsupported (64 or 96)", p->hd);
  VT_REQUIRE(p->B > 0 && p->H > 0 && p->Nq > 0 && p->Nk > 0 && (long long)p->B * p->H <= 65535, "vt_xattn_bwd: bad dims");
  VT_REQUIRE(p->impl >= VT_XATTN_AUTO && p->impl <= VT_XATTN_TCGEN05, "vt_xattn_bwd: bad impl %d", p->impl);
  const bool tc_ok = mma_layout_ok(p->q, p->q_bs, p->q_hs, p->q_rs, p->hd) && mma_layout_ok(p->k, p->k_bs, p->k_hs, p->k_rs, p->hd) &&
                     mma_layout_ok(p->v, p->v_bs, p->v_hs, p->v_rs, p->hd) && mma_layout_ok(p->o, p->o_bs, p->o_hs, p->o_rs, p->hd) &&
                     mma_layout_ok(p->dout, p->o_bs, p->o_hs, p->o_rs, p->hd) && mma_layout_ok(p->dq, p->dq_bs, p->dq_hs, p->dq_rs, p->hd);
  if (p->impl == VT_XATTN_TCGEN05 || (p->impl == VT_XATTN_AUTO && tc_ok)) {
    VT_REQUIRE(mma_layout_ok(p->q, p->q_bs, p->q_hs, p->q_rs, p->hd), "vt_xattn_bwd: unsupported q layout for the tensor-core kernel");
    VT_REQUIRE(tc_ok, "vt_xattn_bwd: unsupported k / v / o / dout / dq layout for the tensor-core kernel");
    MmaAttn a = xattn_operands(p);
    a.dout = static_cast<const __nv_bfloat16*>(p->dout);
    a.delta = p->delta;
    a.dq = static_cast<__nv_bfloat16*>(p->dq);
    a.dq_bs = p->dq_bs; a.dq_hs = p->dq_hs; a.dq_rs = p->dq_rs;
    a.dk32 = p->dk; a.dv32 = p->dv;
    return attn_mma_bwd(a, p->B, p->hd, static_cast<cudaStream_t>(stream));
  }
  const long long ss[15] = {p->q_bs, p->q_hs, p->q_rs, p->k_bs, p->k_hs, p->k_rs, p->v_bs, p->v_hs, p->v_rs, p->o_bs, p->o_hs, p->o_rs,
                            p->dq_bs, p->dq_hs, p->dq_rs};
  VT_REQUIRE(xa_strides_ok(ss, 15), "vt_xattn_bwd: strides must be even");
  VT_REQUIRE(((uintptr_t)p->q | (uintptr_t)p->k | (uintptr_t)p->v | (uintptr_t)p->o | (uintptr_t)p->dout | (uintptr_t)p->dq) % 4 == 0,
             "vt_xattn_bwd: pointers must be 4-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const XaStrides s{p->q_bs, p->q_hs, p->q_rs, p->k_bs, p->k_hs, p->k_rs, p->v_bs, p->v_hs, p->v_rs, p->o_bs, p->o_hs, p->o_rs,
                    p->dq_bs, p->dq_hs, p->dq_rs};
  const size_t kv_bytes = (size_t)p->B * p->H * p->Nk * p->hd * sizeof(float);
  cudaError_t e = cudaMemsetAsync(p->dk, 0, kv_bytes, st);
  VT_REQUIRE(e == cudaSuccess, "vt_xattn_bwd: memset dk: %s", cudaGetErrorString(e));
  e = cudaMemsetAsync(p->dv, 0, kv_bytes, st);
  VT_REQUIRE(e == cudaSuccess, "vt_xattn_bwd: memset dv: %s", cudaGetErrorString(e));
  dim3 gq((p->Nq + XA_QPB - 1) / XA_QPB, p->B * p->H);
  auto dq_kern = p->hd == 96 ? xattn_dq_kernel<96> : xattn_dq_kernel<64>;
  dq_kern<<<gq, 2 * XA_QPB, 0, st>>>(
      static_cast<const __nv_bfloat16*>(p->q), static_cast<const __nv_bfloat16*>(p->k), static_cast<const __nv_bfloat16*>(p->v),
      static_cast<const __nv_bfloat16*>(p->o), static_cast<const __nv_bfloat16*>(p->dout), p->lse, p->delta,
      static_cast<__nv_bfloat16*>(p->dq), s, p->H, p->Nq, p->Nk, p->scale);
  int rc = check_launch("xattn_dq_kernel");
  if (rc) return rc;
  const int qchunks = (p->Nq + XA_QCHUNK - 1) / XA_QCHUNK;
  VT_REQUIRE(qchunks <= 65535, "vt_xattn_bwd: Nq too large");
  dim3 gk((p->Nk + XA_KPB - 1) / XA_KPB, qchunks, p->B * p->H);
  auto dkv_kern = p->hd == 96 ? xattn_dkv_kernel<96> : xattn_dkv_kernel<64>;
  dkv_kern<<<gk, 4 * XA_KPB, 0, st>>>(
      static_cast<const __nv_bfloat16*>(p->q), static_cast<const __nv_bfloat16*>(p->k), static_cast<const __nv_bfloat16*>(p->v),
      static_cast<const __nv_bfloat16*>(p->dout), p->lse, p->delta, p->dk, p->dv, s, p->H, p->Nq, p->Nk, p->scale);
  return check_launch("xattn_dkv_kernel");
}

static int mp_dims_ok(const MpDims& d) {
  return d.kt >= 1 && d.kh >= 1 && d.kw >= 1 && d.kt * d.kh * d.kw < 255 && d.st >= 1 && d.sh >= 1 && d.sw >= 1 &&
         d.To == (d.T + 2 * (d.kt / 2) - d.kt) / d.st + 1 && d.Ho == (d.H + 2 * (d.kh / 2) - d.kh) / d.sh + 1 &&
         d.Wo == (d.W + 2 * (d.kw / 2) - d.kw) / d.sw + 1;
}

extern "C" int vt_maxpool_fwd(const vt_maxpool_fwd_params* p, void* stream) {
  VT_REQUIRE(p && p->x && p->y && p->B > 0 && p->D > 0 && p->D % 4 == 0, "vt_maxpool_fwd: bad params (D %% 4 == 0 required)");
  const MpDims d{p->B, p->D, p->T, p->H, p->W, p->kt, p->kh, p->kw, p->st, p->sh, p->sw, p->To, p->Ho, p->Wo};
  VT_REQUIRE(mp_dims_ok(d), "vt_maxpool_fwd: inconsistent geometry");
  const long long n = (long long)p->B * (1 + (long long)p->To * p->Ho * p->Wo) * (p->D / 4);
  (p->idx ? maxpool_fwd_kernel<true> : maxpool_fwd_kernel<false>)<<<flat_blocks(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      p->x, p->y, p->idx, d);
  return check_launch("maxpool_fwd_kernel");
}

extern "C" int vt_maxpool_bwd(const vt_maxpool_bwd_params* p, void* stream) {
  VT_REQUIRE(p && p->dy && p->idx && p->dx && p->B > 0 && p->D > 0 && p->D % 4 == 0, "vt_maxpool_bwd: bad params (D %% 4 == 0 required)");
  const MpDims d{p->B, p->D, p->T, p->H, p->W, p->kt, p->kh, p->kw, p->st, p->sh, p->sw, p->To, p->Ho, p->Wo};
  VT_REQUIRE(mp_dims_ok(d), "vt_maxpool_bwd: inconsistent geometry");
  const long long n = (long long)p->B * (1 + (long long)p->T * p->H * p->W) * (p->D / 4);
  maxpool_bwd_kernel<<<flat_blocks(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(p->dy, p->idx, p->dx, d);
  return check_launch("maxpool_bwd_kernel");
}

extern "C" int vt_im2col3d_bf16(const vt_im2col3d_params* p, void* stream) {
  VT_REQUIRE(p && p->x && p->cols, "vt_im2col3d_bf16: null pointer");
  VT_REQUIRE(p->To == (p->T + 2 * p->pt - p->kt) / p->st + 1 && p->Ho == (p->H + 2 * p->ph - p->kh) / p->sh + 1 &&
                 p->Wo == (p->W + 2 * p->pw - p->kw) / p->sw + 1, "vt_im2col3d_bf16: output dims inconsistent");
  VT_REQUIRE(p->Kpad >= p->C * p->kt * p->kh * p->kw && p->Kpad % 8 == 0, "vt_im2col3d_bf16: Kpad must cover C*kt*kh*kw and be a multiple of 8");
  const I3Dims d{p->B, p->T, p->C, p->H, p->W, p->kt, p->kh, p->kw, p->st, p->sh, p->sw, p->pt, p->ph, p->pw, p->To, p->Ho, p->Wo, p->Kpad};
  const long long n = (long long)p->B * p->To * p->Ho * p->Wo * ((p->Kpad + p->kw - 1) / p->kw);
  im2col3d_kernel<<<flat_blocks(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(p->x, static_cast<__nv_bfloat16*>(p->cols), d);
  return check_launch("im2col3d_kernel");
}

extern "C" int vt_im2col3d_u8_bf16(const vt_im2col3d_u8_params* p, void* stream) {
  VT_REQUIRE(p && p->x && p->mean && p->std && p->cols, "vt_im2col3d_u8_bf16: null pointer");
  VT_REQUIRE(p->B > 0 && p->T > 0 && p->C > 0 && p->H > 0 && p->W > 0 && p->kt > 0 && p->kh > 0 && p->kw > 0 && p->st > 0 &&
                 p->sh > 0 && p->sw > 0 && p->pt >= 0 && p->ph >= 0 && p->pw >= 0, "vt_im2col3d_u8_bf16: bad dims");
  VT_REQUIRE(p->To == (p->T + 2 * p->pt - p->kt) / p->st + 1 && p->Ho == (p->H + 2 * p->ph - p->kh) / p->sh + 1 &&
                 p->Wo == (p->W + 2 * p->pw - p->kw) / p->sw + 1 && p->To > 0 && p->Ho > 0 && p->Wo > 0,
             "vt_im2col3d_u8_bf16: output dims inconsistent");
  const int kreal = p->C * p->kt * p->kh * p->kw;
  VT_REQUIRE(p->Kpad >= kreal && p->Kpad % 8 == 0, "vt_im2col3d_u8_bf16: Kpad must cover C*kt*kh*kw and be a multiple of 8");
  VT_REQUIRE(reinterpret_cast<uintptr_t>(p->cols) % 16 == 0, "vt_im2col3d_u8_bf16: cols must be 16-byte aligned");
  const int Wp = p->W + 2 * p->pw;
  auto smem_for = [&](int ohb) {
    return (size_t)p->Kpad * sizeof(int) + (size_t)p->C * p->kt * ((ohb - 1) * p->sh + p->kh) * Wp * sizeof(__nv_bfloat16);
  };
  // rows per CTA: the most that keep the window within the default 48 KB (fewer source lines staged twice); one row
  // may take up to I3U8_SMEM_MAX
  constexpr size_t I3U8_SMEM_DEFAULT = 48 * 1024, I3U8_SMEM_MAX = 200 * 1024;
  int ohb = 4;
  while (ohb > 1 && smem_for(ohb) > I3U8_SMEM_DEFAULT) ohb /= 2;
  const size_t smem = smem_for(ohb);
  VT_REQUIRE(smem <= I3U8_SMEM_MAX, "vt_im2col3d_u8_bf16: the staged window (%zu bytes for W=%d, C=%d, kt=%d, kh=%d) does not fit in shared memory",
             smem, p->W, p->C, p->kt, p->kh);
  if (smem > I3U8_SMEM_DEFAULT) {
    static size_t max_set = I3U8_SMEM_DEFAULT;
    if (smem > max_set) {
      cudaError_t e = cudaFuncSetAttribute(im2col3d_u8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)I3U8_SMEM_MAX);
      VT_REQUIRE(e == cudaSuccess, "vt_im2col3d_u8_bf16: smem attribute: %s", cudaGetErrorString(e));
      max_set = I3U8_SMEM_MAX;
    }
  }
  const long long blocks = (long long)p->B * p->To * ((p->Ho + ohb - 1) / ohb);
  VT_REQUIRE(blocks <= 0x7fffffffLL, "vt_im2col3d_u8_bf16: grid too large");
  const I3U8Dims u{{p->B, p->T, p->C, p->H, p->W, p->kt, p->kh, p->kw, p->st, p->sh, p->sw, p->pt, p->ph, p->pw, p->To, p->Ho,
                    p->Wo, p->Kpad},
                   ohb, (ohb - 1) * p->sh + p->kh, Wp, kreal};
  im2col3d_u8_kernel<<<(unsigned)blocks, 256, smem, static_cast<cudaStream_t>(stream)>>>(
      p->x, p->mean, p->std, p->plan, static_cast<__nv_bfloat16*>(p->cols), u);
  return check_launch("im2col3d_u8_kernel");
}

extern "C" int vt_mvit_tokens_fwd(const vt_mvit_tokens_fwd_params* p, void* stream) {
  VT_REQUIRE(p && p->t && p->mask_token && p->cls_token && p->pos_s && p->pos_t && p->pos_cls && p->x, "vt_mvit_tokens_fwd: null pointer");
  VT_REQUIRE(p->B > 0 && p->T > 0 && p->HW > 0 && p->C > 0, "vt_mvit_tokens_fwd: bad dims");
  const long long n = (long long)p->B * (1 + (long long)p->T * p->HW) * p->C;
  mvit_tokens_fwd_kernel<<<flat_blocks(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      p->t, p->wmask, p->mask_token, p->cls_token, p->pos_s, p->pos_t, p->pos_cls, p->x, p->B, p->T, p->HW, p->C);
  return check_launch("mvit_tokens_fwd_kernel");
}

extern "C" int vt_mvit_tokens_bwd(const vt_mvit_tokens_bwd_params* p, void* stream) {
  VT_REQUIRE(p && p->dx && p->dt && p->B > 0 && p->T > 0 && p->HW > 0 && p->C > 0, "vt_mvit_tokens_bwd: bad params");
  const long long n = (long long)p->B * p->T * p->HW * p->C;
  mvit_tokens_bwd_kernel<<<flat_blocks(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      p->dx, p->wmask, static_cast<__nv_bfloat16*>(p->dt), p->B, p->T * p->HW, p->C);
  return check_launch("mvit_tokens_bwd_kernel");
}

extern "C" int vt_mse_blocks(int32_t cells) { return row_blocks(cells, 2); }

extern "C" int vt_mse_fwd(const vt_mse_fwd_params* p, void* stream) {
  VT_REQUIRE(p && p->pred && (p->target || p->target64) && p->mask && (p->num || p->num64) && p->partials, "vt_mse_fwd: null pointer");
  VT_REQUIRE(p->B > 0 && p->t > 0 && p->dt > 0 && p->h > 0 && p->w > 0 && p->dc > 0, "vt_mse_fwd: bad dims");
  VT_REQUIRE(((uintptr_t)p->partials & 15) == 0 && ((uintptr_t)p->num & 15) == 0, "vt_mse_fwd: partials/num must be 16-byte aligned");
  const MseDims d{p->B, p->t, p->dt, p->h, p->w, p->dc};
  const long long cells = (long long)p->B * p->t * p->dt * p->h * p->w;
  VT_REQUIRE(cells < 0x7fffffffll, "vt_mse_fwd: too many cells");
  const int blocks = vt_mse_blocks((int)cells);
  if (p->target64) {
    VT_REQUIRE(p->num64 != nullptr, "vt_mse_fwd: fp64 targets need num64");
    double* part = reinterpret_cast<double*>(p->partials);
    mse_fwd64_kernel<<<blocks, ROW_WARPS * 32, 0, static_cast<cudaStream_t>(stream)>>>(p->pred, p->target64, p->mask, part, d);
    int rc64 = check_launch("mse_fwd64_kernel");
    if (rc64) return rc64;
    mse_sum64_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(part, blocks, p->num64);
    return check_launch("mse_sum64_kernel");
  }
  mse_fwd_kernel<<<blocks, ROW_WARPS * 32, 0, static_cast<cudaStream_t>(stream)>>>(p->pred, p->target, p->mask, p->partials, d);
  int rc = check_launch("mse_fwd_kernel");
  if (rc) return rc;
  vt_reduce_params r{p->partials, p->num, 4, blocks, 4, 0, 1.0f};    // num[0] = sum, num[1..3] = 0
  return vt_reduce_rows(&r, stream);
}

extern "C" int vt_mse_bwd(const vt_mse_bwd_params* p, void* stream) {
  VT_REQUIRE(p && p->pred && (p->target || p->target64) && p->mask && p->coef && p->dpred, "vt_mse_bwd: null pointer");
  VT_REQUIRE(p->B > 0 && p->t > 0 && p->dt > 0 && p->h > 0 && p->w > 0 && p->dc > 0, "vt_mse_bwd: bad dims");
  const MseDims d{p->B, p->t, p->dt, p->h, p->w, p->dc};
  const long long n = (long long)p->B * (1 + (long long)p->t * p->h * p->w) * p->dt * p->dc;
  mse_bwd_kernel<<<flat_blocks(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(p->pred, p->target, p->target64, p->mask,
                                                                                     p->coef, static_cast<__nv_bfloat16*>(p->dpred), d);
  return check_launch("mse_bwd_kernel");
}
