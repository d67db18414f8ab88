// Remainder rows of a GEMM.  M = 12 552 (8 x 1569 tokens: TimeSformer's FFN, MViT's third stage), 50 184 and 200 712 (MViT
// stages 2 and 1) are all 8 rows past a multiple of 128, and those 8 rows cost a whole extra row of 128-row tiles — for
// N = 768 that is 297 tiles instead of 294 for 0.06 % of the work.  vt_gemm therefore runs the
// tensor-core kernel on the first floor(M / 128) * 128 rows and hands the last <= 16 rows to the kernels below: plain
// CUDA-core dot products, bandwidth-bound on one pass over the weight matrix (<= 4.7 MB), same epilogue arithmetic
// (s(m) * (acc + bias[n]) + aux[m, n], bf16 or fp32 out).  Operands are read as stored: B [N, K] ("NT", nn.Linear forward)
// or B [K, N] ("NN", data gradients).  Replaces the same nn.Linear calls as vt_gemm (transformer.py:501-505 and autograd).
#include "vt_common.cuh"

namespace vt {

struct RowsArgs {
  const __nv_bfloat16* a;   // [R, K] row-major, lda
  const __nv_bfloat16* b;
  long long lda, ldb;
  int R, N, K;
  const float* bias;        // [N] or null
  const float* bias2;       // [N] or null: added unscaled (fp32 out with aux)
  const float* row_scale;   // [R] or null
  const float* aux;         // [R, N] fp32 (ldaux) or null
  long long ldaux;
  void* out;                // [R, N] bf16 or fp32
  long long ldo;
  int f32_out;
};

constexpr int ROWS_PER_GROUP = 8;     // rows handled by one blockIdx.y

__device__ __forceinline__ void unpack8(const uint4 v, float (&f)[8]) {
  f[0] = __uint_as_float(v.x << 16); f[1] = __uint_as_float(v.x & 0xffff0000u);
  f[2] = __uint_as_float(v.y << 16); f[3] = __uint_as_float(v.y & 0xffff0000u);
  f[4] = __uint_as_float(v.z << 16); f[5] = __uint_as_float(v.z & 0xffff0000u);
  f[6] = __uint_as_float(v.w << 16); f[7] = __uint_as_float(v.w & 0xffff0000u);
}

__device__ __forceinline__ void rows_store(const RowsArgs& g, int r, int n, float acc) {
  const float s = g.row_scale ? g.row_scale[r] : 1.0f;
  float v = s * (acc + (g.bias ? g.bias[n] : 0.f));
  if (g.f32_out) {
    if (g.aux) v += g.aux[(long long)r * g.ldaux + n];
    if (g.bias2) v += g.bias2[n];
    static_cast<float*>(g.out)[(long long)r * g.ldo + n] = v;
  } else {
    static_cast<__nv_bfloat16*>(g.out)[(long long)r * g.ldo + n] = __float2bfloat16_rn(v);
  }
}

// B [N, K]: one warp per output column, lanes stride over K in 8-element (16-byte) pieces, four pieces in flight; the <= 8
// activation rows are re-read through L1 by every warp (8 x K x 2 bytes <= 48 KB)
constexpr int NT_WARPS = 4;
__global__ void __launch_bounds__(NT_WARPS * 32) rows_nt_kernel(RowsArgs g) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = blockIdx.y * ROWS_PER_GROUP;
  const int nr = min(ROWS_PER_GROUP, g.R - r0);
  const __nv_bfloat16* a = g.a + (long long)r0 * g.lda;
  for (int n = blockIdx.x * NT_WARPS + warp; n < g.N; n += gridDim.x * NT_WARPS) {
    float acc[ROWS_PER_GROUP];
#pragma unroll
    for (int r = 0; r < ROWS_PER_GROUP; ++r) acc[r] = 0.f;
    const __nv_bfloat16* brow = g.b + (long long)n * g.ldb;
    for (int k0 = lane * 8; k0 < g.K; k0 += 4 * 256) {
      uint4 wv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int k = k0 + u * 256;
        wv[u] = k < g.K ? __ldg(reinterpret_cast<const uint4*>(brow + k)) : make_uint4(0u, 0u, 0u, 0u);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int k = k0 + u * 256;
        if (k >= g.K) break;
        float wf[8];
        unpack8(wv[u], wf);
#pragma unroll
        for (int r = 0; r < ROWS_PER_GROUP; ++r) {
          if (r < nr) {
            float af[8];
            unpack8(__ldg(reinterpret_cast<const uint4*>(a + (long long)r * g.lda + k)), af);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[r] = fmaf(af[j], wf[j], acc[r]);
          }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < ROWS_PER_GROUP; ++r) acc[r] = warp_sum(acc[r]);
    float mine = 0.f;
#pragma unroll
    for (int r = 0; r < ROWS_PER_GROUP; ++r)
      if (lane == r) mine = acc[r];
    if (lane < nr) rows_store(g, r0 + lane, n, mine);
  }
}

// B [K, N]: CTA = CG * 8 output columns; thread = (8 consecutive columns) x (one of 256 / CG K slices, 8 consecutive k per
// step); slices are summed by shuffles inside a warp and through shared memory across the 8 warps.  CG is chosen so
// that even N = 768 spreads over 48 CTAs.
template <int CG>
__global__ void __launch_bounds__(256) rows_nn_kernel(RowsArgs g) {
  constexpr int COLS = CG * 8, SLICES = 256 / CG;
  __shared__ float red[8][ROWS_PER_GROUP * COLS];
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int cg = t % CG, ks = t / CG;
  const int r0 = blockIdx.y * ROWS_PER_GROUP;
  const int nr = min(ROWS_PER_GROUP, g.R - r0);
  const __nv_bfloat16* a = g.a + (long long)r0 * g.lda;
  const int n0 = blockIdx.x * COLS + cg * 8;
  const bool col_ok = n0 < g.N;
  float acc[ROWS_PER_GROUP][8];
#pragma unroll
  for (int r = 0; r < ROWS_PER_GROUP; ++r)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[r][j] = 0.f;
  for (int k = ks * 8; k < g.K; k += SLICES * 8) {
    uint4 wv[8];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
      wv[kk] = col_ok ? __ldg(reinterpret_cast<const uint4*>(g.b + (long long)(k + kk) * g.ldb + n0)) : make_uint4(0u, 0u, 0u, 0u);
    float af[ROWS_PER_GROUP][8];
#pragma unroll
    for (int r = 0; r < ROWS_PER_GROUP; ++r) {
      if (r < nr) unpack8(__ldg(reinterpret_cast<const uint4*>(a + (long long)r * g.lda + k)), af[r]);
      else {
#pragma unroll
        for (int j = 0; j < 8; ++j) af[r][j] = 0.f;
      }
    }
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      float wf[8];
      unpack8(wv[kk], wf);
#pragma unroll
      for (int r = 0; r < ROWS_PER_GROUP; ++r)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[r][j] = fmaf(af[r][kk], wf[j], acc[r][j]);
    }
  }
  // lanes cg, cg + CG, cg + 2 CG, ... of a warp hold different K slices of the same columns
#pragma unroll
  for (int r = 0; r < ROWS_PER_GROUP; ++r)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float v = acc[r][j];
#pragma unroll
      for (int o = CG; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      acc[r][j] = v;
    }
  if (lane < CG) {
#pragma unroll
    for (int r = 0; r < ROWS_PER_GROUP; ++r)
#pragma unroll
      for (int j = 0; j < 8; ++j) red[warp][r * COLS + cg * 8 + j] = acc[r][j];
  }
  __syncthreads();
  for (int i = t; i < nr * COLS; i += 256) {
    const int r = i / COLS, c = i - r * COLS;
    const int n = blockIdx.x * COLS + c;
    if (n >= g.N) continue;
    float v = red[0][i];
#pragma unroll
    for (int w = 1; w < 8; ++w) v += red[w][i];
    rows_store(g, r0 + r, n, v);
  }
}

int launch_gemm_rows(const vt_gemm_params* q, int m0, void* stream) {
  const int R = q->M - m0;
  VT_REQUIRE(R > 0 && R <= 2 * ROWS_PER_GROUP && !q->a_mn_major && q->K % 8 == 0 && q->lda % 8 == 0 && q->ldb % 8 == 0,
             "vt_gemm(remainder rows): unsupported call");
  const bool f32 = q->epilogue == VT_EPI_F32;
  RowsArgs g;
  g.a = static_cast<const __nv_bfloat16*>(q->a) + (long long)m0 * q->lda;
  g.b = static_cast<const __nv_bfloat16*>(q->b);
  g.lda = q->lda; g.ldb = q->ldb;
  g.R = R; g.N = q->N; g.K = q->K;
  g.bias = q->bias;
  g.bias2 = q->bias2;
  g.row_scale = q->row_scale ? q->row_scale + m0 : nullptr;
  g.aux = (f32 && q->aux) ? static_cast<const float*>(q->aux) + (long long)m0 * q->ldaux : nullptr;
  g.ldaux = q->ldaux;
  g.out = f32 ? static_cast<void*>(static_cast<float*>(q->out) + (long long)m0 * q->ldo)
              : static_cast<void*>(static_cast<__nv_bfloat16*>(q->out) + (long long)m0 * q->ldo);
  g.ldo = q->ldo;
  g.f32_out = f32 ? 1 : 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int groups = (R + ROWS_PER_GROUP - 1) / ROWS_PER_GROUP;
  if (q->b_mn_major) {
    if (q->N >= 2048) rows_nn_kernel<8><<<dim3((q->N + 63) / 64, groups), 256, 0, st>>>(g);
    else if (q->N >= 1024) rows_nn_kernel<4><<<dim3((q->N + 31) / 32, groups), 256, 0, st>>>(g);
    else rows_nn_kernel<2><<<dim3((q->N + 15) / 16, groups), 256, 0, st>>>(g);
    return check_launch("rows_nn_kernel");
  }
  int blocks = (q->N + NT_WARPS - 1) / NT_WARPS;
  const int cap = sm_count() * 8;
  if (blocks > cap) blocks = cap;
  rows_nt_kernel<<<dim3(blocks, groups), NT_WARPS * 32, 0, st>>>(g);
  return check_launch("rows_nt_kernel");
}

}  // namespace vt
