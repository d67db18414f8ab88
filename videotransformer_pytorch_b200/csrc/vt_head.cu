// Small fp32 kernels around the transformer body:
//   * skinny linear layer (classification head: 8 x 768 -> 400) forward / backward — warp-per-output GEMV, fp32 throughout
//   * softmax cross-entropy (hard labels or soft targets) forward + gradient in one launch
//   * attention probabilities softmax(q k^T * scale) for long sequences (vt_attn_fwd's probs output past 256 tokens:
//     get_last_selfattention of the joint variants), and their cls row alone (vt_attn_cls_probs past 256 tokens)
//   * uint8 clip -> normalised bf16 patch operand with Mixup / CutMix of the flipped batch folded in
//   * top-k hit counters of an evaluation step (view mean, optional softmax, rank of the label)
// All are latency / bandwidth bound warp-primitive kernels (no tensor cores: M <= 64 rows or one-off visualisation work).
#include "vt_common.cuh"
#include "../../include/vt_attn_maps.h"

namespace vt {

// ------------------------------------------------------------------------------------------------
// y[m, n] = sum_k x[m, k] * W[n, k] + b[n]      (fp32; one warp per output column n, 8 rows of x per pass)
// ------------------------------------------------------------------------------------------------
constexpr int LS_ROWS = 8;

__global__ void __launch_bounds__(256)
linear_small_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                        float* __restrict__ y, int M, int N, int K) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * 8 + warp;
  const int m0 = blockIdx.y * LS_ROWS;
  if (n >= N) return;
  float acc[LS_ROWS];
#pragma unroll
  for (int r = 0; r < LS_ROWS; ++r) acc[r] = 0.f;
  const float* wr = w + (long long)n * K;
  for (int k = lane * 4; k < K; k += 128) {
    const float4 wv = __ldg(reinterpret_cast<const float4*>(wr + k));
#pragma unroll
    for (int r = 0; r < LS_ROWS; ++r) {
      if (m0 + r < M) {
        const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (long long)(m0 + r) * K + k));
        acc[r] = fmaf(xv.x, wv.x, fmaf(xv.y, wv.y, fmaf(xv.z, wv.z, fmaf(xv.w, wv.w, acc[r]))));
      }
    }
  }
#pragma unroll
  for (int r = 0; r < LS_ROWS; ++r) acc[r] = warp_sum(acc[r]);
  if (lane == 0) {
    const float bias = b ? b[n] : 0.f;
#pragma unroll
    for (int r = 0; r < LS_ROWS; ++r)
      if (m0 + r < M) y[(long long)(m0 + r) * N + n] = acc[r] + bias;
  }
}

// dW[n, k] = sum_m dy[m, n] x[m, k] ;  db[n] = sum_m dy[m, n]          (one warp per n)
__global__ void __launch_bounds__(256)
linear_small_wgrad_kernel(const float* __restrict__ dy, const float* __restrict__ x, float* __restrict__ dw,
                          float* __restrict__ db, int M, int N, int K) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * 8 + warp;
  if (n >= N) return;
  for (int k = lane * 4; k < K; k += 128) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int m = 0; m < M; ++m) {
      const float g = __ldg(dy + (long long)m * N + n);
      const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (long long)m * K + k));
      acc.x = fmaf(g, xv.x, acc.x); acc.y = fmaf(g, xv.y, acc.y); acc.z = fmaf(g, xv.z, acc.z); acc.w = fmaf(g, xv.w, acc.w);
    }
    *reinterpret_cast<float4*>(dw + (long long)n * K + k) = acc;
  }
  if (db && lane == 0) {
    float s = 0.f;
    for (int m = 0; m < M; ++m) s += dy[(long long)m * N + n];
    db[n] = s;
  }
}

// dx[m, k] = sum_n dy[m, n] W[n, k]: block = 128 columns x 8 rows, the 8 warps split n and merge through shared memory
__global__ void __launch_bounds__(256)
linear_small_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ dx, int M, int N,
                          int K) {
  __shared__ float4 red[8][LS_ROWS][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k = blockIdx.x * 128 + lane * 4;
  const int m0 = blockIdx.y * LS_ROWS;
  float4 acc[LS_ROWS];
#pragma unroll
  for (int r = 0; r < LS_ROWS; ++r) acc[r] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (k < K) {
    for (int n = warp; n < N; n += 8) {
      const float4 wv = __ldg(reinterpret_cast<const float4*>(w + (long long)n * K + k));
#pragma unroll
      for (int r = 0; r < LS_ROWS; ++r) {
        if (m0 + r < M) {
          const float g = __ldg(dy + (long long)(m0 + r) * N + n);
          acc[r].x = fmaf(g, wv.x, acc[r].x); acc[r].y = fmaf(g, wv.y, acc[r].y);
          acc[r].z = fmaf(g, wv.z, acc[r].z); acc[r].w = fmaf(g, wv.w, acc[r].w);
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < LS_ROWS; ++r) red[warp][r][lane] = acc[r];
  __syncthreads();
  if (k < K && warp < LS_ROWS && m0 + warp < M) {          // warp r finalises row r
    float4 s = red[0][warp][lane];
#pragma unroll
    for (int q = 1; q < 8; ++q) {
      const float4 t = red[q][warp][lane];
      s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
    }
    *reinterpret_cast<float4*>(dx + (long long)(m0 + warp) * K + k) = s;
  }
}

// ------------------------------------------------------------------------------------------------
// Softmax cross-entropy, mean over the M rows (nn.CrossEntropyLoss; timm SoftTargetCrossEntropy with `soft`):
//   loss = 1/M sum_m ( log(sum_c e^(z_mc - mx_m)) * sum_c t_mc - sum_c t_mc (z_mc - mx_m) ),   mx_m = max_c z_mc
//   dz_mc = (softmax(z_m)_c * sum_c' t_mc' - t_mc) / M
// The row loss is formed from z - mx, so it does not cancel at the magnitude of the logits, and classes with t = 0 are
// skipped, so a -inf logit that is not the label gives torch's finite loss rather than 0 * -inf = NaN.
// One CTA, rows in sequence (M is the per-GPU batch); deterministic.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
softmax_ce_kernel(const float* __restrict__ z, const int64_t* __restrict__ labels, const float* __restrict__ soft,
                  float* __restrict__ loss, float* __restrict__ row_loss, float* __restrict__ dz, int M, int N) {
  __shared__ float sh[8];
  __shared__ float total;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  auto block_reduce = [&](float v, bool is_max) {
    v = is_max ? warp_max(v) : warp_sum(v);
    __syncthreads();
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    float r = sh[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) r = is_max ? fmaxf(r, sh[i]) : r + sh[i];
    return r;
  };
  if (threadIdx.x == 0) total = 0.f;
  const float inv_m = 1.0f / (float)M;
  for (int m = 0; m < M; ++m) {
    const float* zr = z + (long long)m * N;
    float mx = -INFINITY;
    for (int c = threadIdx.x; c < N; c += 256) mx = fmaxf(mx, zr[c]);
    mx = block_reduce(mx, true);
    float se = 0.f, tz = 0.f, ts = 0.f;
    const long long lab = labels ? (long long)labels[m] : -1;
    for (int c = threadIdx.x; c < N; c += 256) {
      const float d = zr[c] - mx;
      se += expf(d);
      const float t = soft ? soft[(long long)m * N + c] : (c == lab ? 1.f : 0.f);
      if (t != 0.f) tz = fmaf(t, d, tz);
      ts += t;
    }
    se = block_reduce(se, false);
    tz = block_reduce(tz, false);
    ts = block_reduce(ts, false);
    const float inv_se = 1.0f / se;
    for (int c = threadIdx.x; c < N; c += 256) {
      const float t = soft ? soft[(long long)m * N + c] : (c == lab ? 1.f : 0.f);
      dz[(long long)m * N + c] = (expf(zr[c] - mx) * inv_se * ts - t) * inv_m;
    }
    if (threadIdx.x == 0) {
      const float l = logf(se) * ts - tz;
      if (row_loss) row_loss[m] = l;
      total += l;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) loss[0] = total * inv_m;
}

// out[i] = in[i] * s[0]   (chain rule through the scalar loss; s is a device scalar so the step stays graph-capturable)
__global__ void scale_by_scalar_kernel(const float* __restrict__ in, const float* __restrict__ s, float* __restrict__ out,
                                       long long n) {
  const float f = s[0];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = in[i] * f;
}

// ------------------------------------------------------------------------------------------------
// Attention probabilities for any sequence length (head dim 32, 64, 96 or 128): probs[bp, h, i, :] = softmax_j(q_i . k_j * scale)
// CTA = PR_ROWS query rows of one (batch', head): raw scores of those rows live in shared memory (rows x N fp32),
// keys stream through in tiles of 64 (pitch HD + 1 floats: lane = key reads are conflict free); then a row softmax in
// place and coalesced fp32 stores.
// The arithmetic of these probabilities lives in the four functions below, shared with the cls-row kernel: q scaled on
// load, one fmaf per feature in feature order, and a one-warp softmax (max, then exp and sum in lane-strided order,
// then one reciprocal).
// ------------------------------------------------------------------------------------------------
constexpr int PR_ROWS = 8;
constexpr int PR_KT = 64;
constexpr int CLS_KT = 256;    // keys per tile of the cls-row kernel: one per thread

__device__ __forceinline__ float probs_q(__nv_bfloat16 q, float scale) { return __bfloat162float(q) * scale; }

// keys j0 .. j0 + KT - 1 of one head (kbase: key 0's k slice, rows rs elements apart) -> Kt[KT][HD + 1] fp32, zeros past N
template <int HD, int KT>
__device__ __forceinline__ void probs_load_keys(float* Kt, const __nv_bfloat16* kbase, long long rs, int N, int j0) {
  constexpr int KP = HD + 1, CPR = HD / 8;          // key pitch (floats), 16-byte chunks per row
  for (int idx = threadIdx.x; idx < KT * CPR; idx += 256) {       // KT keys x HD / 8 vectors of 8 bf16
    const int j = div_pos<CPR>(idx), c = mod_pos<CPR>(idx);
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (j0 + j < N) v = *reinterpret_cast<const uint4*>(kbase + (long long)(j0 + j) * rs + c * 8);
    float* d = Kt + j * KP + c * 8;
    const float2 a = unpack_bf16x2(v.x), b2 = unpack_bf16x2(v.y), c2 = unpack_bf16x2(v.z), e2 = unpack_bf16x2(v.w);
    d[0] = a.x; d[1] = a.y; d[2] = b2.x; d[3] = b2.y; d[4] = c2.x; d[5] = c2.y; d[6] = e2.x; d[7] = e2.y;
  }
}

// raw score of scaled query q[HD] and key k[HD]
template <int HD>
__device__ __forceinline__ float probs_dot(const float* q, const float* k) {
  float s = 0.f;
#pragma unroll 16
  for (int d = 0; d < HD; ++d) s = fmaf(q[d], k[d], s);
  return s;
}

// one warp: out[0, N) = softmax of the raw scores row[0, N) (row is overwritten with the exponentials)
__device__ __forceinline__ void probs_softmax_row(float* row, int N, int lane, float* out) {
  float mx = -INFINITY;
  for (int j = lane; j < N; j += 32) mx = fmaxf(mx, row[j]);
  mx = warp_max(mx);
  float se = 0.f;
  for (int j = lane; j < N; j += 32) { const float e = expf(row[j] - mx); row[j] = e; se += e; }
  se = warp_sum(se);
  const float inv = 1.0f / se;
  for (int j = lane; j < N; j += 32) out[j] = row[j] * inv;
}

template <int HD>
__global__ void __launch_bounds__(256)
attn_probs_kernel(const __nv_bfloat16* __restrict__ qkv, float* __restrict__ probs, int N, int H, float scale) {
  constexpr int KP = HD + 1;
  extern __shared__ float psm[];
  float* S = psm;                                   // [PR_ROWS][N]
  float* Q = S + (size_t)PR_ROWS * N;               // [PR_ROWS][HD]
  float* Kt = Q + PR_ROWS * HD;                     // [64 keys][HD + 1]
  const int bh = blockIdx.y, bp = bh / H, h = bh - bp * H;
  const int i0 = blockIdx.x * PR_ROWS;
  const long long rs = 3LL * H * HD;
  const __nv_bfloat16* base = qkv + (long long)bp * N * rs + h * HD;
  for (int idx = threadIdx.x; idx < PR_ROWS * HD; idx += 256) {
    const int r = div_pos<HD>(idx), d = mod_pos<HD>(idx);
    Q[idx] = (i0 + r < N) ? probs_q(base[(long long)(i0 + r) * rs + d], scale) : 0.f;
  }
  for (int j0 = 0; j0 < N; j0 += PR_KT) {
    __syncthreads();
    probs_load_keys<HD, PR_KT>(Kt, base + (long long)H * HD, rs, N, j0);
    __syncthreads();
    // 256 threads = 8 rows x 32 lanes; lane handles keys lane and lane + 32 of the tile
    const int r = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float s0 = probs_dot<HD>(Q + r * HD, Kt + lane * KP);
    const float s1 = probs_dot<HD>(Q + r * HD, Kt + (lane + 32) * KP);
    if (j0 + lane < N) S[(size_t)r * N + j0 + lane] = s0;
    if (j0 + lane + 32 < N) S[(size_t)r * N + j0 + lane + 32] = s1;
  }
  __syncthreads();
  const int r = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (i0 + r < N) probs_softmax_row(S + (size_t)r * N, N, lane, probs + ((long long)bh * N + (i0 + r)) * N);
}

// Query row 0 (the cls token) of attn_probs_kernel's probabilities, at any N whose score row fits in shared memory: one
// CTA per (batch', head), keys in tiles of CLS_KT (thread t scores key j0 + t), then warp 0 runs the row softmax into
// out[bh, 0, N).
template <int HD>
__global__ void __launch_bounds__(256)
attn_cls_probs_tiled_kernel(const __nv_bfloat16* __restrict__ qkv, float* __restrict__ out, int N, int H, float scale) {
  constexpr int KP = HD + 1;
  extern __shared__ float psm[];
  float* S = psm;                                   // [N]
  float* Q = S + N;                                 // [HD]
  float* Kt = Q + HD;                               // [CLS_KT keys][HD + 1]
  const int bh = blockIdx.x, bp = bh / H, h = bh - bp * H;
  const long long rs = 3LL * H * HD;
  const __nv_bfloat16* base = qkv + (long long)bp * N * rs + h * HD;
  for (int d = threadIdx.x; d < HD; d += 256) Q[d] = probs_q(base[d], scale);
  for (int j0 = 0; j0 < N; j0 += CLS_KT) {
    __syncthreads();
    probs_load_keys<HD, CLS_KT>(Kt, base + (long long)H * HD, rs, N, j0);
    __syncthreads();
    const float s = probs_dot<HD>(Q, Kt + threadIdx.x * KP);
    if (j0 + (int)threadIdx.x < N) S[j0 + threadIdx.x] = s;
  }
  __syncthreads();
  if (threadIdx.x < 32) probs_softmax_row(S, N, threadIdx.x, out + (long long)bh * N);
}

// ------------------------------------------------------------------------------------------------
// uint8 clip [B, T, H, W, C] -> bf16 patch operand, ToTensor + Normalize fused, with the batch-level Mixup / CutMix of
// reference mixup.py:102-114 folded in: sample b is mixed with sample B-1-b (x.flip(0)).
//   plan = {mode, lam, yl, yh, xl, xh} as floats in device memory (mode 0 none, 1 mixup, 2 cutmix), so a captured graph
//   picks up each step's draw.
// ------------------------------------------------------------------------------------------------
__global__ void im2col_u8_mix_kernel(const uint8_t* __restrict__ x, const float* __restrict__ scale, const float* __restrict__ shift,
                                     const float* __restrict__ plan, __nv_bfloat16* __restrict__ cols, int B, int T, int C,
                                     int H, int W, int tube, int ph, int pw, long long total8) {
  const int Kc = C * tube * ph * pw;
  const int Hp = H / ph, Wp = W / pw, Tp = T / tube;
  const int mode = (int)plan[0];
  const float lam = plan[1];
  const int yl = (int)plan[2], yh = (int)plan[3], xl = (int)plan[4], xh = (int)plan[5];
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
    const int yy = hp * ph + i, xx0 = wp * pw + j;
    const long long off = ((((long long)(tp * tube + dt)) * H + yy) * W + xx0) * C + c;
    const long long clip = (long long)T * H * W * C;
    const uint8_t* src = x + (long long)b * clip + off;
    const uint8_t* oth = x + (long long)(B - 1 - b) * clip + off;
    const float sc = scale[c], sh = shift[c];
    float v[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float a = fmaf((float)src[(long long)q * C], sc, sh);
      if (mode == 1) {
        const float o = fmaf((float)oth[(long long)q * C], sc, sh);
        v[q] = a * lam + o * (1.0f - lam);                           // x.mul_(lam).add_(x.flip(0).mul_(1 - lam))
      } else if (mode == 2) {
        const bool inside = yy >= yl && yy < yh && (xx0 + q) >= xl && (xx0 + q) < xh;
        v[q] = inside ? fmaf((float)oth[(long long)q * C], sc, sh) : a;   // x[:, :, yl:yh, xl:xh] = x.flip(0)[...]
      } else {
        v[q] = a;
      }
    }
    uint4 o;
    o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]);
    o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(cols + e) = o;
  }
}

template <int HD>
static int attn_probs_launch_hd(const void* qkv, float* probs, int Bp, int N, int H, float scale, cudaStream_t st) {
  const size_t smem = ((size_t)PR_ROWS * N + PR_ROWS * HD + PR_KT * (HD + 1)) * sizeof(float);
  VT_REQUIRE(smem <= 200 * 1024, "vt_attn_fwd: N=%d too long for the probs output (%zu bytes of shared memory)", N, smem);
  static size_t max_set = 48 * 1024;
  if (smem > max_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_probs_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    VT_REQUIRE(e == cudaSuccess, "vt_attn_fwd: probs smem attribute: %s", cudaGetErrorString(e));
    max_set = 200 * 1024;
  }
  dim3 grid((N + PR_ROWS - 1) / PR_ROWS, Bp * H);
  attn_probs_kernel<HD><<<grid, 256, smem, st>>>(static_cast<const __nv_bfloat16*>(qkv), probs, N, H, scale);
  return check_launch("attn_probs_kernel");
}

// the probs output of vt_attn_fwd on the tensor-core path (vt_attention.cu); qkv is the packed projection at head dim hd
// (checked by vt_attn_fwd)
int attn_probs_launch(const void* qkv, float* probs, int Bp, int N, int H, int hd, float scale, cudaStream_t st) {
  return with_head_dim(hd, [&](auto d) { return attn_probs_launch_hd<d.value>(qkv, probs, Bp, N, H, scale, st); });
}

template <int HD>
static int attn_cls_probs_tiled_hd(const vt_attn_cls_probs_params* p, cudaStream_t st) {
  constexpr size_t limit = 227 * 1024;   // the largest dynamic shared memory a CTA may opt into on sm_90
  const size_t smem = ((size_t)p->N + HD + CLS_KT * (HD + 1)) * sizeof(float);
  VT_REQUIRE(smem <= limit, "vt_attn_cls_probs: N=%d at head dim %d needs %zu bytes of shared memory (%zu at most)", p->N,
             HD, smem, limit);
  static size_t max_set = 48 * 1024;
  if (smem > max_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_cls_probs_tiled_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)limit);
    VT_REQUIRE(e == cudaSuccess, "vt_attn_cls_probs: smem attribute: %s", cudaGetErrorString(e));
    max_set = limit;
  }
  attn_cls_probs_tiled_kernel<HD><<<p->Bp * p->H, 256, smem, st>>>(static_cast<const __nv_bfloat16*>(p->qkv), p->probs, p->N,
                                                                    p->H, p->scale);
  return check_launch("attn_cls_probs_tiled_kernel");
}

// vt_attn_cls_probs past the generic kernel's N (vt_attention.cu checks the parameters)
int attn_cls_probs_tiled_launch(const vt_attn_cls_probs_params* p, cudaStream_t st) {
  return with_head_dim(p->hd, [&](auto d) { return attn_cls_probs_tiled_hd<d.value>(p, st); });
}

static int grid_1d(long long n, int threads) {
  long long b = (n + threads - 1) / threads;
  const long long cap = (long long)sm_count() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace vt

using namespace vt;

extern "C" int vt_linear_small_fwd(const vt_linear_small_params* p, void* stream) {
  VT_REQUIRE(p && p->x && p->w && p->y, "vt_linear_small_fwd: null pointer");
  VT_REQUIRE(p->M > 0 && p->N > 0 && p->K > 0 && p->K % 4 == 0, "vt_linear_small_fwd: bad shape M=%d N=%d K=%d (K %% 4 == 0)", p->M, p->N, p->K);
  VT_REQUIRE(p->M <= 4096, "vt_linear_small_fwd: M=%d is not skinny (use vt_gemm)", p->M);
  VT_REQUIRE(((reinterpret_cast<uintptr_t>(p->x) | reinterpret_cast<uintptr_t>(p->w)) & 15) == 0,
             "vt_linear_small_fwd: x and w must be 16-byte aligned");
  dim3 grid((p->N + 7) / 8, (p->M + LS_ROWS - 1) / LS_ROWS);
  linear_small_fwd_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(p->x, p->w, p->b, p->y, p->M, p->N, p->K);
  return check_launch("linear_small_fwd_kernel");
}

extern "C" int vt_linear_small_bwd(const vt_linear_small_bwd_params* p, void* stream) {
  VT_REQUIRE(p && p->dy && p->x && p->w, "vt_linear_small_bwd: null pointer");
  VT_REQUIRE(p->M > 0 && p->N > 0 && p->K > 0 && p->K % 4 == 0, "vt_linear_small_bwd: bad shape");
  VT_REQUIRE(p->M <= 4096, "vt_linear_small_bwd: M=%d is not skinny", p->M);
  VT_REQUIRE(((reinterpret_cast<uintptr_t>(p->x) | reinterpret_cast<uintptr_t>(p->w) | reinterpret_cast<uintptr_t>(p->dw) |
               reinterpret_cast<uintptr_t>(p->dx)) & 15) == 0,
             "vt_linear_small_bwd: x, w, dw and dx must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (p->dw) {
    linear_small_wgrad_kernel<<<(p->N + 7) / 8, 256, 0, st>>>(p->dy, p->x, p->dw, p->db, p->M, p->N, p->K);
    int rc = check_launch("linear_small_wgrad_kernel");
    if (rc) return rc;
  }
  if (p->dx) {
    dim3 grid((p->K + 127) / 128, (p->M + LS_ROWS - 1) / LS_ROWS);
    linear_small_dgrad_kernel<<<grid, 256, 0, st>>>(p->dy, p->w, p->dx, p->M, p->N, p->K);
    return check_launch("linear_small_dgrad_kernel");
  }
  return 0;
}

extern "C" int vt_softmax_ce(const vt_softmax_ce_params* p, void* stream) {
  VT_REQUIRE(p && p->logits && p->loss && p->dlogits, "vt_softmax_ce: null pointer");
  VT_REQUIRE((p->labels != nullptr) != (p->soft_targets != nullptr), "vt_softmax_ce: give labels or soft_targets (exactly one)");
  VT_REQUIRE(p->M > 0 && p->M <= 4096 && p->N > 0, "vt_softmax_ce: bad shape M=%d N=%d", p->M, p->N);
  softmax_ce_kernel<<<1, 256, 0, static_cast<cudaStream_t>(stream)>>>(p->logits, p->labels, p->soft_targets, p->loss,
                                                                       p->row_loss, p->dlogits, p->M, p->N);
  return check_launch("softmax_ce_kernel");
}

extern "C" int vt_scale_by_scalar(const vt_scale_params* p, void* stream) {
  VT_REQUIRE(p && p->in && p->scalar && p->out && p->n > 0, "vt_scale_by_scalar: bad params");
  scale_by_scalar_kernel<<<grid_1d(p->n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(p->in, p->scalar, p->out, p->n);
  return check_launch("scale_by_scalar_kernel");
}

extern "C" int vt_im2col_u8_mix_bf16(const vt_im2col_u8_mix_params* p, void* stream) {
  VT_REQUIRE(p && p->x && p->scale && p->shift && p->cols && p->plan, "vt_im2col_u8_mix_bf16: null pointer");
  VT_REQUIRE(p->pw % 8 == 0 && p->W % p->pw == 0 && p->H % p->ph == 0 && p->T % p->tube == 0, "vt_im2col_u8_mix_bf16: unsupported geometry");
  const long long total8 = (long long)p->B * p->T * p->C * p->H * p->W / 8;
  im2col_u8_mix_kernel<<<grid_1d(total8, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      p->x, p->scale, p->shift, p->plan, static_cast<__nv_bfloat16*>(p->cols), p->B, p->T, p->C, p->H, p->W, p->tube, p->ph,
      p->pw, total8);
  return check_launch("im2col_u8_mix_kernel");
}

// ------------------------------------------------------------------------------------------------
// Top-k hits of one evaluation batch: one CTA per clip.  The clip's V view rows are averaged into shared memory (summed
// in view order, then scaled by 1/V as torch's mean does: preds.view(-1, V, C).mean(1)); rank = number of classes whose mean is strictly
// greater than the label's; counter i gains 1 when rank < k[i].  Integer atomics: the totals do not depend on the order
// the CTAs finish in, and nothing is allocated or synchronised, so the kernel can be captured in a CUDA graph.
// ------------------------------------------------------------------------------------------------
namespace vt {
constexpr int TK_THREADS = 256;

__global__ void __launch_bounds__(TK_THREADS)
topk_hits_kernel(const float* __restrict__ logits, const int64_t* __restrict__ labels, float* __restrict__ probs,
                 unsigned long long* __restrict__ hits, unsigned long long* __restrict__ samples, int B, int V, int C,
                 int4 ks, int n_k) {
  extern __shared__ float tk_mean[];
  __shared__ float red_f[TK_THREADS / 32];
  __shared__ int red_i[TK_THREADS / 32];
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* z = logits + (long long)b * V * C;
  const float inv_v = 1.0f / (float)V;
  for (int c = threadIdx.x; c < C; c += TK_THREADS) {
    float m = z[c];
    for (int v = 1; v < V; ++v) m += z[(long long)v * C + c];
    tk_mean[c] = m * inv_v;
  }
  __syncthreads();
  const long long lab = labels[b];
  const bool lab_ok = lab >= 0 && lab < C;
  const float ml = lab_ok ? tk_mean[lab] : 0.f;
  int above = 0;
  for (int c = threadIdx.x; c < C; c += TK_THREADS) above += tk_mean[c] > ml;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) above += __shfl_xor_sync(0xffffffffu, above, o);
  if (lane == 0) red_i[warp] = above;
  if (probs) {
    float mx = -INFINITY;
    for (int c = threadIdx.x; c < C; c += TK_THREADS) mx = fmaxf(mx, tk_mean[c]);
    mx = warp_max(mx);
    if (lane == 0) red_f[warp] = mx;
    __syncthreads();
    mx = red_f[0];
#pragma unroll
    for (int i = 1; i < TK_THREADS / 32; ++i) mx = fmaxf(mx, red_f[i]);
    float se = 0.f;
    for (int c = threadIdx.x; c < C; c += TK_THREADS) se += expf(tk_mean[c] - mx);
    se = warp_sum(se);
    __syncthreads();
    if (lane == 0) red_f[warp] = se;
    __syncthreads();
    se = red_f[0];
#pragma unroll
    for (int i = 1; i < TK_THREADS / 32; ++i) se += red_f[i];
    const float inv = 1.0f / se;
    for (int c = threadIdx.x; c < C; c += TK_THREADS) probs[(long long)b * C + c] = expf(tk_mean[c] - mx) * inv;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int rank = 0;
#pragma unroll
    for (int i = 0; i < TK_THREADS / 32; ++i) rank += red_i[i];
    if (!lab_ok || ml != ml) rank = C;             // label out of range or NaN score: a miss for every k
    const int kk[4] = {ks.x, ks.y, ks.z, ks.w};
    for (int i = 0; i < n_k; ++i)
      if (rank < kk[i]) atomicAdd(hits + i, 1ull);
    if (b == 0) atomicAdd(samples, (unsigned long long)B);
  }
}
}  // namespace vt

extern "C" int vt_topk_hits(const vt_topk_hits_params* p, void* stream) {
  using namespace vt;
  VT_REQUIRE(p && p->logits && p->labels && p->hits && p->samples, "vt_topk_hits: null pointer");
  VT_REQUIRE(p->B > 0 && p->V > 0 && p->C > 0, "vt_topk_hits: bad shape B=%d V=%d C=%d", p->B, p->V, p->C);
  VT_REQUIRE(p->C <= 12000, "vt_topk_hits: C=%d classes unsupported (<= 12000)", p->C);   // the means fit 48 KiB of shared memory
  VT_REQUIRE(p->n_k >= 0 && p->n_k <= 4, "vt_topk_hits: n_k=%d (0..4)", p->n_k);
  VT_REQUIRE(((reinterpret_cast<uintptr_t>(p->hits) | reinterpret_cast<uintptr_t>(p->samples)) & 7) == 0,
             "vt_topk_hits: counters must be 8-byte aligned");
  const int4 ks = make_int4(p->k[0], p->k[1], p->k[2], p->k[3]);
  topk_hits_kernel<<<p->B, TK_THREADS, p->C * sizeof(float), static_cast<cudaStream_t>(stream)>>>(
      p->logits, p->labels, p->probs, reinterpret_cast<unsigned long long*>(p->hits),
      reinterpret_cast<unsigned long long*>(p->samples), p->B, p->V, p->C, ks, p->n_k);
  return check_launch("topk_hits_kernel");
}

// ------------------------------------------------------------------------------------------------
// cls rows of the divided space-time blocks: dst[b, :] = src[b, :] + scale * sum_t extra[b, t, :]
// (extra == NULL: plain row copy).  One launch for what autograd spells as mean / sum + add + strided copy
// (transformer.py:282-283 cls passthrough of the temporal block, :371-377 mean over the per-frame cls replicas).
// ------------------------------------------------------------------------------------------------
namespace vt {
__global__ void cls_rows_kernel(const float* __restrict__ src, long long src_stride, const float* __restrict__ extra,
                                long long extra_bs, int T, float scale, float* __restrict__ dst, long long dst_stride, int B, int D4) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B * D4; i += gridDim.x * blockDim.x) {
    const int b = i / D4, j = i - b * D4;
    float4 v = reinterpret_cast<const float4*>(src + (long long)b * src_stride)[j];
    if (extra) {
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int t = 0; t < T; ++t) {
        const float4 e = reinterpret_cast<const float4*>(extra + (long long)b * extra_bs + (long long)t * D4 * 4)[j];
        a.x += e.x; a.y += e.y; a.z += e.z; a.w += e.w;
      }
      v.x = fmaf(scale, a.x, v.x); v.y = fmaf(scale, a.y, v.y); v.z = fmaf(scale, a.z, v.z); v.w = fmaf(scale, a.w, v.w);
    }
    reinterpret_cast<float4*>(dst + (long long)b * dst_stride)[j] = v;
  }
}
}  // namespace vt

extern "C" int vt_cls_rows(const vt_cls_rows_params* p, void* stream) {
  using namespace vt;
  VT_REQUIRE(p && p->src && p->dst && p->B > 0 && p->D > 0, "vt_cls_rows: bad params");
  VT_REQUIRE(p->D % 4 == 0 && p->src_stride % 4 == 0 && p->dst_stride % 4 == 0 && (!p->extra || (p->extra_bs % 4 == 0 && p->T > 0)),
             "vt_cls_rows: D and strides must be multiples of 4");
  VT_REQUIRE(((reinterpret_cast<uintptr_t>(p->src) | reinterpret_cast<uintptr_t>(p->dst) | reinterpret_cast<uintptr_t>(p->extra)) & 15) == 0,
             "vt_cls_rows: pointers must be 16-byte aligned");
  const int n = p->B * (p->D / 4);
  int blocks = (n + 255) / 256;
  if (blocks > 1024) blocks = 1024;
  cls_rows_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(p->src, p->src_stride, p->extra, p->extra_bs, p->T, p->scale,
                                                                        p->dst, p->dst_stride, p->B, p->D / 4);
  return check_launch("cls_rows_kernel");
}

