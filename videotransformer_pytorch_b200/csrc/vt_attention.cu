// Softmax attention core on packed qkv (bf16 [Bp, N, 3, H, hd], hd = 32, 64, 96 or 128) — generic warp-primitive kernels.
// One CTA per (batch', head); Q/K/V/dO rows live in shared memory with a pitch of hd / 2 + 1 words (odd: 17, 33, 49, 65)
// so that both "lane = key/query index" and "lane = feature pair" access patterns are bank-conflict free.  A lane owns the
// feature pairs lane, lane + 32, .. of a row (at hd 32, and for the second pair at hd 96, lanes 16..31 have none).
// Used for the temporal pass of ViViT (N = 9), the probability output at N <= 256 and the other N <= 32; N > 32 runs on
// the tensor-core kernels (vt_attention_mma.cu), N = 8 on the warp-per-problem kernel (vt_attention_small.cu).
#include "vt_attention_mma.cuh"
#include "../../include/vt_attn_maps.h"

namespace vt {

constexpr int AT_WARPS = 8;
constexpr int AT_THREADS = AT_WARPS * 32;
constexpr int MAX_N = 256;
constexpr int SMEM_OPTIN = 227 * 1024;   // the largest dynamic shared memory a CTA may opt into on sm_90

// rows of HD bf16 -> dst[row][HD / 2 + 1] words
template <int HD>
__device__ __forceinline__ void load_rows_to_smem(uint32_t* dst, const __nv_bfloat16* base, long long row_stride, int N) {
  constexpr int CPR = HD / 8, PITCH = HD / 2 + 1;   // 16-byte chunks per row
  for (int idx = threadIdx.x; idx < N * CPR; idx += AT_THREADS) {
    const int row = div_pos<CPR>(idx), c = mod_pos<CPR>(idx);
    const uint4 v = *reinterpret_cast<const uint4*>(base + (long long)row * row_stride + c * 8);
    uint32_t* d = dst + row * PITCH + c * 4;
    d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
  }
}

// Softmax probabilities of one query row (qrow: its hd / 2 words of q in global memory) against the N keys staged in
// Ks, written by one warp to P[0, N) (shared or global memory); the row max and the sum of exponentials come back in
// mx / l (lse = mx + log l).  The probabilities of the generic kernel are defined here once: attn_fwd_kernel's rows and
// the cls-row kernel both call it.
template <int HD>
__device__ __forceinline__ void generic_probs_row(const uint32_t* qrow, const uint32_t* Ks, int N, float scale, int lane,
                                                  float* P, float& mx, float& l) {
  constexpr int NW = HD / 2, PITCH = NW + 1;
  float s[MAX_N / 32];
#pragma unroll
  for (int jj = 0; jj < MAX_N / 32; ++jj) s[jj] = 0.f;
#pragma unroll 4
  for (int w = 0; w < NW; ++w) {
    const float2 q = unpack_bf16x2(__ldg(qrow + w));
#pragma unroll
    for (int jj = 0; jj < MAX_N / 32; ++jj) {
      const int j = lane + 32 * jj;
      if (j < N) {
        const float2 k = unpack_bf16x2(Ks[j * PITCH + w]);
        s[jj] = fmaf(q.x, k.x, fmaf(q.y, k.y, s[jj]));
      }
    }
  }
  mx = -INFINITY;
#pragma unroll
  for (int jj = 0; jj < MAX_N / 32; ++jj) {
    const int j = lane + 32 * jj;
    s[jj] = (j < N) ? s[jj] * scale : -INFINITY;
    mx = fmaxf(mx, s[jj]);
  }
  mx = warp_max(mx);
  l = 0.f;
#pragma unroll
  for (int jj = 0; jj < MAX_N / 32; ++jj) {
    const int j = lane + 32 * jj;
    s[jj] = (j < N) ? __expf(s[jj] - mx) : 0.f;
    l += s[jj];
  }
  l = warp_sum(l);
  const float inv = 1.0f / l;
#pragma unroll
  for (int jj = 0; jj < MAX_N / 32; ++jj) {
    const int j = lane + 32 * jj;
    if (j < N) P[j] = s[jj] * inv;
  }
}

template <int HD>
__global__ void __launch_bounds__(AT_THREADS)
attn_fwd_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ ctx, float* __restrict__ lse,
                float* __restrict__ probs, int N, int H, float scale) {
  constexpr int NW = HD / 2, PITCH = NW + 1, WPL = (NW + 31) / 32;   // words per row, pitch, words per lane
  extern __shared__ uint32_t sm[];
  const int npad = (N + 31) & ~31;
  uint32_t* Ks = sm;
  uint32_t* Vs = Ks + N * PITCH;
  float* Ps = reinterpret_cast<float*>(Vs + N * PITCH);  // [AT_WARPS][npad]
  const int bh = blockIdx.x, bp = bh / H, h = bh - bp * H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long rs = 3LL * H * HD;  // qkv row stride (elements)
  const __nv_bfloat16* qbase = qkv + (long long)bp * N * rs + h * HD;
  load_rows_to_smem<HD>(Ks, qbase + (long long)H * HD, rs, N);
  load_rows_to_smem<HD>(Vs, qbase + 2LL * H * HD, rs, N);
  __syncthreads();
  float* P = Ps + warp * npad;
  for (int i = warp; i < N; i += AT_WARPS) {
    const uint32_t* qrow = reinterpret_cast<const uint32_t*>(qbase + (long long)i * rs);
    float mx, l;
    generic_probs_row<HD>(qrow, Ks, N, scale, lane, P, mx, l);
    if (lane == 0 && lse) lse[(long long)bh * N + i] = mx + __logf(l);
    __syncwarp();
    float o[WPL][2];
#pragma unroll
    for (int u = 0; u < WPL; ++u) { o[u][0] = 0.f; o[u][1] = 0.f; }
    for (int j = 0; j < N; ++j) {
      const float p = P[j];
#pragma unroll
      for (int u = 0; u < WPL; ++u) {
        if (lane + 32 * u < NW) {
          const float2 v = unpack_bf16x2(Vs[j * PITCH + lane + 32 * u]);
          o[u][0] = fmaf(p, v.x, o[u][0]);
          o[u][1] = fmaf(p, v.y, o[u][1]);
        }
      }
    }
    uint32_t* crow = reinterpret_cast<uint32_t*>(ctx + ((long long)bp * N + i) * H * HD + h * HD);
#pragma unroll
    for (int u = 0; u < WPL; ++u)
      if (lane + 32 * u < NW) crow[lane + 32 * u] = pack_bf16x2(o[u][0], o[u][1]);
    if (probs) {
      float* pr = probs + ((long long)bh * N + i) * N;
      for (int j = lane; j < N; j += 32) pr[j] = P[j];
    }
    __syncwarp();
  }
}

// Query row 0 (the cls token) of the generic kernel's probabilities: one CTA per (batch', head) stages K and one warp
// writes the row straight to out[bh, 0, N).
template <int HD>
__global__ void __launch_bounds__(AT_THREADS)
attn_cls_probs_kernel(const __nv_bfloat16* __restrict__ qkv, float* __restrict__ out, int N, int H, float scale) {
  extern __shared__ uint32_t sm[];
  const int bh = blockIdx.x, bp = bh / H, h = bh - bp * H;
  const long long rs = 3LL * H * HD;
  const __nv_bfloat16* qbase = qkv + (long long)bp * N * rs + h * HD;
  load_rows_to_smem<HD>(sm, qbase + (long long)H * HD, rs, N);
  __syncthreads();
  if (threadIdx.x < 32) {
    float mx, l;
    generic_probs_row<HD>(reinterpret_cast<const uint32_t*>(qbase), sm, N, scale, threadIdx.x, out + (long long)bh * N, mx, l);
  }
}

template <int HD>
__global__ void __launch_bounds__(AT_THREADS)
attn_bwd_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ ctx,
                const __nv_bfloat16* __restrict__ dctx, const float* __restrict__ lse, __nv_bfloat16* __restrict__ dqkv,
                int N, int H, float scale) {
  constexpr int NW = HD / 2, PITCH = NW + 1, WPL = (NW + 31) / 32;
  extern __shared__ uint32_t sm[];
  const int npad = (N + 31) & ~31;
  uint32_t* Qs = sm;
  uint32_t* Ks = Qs + N * PITCH;
  uint32_t* Vs = Ks + N * PITCH;
  uint32_t* Ds = Vs + N * PITCH;
  float* lse_s = reinterpret_cast<float*>(Ds + N * PITCH);
  float* del_s = lse_s + npad;
  float* rowA = del_s + npad;            // [AT_WARPS][npad]
  float* rowB = rowA + AT_WARPS * npad;  // [AT_WARPS][npad]
  const int bh = blockIdx.x, bp = bh / H, h = bh - bp * H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long rs = 3LL * H * HD;
  const long long cs = (long long)H * HD;
  const __nv_bfloat16* qbase = qkv + (long long)bp * N * rs + h * HD;
  const __nv_bfloat16* obase = ctx + (long long)bp * N * cs + h * HD;
  const __nv_bfloat16* dbase = dctx + (long long)bp * N * cs + h * HD;
  load_rows_to_smem<HD>(Qs, qbase, rs, N);
  load_rows_to_smem<HD>(Ks, qbase + cs, rs, N);
  load_rows_to_smem<HD>(Vs, qbase + 2 * cs, rs, N);
  load_rows_to_smem<HD>(Ds, dbase, cs, N);
  for (int i = warp; i < N; i += AT_WARPS) {
    float od = 0.f;
#pragma unroll
    for (int u = 0; u < WPL; ++u) {
      if (lane + 32 * u < NW) {
        const float2 o = unpack_bf16x2(reinterpret_cast<const uint32_t*>(obase + (long long)i * cs)[lane + 32 * u]);
        const float2 d = unpack_bf16x2(reinterpret_cast<const uint32_t*>(dbase + (long long)i * cs)[lane + 32 * u]);
        od = u == 0 ? o.x * d.x + o.y * d.y : od + (o.x * d.x + o.y * d.y);
      }
    }
    const float t = warp_sum(od);
    if (lane == 0) {
      del_s[i] = t;
      lse_s[i] = lse[(long long)bh * N + i];
    }
  }
  __syncthreads();
  float* A = rowA + warp * npad;
  float* Bv = rowB + warp * npad;
  __nv_bfloat16* dq_base = dqkv + (long long)bp * N * rs + h * HD;

  // pass A: one warp per query row -> dQ
  for (int i = warp; i < N; i += AT_WARPS) {
    float s[MAX_N / 32], dp[MAX_N / 32];
#pragma unroll
    for (int jj = 0; jj < MAX_N / 32; ++jj) { s[jj] = 0.f; dp[jj] = 0.f; }
#pragma unroll 4
    for (int w = 0; w < NW; ++w) {
      const float2 q = unpack_bf16x2(Qs[i * PITCH + w]);
      const float2 g = unpack_bf16x2(Ds[i * PITCH + w]);
#pragma unroll
      for (int jj = 0; jj < MAX_N / 32; ++jj) {
        const int j = lane + 32 * jj;
        if (j < N) {
          const float2 k = unpack_bf16x2(Ks[j * PITCH + w]);
          const float2 v = unpack_bf16x2(Vs[j * PITCH + w]);
          s[jj] = fmaf(q.x, k.x, fmaf(q.y, k.y, s[jj]));
          dp[jj] = fmaf(g.x, v.x, fmaf(g.y, v.y, dp[jj]));
        }
      }
    }
    const float li = lse_s[i], di = del_s[i];
#pragma unroll
    for (int jj = 0; jj < MAX_N / 32; ++jj) {
      const int j = lane + 32 * jj;
      if (j < N) {
        const float p = __expf(s[jj] * scale - li);
        A[j] = p * (dp[jj] - di) * scale;
      }
    }
    __syncwarp();
    float a[WPL][2];
#pragma unroll
    for (int u = 0; u < WPL; ++u) { a[u][0] = 0.f; a[u][1] = 0.f; }
    for (int j = 0; j < N; ++j) {
      const float ds = A[j];
#pragma unroll
      for (int u = 0; u < WPL; ++u) {
        if (lane + 32 * u < NW) {
          const float2 k = unpack_bf16x2(Ks[j * PITCH + lane + 32 * u]);
          a[u][0] = fmaf(ds, k.x, a[u][0]);
          a[u][1] = fmaf(ds, k.y, a[u][1]);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < WPL; ++u)
      if (lane + 32 * u < NW) reinterpret_cast<uint32_t*>(dq_base + (long long)i * rs)[lane + 32 * u] = pack_bf16x2(a[u][0], a[u][1]);
    __syncwarp();
  }

  // pass B: one warp per key row -> dK, dV
  for (int j = warp; j < N; j += AT_WARPS) {
    float s[MAX_N / 32], dp[MAX_N / 32];
#pragma unroll
    for (int ii = 0; ii < MAX_N / 32; ++ii) { s[ii] = 0.f; dp[ii] = 0.f; }
#pragma unroll 4
    for (int w = 0; w < NW; ++w) {
      const float2 k = unpack_bf16x2(Ks[j * PITCH + w]);
      const float2 v = unpack_bf16x2(Vs[j * PITCH + w]);
#pragma unroll
      for (int ii = 0; ii < MAX_N / 32; ++ii) {
        const int i = lane + 32 * ii;
        if (i < N) {
          const float2 q = unpack_bf16x2(Qs[i * PITCH + w]);
          const float2 g = unpack_bf16x2(Ds[i * PITCH + w]);
          s[ii] = fmaf(q.x, k.x, fmaf(q.y, k.y, s[ii]));
          dp[ii] = fmaf(g.x, v.x, fmaf(g.y, v.y, dp[ii]));
        }
      }
    }
#pragma unroll
    for (int ii = 0; ii < MAX_N / 32; ++ii) {
      const int i = lane + 32 * ii;
      if (i < N) {
        const float p = __expf(s[ii] * scale - lse_s[i]);
        A[i] = p * (dp[ii] - del_s[i]) * scale;
        Bv[i] = p;
      }
    }
    __syncwarp();
    float kk[WPL][2], vv[WPL][2];
#pragma unroll
    for (int u = 0; u < WPL; ++u) { kk[u][0] = 0.f; kk[u][1] = 0.f; vv[u][0] = 0.f; vv[u][1] = 0.f; }
    for (int i = 0; i < N; ++i) {
      const float ds = A[i], p = Bv[i];
#pragma unroll
      for (int u = 0; u < WPL; ++u) {
        if (lane + 32 * u < NW) {
          const float2 q = unpack_bf16x2(Qs[i * PITCH + lane + 32 * u]);
          const float2 g = unpack_bf16x2(Ds[i * PITCH + lane + 32 * u]);
          kk[u][0] = fmaf(ds, q.x, kk[u][0]); kk[u][1] = fmaf(ds, q.y, kk[u][1]);
          vv[u][0] = fmaf(p, g.x, vv[u][0]);  vv[u][1] = fmaf(p, g.y, vv[u][1]);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < WPL; ++u) {
      if (lane + 32 * u < NW) {
        reinterpret_cast<uint32_t*>(dq_base + (long long)j * rs + cs)[lane + 32 * u] = pack_bf16x2(kk[u][0], kk[u][1]);
        reinterpret_cast<uint32_t*>(dq_base + (long long)j * rs + 2 * cs)[lane + 32 * u] = pack_bf16x2(vv[u][0], vv[u][1]);
      }
    }
    __syncwarp();
  }
}

int attn8_fwd_launch(const vt_attn_fwd_params* p, cudaStream_t st);
int attn8_bwd_launch(const vt_attn_bwd_params* p, cudaStream_t st);
int attn_probs_launch(const void* qkv, float* probs, int Bp, int N, int H, int hd, float scale, cudaStream_t st);
int attn_cls_probs_tiled_launch(const vt_attn_cls_probs_params* p, cudaStream_t st);

// past the generic kernel's N the tensor-core kernels take every call, probabilities included (the 64-row tiles: the
// whole-problem kernels stop at N = 256)
static int pick_impl(int impl, int N, bool probs) {
  if (impl != VT_ATTN_AUTO) return impl;
  if (N > MAX_N) return VT_ATTN_TCGEN05;
  if (probs) return VT_ATTN_GENERIC;
  if (N == 8) return VT_ATTN_WARP8;
  if (N > 32) return VT_ATTN_TCGEN05;
  return VT_ATTN_GENERIC;
}

// packed qkv [Bp, N, 3, H, hd] / ctx [Bp, N, H, hd] as strided q / k / v / o operands of the tensor-core kernels
static MmaAttn packed_operands(const void* qkv, const void* ctx, const float* lse, int N, int H, int hd, float scale) {
  MmaAttn a{};
  const long long rs = 3LL * H * hd, cs = (long long)H * hd;
  const __nv_bfloat16* q = static_cast<const __nv_bfloat16*>(qkv);
  a.q = q; a.k = q + cs; a.v = q + 2 * cs;
  a.q_bs = a.k_bs = a.v_bs = (long long)N * rs;
  a.q_hs = a.k_hs = a.v_hs = hd;
  a.q_rs = a.k_rs = a.v_rs = rs;
  a.o = static_cast<const __nv_bfloat16*>(ctx);
  a.o_bs = (long long)N * cs; a.o_hs = hd; a.o_rs = cs;
  a.lse = const_cast<float*>(lse);
  a.H = H; a.Nq = N; a.Nk = N; a.scale = scale;
  return a;
}

// the tensor-core kernels that own a whole problem per CTA where they cover N (head dim 64 only); VT_ATTN_WHOLE=0 keeps
// the 64-row tiles
static bool use_whole(const MmaAttn& a, int hd) { return feature_on("VT_ATTN_WHOLE", true) && attn_whole_ok(a, hd); }

// raises `kern`'s dynamic shared-memory limit to at least `floor` bytes (and to `smem` where that is more) once a launch
// needs more than the default 48 KB; `max_set` is the limit set so far
template <class K>
static int raise_smem(K kern, int smem, int floor, int& max_set, const char* what) {
  if (smem <= 48 * 1024 || smem <= max_set) return 0;
  const int lim = smem > floor ? smem : floor;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, lim);
  VT_REQUIRE(e == cudaSuccess, "%s: smem attribute: %s", what, cudaGetErrorString(e));
  max_set = lim;
  return 0;
}

template <int HD>
static int generic_fwd(const vt_attn_fwd_params* p, cudaStream_t st) {
  const int npad = (p->N + 31) & ~31;
  const int smem = (2 * p->N * (HD / 2 + 1) + AT_WARPS * npad) * 4;
  static int max_set = 0;
  if (raise_smem(attn_fwd_kernel<HD>, smem, 100 * 1024, max_set, "vt_attn_fwd")) return 1;
  attn_fwd_kernel<HD><<<p->Bp * p->H, AT_THREADS, smem, st>>>(
      static_cast<const __nv_bfloat16*>(p->qkv), static_cast<__nv_bfloat16*>(p->ctx), p->lse, p->probs, p->N, p->H, p->scale);
  return check_launch("attn_fwd_kernel");
}

template <int HD>
static int generic_bwd(const vt_attn_bwd_params* p, cudaStream_t st) {
  const int npad = (p->N + 31) & ~31;
  const int smem = (4 * p->N * (HD / 2 + 1) + 2 * npad + 2 * AT_WARPS * npad) * 4;
  VT_REQUIRE(smem <= SMEM_OPTIN, "vt_attn_bwd: N=%d at head dim %d needs %d bytes of shared memory in the generic kernel",
             p->N, HD, smem);
  static int max_set = 0;
  if (raise_smem(attn_bwd_kernel<HD>, smem, 200 * 1024, max_set, "vt_attn_bwd")) return 1;
  attn_bwd_kernel<HD><<<p->Bp * p->H, AT_THREADS, smem, st>>>(
      static_cast<const __nv_bfloat16*>(p->qkv), static_cast<const __nv_bfloat16*>(p->ctx),
      static_cast<const __nv_bfloat16*>(p->dctx), p->lse, static_cast<__nv_bfloat16*>(p->dqkv), p->N, p->H, p->scale);
  return check_launch("attn_bwd_kernel");
}

template <int HD>
static int generic_cls_probs(const vt_attn_cls_probs_params* p, cudaStream_t st) {
  const int smem = p->N * (HD / 2 + 1) * 4;
  static int max_set = 0;
  if (raise_smem(attn_cls_probs_kernel<HD>, smem, 100 * 1024, max_set, "vt_attn_cls_probs")) return 1;
  attn_cls_probs_kernel<HD><<<p->Bp * p->H, AT_THREADS, smem, st>>>(static_cast<const __nv_bfloat16*>(p->qkv), p->probs,
                                                                   p->N, p->H, p->scale);
  return check_launch("attn_cls_probs_kernel");
}

}  // namespace vt

using namespace vt;

extern "C" int vt_attn_fwd(const vt_attn_fwd_params* p, void* stream) {
  VT_REQUIRE(p && p->qkv && p->ctx, "vt_attn_fwd: null pointer");   // lse may be NULL (not written)
  VT_REQUIRE(attn_head_dim_ok(p->hd), "vt_attn_fwd: head dim %d unsupported (32, 64, 96 or 128)", p->hd);
  VT_REQUIRE(p->N >= 1, "vt_attn_fwd: N=%d unsupported", p->N);
  VT_REQUIRE(p->Bp > 0 && p->H > 0, "vt_attn_fwd: bad Bp/H");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int impl = pick_impl(p->impl, p->N, p->probs != nullptr);
  if (impl == VT_ATTN_TCGEN05) {
    VT_REQUIRE((((uintptr_t)p->qkv | (uintptr_t)p->ctx) & 15) == 0, "vt_attn_fwd: qkv / ctx must be 16-byte aligned");
    if (p->probs) {   // the tensor-core kernels write no probabilities: the row-tile softmax kernel does
      const int rc = attn_probs_launch(p->qkv, p->probs, p->Bp, p->N, p->H, p->hd, p->scale, st);
      if (rc) return rc;
    }
    MmaAttn a = packed_operands(p->qkv, p->ctx, p->lse, p->N, p->H, p->hd, p->scale);
    a.o_out = static_cast<__nv_bfloat16*>(p->ctx);
    if (use_whole(a, p->hd)) return attn_whole_fwd(a, p->Bp, st);
    return attn_mma_fwd(a, p->Bp, p->hd, st);
  }
  if (impl == VT_ATTN_WARP8) {
    VT_REQUIRE(p->probs == nullptr && p->N == 8, "vt_attn_fwd: warp8 kernel needs N == 8 and no probs output");
    return attn8_fwd_launch(p, st);
  }
  VT_REQUIRE(p->N <= MAX_N, "vt_attn_fwd: N=%d unsupported by the generic kernel (1..%d)", p->N, MAX_N);
  return with_head_dim(p->hd, [&](auto hd) { return generic_fwd<hd.value>(p, st); });
}

extern "C" int vt_attn_bwd(const vt_attn_bwd_params* p, void* stream) {
  VT_REQUIRE(p && p->qkv && p->ctx && p->dctx && p->lse && p->dqkv, "vt_attn_bwd: null pointer");
  VT_REQUIRE(attn_head_dim_ok(p->hd), "vt_attn_bwd: head dim %d unsupported (32, 64, 96 or 128)", p->hd);
  VT_REQUIRE(p->N >= 1, "vt_attn_bwd: N=%d unsupported", p->N);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int impl = pick_impl(p->impl, p->N, false);
  if (impl == VT_ATTN_TCGEN05) {
    VT_REQUIRE((((uintptr_t)p->qkv | (uintptr_t)p->ctx | (uintptr_t)p->dctx | (uintptr_t)p->dqkv) & 15) == 0,
               "vt_attn_bwd: qkv / ctx / dctx / dqkv must be 16-byte aligned");
    MmaAttn a = packed_operands(p->qkv, p->ctx, p->lse, p->N, p->H, p->hd, p->scale);
    a.dout = static_cast<const __nv_bfloat16*>(p->dctx);
    __nv_bfloat16* d = static_cast<__nv_bfloat16*>(p->dqkv);
    const long long cs = (long long)p->H * p->hd;
    a.dq = d; a.dk16 = d + cs; a.dv16 = d + 2 * cs;
    a.dq_bs = a.dk_bs = a.dv_bs = a.q_bs;
    a.dq_hs = a.dk_hs = a.dv_hs = p->hd;
    a.dq_rs = a.dk_rs = a.dv_rs = a.q_rs;
    if (use_whole(a, p->hd)) return attn_whole_bwd(a, p->Bp, st);
    return attn_mma_bwd(a, p->Bp, p->hd, st);
  }
  if (impl == VT_ATTN_WARP8) {
    VT_REQUIRE(p->N == 8, "vt_attn_bwd: warp8 kernel needs N == 8");
    return attn8_bwd_launch(p, st);
  }
  VT_REQUIRE(p->N <= MAX_N, "vt_attn_bwd: N=%d unsupported by the generic kernel (1..%d)", p->N, MAX_N);
  return with_head_dim(p->hd, [&](auto hd) { return generic_bwd<hd.value>(p, st); });
}

// Row 0 of vt_attn_fwd's probs output from the same device code as the route vt_attn_fwd takes at this N: the generic
// kernel's row function up to MAX_N, the row-tile softmax kernel's score and softmax functions (vt_head.cu) past it.
extern "C" int vt_attn_cls_probs(const vt_attn_cls_probs_params* p, void* stream) {
  VT_REQUIRE(p && p->qkv && p->probs, "vt_attn_cls_probs: null pointer");
  VT_REQUIRE(attn_head_dim_ok(p->hd), "vt_attn_cls_probs: head dim %d unsupported (32, 64, 96 or 128)", p->hd);
  VT_REQUIRE(p->N >= 1, "vt_attn_cls_probs: N=%d unsupported", p->N);
  VT_REQUIRE(p->Bp > 0 && p->H > 0 && (long long)p->Bp * p->H <= 0x7fffffffLL, "vt_attn_cls_probs: bad Bp=%d / H=%d",
             p->Bp, p->H);
  VT_REQUIRE(((uintptr_t)p->qkv & 15) == 0, "vt_attn_cls_probs: qkv must be 16-byte aligned");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (p->N > MAX_N) return attn_cls_probs_tiled_launch(p, st);
  return with_head_dim(p->hd, [&](auto hd) { return generic_cls_probs<hd.value>(p, st); });
}
