// Softmax attention core on packed qkv (bf16 [Bp, N, 3, H, 64]) — generic warp-primitive kernels.
// One CTA per (batch', head); Q/K/V/dO rows live in shared memory with a 33-word row pitch so that both
// "lane = key/query index" and "lane = feature pair" access patterns are bank-conflict free.
// Used for the temporal pass of ViViT (N = 9), the probability output at N <= 256 and the other N <= 32; N > 32 runs on
// the tensor-core kernels (vt_attention_mma.cu), N = 8 on the warp-per-problem kernel (vt_attention_small.cu).
#include "vt_attention_mma.cuh"

namespace vt {

constexpr int AT_WARPS = 8;
constexpr int AT_THREADS = AT_WARPS * 32;
constexpr int HD = 64;
constexpr int PITCH = 33;      // 32 bf16x2 words + 1 pad
constexpr int MAX_N = 256;

__device__ __forceinline__ void load_rows_to_smem(uint32_t* dst, const __nv_bfloat16* base, long long row_stride, int N) {
  // rows of 64 bf16 (128 B) -> dst[row][PITCH] words
  for (int idx = threadIdx.x; idx < N * 8; idx += AT_THREADS) {
    const int row = idx >> 3, c = idx & 7;
    const uint4 v = *reinterpret_cast<const uint4*>(base + (long long)row * row_stride + c * 8);
    uint32_t* d = dst + row * PITCH + c * 4;
    d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
  }
}

__global__ void __launch_bounds__(AT_THREADS)
attn_fwd_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ ctx, float* __restrict__ lse,
                float* __restrict__ probs, int N, int H, float scale) {
  extern __shared__ uint32_t sm[];
  const int npad = (N + 31) & ~31;
  uint32_t* Ks = sm;
  uint32_t* Vs = Ks + N * PITCH;
  float* Ps = reinterpret_cast<float*>(Vs + N * PITCH);  // [AT_WARPS][npad]
  const int bh = blockIdx.x, bp = bh / H, h = bh - bp * H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long rs = 3LL * H * HD;  // qkv row stride (elements)
  const __nv_bfloat16* qbase = qkv + (long long)bp * N * rs + h * HD;
  load_rows_to_smem(Ks, qbase + (long long)H * HD, rs, N);
  load_rows_to_smem(Vs, qbase + 2LL * H * HD, rs, N);
  __syncthreads();
  float* P = Ps + warp * npad;
  for (int i = warp; i < N; i += AT_WARPS) {
    const uint32_t* qrow = reinterpret_cast<const uint32_t*>(qbase + (long long)i * rs);
    float s[MAX_N / 32];
#pragma unroll
    for (int jj = 0; jj < MAX_N / 32; ++jj) s[jj] = 0.f;
#pragma unroll 4
    for (int w = 0; w < 32; ++w) {
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
    float mx = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < MAX_N / 32; ++jj) {
      const int j = lane + 32 * jj;
      s[jj] = (j < N) ? s[jj] * scale : -INFINITY;
      mx = fmaxf(mx, s[jj]);
    }
    mx = warp_max(mx);
    float l = 0.f;
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
    if (lane == 0 && lse) lse[(long long)bh * N + i] = mx + __logf(l);
    __syncwarp();
    float o0 = 0.f, o1 = 0.f;
    for (int j = 0; j < N; ++j) {
      const float p = P[j];
      const float2 v = unpack_bf16x2(Vs[j * PITCH + lane]);
      o0 = fmaf(p, v.x, o0);
      o1 = fmaf(p, v.y, o1);
    }
    reinterpret_cast<uint32_t*>(ctx + ((long long)bp * N + i) * H * HD + h * HD)[lane] = pack_bf16x2(o0, o1);
    if (probs) {
      float* pr = probs + ((long long)bh * N + i) * N;
      for (int j = lane; j < N; j += 32) pr[j] = P[j];
    }
    __syncwarp();
  }
}

__global__ void __launch_bounds__(AT_THREADS)
attn_bwd_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ ctx,
                const __nv_bfloat16* __restrict__ dctx, const float* __restrict__ lse, __nv_bfloat16* __restrict__ dqkv,
                int N, int H, float scale) {
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
  load_rows_to_smem(Qs, qbase, rs, N);
  load_rows_to_smem(Ks, qbase + cs, rs, N);
  load_rows_to_smem(Vs, qbase + 2 * cs, rs, N);
  load_rows_to_smem(Ds, dbase, cs, N);
  for (int i = warp; i < N; i += AT_WARPS) {
    const float2 o = unpack_bf16x2(reinterpret_cast<const uint32_t*>(obase + (long long)i * cs)[lane]);
    const float2 d = unpack_bf16x2(reinterpret_cast<const uint32_t*>(dbase + (long long)i * cs)[lane]);
    const float t = warp_sum(o.x * d.x + o.y * d.y);
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
    for (int w = 0; w < 32; ++w) {
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
    float a0 = 0.f, a1 = 0.f;
    for (int j = 0; j < N; ++j) {
      const float ds = A[j];
      const float2 k = unpack_bf16x2(Ks[j * PITCH + lane]);
      a0 = fmaf(ds, k.x, a0);
      a1 = fmaf(ds, k.y, a1);
    }
    reinterpret_cast<uint32_t*>(dq_base + (long long)i * rs)[lane] = pack_bf16x2(a0, a1);
    __syncwarp();
  }

  // pass B: one warp per key row -> dK, dV
  for (int j = warp; j < N; j += AT_WARPS) {
    float s[MAX_N / 32], dp[MAX_N / 32];
#pragma unroll
    for (int ii = 0; ii < MAX_N / 32; ++ii) { s[ii] = 0.f; dp[ii] = 0.f; }
#pragma unroll 4
    for (int w = 0; w < 32; ++w) {
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
    float k0 = 0.f, k1 = 0.f, v0 = 0.f, v1 = 0.f;
    for (int i = 0; i < N; ++i) {
      const float ds = A[i], p = Bv[i];
      const float2 q = unpack_bf16x2(Qs[i * PITCH + lane]);
      const float2 g = unpack_bf16x2(Ds[i * PITCH + lane]);
      k0 = fmaf(ds, q.x, k0); k1 = fmaf(ds, q.y, k1);
      v0 = fmaf(p, g.x, v0);  v1 = fmaf(p, g.y, v1);
    }
    reinterpret_cast<uint32_t*>(dq_base + (long long)j * rs + cs)[lane] = pack_bf16x2(k0, k1);
    reinterpret_cast<uint32_t*>(dq_base + (long long)j * rs + 2 * cs)[lane] = pack_bf16x2(v0, v1);
    __syncwarp();
  }
}

int attn8_fwd_launch(const vt_attn_fwd_params* p, cudaStream_t st);
int attn8_bwd_launch(const vt_attn_bwd_params* p, cudaStream_t st);
int attn_probs_launch(const void* qkv, float* probs, int Bp, int N, int H, float scale, cudaStream_t st);

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

// packed qkv [Bp, N, 3, H, 64] / ctx [Bp, N, H, 64] as strided q / k / v / o operands of the tensor-core kernels
static MmaAttn packed_operands(const void* qkv, const void* ctx, const float* lse, int Bp, int N, int H, float scale) {
  MmaAttn a{};
  const long long rs = 3LL * H * HD, cs = (long long)H * HD;
  const __nv_bfloat16* q = static_cast<const __nv_bfloat16*>(qkv);
  a.q = q; a.k = q + cs; a.v = q + 2 * cs;
  a.q_bs = a.k_bs = a.v_bs = (long long)N * rs;
  a.q_hs = a.k_hs = a.v_hs = HD;
  a.q_rs = a.k_rs = a.v_rs = rs;
  a.o = static_cast<const __nv_bfloat16*>(ctx);
  a.o_bs = (long long)N * cs; a.o_hs = HD; a.o_rs = cs;
  a.lse = const_cast<float*>(lse);
  a.H = H; a.Nq = N; a.Nk = N; a.scale = scale;
  (void)Bp;
  return a;
}

// the tensor-core kernels that own a whole problem per CTA where they cover N; VT_ATTN_WHOLE=0 keeps the 64-row tiles
static bool use_whole(const MmaAttn& a) { return feature_on("VT_ATTN_WHOLE", true) && attn_whole_ok(a, HD); }

}  // namespace vt

using namespace vt;

extern "C" int vt_attn_fwd(const vt_attn_fwd_params* p, void* stream) {
  VT_REQUIRE(p && p->qkv && p->ctx, "vt_attn_fwd: null pointer");   // lse may be NULL (not written)
  VT_REQUIRE(p->hd == HD, "vt_attn_fwd: head dim %d unsupported (64 only)", p->hd);
  VT_REQUIRE(p->N >= 1, "vt_attn_fwd: N=%d unsupported", p->N);
  VT_REQUIRE(p->Bp > 0 && p->H > 0, "vt_attn_fwd: bad Bp/H");
  const int impl = pick_impl(p->impl, p->N, p->probs != nullptr);
  if (impl == VT_ATTN_TCGEN05) {
    VT_REQUIRE((((uintptr_t)p->qkv | (uintptr_t)p->ctx) & 15) == 0, "vt_attn_fwd: qkv / ctx must be 16-byte aligned");
    if (p->probs) {   // the tensor-core kernels write no probabilities: the row-tile softmax kernel does
      const int rc = attn_probs_launch(p->qkv, p->probs, p->Bp, p->N, p->H, p->scale, static_cast<cudaStream_t>(stream));
      if (rc) return rc;
    }
    MmaAttn a = packed_operands(p->qkv, p->ctx, p->lse, p->Bp, p->N, p->H, p->scale);
    a.o_out = static_cast<__nv_bfloat16*>(p->ctx);
    if (use_whole(a)) return attn_whole_fwd(a, p->Bp, static_cast<cudaStream_t>(stream));
    return attn_mma_fwd(a, p->Bp, HD, static_cast<cudaStream_t>(stream));
  }
  if (impl == VT_ATTN_WARP8) {
    VT_REQUIRE(p->probs == nullptr && p->N == 8, "vt_attn_fwd: warp8 kernel needs N == 8 and no probs output");
    return attn8_fwd_launch(p, static_cast<cudaStream_t>(stream));
  }
  VT_REQUIRE(p->N <= MAX_N, "vt_attn_fwd: N=%d unsupported by the generic kernel (1..%d)", p->N, MAX_N);
  const int npad = (p->N + 31) & ~31;
  const int smem = (2 * p->N * PITCH + AT_WARPS * npad) * 4;
  static int max_set = 0;
  if (smem > 48 * 1024 && smem > max_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    VT_REQUIRE(e == cudaSuccess, "vt_attn_fwd: smem attribute: %s", cudaGetErrorString(e));
    max_set = 100 * 1024;
  }
  attn_fwd_kernel<<<p->Bp * p->H, AT_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(p->qkv), static_cast<__nv_bfloat16*>(p->ctx), p->lse, p->probs, p->N, p->H, p->scale);
  return check_launch("attn_fwd_kernel");
}

extern "C" int vt_attn_bwd(const vt_attn_bwd_params* p, void* stream) {
  VT_REQUIRE(p && p->qkv && p->ctx && p->dctx && p->lse && p->dqkv, "vt_attn_bwd: null pointer");
  VT_REQUIRE(p->hd == HD, "vt_attn_bwd: head dim %d unsupported (64 only)", p->hd);
  VT_REQUIRE(p->N >= 1, "vt_attn_bwd: N=%d unsupported", p->N);
  const int impl = pick_impl(p->impl, p->N, false);
  if (impl == VT_ATTN_TCGEN05) {
    VT_REQUIRE((((uintptr_t)p->qkv | (uintptr_t)p->ctx | (uintptr_t)p->dctx | (uintptr_t)p->dqkv) & 15) == 0,
               "vt_attn_bwd: qkv / ctx / dctx / dqkv must be 16-byte aligned");
    MmaAttn a = packed_operands(p->qkv, p->ctx, p->lse, p->Bp, p->N, p->H, p->scale);
    a.dout = static_cast<const __nv_bfloat16*>(p->dctx);
    __nv_bfloat16* d = static_cast<__nv_bfloat16*>(p->dqkv);
    const long long cs = (long long)p->H * HD;
    a.dq = d; a.dk16 = d + cs; a.dv16 = d + 2 * cs;
    a.dq_bs = a.dk_bs = a.dv_bs = a.q_bs;
    a.dq_hs = a.dk_hs = a.dv_hs = HD;
    a.dq_rs = a.dk_rs = a.dv_rs = a.q_rs;
    if (use_whole(a)) return attn_whole_bwd(a, p->Bp, static_cast<cudaStream_t>(stream));
    return attn_mma_bwd(a, p->Bp, HD, static_cast<cudaStream_t>(stream));
  }
  if (impl == VT_ATTN_WARP8) {
    VT_REQUIRE(p->N == 8, "vt_attn_bwd: warp8 kernel needs N == 8");
    return attn8_bwd_launch(p, static_cast<cudaStream_t>(stream));
  }
  VT_REQUIRE(p->N <= MAX_N, "vt_attn_bwd: N=%d unsupported by the generic kernel (1..%d)", p->N, MAX_N);
  const int npad = (p->N + 31) & ~31;
  const int smem = (4 * p->N * PITCH + 2 * npad + 2 * AT_WARPS * npad) * 4;
  static int max_set = 0;
  if (smem > 48 * 1024 && smem > max_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    VT_REQUIRE(e == cudaSuccess, "vt_attn_bwd: smem attribute: %s", cudaGetErrorString(e));
    max_set = 200 * 1024;
  }
  attn_bwd_kernel<<<p->Bp * p->H, AT_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(p->qkv), static_cast<const __nv_bfloat16*>(p->ctx),
      static_cast<const __nv_bfloat16*>(p->dctx), p->lse, static_cast<__nv_bfloat16*>(p->dqkv), p->N, p->H, p->scale);
  return check_launch("attn_bwd_kernel");
}
