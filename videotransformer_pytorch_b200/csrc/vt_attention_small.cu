// Temporal attention of the divided space-time block: 8 frames x 8 frames per (sample, patch, head) —
// 18 816 independent 8x8x64 problems per layer at batch 8.  0.1 % of the FLOPs, so the kernel is built
// to be bandwidth/latency lean instead of tensor-core shaped: one warp per problem, Q/K/V (and dO) rows
// staged in shared memory (33-word pitch, conflict-free), lane (i, g) = query row i = lane/4 and quarter
// g = lane%4:  scores for keys {2g, 2g+1} (full 64-dim dots), softmax across the 4 lanes of a row with two
// shuffles, then the lane owns features [16g, 16g+16) of its output row.  Backward uses the same mapping
// (dQ rows, then dK/dV rows) and recomputes P from the saved log-sum-exp.
#include "vt_common.cuh"

namespace vt {

constexpr int SM_N = 8;
constexpr int SM_HD = 64;
constexpr int SM_PITCH = 33;
constexpr int SM_WARPS = 8;

// software pipelining: the next problem's rows are fetched into registers while the current one is computed
struct Rows8 { uint4 v[2]; };
__device__ __forceinline__ Rows8 fetch_rows8(const __nv_bfloat16* base, long long row_stride, int lane) {
  Rows8 r;
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const int row = (lane >> 3) + 4 * it, c = lane & 7;
    r.v[it] = *reinterpret_cast<const uint4*>(base + (long long)row * row_stride + c * 8);
  }
  return r;
}
__device__ __forceinline__ void put_rows8(uint32_t* dst, const Rows8& r, int lane) {
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const int row = (lane >> 3) + 4 * it, c = lane & 7;
    uint32_t* d = dst + row * SM_PITCH + c * 4;
    d[0] = r.v[it].x; d[1] = r.v[it].y; d[2] = r.v[it].z; d[3] = r.v[it].w;
  }
}

__global__ void __launch_bounds__(SM_WARPS * 32)
attn8_fwd_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ ctx, float* __restrict__ lse,
                 int nprob, int H, float scale) {
  __shared__ uint32_t sh[SM_WARPS][3][SM_N * SM_PITCH];
  __shared__ float shp[SM_WARPS][SM_N * 9];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t* Qs = sh[warp][0];
  uint32_t* Ks = sh[warp][1];
  uint32_t* Vs = sh[warp][2];
  float* Ps = shp[warp];
  const long long rs = 3LL * H * SM_HD, cs = (long long)H * SM_HD;
  const int i = lane >> 2, g = lane & 3;
  const int pstep = gridDim.x * SM_WARPS;
  int prob = blockIdx.x * SM_WARPS + warp;
  Rows8 rq, rk, rv;
  if (prob < nprob) {
    const __nv_bfloat16* b0 = qkv + (long long)(prob / H) * SM_N * rs + (prob % H) * SM_HD;
    rq = fetch_rows8(b0, rs, lane); rk = fetch_rows8(b0 + cs, rs, lane); rv = fetch_rows8(b0 + 2 * cs, rs, lane);
  }
  for (; prob < nprob; prob += pstep) {
    const int bp = prob / H, h = prob - bp * H;
    put_rows8(Qs, rq, lane); put_rows8(Ks, rk, lane); put_rows8(Vs, rv, lane);
    __syncwarp();
    if (prob + pstep < nprob) {
      const int np = prob + pstep;
      const __nv_bfloat16* b1 = qkv + (long long)(np / H) * SM_N * rs + (np % H) * SM_HD;
      rq = fetch_rows8(b1, rs, lane); rk = fetch_rows8(b1 + cs, rs, lane); rv = fetch_rows8(b1 + 2 * cs, rs, lane);
    }
    float s0 = 0.f, s1 = 0.f;
#pragma unroll 8
    for (int w = 0; w < 32; ++w) {
      const float2 q = unpack_bf16x2(Qs[i * SM_PITCH + w]);
      const float2 k0 = unpack_bf16x2(Ks[(2 * g) * SM_PITCH + w]);
      const float2 k1 = unpack_bf16x2(Ks[(2 * g + 1) * SM_PITCH + w]);
      s0 = fmaf(q.x, k0.x, fmaf(q.y, k0.y, s0));
      s1 = fmaf(q.x, k1.x, fmaf(q.y, k1.y, s1));
    }
    s0 *= scale; s1 *= scale;
    float m = fmaxf(s0, s1);
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    const float e0 = __expf(s0 - m), e1 = __expf(s1 - m);
    float l = e0 + e1;
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.0f / l;
    Ps[i * 9 + 2 * g] = e0 * inv;
    Ps[i * 9 + 2 * g + 1] = e1 * inv;
    if (g == 0 && lse) lse[(long long)prob * SM_N + i] = m + __logf(l);
    __syncwarp();
    float acc[16];
#pragma unroll
    for (int d = 0; d < 16; ++d) acc[d] = 0.f;
#pragma unroll
    for (int j = 0; j < SM_N; ++j) {
      const float p = Ps[i * 9 + j];
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        const float2 v = unpack_bf16x2(Vs[j * SM_PITCH + g * 8 + w]);
        acc[2 * w] = fmaf(p, v.x, acc[2 * w]);
        acc[2 * w + 1] = fmaf(p, v.y, acc[2 * w + 1]);
      }
    }
    uint4 o0, o1;
    o0.x = pack_bf16x2(acc[0], acc[1]);   o0.y = pack_bf16x2(acc[2], acc[3]);
    o0.z = pack_bf16x2(acc[4], acc[5]);   o0.w = pack_bf16x2(acc[6], acc[7]);
    o1.x = pack_bf16x2(acc[8], acc[9]);   o1.y = pack_bf16x2(acc[10], acc[11]);
    o1.z = pack_bf16x2(acc[12], acc[13]); o1.w = pack_bf16x2(acc[14], acc[15]);
    uint4* dst = reinterpret_cast<uint4*>(ctx + ((long long)bp * SM_N + i) * cs + h * SM_HD + g * 16);
    dst[0] = o0;
    dst[1] = o1;
    __syncwarp();
  }
}

__global__ void __launch_bounds__(SM_WARPS * 32)
attn8_bwd_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ ctx,
                 const __nv_bfloat16* __restrict__ dctx, const float* __restrict__ lse, __nv_bfloat16* __restrict__ dqkv,
                 int nprob, int H, float scale) {
  __shared__ uint32_t sh[SM_WARPS][4][SM_N * SM_PITCH];
  __shared__ float shp[SM_WARPS][2][SM_N * 9];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t* Qs = sh[warp][0];
  uint32_t* Ks = sh[warp][1];
  uint32_t* Vs = sh[warp][2];
  uint32_t* Gs = sh[warp][3];   // dO
  float* Ps = shp[warp][0];
  float* Ds = shp[warp][1];     // dS
  const long long rs = 3LL * H * SM_HD, cs = (long long)H * SM_HD;
  const int i = lane >> 2, g = lane & 3;
  const int pstep = gridDim.x * SM_WARPS;
  int prob = blockIdx.x * SM_WARPS + warp;
  Rows8 rq, rk, rv, rg;
  if (prob < nprob) {
    const __nv_bfloat16* b0 = qkv + (long long)(prob / H) * SM_N * rs + (prob % H) * SM_HD;
    rq = fetch_rows8(b0, rs, lane); rk = fetch_rows8(b0 + cs, rs, lane); rv = fetch_rows8(b0 + 2 * cs, rs, lane);
    rg = fetch_rows8(dctx + (long long)(prob / H) * SM_N * cs + (prob % H) * SM_HD, cs, lane);
  }
  for (; prob < nprob; prob += pstep) {
    const int bp = prob / H, h = prob - bp * H;
    put_rows8(Qs, rq, lane); put_rows8(Ks, rk, lane); put_rows8(Vs, rv, lane); put_rows8(Gs, rg, lane);
    __syncwarp();
    if (prob + pstep < nprob) {
      const int np = prob + pstep;
      const __nv_bfloat16* b1 = qkv + (long long)(np / H) * SM_N * rs + (np % H) * SM_HD;
      rq = fetch_rows8(b1, rs, lane); rk = fetch_rows8(b1 + cs, rs, lane); rv = fetch_rows8(b1 + 2 * cs, rs, lane);
      rg = fetch_rows8(dctx + (long long)(np / H) * SM_N * cs + (np % H) * SM_HD, cs, lane);
    }
    // delta_i = dO_i . O_i  (each lane: its 16 features, then reduce over the 4 lanes of the row)
    float del = 0.f;
    {
      const uint4* o4 = reinterpret_cast<const uint4*>(ctx + ((long long)bp * SM_N + i) * cs + h * SM_HD + g * 16);
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const uint4 o = o4[u];
        const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          const float2 a = unpack_bf16x2(ow[w]);
          const float2 b = unpack_bf16x2(Gs[i * SM_PITCH + g * 8 + u * 4 + w]);
          del = fmaf(a.x, b.x, fmaf(a.y, b.y, del));
        }
      }
      del += __shfl_xor_sync(0xffffffffu, del, 1);
      del += __shfl_xor_sync(0xffffffffu, del, 2);
    }
    float s0 = 0.f, s1 = 0.f, p0 = 0.f, p1 = 0.f;   // scores and dP for keys 2g, 2g+1
#pragma unroll 8
    for (int w = 0; w < 32; ++w) {
      const float2 q = unpack_bf16x2(Qs[i * SM_PITCH + w]);
      const float2 d = unpack_bf16x2(Gs[i * SM_PITCH + w]);
      const float2 k0 = unpack_bf16x2(Ks[(2 * g) * SM_PITCH + w]);
      const float2 k1 = unpack_bf16x2(Ks[(2 * g + 1) * SM_PITCH + w]);
      const float2 v0 = unpack_bf16x2(Vs[(2 * g) * SM_PITCH + w]);
      const float2 v1 = unpack_bf16x2(Vs[(2 * g + 1) * SM_PITCH + w]);
      s0 = fmaf(q.x, k0.x, fmaf(q.y, k0.y, s0));
      s1 = fmaf(q.x, k1.x, fmaf(q.y, k1.y, s1));
      p0 = fmaf(d.x, v0.x, fmaf(d.y, v0.y, p0));
      p1 = fmaf(d.x, v1.x, fmaf(d.y, v1.y, p1));
    }
    const float li = lse[(long long)prob * SM_N + i];
    const float e0 = __expf(s0 * scale - li), e1 = __expf(s1 * scale - li);
    Ps[i * 9 + 2 * g] = e0;
    Ps[i * 9 + 2 * g + 1] = e1;
    Ds[i * 9 + 2 * g] = e0 * (p0 - del) * scale;
    Ds[i * 9 + 2 * g + 1] = e1 * (p1 - del) * scale;
    __syncwarp();
    float aq[16], ak[16], av[16];
#pragma unroll
    for (int d = 0; d < 16; ++d) { aq[d] = 0.f; ak[d] = 0.f; av[d] = 0.f; }
    // lane (i,g): dQ_i[16g..] = sum_j dS[i][j] K_j ;  as key row i: dK_i = sum_q dS[q][i] Q_q ; dV_i = sum_q P[q][i] dO_q
#pragma unroll
    for (int j = 0; j < SM_N; ++j) {
      const float dsq = Ds[i * 9 + j];
      const float dsk = Ds[j * 9 + i];
      const float pk = Ps[j * 9 + i];
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        const float2 k = unpack_bf16x2(Ks[j * SM_PITCH + g * 8 + w]);
        const float2 q = unpack_bf16x2(Qs[j * SM_PITCH + g * 8 + w]);
        const float2 d = unpack_bf16x2(Gs[j * SM_PITCH + g * 8 + w]);
        aq[2 * w] = fmaf(dsq, k.x, aq[2 * w]); aq[2 * w + 1] = fmaf(dsq, k.y, aq[2 * w + 1]);
        ak[2 * w] = fmaf(dsk, q.x, ak[2 * w]); ak[2 * w + 1] = fmaf(dsk, q.y, ak[2 * w + 1]);
        av[2 * w] = fmaf(pk, d.x, av[2 * w]);  av[2 * w + 1] = fmaf(pk, d.y, av[2 * w + 1]);
      }
    }
    __nv_bfloat16* obase = dqkv + ((long long)bp * SM_N + i) * rs + h * SM_HD + g * 16;
#pragma unroll
    for (int slot = 0; slot < 3; ++slot) {
      const float* a = slot == 0 ? aq : (slot == 1 ? ak : av);
      uint4 o0, o1;
      o0.x = pack_bf16x2(a[0], a[1]);   o0.y = pack_bf16x2(a[2], a[3]);
      o0.z = pack_bf16x2(a[4], a[5]);   o0.w = pack_bf16x2(a[6], a[7]);
      o1.x = pack_bf16x2(a[8], a[9]);   o1.y = pack_bf16x2(a[10], a[11]);
      o1.z = pack_bf16x2(a[12], a[13]); o1.w = pack_bf16x2(a[14], a[15]);
      uint4* dst = reinterpret_cast<uint4*>(obase + slot * cs);
      dst[0] = o0;
      dst[1] = o1;
    }
    __syncwarp();
  }
}

// persistent grid = resident CTAs (register-limited: 3/SM forward, 2/SM backward) so that every warp walks several
// problems and the register prefetch of the next problem overlaps the current one
static int small_grid(int nprob, int ctas_per_sm) {
  int blocks = (nprob + SM_WARPS - 1) / SM_WARPS;
  const int cap = sm_count() * ctas_per_sm;
  return blocks < cap ? blocks : cap;
}

int attn8_fwd_launch(const vt_attn_fwd_params* p, cudaStream_t st) {
  const int nprob = p->Bp * p->H;
  attn8_fwd_kernel<<<small_grid(nprob, 3), SM_WARPS * 32, 0, st>>>(static_cast<const __nv_bfloat16*>(p->qkv),
                                                                static_cast<__nv_bfloat16*>(p->ctx), p->lse, nprob, p->H, p->scale);
  return check_launch("attn8_fwd_kernel");
}

int attn8_bwd_launch(const vt_attn_bwd_params* p, cudaStream_t st) {
  const int nprob = p->Bp * p->H;
  attn8_bwd_kernel<<<small_grid(nprob, 2), SM_WARPS * 32, 0, st>>>(
      static_cast<const __nv_bfloat16*>(p->qkv), static_cast<const __nv_bfloat16*>(p->ctx),
      static_cast<const __nv_bfloat16*>(p->dctx), p->lse, static_cast<__nv_bfloat16*>(p->dqkv), nprob, p->H, p->scale);
  return check_launch("attn8_bwd_kernel");
}

}  // namespace vt
