// Temporal attention of the divided space-time block: 8 frames x 8 frames per (sample, patch, head) —
// 18 816 independent 8x8x64 problems per layer at batch 8.  0.1 % of the FLOPs, so the kernel is built
// to be bandwidth/latency lean instead of tensor-core shaped: one warp per problem, Q/K/V (and dO) rows
// staged in shared memory (HD / 2 + 1-word pitch, odd: conflict-free), lane (i, g) = query row i = lane/4 and quarter
// g = lane%4:  scores for keys {2g, 2g+1} (full HD-dim dots), softmax across the 4 lanes of a row with two
// shuffles, then the lane owns features [g HD/4, (g+1) HD/4) of its output row.  Backward uses the same mapping
// (dQ rows, then dK/dV rows) and recomputes P from the saved log-sum-exp.  Instantiated at head dims 32, 64, 96 and 128;
// at 96 and 128 a CTA has 4 warps so that the backward's staged rows stay within 48 KB of static shared memory.
#include "vt_common.cuh"

namespace vt {

constexpr int SM_N = 8;

template <int HD>
struct Attn8 {
  static constexpr int PITCH = HD / 2 + 1;     // words per staged row
  static constexpr int FW = HD / 8;            // words of a lane's quarter of a row
  static constexpr int CPR = HD / 8;           // 16-byte chunks per row
  static constexpr int RPL = SM_N * CPR / 32;  // chunks of an 8-row operand per lane
  static constexpr int WARPS = HD <= 64 ? 8 : 4;
  // row and 16-byte chunk of chunk lane + 32 it of an 8-row operand (a whole number of rows per 32 chunks but at 96)
  static __device__ __forceinline__ int row(int lane, int it) {
    return 32 % CPR == 0 ? lane / CPR + 32 / CPR * it : (lane + 32 * it) / CPR;
  }
  static __device__ __forceinline__ int col(int lane, int it) { return 32 % CPR == 0 ? lane % CPR : (lane + 32 * it) % CPR; }
};

// software pipelining: the next problem's rows are fetched into registers while the current one is computed
template <int HD>
struct Rows8 { uint4 v[Attn8<HD>::RPL]; };
template <int HD>
__device__ __forceinline__ Rows8<HD> fetch_rows8(const __nv_bfloat16* base, long long row_stride, int lane) {
  using C = Attn8<HD>;
  Rows8<HD> r;
#pragma unroll
  for (int it = 0; it < C::RPL; ++it) {
    const int row = C::row(lane, it), c = C::col(lane, it);
    r.v[it] = *reinterpret_cast<const uint4*>(base + (long long)row * row_stride + c * 8);
  }
  return r;
}
template <int HD>
__device__ __forceinline__ void put_rows8(uint32_t* dst, const Rows8<HD>& r, int lane) {
  using C = Attn8<HD>;
#pragma unroll
  for (int it = 0; it < C::RPL; ++it) {
    const int row = C::row(lane, it), c = C::col(lane, it);
    uint32_t* d = dst + row * C::PITCH + c * 4;
    d[0] = r.v[it].x; d[1] = r.v[it].y; d[2] = r.v[it].z; d[3] = r.v[it].w;
  }
}

template <int HD>
__global__ void __launch_bounds__(Attn8<HD>::WARPS * 32)
attn8_fwd_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ ctx, float* __restrict__ lse,
                 int nprob, int H, float scale) {
  using C = Attn8<HD>;
  constexpr int SM_WARPS = C::WARPS, SM_PITCH = C::PITCH, FW = C::FW;
  __shared__ uint32_t sh[SM_WARPS][3][SM_N * SM_PITCH];
  __shared__ float shp[SM_WARPS][SM_N * 9];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t* Qs = sh[warp][0];
  uint32_t* Ks = sh[warp][1];
  uint32_t* Vs = sh[warp][2];
  float* Ps = shp[warp];
  const long long rs = 3LL * H * HD, cs = (long long)H * HD;
  const int i = lane >> 2, g = lane & 3;
  const int pstep = gridDim.x * SM_WARPS;
  int prob = blockIdx.x * SM_WARPS + warp;
  Rows8<HD> rq, rk, rv;
  if (prob < nprob) {
    const __nv_bfloat16* b0 = qkv + (long long)(prob / H) * SM_N * rs + (prob % H) * HD;
    rq = fetch_rows8<HD>(b0, rs, lane); rk = fetch_rows8<HD>(b0 + cs, rs, lane); rv = fetch_rows8<HD>(b0 + 2 * cs, rs, lane);
  }
  for (; prob < nprob; prob += pstep) {
    const int bp = prob / H, h = prob - bp * H;
    put_rows8<HD>(Qs, rq, lane); put_rows8<HD>(Ks, rk, lane); put_rows8<HD>(Vs, rv, lane);
    __syncwarp();
    if (prob + pstep < nprob) {
      const int np = prob + pstep;
      const __nv_bfloat16* b1 = qkv + (long long)(np / H) * SM_N * rs + (np % H) * HD;
      rq = fetch_rows8<HD>(b1, rs, lane); rk = fetch_rows8<HD>(b1 + cs, rs, lane); rv = fetch_rows8<HD>(b1 + 2 * cs, rs, lane);
    }
    float s0 = 0.f, s1 = 0.f;
#pragma unroll 8
    for (int w = 0; w < HD / 2; ++w) {
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
    float acc[2 * FW];
#pragma unroll
    for (int d = 0; d < 2 * FW; ++d) acc[d] = 0.f;
#pragma unroll
    for (int j = 0; j < SM_N; ++j) {
      const float p = Ps[i * 9 + j];
#pragma unroll
      for (int w = 0; w < FW; ++w) {
        const float2 v = unpack_bf16x2(Vs[j * SM_PITCH + g * FW + w]);
        acc[2 * w] = fmaf(p, v.x, acc[2 * w]);
        acc[2 * w + 1] = fmaf(p, v.y, acc[2 * w + 1]);
      }
    }
    uint4 o[FW / 4];
#pragma unroll
    for (int u = 0; u < FW / 4; ++u) {
      o[u].x = pack_bf16x2(acc[8 * u], acc[8 * u + 1]);     o[u].y = pack_bf16x2(acc[8 * u + 2], acc[8 * u + 3]);
      o[u].z = pack_bf16x2(acc[8 * u + 4], acc[8 * u + 5]); o[u].w = pack_bf16x2(acc[8 * u + 6], acc[8 * u + 7]);
    }
    uint4* dst = reinterpret_cast<uint4*>(ctx + ((long long)bp * SM_N + i) * cs + h * HD + g * (HD / 4));
#pragma unroll
    for (int u = 0; u < FW / 4; ++u) dst[u] = o[u];
    __syncwarp();
  }
}

template <int HD>
__global__ void __launch_bounds__(Attn8<HD>::WARPS * 32)
attn8_bwd_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ ctx,
                 const __nv_bfloat16* __restrict__ dctx, const float* __restrict__ lse, __nv_bfloat16* __restrict__ dqkv,
                 int nprob, int H, float scale) {
  using C = Attn8<HD>;
  constexpr int SM_WARPS = C::WARPS, SM_PITCH = C::PITCH, FW = C::FW;
  __shared__ uint32_t sh[SM_WARPS][4][SM_N * SM_PITCH];
  __shared__ float shp[SM_WARPS][2][SM_N * 9];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t* Qs = sh[warp][0];
  uint32_t* Ks = sh[warp][1];
  uint32_t* Vs = sh[warp][2];
  uint32_t* Gs = sh[warp][3];   // dO
  float* Ps = shp[warp][0];
  float* Ds = shp[warp][1];     // dS
  const long long rs = 3LL * H * HD, cs = (long long)H * HD;
  const int i = lane >> 2, g = lane & 3;
  const int pstep = gridDim.x * SM_WARPS;
  int prob = blockIdx.x * SM_WARPS + warp;
  Rows8<HD> rq, rk, rv, rg;
  if (prob < nprob) {
    const __nv_bfloat16* b0 = qkv + (long long)(prob / H) * SM_N * rs + (prob % H) * HD;
    rq = fetch_rows8<HD>(b0, rs, lane); rk = fetch_rows8<HD>(b0 + cs, rs, lane); rv = fetch_rows8<HD>(b0 + 2 * cs, rs, lane);
    rg = fetch_rows8<HD>(dctx + (long long)(prob / H) * SM_N * cs + (prob % H) * HD, cs, lane);
  }
  for (; prob < nprob; prob += pstep) {
    const int bp = prob / H, h = prob - bp * H;
    put_rows8<HD>(Qs, rq, lane); put_rows8<HD>(Ks, rk, lane); put_rows8<HD>(Vs, rv, lane); put_rows8<HD>(Gs, rg, lane);
    __syncwarp();
    if (prob + pstep < nprob) {
      const int np = prob + pstep;
      const __nv_bfloat16* b1 = qkv + (long long)(np / H) * SM_N * rs + (np % H) * HD;
      rq = fetch_rows8<HD>(b1, rs, lane); rk = fetch_rows8<HD>(b1 + cs, rs, lane); rv = fetch_rows8<HD>(b1 + 2 * cs, rs, lane);
      rg = fetch_rows8<HD>(dctx + (long long)(np / H) * SM_N * cs + (np % H) * HD, cs, lane);
    }
    // delta_i = dO_i . O_i  (each lane: its HD / 4 features, then reduce over the 4 lanes of the row)
    float del = 0.f;
    {
      const uint4* o4 = reinterpret_cast<const uint4*>(ctx + ((long long)bp * SM_N + i) * cs + h * HD + g * (HD / 4));
#pragma unroll
      for (int u = 0; u < FW / 4; ++u) {
        const uint4 o = o4[u];
        const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          const float2 a = unpack_bf16x2(ow[w]);
          const float2 b = unpack_bf16x2(Gs[i * SM_PITCH + g * FW + u * 4 + w]);
          del = fmaf(a.x, b.x, fmaf(a.y, b.y, del));
        }
      }
      del += __shfl_xor_sync(0xffffffffu, del, 1);
      del += __shfl_xor_sync(0xffffffffu, del, 2);
    }
    float s0 = 0.f, s1 = 0.f, p0 = 0.f, p1 = 0.f;   // scores and dP for keys 2g, 2g+1
#pragma unroll 8
    for (int w = 0; w < HD / 2; ++w) {
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
    float aq[2 * FW], ak[2 * FW], av[2 * FW];
#pragma unroll
    for (int d = 0; d < 2 * FW; ++d) { aq[d] = 0.f; ak[d] = 0.f; av[d] = 0.f; }
    // lane (i,g): dQ_i[g HD/4..] = sum_j dS[i][j] K_j ;  as key row i: dK_i = sum_q dS[q][i] Q_q ; dV_i = sum_q P[q][i] dO_q
#pragma unroll
    for (int j = 0; j < SM_N; ++j) {
      const float dsq = Ds[i * 9 + j];
      const float dsk = Ds[j * 9 + i];
      const float pk = Ps[j * 9 + i];
#pragma unroll
      for (int w = 0; w < FW; ++w) {
        const float2 k = unpack_bf16x2(Ks[j * SM_PITCH + g * FW + w]);
        const float2 q = unpack_bf16x2(Qs[j * SM_PITCH + g * FW + w]);
        const float2 d = unpack_bf16x2(Gs[j * SM_PITCH + g * FW + w]);
        aq[2 * w] = fmaf(dsq, k.x, aq[2 * w]); aq[2 * w + 1] = fmaf(dsq, k.y, aq[2 * w + 1]);
        ak[2 * w] = fmaf(dsk, q.x, ak[2 * w]); ak[2 * w + 1] = fmaf(dsk, q.y, ak[2 * w + 1]);
        av[2 * w] = fmaf(pk, d.x, av[2 * w]);  av[2 * w + 1] = fmaf(pk, d.y, av[2 * w + 1]);
      }
    }
    __nv_bfloat16* obase = dqkv + ((long long)bp * SM_N + i) * rs + h * HD + g * (HD / 4);
#pragma unroll
    for (int slot = 0; slot < 3; ++slot) {
      const float* a = slot == 0 ? aq : (slot == 1 ? ak : av);
      uint4* dst = reinterpret_cast<uint4*>(obase + slot * cs);
#pragma unroll
      for (int u = 0; u < FW / 4; ++u) {
        const float* b = a + 8 * u;
        dst[u] = make_uint4(pack_bf16x2(b[0], b[1]), pack_bf16x2(b[2], b[3]), pack_bf16x2(b[4], b[5]), pack_bf16x2(b[6], b[7]));
      }
    }
    __syncwarp();
  }
}

// persistent grid = resident CTAs (register-limited; at head dim 64 3/SM forward, 2/SM backward) so that every warp walks
// several problems and the register prefetch of the next problem overlaps the current one
template <int HD>
static int small_grid(int nprob, int ctas_per_sm) {
  constexpr int SM_WARPS = Attn8<HD>::WARPS;
  int blocks = (nprob + SM_WARPS - 1) / SM_WARPS;
  const int cap = sm_count() * ctas_per_sm;
  return blocks < cap ? blocks : cap;
}

// resident CTAs per SM of the forward / backward at each head dim, from their ptxas register counts (forward 48, 64, 128,
// 128 registers; backward 64, 80, 128, 168 at head dim 32, 64, 96, 128; 8 warps per CTA up to 64, 4 above)
template <int HD> constexpr int attn8_fwd_ctas() { return HD == 32 ? 5 : HD == 64 ? 3 : 4; }
template <int HD> constexpr int attn8_bwd_ctas() { return HD == 32 ? 4 : HD == 64 ? 2 : HD == 96 ? 4 : 3; }

int attn8_fwd_launch(const vt_attn_fwd_params* p, cudaStream_t st) {
  const int nprob = p->Bp * p->H;
  return with_head_dim(p->hd, [&](auto hd) {
    constexpr int HD = hd.value;
    attn8_fwd_kernel<HD><<<small_grid<HD>(nprob, attn8_fwd_ctas<HD>()), Attn8<HD>::WARPS * 32, 0, st>>>(
        static_cast<const __nv_bfloat16*>(p->qkv), static_cast<__nv_bfloat16*>(p->ctx), p->lse, nprob, p->H, p->scale);
    return check_launch("attn8_fwd_kernel");
  });
}

int attn8_bwd_launch(const vt_attn_bwd_params* p, cudaStream_t st) {
  const int nprob = p->Bp * p->H;
  return with_head_dim(p->hd, [&](auto hd) {
    constexpr int HD = hd.value;
    attn8_bwd_kernel<HD><<<small_grid<HD>(nprob, attn8_bwd_ctas<HD>()), Attn8<HD>::WARPS * 32, 0, st>>>(
        static_cast<const __nv_bfloat16*>(p->qkv), static_cast<const __nv_bfloat16*>(p->ctx),
        static_cast<const __nv_bfloat16*>(p->dctx), p->lse, static_cast<__nv_bfloat16*>(p->dqkv), nprob, p->H, p->scale);
    return check_launch("attn8_bwd_kernel");
  });
}

}  // namespace vt
