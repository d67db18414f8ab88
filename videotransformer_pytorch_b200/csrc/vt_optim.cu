// Fused gradient clipping + optimizer update (SURVEY §8f rank 1).
//
// The reference clips every parameter's gradient to `clip_grad` by its own L2 norm (model_trainer.py:155-170: one
// torch.norm launch + one host comparison per parameter, 247 of them for TimeSformer-B) and then runs torch.optim
// SGD(momentum 0.9, nesterov) or AdamW (optimizer.py:33-38).  Here that is two launches for the whole model:
//   1. multi_norm2 + norm2_finish: squared L2 norm of every gradient tensor (one partial per chunk, then each tensor's
//      partials summed in chunk order: the same inputs give the same bits on every call)
//   2. fused update: per element g = grad * min(1, clip / (norm + 1e-6)), then the SGD-nesterov or AdamW step.
// Tensors are addressed through device arrays of pointers (multi-tensor apply), so parameters, gradients (per-tensor
// .grad or views of the DDP flat buckets) and optimizer state stay wherever PyTorch put them.
// The per-step scalars (clip, bias corrections, first-step flag) are kernel arguments, or, when `hyper` is given, read
// from that device block: a CUDA graph that recorded the update then takes each step's values from the block, which the
// host rewrites between replays.  The host computes the values in both forms, so both give the same bits.
#include <math.h>

#include "vt_common.cuh"

namespace vt {

constexpr int OPT_THREADS = 256;

struct OptChunk {
  int32_t tensor;
  int32_t len;
  long long offset;
};
static_assert(sizeof(OptChunk) == 16, "chunk table layout");

__global__ void __launch_bounds__(OPT_THREADS)
multi_norm2_kernel(const OptChunk* __restrict__ chunks, const long long* __restrict__ gptr, float* __restrict__ partials) {
  const OptChunk c = chunks[blockIdx.x];
  const float* g = reinterpret_cast<const float*>(gptr[c.tensor]) + c.offset;
  float s = 0.f;
  if ((reinterpret_cast<uintptr_t>(g) & 15) == 0) {
    const int n4 = c.len >> 2;
    const float4* g4 = reinterpret_cast<const float4*>(g);
    for (int i = threadIdx.x; i < n4; i += OPT_THREADS) {
      const float4 v = g4[i];
      s += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
    }
    for (int i = (n4 << 2) + threadIdx.x; i < c.len; i += OPT_THREADS) s += g[i] * g[i];
  } else {
    for (int i = threadIdx.x; i < c.len; i += OPT_THREADS) s += g[i] * g[i];
  }
  s = warp_sum(s);
  __shared__ float sh[OPT_THREADS / 32];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f;
    for (int i = 0; i < OPT_THREADS / 32; ++i) a += sh[i];
    partials[blockIdx.x] = a;
  }
}

// norm2[t] = the partials of tensor t's chunks added in table order; one thread per chunk, the thread of a tensor's first
// chunk walks its run (a tensor's chunks are consecutive in the table)
__global__ void norm2_finish_kernel(const OptChunk* __restrict__ chunks, const float* __restrict__ partials,
                                    float* __restrict__ norm2, int n_chunks) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_chunks) return;
  const int t = chunks[c].tensor;
  if (c > 0 && chunks[c - 1].tensor == t) return;
  float s = partials[c];
  for (int j = c + 1; j < n_chunks && chunks[j].tensor == t; ++j) s += partials[j];
  norm2[t] = s;
}

struct OptArgs {
  const OptChunk* chunks;
  const long long* pptr;
  const long long* gptr;
  const long long* s1ptr;   // momentum buffer / exp_avg
  const long long* s2ptr;   // exp_avg_sq (AdamW)
  const float* norm2;       // NULL => no clipping
  const float* lr;          // per tensor
  const float* wd;          // per tensor
  const float* hyper;       // NULL, or the device block {clip, bc1, bc2, first_step, spare} replacing the scalars below
  float clip;
  float momentum, beta1, beta2, eps, bc1, bc2;
  int nesterov, first_step;
};

__device__ __forceinline__ float clip_coef(const OptArgs& a, float clip, int t) {
  if (a.norm2 == nullptr || clip <= 0.f) return 1.0f;
  const float c = clip / (sqrtf(a.norm2[t]) + 1e-6f);
  return c < 1.0f ? c : 1.0f;
}

__global__ void __launch_bounds__(OPT_THREADS) fused_sgd_kernel(const OptArgs a) {
  const OptChunk c = a.chunks[blockIdx.x];
  float* p = reinterpret_cast<float*>(a.pptr[c.tensor]) + c.offset;
  const float* g = reinterpret_cast<const float*>(a.gptr[c.tensor]) + c.offset;
  float* buf = reinterpret_cast<float*>(a.s1ptr[c.tensor]) + c.offset;
  const float clip = a.hyper ? a.hyper[VT_OPT_HYPER_CLIP] : a.clip;
  const bool first_step = a.hyper ? a.hyper[VT_OPT_HYPER_FIRST_STEP] != 0.f : a.first_step != 0;
  const float coef = clip_coef(a, clip, c.tensor), lr = a.lr[c.tensor], wd = a.wd[c.tensor];
  for (int i = threadIdx.x; i < c.len; i += OPT_THREADS) {
    const float w = p[i];
    float d = fmaf(wd, w, g[i] * coef);
    const float b = first_step ? d : fmaf(a.momentum, buf[i], d);
    buf[i] = b;
    d = a.nesterov ? fmaf(a.momentum, b, d) : b;
    p[i] = fmaf(-lr, d, w);
  }
}

__global__ void __launch_bounds__(OPT_THREADS) fused_adamw_kernel(const OptArgs a) {
  const OptChunk c = a.chunks[blockIdx.x];
  float* p = reinterpret_cast<float*>(a.pptr[c.tensor]) + c.offset;
  const float* g = reinterpret_cast<const float*>(a.gptr[c.tensor]) + c.offset;
  float* m = reinterpret_cast<float*>(a.s1ptr[c.tensor]) + c.offset;
  float* v = reinterpret_cast<float*>(a.s2ptr[c.tensor]) + c.offset;
  const float clip = a.hyper ? a.hyper[VT_OPT_HYPER_CLIP] : a.clip;
  const float bc1 = a.hyper ? a.hyper[VT_OPT_HYPER_BC1] : a.bc1, bc2 = a.hyper ? a.hyper[VT_OPT_HYPER_BC2] : a.bc2;
  const float coef = clip_coef(a, clip, c.tensor), lr = a.lr[c.tensor], wd = a.wd[c.tensor];
  const float step_size = lr / bc1, inv_sqrt_bc2 = rsqrtf(bc2);
  for (int i = threadIdx.x; i < c.len; i += OPT_THREADS) {
    const float gi = g[i] * coef;
    const float w = p[i] * (1.0f - lr * wd);
    const float mi = fmaf(a.beta1, m[i], (1.0f - a.beta1) * gi);
    const float vi = fmaf(a.beta2, v[i], (1.0f - a.beta2) * gi * gi);
    m[i] = mi;
    v[i] = vi;
    p[i] = w - step_size * mi / (sqrtf(vi) * inv_sqrt_bc2 + a.eps);
  }
}

}  // namespace vt

using namespace vt;

extern "C" int vt_opt_norm2(const vt_opt_params* p, void* stream) {
  VT_REQUIRE(p && p->chunks && p->gptr && p->norm2 && p->n_chunks > 0 && p->n_tensors > 0, "vt_opt_norm2: bad params");
  VT_REQUIRE(p->partials, "vt_opt_norm2: partials workspace (n_chunks floats) missing");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(p->norm2, 0, sizeof(float) * p->n_tensors, st);   // tensors without chunks
  VT_REQUIRE(e == cudaSuccess, "vt_opt_norm2: memset: %s", cudaGetErrorString(e));
  const OptChunk* chunks = static_cast<const OptChunk*>(p->chunks);
  multi_norm2_kernel<<<p->n_chunks, OPT_THREADS, 0, st>>>(chunks, reinterpret_cast<const long long*>(p->gptr), p->partials);
  int rc = check_launch("multi_norm2_kernel");
  if (rc) return rc;
  norm2_finish_kernel<<<(p->n_chunks + 255) / 256, 256, 0, st>>>(chunks, p->partials, p->norm2, p->n_chunks);
  return check_launch("norm2_finish_kernel");
}

static int opt_args(const vt_opt_params* p, OptArgs* a, const char* who, bool need_s2) {
  VT_REQUIRE(p && p->chunks && p->pptr && p->gptr && p->s1ptr && p->lr && p->wd && p->n_chunks > 0, "%s: bad params", who);
  VT_REQUIRE(!need_s2 || p->s2ptr, "%s: second moment buffers missing", who);
  a->chunks = static_cast<const OptChunk*>(p->chunks);
  a->pptr = reinterpret_cast<const long long*>(p->pptr);
  a->gptr = reinterpret_cast<const long long*>(p->gptr);
  a->s1ptr = reinterpret_cast<const long long*>(p->s1ptr);
  a->s2ptr = reinterpret_cast<const long long*>(p->s2ptr);
  // with `hyper` the clip value is only known on the device: the kernels test it there
  VT_REQUIRE(!p->hyper || p->norm2, "%s: the hyper block needs the norm2 array", who);
  a->norm2 = (p->hyper || p->clip > 0.f) ? p->norm2 : nullptr;
  a->lr = p->lr;
  a->wd = p->wd;
  a->hyper = p->hyper;
  a->clip = p->clip;
  a->momentum = p->momentum; a->beta1 = p->beta1; a->beta2 = p->beta2; a->eps = p->eps; a->bc1 = p->bc1; a->bc2 = p->bc2;
  a->nesterov = p->nesterov;
  a->first_step = p->first_step;
  return 0;
}

extern "C" int vt_opt_sgd(const vt_opt_params* p, void* stream) {
  OptArgs a;
  int rc = opt_args(p, &a, "vt_opt_sgd", false);
  if (rc) return rc;
  fused_sgd_kernel<<<p->n_chunks, OPT_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(a);
  return check_launch("fused_sgd_kernel");
}

extern "C" int vt_opt_adamw(const vt_opt_params* p, void* stream) {
  OptArgs a;
  int rc = opt_args(p, &a, "vt_opt_adamw", true);
  if (rc) return rc;
  VT_REQUIRE(p->hyper || (p->bc1 > 0.f && p->bc2 > 0.f), "vt_opt_adamw: bias corrections must be positive");
  fused_adamw_kernel<<<p->n_chunks, OPT_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(a);
  return check_launch("fused_adamw_kernel");
}
