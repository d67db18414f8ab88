// Clip transforms on decode-resolution uint8 frames: torchvision's resized crop / resize + crop (+ flip) and ColorJitter,
// as the reference's DataLoader applies them (data_transform.py:495-615) to a uint8 T C H W clip.  See vt_b200.h.
//
// Resize.  torchvision casts uint8 to fp32 and calls F.interpolate(antialias=True), whose CPU kernel computes, per output
// index i of an axis with scale = in / out (fp32):
//   center = scale * (i + 0.5), support = taps/2 * max(scale, 1), invscale = 1 / max(scale, 1)    (fp32)
//   taps j in [int(center - support + 0.5), int(center + support + 0.5)) clamped to the axis
//   w_j = filter((j - center + 0.5) * invscale), then each w_j divided by their fp32 sum
// and applies the width pass first, then the height pass, each a sequential fp32 sum starting at the first tap.  The
// weights here are computed with the same fp32 roundings (center rounded to fp32 is what moves them up to 1.6e-5 away
// from an exact-arithmetic restatement).  Every product and sum is rounded separately (__fmul_rn / __fadd_rn), so the
// result is the CPU twin's in tests/emu_augment.py bit for bit; against torch itself it may differ in the last bits
// where the compiler contracted torch's expressions into FMAs.
//
// One CTA computes CROP_ROWS output rows of one frame.  It builds the weights of all S output columns and of its rows in
// shared memory, then each thread computes whole pixels (3 channels) as sum_i wy_i * (sum_j wx_j * src): the width-pass
// value of a tap row is recomputed by every output row that uses it instead of being staged, which keeps the shared
// memory independent of the scale factor and gives the separable result exactly (same operations, same order).
//
// ColorJitter.  One CTA per frame holds the S x S x 3 frame in shared memory and applies the clip's ops in order.  The
// contrast mean is torch.mean over the fp32 grayscale frame: an integer sum (exact in fp32 up to 254 * 256 * 256 < 2^24)
// divided by S * S.
//
// RandAugment.  The same one-CTA-per-frame layout, with torchvision's 14 ops applied in the drawn order.  Pointwise ops
// and the per-frame statistics (grayscale sum, per-channel min / max and histograms: warp reductions, then shared
// atomics) work on the frame in shared memory.  Ops that read other pixels (shears, translations, rotation, sharpness)
// gather from shared memory into the frame's global output, which is reloaded only if another op follows.
#include "vt_common.cuh"

namespace vt {

constexpr int CROP_ROWS = 8;
constexpr int CROP_THREADS = 256;
constexpr int MAXT = VT_CROP_MAX_TAPS;

__device__ __forceinline__ float aa_filter(float x, int filter) {
  x = fabsf(x);
  if (filter == 1) return x < 1.f ? __fsub_rn(1.f, x) : 0.f;
  if (x < 1.f)        // ((a + 2) x - (a + 3)) x x + 1, a = -0.5
    return __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(1.5f, x), 2.5f), x), x), 1.f);
  if (x < 2.f)        // ((a x - 5 a) x + 8 a) x - 4 a
    return __fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(-0.5f, x), 2.5f), x), 4.f), x), 2.f);
  return 0.f;
}

__device__ __forceinline__ float axis_support(int in, int out, int filter) {
  const float scale = __fdiv_rn((float)in, (float)out);
  const float half = filter == 0 ? 2.f : 1.f;
  return scale >= 1.f ? half * scale : half;
}

__device__ __forceinline__ int axis_max_taps(float support) { return 2 * (int)ceilf(support) + 1; }

// taps of output index i (in the resized axis of `out` cells) over an input axis of `in` cells: w[j * ws], j < *n
__device__ void axis_taps(int i, int in, int out, int filter, float* w, int ws, int* lo_out, int* n_out) {
  const float scale = __fdiv_rn((float)in, (float)out);
  const float support = axis_support(in, out, filter);
  const float invscale = scale >= 1.f ? (float)(1.0 / (double)scale) : 1.f;
  const float center = __fmul_rn(scale, (float)i + 0.5f);
  const int lo = max((int)((double)__fsub_rn(center, support) + 0.5), 0);
  const int hi = min((int)((double)__fadd_rn(center, support) + 0.5), in);
  const int n = min(max(hi - lo, 0), min(axis_max_taps(support), MAXT));   // torch clips to 2 ceil(support) + 1
  float total = 0.f;
  for (int j = 0; j < n; ++j) {
    const float x = (float)(((double)__fsub_rn((float)(j + lo), center) + 0.5) * (double)invscale);
    const float v = aa_filter(x, filter);
    w[j * ws] = v;
    total = __fadd_rn(total, v);
  }
  if (total != 0.f)
    for (int j = 0; j < n; ++j) w[j * ws] = __fdiv_rn(w[j * ws], total);
  *lo_out = lo;
  *n_out = n;
}

__device__ bool desc_ok(const vt_crop_desc& d, int T, int S, int64_t src_bytes) {
  if (d.H <= 0 || d.W <= 0 || d.pitch < 3 * d.W || d.src_offset < 0) return false;
  if (d.crop_y < 0 || d.crop_x < 0 || d.crop_h <= 0 || d.crop_w <= 0) return false;
  if (d.crop_y + d.crop_h > d.H || d.crop_x + d.crop_w > d.W) return false;
  if (d.RH <= 0 || d.RW <= 0 || d.oy < 0 || d.ox < 0 || d.oy + S > d.RH || d.ox + S > d.RW) return false;
  if (d.filter != 0 && d.filter != 1) return false;
  if (axis_max_taps(axis_support(d.crop_h, d.RH, d.filter)) > MAXT) return false;
  if (axis_max_taps(axis_support(d.crop_w, d.RW, d.filter)) > MAXT) return false;
  const int64_t last = d.src_offset + (int64_t)T * d.H * d.pitch - d.pitch + 3ll * d.W;   // one past the last byte
  return last <= src_bytes;
}

__global__ void __launch_bounds__(CROP_THREADS)
resized_crop_u8_kernel(const uint8_t* __restrict__ src, int64_t src_bytes, const vt_crop_desc* __restrict__ descs,
                       uint8_t* __restrict__ out, int32_t* err, int T, int S) {
  extern __shared__ float sm[];
  float* xw = sm;                                  // [MAXT][S]
  float* yw = xw + MAXT * S;                       // [MAXT][CROP_ROWS]
  int* xlo = reinterpret_cast<int*>(yw + MAXT * CROP_ROWS);
  int* xn = xlo + S;
  int* ylo = xn + S;
  int* yn = ylo + CROP_ROWS;
  __shared__ vt_crop_desc d;
  __shared__ int ok;
  const int clip = blockIdx.x / T, t = blockIdx.x % T;
  const int r0 = blockIdx.y * CROP_ROWS;
  const int rows = min(CROP_ROWS, S - r0);
  if (threadIdx.x == 0) {
    d = descs[clip];
    ok = desc_ok(d, T, S, src_bytes);
    if (!ok && err) *err = 1;
  }
  __syncthreads();
  uint8_t* o = out + (((int64_t)clip * T + t) * S + r0) * S * 3;
  if (!ok) {
    for (int k = threadIdx.x; k < rows * S * 3; k += blockDim.x) o[k] = 0;
    return;
  }
  for (int c = threadIdx.x; c < S + rows; c += blockDim.x) {
    if (c < S) axis_taps(d.ox + c, d.crop_w, d.RW, d.filter, xw + c, S, xlo + c, xn + c);
    else axis_taps(d.oy + r0 + (c - S), d.crop_h, d.RH, d.filter, yw + (c - S), CROP_ROWS, ylo + (c - S), yn + (c - S));
  }
  __syncthreads();
  const uint8_t* frame = src + d.src_offset + (int64_t)t * d.H * d.pitch + (int64_t)d.crop_y * d.pitch + 3ll * d.crop_x;
  for (int k = threadIdx.x; k < rows * S; k += blockDim.x) {
    const int r = k / S, x = k % S;
    const int c = d.flip ? S - 1 - x : x;          // resized column this output pixel shows
    const int nx = xn[c], x0 = xlo[c], ny = yn[r];
    const uint8_t* base = frame + (int64_t)ylo[r] * d.pitch + 3ll * x0;
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f;
    for (int i = 0; i < ny; ++i) {
      const uint8_t* row = base + (int64_t)i * d.pitch;
      float h0 = 0.f, h1 = 0.f, h2 = 0.f;
      for (int j = 0; j < nx; ++j) {
        const float w = xw[j * S + c];
        const float p0 = __fmul_rn((float)__ldg(row + 3 * j), w);
        const float p1 = __fmul_rn((float)__ldg(row + 3 * j + 1), w);
        const float p2 = __fmul_rn((float)__ldg(row + 3 * j + 2), w);
        h0 = j ? __fadd_rn(h0, p0) : p0;
        h1 = j ? __fadd_rn(h1, p1) : p1;
        h2 = j ? __fadd_rn(h2, p2) : p2;
      }
      const float w = yw[i * CROP_ROWS + r];
      acc0 = i ? __fadd_rn(acc0, __fmul_rn(h0, w)) : __fmul_rn(h0, w);
      acc1 = i ? __fadd_rn(acc1, __fmul_rn(h1, w)) : __fmul_rn(h1, w);
      acc2 = i ? __fadd_rn(acc2, __fmul_rn(h2, w)) : __fmul_rn(h2, w);
    }
    uint8_t* q = o + (int64_t)k * 3;
    q[0] = (uint8_t)rintf(fminf(fmaxf(acc0, 0.f), 255.f));
    q[1] = (uint8_t)rintf(fminf(fmaxf(acc1, 0.f), 255.f));
    q[2] = (uint8_t)rintf(fminf(fmaxf(acc2, 0.f), 255.f));
  }
}

__device__ __forceinline__ float gray_u8(float r, float g, float b) {
  return truncf(__fadd_rn(__fadd_rn(__fmul_rn(0.2989f, r), __fmul_rn(0.587f, g)), __fmul_rn(0.114f, b)));
}

__device__ __forceinline__ uint8_t blend_u8(float x, float y, float r, float rc) {
  return (uint8_t)__float2uint_rz(fminf(fmaxf(__fadd_rn(__fmul_rn(r, x), __fmul_rn(rc, y)), 0.f), 255.f));
}

constexpr int JITTER_THREADS = 512;

__global__ void __launch_bounds__(JITTER_THREADS)
color_jitter_u8_kernel(uint8_t* __restrict__ frames, const vt_jitter_desc* __restrict__ descs, int T, int S) {
  extern __shared__ __align__(16) uint8_t px[];
  __shared__ unsigned int gray_sum;
  const vt_jitter_desc d = descs[blockIdx.x / T];
  if (d.n_ops <= 0) return;
  const int npx = S * S;
  const int nbytes = npx * 3;
  uint8_t* g = frames + (int64_t)blockIdx.x * nbytes;
  const bool vec = (nbytes % 16) == 0 && (reinterpret_cast<uintptr_t>(g) % 16) == 0;
  if (vec) {
    for (int k = threadIdx.x; k < nbytes / 16; k += blockDim.x) reinterpret_cast<uint4*>(px)[k] = reinterpret_cast<const uint4*>(g)[k];
  } else {
    for (int k = threadIdx.x; k < nbytes; k += blockDim.x) px[k] = g[k];
  }
  __syncthreads();
  for (int s = 0; s < d.n_ops && s < 3; ++s) {
    const int op = d.op[s];
    const float r = d.factor[s], rc = d.one_minus[s];
    float mean = 0.f;
    if (op == 1) {
      if (threadIdx.x == 0) gray_sum = 0;
      __syncthreads();
      unsigned int part = 0;
      for (int p = threadIdx.x; p < npx; p += blockDim.x)
        part += (unsigned int)gray_u8(px[3 * p], px[3 * p + 1], px[3 * p + 2]);
      part = __reduce_add_sync(0xffffffffu, part);
      if ((threadIdx.x & 31) == 0) atomicAdd(&gray_sum, part);
      __syncthreads();
      mean = __fdiv_rn((float)gray_sum, (float)npx);
    }
    for (int p = threadIdx.x; p < npx; p += blockDim.x) {
      const float c0 = px[3 * p], c1 = px[3 * p + 1], c2 = px[3 * p + 2];
      const float y = op == 0 ? 0.f : op == 1 ? mean : gray_u8(c0, c1, c2);
      px[3 * p] = blend_u8(c0, y, r, rc);
      px[3 * p + 1] = blend_u8(c1, y, r, rc);
      px[3 * p + 2] = blend_u8(c2, y, r, rc);
    }
    __syncthreads();
  }
  if (vec) {
    for (int k = threadIdx.x; k < nbytes / 16; k += blockDim.x) reinterpret_cast<uint4*>(g)[k] = reinterpret_cast<const uint4*>(px)[k];
  } else {
    for (int k = threadIdx.x; k < nbytes; k += blockDim.x) g[k] = px[k];
  }
}

enum RandAugOp {
  RA_IDENTITY, RA_SHEAR_X, RA_SHEAR_Y, RA_TRANSLATE_X, RA_TRANSLATE_Y, RA_ROTATE, RA_BRIGHTNESS, RA_COLOR, RA_CONTRAST,
  RA_SHARPNESS, RA_POSTERIZE, RA_SOLARIZE, RA_AUTOCONTRAST, RA_EQUALIZE, RA_NUM_OPS
};

constexpr int RA_THREADS = 512;

__device__ __forceinline__ void copy_frame(uint8_t* dst, const uint8_t* src, int nbytes, bool vec) {
  if (vec) {
    for (int k = threadIdx.x; k < nbytes / 16; k += blockDim.x) reinterpret_cast<uint4*>(dst)[k] = reinterpret_cast<const uint4*>(src)[k];
  } else {
    for (int k = threadIdx.x; k < nbytes; k += blockDim.x) dst[k] = src[k];
  }
}

// source coordinate of output index i along an axis: ((g + 1) * S - 1) / 2, nearest (half to even); -1 when outside
__device__ __forceinline__ int nearest_source(float g, int S) {
  const float u = rintf(__fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(g, 1.f), (float)S), 1.f), 0.5f));
  return u >= 0.f && u <= (float)(S - 1) ? (int)u : -1;
}

// Equalize table of channel `c` (one warp): lane l owns bins 8l .. 8l + 7 of hist and writes the same entries of lut.
__device__ void equalize_lut(const unsigned int* hist, uint8_t* lut, int npx) {
  const int lane = threadIdx.x & 31;
  unsigned int h[8], local = 0;
  int top = -1;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    h[k] = hist[8 * lane + k];
    local += h[k];
    if (h[k]) top = 8 * lane + k;
  }
  top = __reduce_max_sync(0xffffffffu, top + 1) - 1;      // the highest occupied bin (npx > 0, so one exists)
  const unsigned int step = (unsigned int)(npx - (int)hist[top]) / 255u;
  unsigned int incl = local;                               // inclusive scan of the lanes' totals
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  unsigned int before = incl - local;                      // pixels in bins below 8 * lane
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int i = 8 * lane + k;
    lut[i] = step == 0 ? (uint8_t)i : i == 0 ? 0 : (uint8_t)min((before + step / 2) / step, 255u);
    before += h[k];
  }
}

// The frame buffer is written by this CTA and read back by it after a gather op, so it is not read through the
// read-only path (no const __restrict__ / __ldg).
__global__ void __launch_bounds__(RA_THREADS)
rand_augment_u8_kernel(uint8_t* frames, const vt_randaug_desc* __restrict__ descs, int32_t* err, int T, int S) {
  extern __shared__ __align__(16) uint8_t px[];
  __shared__ unsigned int stat[3 * 256];                   // histograms, or the grayscale sum / per-channel min, max
  __shared__ uint8_t lut[3 * 256];
  const vt_randaug_desc& d = descs[blockIdx.x / T];
  const int npx = S * S;
  const int nbytes = npx * 3;
  uint8_t* g = frames + (int64_t)blockIdx.x * nbytes;
  const int n_ops = d.n_ops;
  bool ok = n_ops >= 0 && n_ops <= VT_RANDAUG_MAX_OPS;
  for (int s = 0; ok && s < n_ops; ++s) ok = d.op[s] >= 0 && d.op[s] < RA_NUM_OPS;
  if (!ok) {
    if (threadIdx.x == 0 && err) *err = 1;
    for (int k = threadIdx.x; k < nbytes; k += blockDim.x) g[k] = 0;
    return;
  }
  const bool vec = (nbytes % 16) == 0 && (reinterpret_cast<uintptr_t>(g) % 16) == 0;
  bool loaded = false, dirty = false;                      // px holds the frame / px is newer than g
  const float off = __fsub_rn(0.5f, __fmul_rn(0.5f, (float)S));        // x of column 0: -S/2 + 0.5
  for (int s = 0; s < n_ops; ++s) {
    const int op = d.op[s];
    if (op == RA_IDENTITY || (op == RA_SHARPNESS && S <= 2)) continue;
    if (!loaded) {
      copy_frame(px, g, nbytes, vec);
      __syncthreads();
      loaded = true;
    }
    const float r = d.arg[s], rc = d.one_minus[s];
    if (op <= RA_ROTATE || op == RA_SHARPNESS) {           // gather from px into g, then reload px if an op follows
      const float* th = d.theta[s];
      for (int p = threadIdx.x; p < npx; p += blockDim.x) {
        const int row = p / S, col = p % S;
        const uint8_t* q = px + 3 * p;
        uint8_t o0, o1, o2;
        if (op == RA_SHARPNESS) {
          const float c0 = q[0], c1 = q[1], c2 = q[2];
          float y0 = c0, y1 = c1, y2 = c2;
          if (row > 0 && row < S - 1 && col > 0 && col < S - 1) {
            int n0 = 0, n1 = 0, n2 = 0;                    // 3 x 3 sum plus 4 x centre: 13 x the blur
            for (int dy = -1; dy <= 1; ++dy)
              for (int dx = -1; dx <= 1; ++dx) {
                const uint8_t* e = q + 3 * (dy * S + dx);
                n0 += e[0], n1 += e[1], n2 += e[2];
              }
            n0 += 4 * q[0], n1 += 4 * q[1], n2 += 4 * q[2];
            y0 = (float)((2 * n0 + 13) / 26), y1 = (float)((2 * n1 + 13) / 26), y2 = (float)((2 * n2 + 13) / 26);
          }
          o0 = blend_u8(c0, y0, r, rc), o1 = blend_u8(c1, y1, r, rc), o2 = blend_u8(c2, y2, r, rc);
        } else {
          const float x = __fadd_rn((float)col, off), y = __fadd_rn((float)row, off);
          const int sx = nearest_source(__fadd_rn(__fadd_rn(__fmul_rn(x, th[0]), __fmul_rn(y, th[1])), th[2]), S);
          const int sy = nearest_source(__fadd_rn(__fadd_rn(__fmul_rn(x, th[3]), __fmul_rn(y, th[4])), th[5]), S);
          if (sx >= 0 && sy >= 0) {
            const uint8_t* e = px + 3 * (sy * S + sx);
            o0 = e[0], o1 = e[1], o2 = e[2];
          } else {
            o0 = o1 = o2 = 0;
          }
        }
        g[3 * p] = o0, g[3 * p + 1] = o1, g[3 * p + 2] = o2;
      }
      __syncthreads();
      dirty = false;
      loaded = false;
      continue;
    }
    float mean = 0.f;
    if (op == RA_CONTRAST || op == RA_AUTOCONTRAST || op == RA_EQUALIZE) {
      for (int k = threadIdx.x; k < 3 * 256; k += blockDim.x) stat[k] = op == RA_AUTOCONTRAST && k < 3 ? 255u : 0u;
      __syncthreads();
      if (op == RA_CONTRAST) {
        unsigned int part = 0;
        for (int p = threadIdx.x; p < npx; p += blockDim.x) part += (unsigned int)gray_u8(px[3 * p], px[3 * p + 1], px[3 * p + 2]);
        part = __reduce_add_sync(0xffffffffu, part);
        if ((threadIdx.x & 31) == 0) atomicAdd(&stat[0], part);
      } else if (op == RA_AUTOCONTRAST) {
        unsigned int mn0 = 255, mn1 = 255, mn2 = 255, mx0 = 0, mx1 = 0, mx2 = 0;
        for (int p = threadIdx.x; p < npx; p += blockDim.x) {
          const unsigned int c0 = px[3 * p], c1 = px[3 * p + 1], c2 = px[3 * p + 2];
          mn0 = min(mn0, c0), mn1 = min(mn1, c1), mn2 = min(mn2, c2);
          mx0 = max(mx0, c0), mx1 = max(mx1, c1), mx2 = max(mx2, c2);
        }
        mn0 = __reduce_min_sync(0xffffffffu, mn0), mn1 = __reduce_min_sync(0xffffffffu, mn1);
        mn2 = __reduce_min_sync(0xffffffffu, mn2), mx0 = __reduce_max_sync(0xffffffffu, mx0);
        mx1 = __reduce_max_sync(0xffffffffu, mx1), mx2 = __reduce_max_sync(0xffffffffu, mx2);
        if ((threadIdx.x & 31) == 0) {
          atomicMin(&stat[0], mn0), atomicMin(&stat[1], mn1), atomicMin(&stat[2], mn2);
          atomicMax(&stat[3], mx0), atomicMax(&stat[4], mx1), atomicMax(&stat[5], mx2);
        }
      } else {
        for (int p = threadIdx.x; p < npx; p += blockDim.x) {
          atomicAdd(&stat[px[3 * p]], 1u);
          atomicAdd(&stat[256 + px[3 * p + 1]], 1u);
          atomicAdd(&stat[512 + px[3 * p + 2]], 1u);
        }
      }
      __syncthreads();
      if (op == RA_CONTRAST) mean = __fdiv_rn((float)stat[0], (float)npx);
      if (op == RA_EQUALIZE) {
        if (threadIdx.x < 96) equalize_lut(stat + 256 * (threadIdx.x >> 5), lut + 256 * (threadIdx.x >> 5), npx);
        __syncthreads();
      }
    }
    const unsigned int mask = op == RA_POSTERIZE ? (unsigned int)r : 0u;
    for (int p = threadIdx.x; p < npx; p += blockDim.x) {
      uint8_t* q = px + 3 * p;
      if (op == RA_POSTERIZE) {
        q[0] &= mask, q[1] &= mask, q[2] &= mask;
      } else if (op == RA_SOLARIZE) {
        for (int c = 0; c < 3; ++c) q[c] = (float)q[c] >= r ? 255 - q[c] : q[c];
      } else if (op == RA_AUTOCONTRAST) {
        for (int c = 0; c < 3; ++c) {
          const unsigned int mn = stat[c], mx = stat[3 + c];
          if (mx != mn) {
            // torch evaluates 255 / (max - min) as reciprocal(max - min) * 255
            const float v = __fmul_rn((float)(q[c] - mn), __fmul_rn(__frcp_rn((float)(mx - mn)), 255.f));
            q[c] = (uint8_t)__float2uint_rz(fminf(fmaxf(v, 0.f), 255.f));
          }
        }
      } else if (op == RA_EQUALIZE) {
        q[0] = lut[q[0]], q[1] = lut[256 + q[1]], q[2] = lut[512 + q[2]];
      } else {                                             // brightness, color (saturation), contrast
        const float c0 = q[0], c1 = q[1], c2 = q[2];
        const float y = op == RA_BRIGHTNESS ? 0.f : op == RA_CONTRAST ? mean : gray_u8(c0, c1, c2);
        q[0] = blend_u8(c0, y, r, rc), q[1] = blend_u8(c1, y, r, rc), q[2] = blend_u8(c2, y, r, rc);
      }
    }
    __syncthreads();
    dirty = true;
  }
  if (dirty) copy_frame(g, px, nbytes, vec);
}

}  // namespace vt

extern "C" int vt_resized_crop_u8(const vt_resized_crop_params* p, void* stream) {
  using namespace vt;
  VT_REQUIRE(p && p->src && p->desc && p->out, "vt_resized_crop_u8: null pointer");
  VT_REQUIRE(p->n > 0 && p->T > 0 && p->S > 0 && p->S <= 512, "vt_resized_crop_u8: bad sizes n=%d T=%d S=%d (S <= 512)",
             p->n, p->T, p->S);
  VT_REQUIRE((int64_t)p->n * p->T < (1ll << 31), "vt_resized_crop_u8: too many frames");
  const size_t smem = (size_t)MAXT * (p->S + CROP_ROWS) * sizeof(float) + (size_t)(2 * p->S + 2 * CROP_ROWS) * sizeof(int);
  cudaFuncSetAttribute(resized_crop_u8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  dim3 grid(p->n * p->T, (p->S + CROP_ROWS - 1) / CROP_ROWS);
  resized_crop_u8_kernel<<<grid, CROP_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      p->src, p->src_bytes, p->desc, p->out, p->err, p->T, p->S);
  return check_launch("resized_crop_u8_kernel");
}

extern "C" int vt_color_jitter_u8(const vt_color_jitter_params* p, void* stream) {
  using namespace vt;
  VT_REQUIRE(p && p->frames && p->desc, "vt_color_jitter_u8: null pointer");
  VT_REQUIRE(p->n > 0 && p->T > 0 && p->S > 0, "vt_color_jitter_u8: bad sizes n=%d T=%d S=%d", p->n, p->T, p->S);
  VT_REQUIRE(p->S <= 256, "vt_color_jitter_u8: S=%d > 256 (the frame must fit in shared memory and its grayscale sum in "
             "fp32's exact integers)", p->S);
  const size_t smem = (size_t)p->S * p->S * 3;
  cudaFuncSetAttribute(color_jitter_u8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  color_jitter_u8_kernel<<<p->n * p->T, JITTER_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      p->frames, p->desc, p->T, p->S);
  return check_launch("color_jitter_u8_kernel");
}

extern "C" int vt_rand_augment_u8(const vt_rand_augment_params* p, void* stream) {
  using namespace vt;
  VT_REQUIRE(p && p->frames && p->desc, "vt_rand_augment_u8: null pointer");
  VT_REQUIRE(p->n > 0 && p->T > 0 && p->S > 0, "vt_rand_augment_u8: bad sizes n=%d T=%d S=%d", p->n, p->T, p->S);
  VT_REQUIRE(p->S <= 256, "vt_rand_augment_u8: S=%d > 256 (the frame must fit in shared memory and its grayscale sum in "
             "fp32's exact integers)", p->S);
  VT_REQUIRE((int64_t)p->n * p->T < (1ll << 31), "vt_rand_augment_u8: too many frames");
  const size_t smem = (size_t)p->S * p->S * 3;
  cudaFuncSetAttribute(rand_augment_u8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  rand_augment_u8_kernel<<<p->n * p->T, RA_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      p->frames, p->desc, p->err, p->T, p->S);
  return check_launch("rand_augment_u8_kernel");
}
