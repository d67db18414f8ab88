/*
 * vt_b200.h — C ABI of the H100 (sm_90a) video-transformer hot-path kernels.
 *
 * Drop-in boundary (SURVEY.md §8b): the reference has no FFI layer of its own — its hot path is the
 * forward/backward of the nn.Modules in transformer.py / video_transformer.py, executed by stock
 * ATen/cuBLAS/cuDNN calls.  This library is what a maintainer binds *underneath* those modules
 * (ctypes stub in INTEGRATION.md); each entry point names the reference call site it replaces
 * (paths relative to the reference repo root).
 *
 * Conventions
 *  - every function: int fn(const <params>*, void* cuda_stream); 0 = ok, non-zero = error
 *    (message via vt_last_error).  No exceptions, no abort, no fallback: unsupported shapes are errors.
 *  - all pointers are device pointers owned by the caller (PyTorch caching allocator); kernels are
 *    enqueued on `cuda_stream` and never allocate, free, synchronise or retain pointers.
 *  - bf16 = raw uint16 storage of __nv_bfloat16; "rows" are contiguous along the last dimension.
 *  - re-entrant: callable from the Python main thread (forward) and the autograd thread (backward).
 */
#ifndef VT_B200_H
#define VT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VT_ABI_VERSION 1

int vt_version(void);
/* copies the calling thread's last error message (NUL terminated) into buf; returns its length */
int vt_last_error(char* buf, size_t buf_bytes);
/* number of SMs of the current device (grid sizing is done inside the library) */
int vt_sm_count(void);
/* run the persistent GEMM on vt_sm_count() - n SMs (grid size, tile shape and split-K planned for that many); 0 restores the
 * default.  The other n SMs stay free for concurrent kernels (the NCCL all-reduce overlapped with the backward) */
int vt_set_reserved_sms(int n);
/* number of kernels this library has launched in this process (mod 2^31); bench.py's gpu_launches */
int vt_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * GEMM on Hopper tensor cores (wgmma):  acc[M,N] = sum_k A[m,k] * B[n,k]   (bf16 x bf16 -> fp32 in registers)
 * Operands are fed by TMA into 128B-swizzled shared memory.
 *   a_mn_major = 0 : A stored row-major [M, K] (leading dim lda)      "K-major"
 *   a_mn_major = 1 : A stored row-major [K, M] (leading dim lda)      "MN-major" (no transpose copy)
 *   b_mn_major = 0 : B stored row-major [N, K] (leading dim ldb)      (nn.Linear weight layout)
 *   b_mn_major = 1 : B stored row-major [K, N]
 * Replaces: nn.Linear forward (F.linear -> cuBLASLt addmm) at transformer.py:167 (qkv), :175 (proj),
 *   :267 (temporal_fc), :501-505 (FFN), the Conv2d/Conv3d patch projection :116-126 after im2col,
 *   and autograd's dgrad / wgrad GEMMs of the same layers.
 *
 * Epilogues (fused, applied to the accumulator registers):
 *   VT_EPI_BF16  : out_bf16[orow(m), n]  = s(m) * (acc + bias[n])
 *   VT_EPI_F32   : out_f32 [orow(m), n]  = s(m) * (acc + bias[n]) + (aux ? aux_f32[arow(m), n] : 0)
 *                  (residual add / pos+time-embed add / fp32 gradients)
 *   VT_EPI_GELU_H: out_bf16[orow(m), n] = gelu_erf(bf16(s(m) * (acc + bias[n])))  — forward-only FC1: h alone, z is not
 *                  written.  Bit for bit VT_EPI_BF16 followed by vt_gelu_fwd_bf16 (same per-element code, same tiles).
 * orow(m) = out_row ? out_row[m] : m  (negative => row skipped);  arow likewise (negative => no addend);  s(m) = row_scale ? row_scale[m] : 1
 * (row_scale carries DropPath's per-row mask/keep factor, transformer.py:34-42, and the 1/T of the cls mean :371-373).
 *
 * Split-K: when `workspace` is given and the tile count under-fills the GPU (weight gradients:
 * K = tokens), K is split; partial tiles go to the fp32 workspace and are summed by a second kernel.
 * Only with VT_EPI_F32, no row maps.
 *
 * Epilogue values 2 and 3 are unassigned and rejected; the others keep their numbers for ABI compatibility.
 * ------------------------------------------------------------------------------------------- */
enum { VT_EPI_BF16 = 0, VT_EPI_F32 = 1, VT_EPI_GELU_H = 4 };

typedef struct {
  const void* a;      /* bf16 */
  const void* b;      /* bf16 */
  int64_t lda, ldb;   /* leading dims in elements (multiples of 8) */
  int32_t M, N, K;
  int32_t a_mn_major, b_mn_major;
  int32_t epilogue;
  const float* bias;       /* [N] or NULL */
  void* out;               /* bf16 or fp32 per epilogue */
  void* out2;              /* unused; kept for ABI compatibility */
  const void* aux;         /* fp32, VT_EPI_F32 only (rejected with the other epilogues), or NULL */
  int64_t ldo, ldo2, ldaux;  /* ldo2: unused; kept for ABI compatibility */
  const int32_t* out_row;  /* [M] or NULL */
  const int32_t* aux_row;  /* [M] or NULL */
  const float* row_scale;  /* [M] or NULL */
  void* workspace;         /* fp32 scratch for split-K or NULL */
  int64_t workspace_bytes;
  int32_t force_splits;    /* 0 = heuristic, >0 = exactly this many K splits (tests) */
  int32_t force_bn;        /* 0 = heuristic, 128 / 192 / 256 (tests) */
  int32_t force_cluster;   /* unused; kept for ABI compatibility */
  void* debug;             /* unused; kept for ABI compatibility */
  /* Affine description of out_row / aux_row for VT_EPI_F32 with aux (the residual scatter of the divided space-time blocks),
   * map_period = 0: none.  GEMM row m -> outer = m / map_period, inner = m % map_period.  Rows with inner < map_skip are
   * "special" (the per-frame cls replicas of the spatial pass): no addend, written to out + map_special_base +
   * outer * map_special_stride (dropped when map_special_base < 0).  Every other row reads its addend from / writes its
   * result to element offset  map_base + (outer % map_tcount) * map_stride_t + (inner - map_skip) * map_stride_p +
   * (outer / map_tcount) * map_stride_b  of aux / out: the einops regroupings of the token stream (reference
   * transformer.py:250, :279-280, :352-356, :375-377) computed in the epilogue instead of read from index arrays; the
   * out_row / aux_row arrays, when also given, must describe the same mapping. */
  int32_t map_period, map_skip, map_tcount;
  int32_t force_tail;      /* unused; kept for ABI compatibility */
  int64_t map_stride_t, map_stride_p, map_stride_b, map_base;
  int64_t map_special_base, map_special_stride;
  const float* bias2;      /* VT_EPI_F32 with aux only: out = s(m) * (acc + bias[n]) + bias2[n] + aux — the bias of a second
                              linear layer folded into this GEMM (temporal_fc after proj, transformer.py:264-267) */
  int32_t out_zeroed;      /* accepted for ABI compatibility: split-K partials are summed from `workspace` into `out` */
} vt_gemm_params;

int vt_gemm(const vt_gemm_params* p, void* stream);

/* ---------------------------------------------------------------------------------------------
 * FP8 forward GEMM (inference forms of the block linears):  acc[M,N] = sum_k A[m,k] * B[n,k] with e4m3 operands, then
 *   acc <- acc * (a_scale[m] * b_scale[n])   (per-token scale of A, per-output-channel scale of B)
 * followed by the per-element code of VT_EPI_BF16 / VT_EPI_F32 / VT_EPI_GELU_H exactly as vt_gemm applies it (bias,
 * bias2, row_scale, row maps, affine map, staged or register epilogue).  g.a / g.b point to e4m3 bytes (raw
 * __nv_fp8_e4m3), lda / ldb in elements; both operands K-major (a_mn_major = b_mn_major = 0).  Each 128-wide k-block
 * is accumulated by 4 x wgmma k32 into a fresh fp32 register tile and then added on the CUDA cores to the tile's fp32
 * accumulator.  K % 16 == 0, lda % 16 == 0, ldb % 16 == 0, 16-byte aligned bases.  No split-K: workspace is ignored.
 * sm_90 only.
 * ------------------------------------------------------------------------------------------- */
typedef struct { vt_gemm_params g; const float* a_scale; const float* b_scale; } vt_gemm_e4m3_params;
int vt_gemm_e4m3(const vt_gemm_e4m3_params* p, void* stream);

/* Row quantiser of the fp8 forms: x bf16 (x_fp32 = 0) or fp32 [M, K] (leading dim ldx) -> q e4m3 [M, K] (leading dim
 * ldq) and scale fp32 [M], one warp per row:
 *   amax = max_k |x[m,k]|;  scale[m] = 2^ceil(log2(amax / 448)) clamped to [2^-126, 2^127], 1 for an all-zero row;
 *   q[m,k] = e4m3_rn_satfinite(x[m,k] / scale[m])   (x / scale is exact: the cast is the only rounding).
 * Serves activations (per token) and weights (per output channel).  K % 16 == 0; x and q rows 16-byte aligned. */
typedef struct { const void* x; int32_t x_fp32; int64_t ldx; void* q; int64_t ldq; float* scale; int32_t M, K; } vt_quant_rows_params;
int vt_quant_rows_e4m3(const vt_quant_rows_params* p, void* stream);

/* ---------------------------------------------------------------------------------------------
 * LayerNorm over the last dim (biased variance), fp32 statistics, one warp per row.
 * Replaces nn.LayerNorm at transformer.py:257 / :359 / :439 / :519 and video_transformer.py:251,
 * fused with the einops regroupings around it (transformer.py:250, :352-356): row m of the output
 * is the normalised row in_row[m] of x, so '(b t) p' / '(b p) t' orders and the per-frame cls copy
 * cost no separate pass.
 *   y_bf16[m,:] = (x[in_row ? in_row[m] : m, :] - mean) * rstd * gamma + beta ;  mean/rstd saved.
 * mean / rstd may both be NULL: not written (forward-only calls; only the backward reads them).
 * D must be a multiple of 128 and <= 1024.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  const float* x; int64_t ldx;
  const int32_t* in_row;
  const float* gamma; const float* beta;
  void* y;            /* bf16 [rows, D] (or fp32 when y_fp32 != 0) */
  float* mean; float* rstd;   /* [rows] */
  int32_t rows, D;
  float eps;
  int32_t y_fp32;
} vt_ln_fwd_params;
int vt_layernorm_fwd(const vt_ln_fwd_params* p, void* stream);

/* LayerNorm backward.  g = dy*gamma ; dx = rstd*(g - mean(g) - xhat*mean(g*xhat)).
 * Scatter: t = out_row ? out_row[m] : m.
 *   t >= 0 : dx[t,:]        = dx_row + (dres ? dres[t,:] : 0)      (adds the residual-path gradient)
 *   t <  0 : dx_aux[-t-1,:] = dx_row                                (replicated cls rows, summed by caller)
 * dgamma/dbeta: per-CTA partials into `partials` ([blocks, 2, D] fp32, blocks = vt_ln_bwd_blocks()),
 * then reduce with vt_reduce_rows. */
typedef struct {
  const void* dy; int32_t dy_fp32;      /* bf16 [rows, D] (fp32 if dy_fp32) */
  const float* x; int64_t ldx; const int32_t* in_row;
  const float* mean; const float* rstd; const float* gamma;
  const float* dres; float* dx; int64_t lddx;
  float* dx_aux;
  const int32_t* out_row;
  float* partials;
  int32_t rows, D;
} vt_ln_bwd_params;
int vt_ln_bwd_blocks(int32_t rows);
int vt_layernorm_bwd(const vt_ln_bwd_params* p, void* stream);

/* out[j] = (accumulate ? out[j] : 0) + scale * sum_{s<S} in[s*stride + j],  j < n (n % 4 == 0) */
typedef struct { const float* in; float* out; int64_t stride; int32_t S; int64_t n; int32_t accumulate; float scale; } vt_reduce_params;
int vt_reduce_rows(const vt_reduce_params* p, void* stream);

/* Column sums of a bf16 [M,N] matrix (bias gradients): out_f32[n] = sum_m in[m,n].
 * workspace: fp32 [vt_colsum_chunks(M), N].  Deterministic (fixed summation order) in both forms. */
typedef struct { const void* in; int64_t ld; int32_t M, N; float* out; float* workspace;
                 int32_t* counters; /* optional: >= ceil(N/64) zeroed ints -> single-launch form (the last CTA sums the partials and
                                       re-zeroes its counter); NULL -> partials are reduced by a second launch */ } vt_colsum_params;
int vt_colsum_chunks(int32_t M);
int vt_colsum_bf16(const vt_colsum_params* p, void* stream);

/* fp32 -> bf16 casts.  vt_cast: flat.  vt_gather_cast: out[m,:] = bf16(src[in_row[m],:] * row_scale[m])
 * (gradient of the residual scatter + DropPath scale; in_row < 0 => zeros). */
typedef struct { const float* src; void* dst; int64_t n; } vt_cast_params;
int vt_cast_f32_bf16(const vt_cast_params* p, void* stream);
typedef struct { const float* src; int64_t lds; const int32_t* in_row; const float* row_scale; void* dst; int32_t rows, D; } vt_gather_cast_params;
int vt_gather_cast_bf16(const vt_gather_cast_params* p, void* stream);

/* Exact-erf GELU on bf16 (nn.GELU default, transformer.py:483 / :502) as stand-alone bandwidth kernels:
 *   vt_gelu_fwd_bf16: out = gelu(z)            vt_gelu_bwd_bf16: out = dh * gelu'(z)
 * These are the FFN's activation in training: FC1 writes z with VT_EPI_BF16 and vt_gelu_fwd_bf16 computes h from it;
 * the backward takes dz from vt_gelu_bwd_bf16, or from vt_gelu_bwd_colsum_bf16 together with FC1's bias gradient.  Only
 * the forward-only FC1 computes h in the GEMM (VT_EPI_GELU_H).  n = element count (n % 8 == 0). */
typedef struct { const void* z; const void* dh; void* out; int64_t n; } vt_gelu_params;
int vt_gelu_fwd_bf16(const vt_gelu_params* p, void* stream);
int vt_gelu_bwd_bf16(const vt_gelu_params* p, void* stream);

/* cls rows of the divided space-time blocks in one launch:  dst[b, :] = src[b, :] + scale * sum_t extra[b, t, :]
 * (extra NULL: row copy).  src / dst: fp32 rows b * stride apart; extra: fp32 [B, T, D] with batch stride extra_bs.
 * Replaces the cls passthrough of the temporal block and `cls + mean_t(cls replicas)` of the spatial block
 * (transformer.py:282-283, :371-377) and their adjoints. */
typedef struct { const float* src; int64_t src_stride; const float* extra; int64_t extra_bs; int32_t T; float scale;
                 float* dst; int64_t dst_stride; int32_t B, D; } vt_cls_rows_params;
int vt_cls_rows(const vt_cls_rows_params* p, void* stream);

/* The two producers of a layer's dY that also emit its column sums (= the bias gradient autograd's sum over tokens gives
 * nn.Linear, transformer.py:175 / :267 / :505 / :501): vt_gather_cast_bf16 + vt_colsum_bf16, and vt_gelu_bwd_bf16 +
 * vt_colsum_bf16, in one pass each.  colsum fp32 [D] / [N]; workspace fp32 [workspace_rows, D] with workspace_rows >=
 * vt_*_blocks(rows).  Sums are over the bf16-rounded outputs, in a fixed order. */
typedef struct { const float* src; int64_t lds; const int32_t* in_row; const float* row_scale; void* dst; int32_t rows, D;
                 float* colsum; float* workspace; int32_t workspace_rows;
                 int32_t unscaled_sums;   /* 1: colsum is [2, D] — row 1 = sums of the rows before row_scale; workspace [rows, 2 D] */
               } vt_gather_cast_colsum_params;
int vt_gather_cast_colsum_blocks(int32_t rows);
int vt_gather_cast_colsum_bf16(const vt_gather_cast_colsum_params* p, void* stream);
typedef struct { const void* z; const void* dh; void* out; int32_t M, N; float* colsum; float* workspace;
                 int32_t workspace_rows; } vt_gelu_bwd_colsum_params;
int vt_gelu_bwd_colsum_blocks(int32_t M);
int vt_gelu_bwd_colsum_bf16(const vt_gelu_bwd_colsum_params* p, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Multi-head softmax attention core on a packed qkv tensor (no projection):
 *   qkv bf16 [Bp, N, 3, H, hd] (the layout produced by transformer.py:167's reshape), hd = 32, 64, 96 or 128 (every
 *   kernel below at each; other widths are refused)
 *   ctx bf16 [Bp, N, H*hd] = softmax(q k^T * scale) v      (transformer.py:170-174)
 *   lse fp32 [Bp, H, N]   (saved for backward; NULL = not written, for every implementation);
 *   probs fp32 [Bp,H,N,N] optional (Attention returns it, :177; get_last_selfattention, video_transformer.py:258-261)
 * Three kernels behind one entry point: tensor-core flash kernels for any N > 32 (the spatial pass N = 197, the joint
 * space-time pass N = 1569; mma.sync bf16 with fp32 accumulators, K/V tiles double-buffered in shared memory by cp.async,
 * vt_attention_mma.cu), a warp-per-problem kernel for the temporal pass (N = 8, 18 816 problems/layer), and a generic
 * warp-per-query kernel for N <= 256 (ViViT N = 9, probs output; its backward at hd 128 holds up to N = 208).  The
 * whole-problem tensor-core kernels take hd 64 only; other widths run the 64-row tiles.  With the tensor-core kernels the
 * probs output comes from a row-tile softmax kernel that fits 8 rows of scores in shared memory (N <= ~5000).
 * VT_ATTN_TCGEN05 selects the tensor-core kernel (the name is kept for ABI compatibility).
 * ------------------------------------------------------------------------------------------- */
enum { VT_ATTN_AUTO = 0, VT_ATTN_GENERIC = 1, VT_ATTN_TCGEN05 = 2, VT_ATTN_WARP8 = 3 };
typedef struct {
  const void* qkv; void* ctx; float* lse; float* probs;
  int32_t Bp, N, H, hd; float scale;
  int32_t impl;   /* VT_ATTN_AUTO picks: N > 256 -> tensor-core kernel (probs included); else probs -> generic;
                     N == 8 -> warp-per-problem kernel; N > 32 -> tensor-core kernel; else generic */
} vt_attn_fwd_params;
int vt_attn_fwd(const vt_attn_fwd_params* p, void* stream);
typedef struct {
  const void* qkv; const void* ctx; const void* dctx; const float* lse; void* dqkv;
  int32_t Bp, N, H, hd; float scale;
  int32_t impl;
} vt_attn_bwd_params;
int vt_attn_bwd(const vt_attn_bwd_params* p, void* stream);
/* The cls row of the probs output alone and show_attn's threshold masks: vt_attn_maps.h. */

/* ---------------------------------------------------------------------------------------------
 * Patch / tubelet embedding operand: non-overlapping Conv2d k16 s16 (transformer.py:116-120,:145-147)
 * or Conv3d k(tube,16,16) (:122-126,:141-143) == im2col + GEMM.
 *   x fp32 [B, T, C, H, W] -> cols bf16 [B*(T/tube)*(H/ph)*(W/pw), C*tube*ph*pw], k = ((c*tube+dt)*ph+i)*pw+j
 * vt_col2im is its adjoint (gradient w.r.t. the clip), fp32 out, from fp32 cols.
 * ------------------------------------------------------------------------------------------- */
typedef struct { const float* x; void* cols; int32_t B, T, C, H, W, tube, ph, pw; } vt_im2col_params;
int vt_im2col_bf16(const vt_im2col_params* p, void* stream);
/* Same operand from the decoder's uint8 clip (SURVEY §8f rank 2; data_transform.py:52-64 ToTensor + :534-539 Normalize fused in):
 *   x u8 [B, T, H, W, C] (channels last) -> cols[row, k] = bf16(x * scale[c] + shift[c]),  scale = 1/(255 std), shift = -mean/std */
typedef struct { const uint8_t* x; const float* scale; const float* shift; void* cols; int32_t B, T, C, H, W, tube, ph, pw; } vt_im2col_u8_params;
int vt_im2col_u8_bf16(const vt_im2col_u8_params* p, void* stream);
typedef struct { const float* cols; float* dx; int32_t B, T, C, H, W, tube, ph, pw; } vt_col2im_params;
int vt_col2im_f32(const vt_col2im_params* p, void* stream);

/* ---------------------------------------------------------------------------------------------
 * MaskFeat HOG target (dataset.py:39-45 -> skimage.feature.hog x3 + 2x2 cell regroup).
 *   frames u8 [F, H, W, 3] (H, W multiples of 16) -> feat fp32 [F, H/16, W/16, 108]
 *   bins (optional) u8 [F, 3, H, W]: orientation bin 0..8 per pixel/channel, 9 = no bin
 *   lut u8 [511*511]: bin of integer gradient (gy+255, gx+255), built on the host with numpy
 * ------------------------------------------------------------------------------------------- */
typedef struct { const uint8_t* frames; const uint8_t* lut; float* feat; uint8_t* bins; int32_t F, H, W; } vt_hog_params;
int vt_hog(const vt_hog_params* p, void* stream);

/* =============================================================================================
 * MaskFeat / MViT path (SURVEY §8 a13-a15).  Block arithmetic = pytorchvideo MultiScaleBlock as configured at
 * video_transformer.py:764-785 (restated in oracle/mvit_oracle.py); head dim is 96 in every block.
 * vt_layernorm_fwd/bwd additionally accept D = 32..256 in steps of 32 (block widths 96 and 192) without row maps.
 * ============================================================================================= */

/* Depthwise Conv3d pooling of one of q/k/v + LayerNorm(hd)  (pytorchvideo _attention_pool, pool_mode="conv"):
 *   element (b, n, h, c) of the input lives at in[b*in_bs + n*in_rs + h*hd + c] (bf16; n = 0 is the cls row, rows
 *   1.. are the (T,Hin,Win) tokens, t-major) — i.e. a q/k/v slice of the fused projection output is read in place.
 *   pooled fp32 [B,H,1+Lo,hd] = cls row copied, other rows conv3d(kernel 3x3x3, stride (st,sh,sw), padding 1, groups=hd)
 *   out    bf16 [B,H,1+Lo,hd] = LayerNorm(pooled; gamma, beta, eps) over hd;  mean/rstd [B*H*(1+Lo)] saved.
 * Lo = To*Ho*Wo with To = (T + 2 - 3)/st + 1 etc.   w: fp32 [hd, 27] (nn.Conv3d weight [hd,1,3,3,3]).
 * pooled, mean and rstd are only read by vt_pool_bwd: all three NULL = none written (forward-only calls). */
typedef struct {
  const void* in; int64_t in_bs, in_rs;
  const float* w; const float* gamma; const float* beta;
  float* pooled; void* out; float* mean; float* rstd;
  int32_t B, H, hd, T, Hin, Win, st, sh, sw, To, Ho, Wo;
  float eps;
} vt_pool_fwd_params;
int vt_pool_fwd(const vt_pool_fwd_params* p, void* stream);

/* Backward of vt_pool_fwd.  dout: gradient of `out` (bf16, or fp32 if dout_fp32).  Produces
 *   din (bf16, addressed like `in` with din_bs/din_rs: every (b,n,h,:) is written), dw [hd,27], dgamma, dbeta [hd].
 * scratch: fp32, at least vt_pool_bwd_scratch(rows_out, hd) floats (dpooled + per-CTA partial sums). */
typedef struct {
  const void* dout; int32_t dout_fp32;
  const float* pooled; const float* mean; const float* rstd; const float* gamma;
  const void* in; int64_t in_bs, in_rs; const float* w;
  void* din; int64_t din_bs, din_rs;
  float* dw; float* dgamma; float* dbeta;
  float* scratch; int64_t scratch_floats;
  int32_t B, H, hd, T, Hin, Win, st, sh, sw, To, Ho, Wo;
} vt_pool_bwd_params;
int vt_pool_bwd_scratch(int32_t rows_out, int32_t hd);   /* floats */
int vt_pool_bwd(const vt_pool_bwd_params* p, void* stream);

/* Softmax attention with separate, strided Q / K / V and Nq != Nk (pooling attention):
 *   element (b, h, n, c) of q at q[b*q_bs + h*q_hs + n*q_rs + c] (bf16), same for k, v, o (and dout, dq).
 *   o = softmax(scale * q k^T) v ;  lse fp32 [B,H,Nq] = log sum exp(scale * q k^T)  (NULL = not written, both kernels).
 * Two implementations, head dim 64 or 96: tensor-core flash kernels (vt_attention_mma.cu, VT_XATTN_TCGEN05 — the name is
 * kept for ABI compatibility) and CUDA-core kernels for arbitrary strides (two threads per query row, K/V tiles staged in
 * shared memory). */
enum { VT_XATTN_AUTO = 0, VT_XATTN_SIMT = 1, VT_XATTN_TCGEN05 = 2 };
typedef struct {
  const void* q; const void* k; const void* v; void* o; float* lse;
  int64_t q_bs, q_hs, q_rs, k_bs, k_hs, k_rs, v_bs, v_hs, v_rs, o_bs, o_hs, o_rs;
  int32_t B, H, Nq, Nk, hd; float scale;
  int32_t impl;   /* VT_XATTN_AUTO: tensor-core kernels when every operand is token-major ([B,N,H*hd] slices) or head-major
                     contiguous ([B,H,N,hd]) with 16-byte aligned rows, else the CUDA-core kernels */
} vt_xattn_fwd_params;
int vt_xattn_fwd(const vt_xattn_fwd_params* p, void* stream);
/* dq: bf16 with its own strides.  dk, dv: fp32 [B,H,Nk,hd] contiguous (every element written by the call).
 * delta: fp32 scratch [B,H,Nq]. */
typedef struct {
  const void* q; const void* k; const void* v; const void* o; const void* dout; const float* lse;
  float* delta; void* dq; float* dk; float* dv;
  int64_t q_bs, q_hs, q_rs, k_bs, k_hs, k_rs, v_bs, v_hs, v_rs, o_bs, o_hs, o_rs, dq_bs, dq_hs, dq_rs;
  int32_t B, H, Nq, Nk, hd; float scale;
  int32_t impl;
} vt_xattn_bwd_params;
int vt_xattn_bwd(const vt_xattn_bwd_params* p, void* stream);

/* Skip-path MaxPool3d on the fp32 token stream (pytorchvideo MultiScaleBlock.pool_skip: kernel s+1, stride s, padding
 * k//2 per axis; cls row copied).  x [B,1+T*H*W,D] -> y [B,1+To*Ho*Wo,D]; idx u8 same shape as y = winning tap
 * ((dt*kh+dh)*kw+dw, first maximum in scan order like torch).  Backward routes dy to the winners.  idx NULL = winners not
 * recorded (forward-only calls). */
typedef struct {
  const float* x; float* y; uint8_t* idx;
  int32_t B, D, T, H, W, kt, kh, kw, st, sh, sw, To, Ho, Wo;
} vt_maxpool_fwd_params;
int vt_maxpool_fwd(const vt_maxpool_fwd_params* p, void* stream);
typedef struct {
  const float* dy; const uint8_t* idx; float* dx;
  int32_t B, D, T, H, W, kt, kh, kw, st, sh, sw, To, Ho, Wo;
} vt_maxpool_bwd_params;
int vt_maxpool_bwd(const vt_maxpool_bwd_params* p, void* stream);

/* Overlapping Conv3d patch embedding operand (create_conv_patch_embed, video_transformer.py:585-618: kernel (3,7,7),
 * stride (2,4,4), padding (1,3,3)):  x fp32 [B,T,C,H,W] (the clip as the reference receives it, before its
 * transpose(1,2) at :912) -> cols bf16 [B*To*Ho*Wo, Kpad], column ((c*kt+dt)*kh+dh)*kw+dw, zero padded to Kpad. */
typedef struct {
  const float* x; void* cols;
  int32_t B, T, C, H, W, kt, kh, kw, st, sh, sw, pt, ph, pw, To, Ho, Wo, Kpad;
} vt_im2col3d_params;
int vt_im2col3d_bf16(const vt_im2col3d_params* p, void* stream);
/* The same operand from the decoder's uint8 clip x [B,T,H,W,C] (channels last), in the reference's order:
 *   ToTensor + Normalize (data_transform.py:62-64, :534-539), v = ((u / 255) - mean[c]) / std[c], each op rounded to
 *   nearest in fp32 (bit for bit the reference's float clip);
 *   then the batch-level Mixup / CutMix of mixup.py:102-114 against sample B-1-b when plan != NULL (plan = device
 *   float[6] {mode, lam, yl, yh, xl, xh} as in vt_im2col_u8_mix_params; mode 1: v*lam + o*(1-lam) with (1-lam) taken
 *   in fp32, mode 2: o inside rows [yl,yh) x cols [xl,xh));
 *   then the transpose and Conv3d zero padding (video_transformer.py:912): a tap outside the clip is 0 in normalised space.
 *   Each value is rounded to bf16 once, after the blend.  cols as in vt_im2col3d_bf16 (16-byte aligned, Kpad % 8 == 0). */
typedef struct {
  const uint8_t* x; const float* mean; const float* std; const float* plan; void* cols;
  int32_t B, T, C, H, W, kt, kh, kw, st, sh, sw, pt, ph, pw, To, Ho, Wo, Kpad;
} vt_im2col3d_u8_params;
int vt_im2col3d_u8_bf16(const vt_im2col3d_u8_params* p, void* stream);

/* Token preparation (MaskFeat.forward_features :915-919 + SpatioTemporalClsPositionalEncoding):
 *   x[b,0,:]   = cls_token + pos_cls
 *   x[b,1+l,:] = t[b,l,:]*(1-w[b,l]) + mask_token*w[b,l] + pos_s[l % HW,:] + pos_t[l / HW,:]      (w NULL => 0)
 * t fp32 [B*L, C] (conv output incl. bias), x fp32 [B,1+L,C], L = T*HW.
 * Backward: dt bf16 [B*L, C] = dx[b,1+l,:]*(1-w[b,l]) (parameter-table gradients are plain reductions of dx). */
typedef struct {
  const float* t; const float* wmask; const float* mask_token; const float* cls_token;
  const float* pos_s; const float* pos_t; const float* pos_cls; float* x;
  int32_t B, T, HW, C;
} vt_mvit_tokens_fwd_params;
int vt_mvit_tokens_fwd(const vt_mvit_tokens_fwd_params* p, void* stream);
typedef struct { const float* dx; const float* wmask; void* dt; int32_t B, T, HW, C; } vt_mvit_tokens_bwd_params;
int vt_mvit_tokens_bwd(const vt_mvit_tokens_bwd_params* p, void* stream);

/* Masked MSE of MaskFeat.forward (video_transformer.py:882-901):
 *   pred fp32 [B, 1+t*h*w, dt*dc] (decoder output incl. the cls row), target fp32 [B, t*dt, h, w, dc],
 *   mask fp32 [B, t*dt, h, w] (already restricted to the cube centre frames, :889-896)
 *   num[0] = sum_{cells} mask * mean_dc (pred - target)^2        (the caller divides by mask.sum() + 1e-5)
 * Backward: dpred bf16 [B*(1+t*h*w), dt*dc] = coef[0] * mask * (pred - target), cls rows zero; coef is a device
 * scalar (2 * dloss / (dc * (mask.sum() + 1e-5))).  partials: fp32 scratch [vt_mse_blocks(cells) * 4]. */
typedef struct {
  const float* pred; const float* target; const float* mask; float* num; float* partials;
  int32_t B, t, dt, h, w, dc;
  /* fp64 variant (the reference's targets are fp64 numpy arrays, dataset.py:190, which makes its loss fp64,
   * video_transformer.py:899-901): target64 != NULL replaces `target`; differences, squares and all sums are then taken in
   * fp64 and the sum goes to num64[0]; `partials` must hold vt_mse_blocks(cells) * 4 doubles. */
  const double* target64; double* num64;
} vt_mse_fwd_params;
int vt_mse_blocks(int32_t cells);
int vt_mse_fwd(const vt_mse_fwd_params* p, void* stream);
typedef struct {
  const float* pred; const float* target; const float* mask; const float* coef; void* dpred;
  int32_t B, t, dt, h, w, dc;
  const double* target64;   /* fp64 targets (replaces `target`) or NULL */
} vt_mse_bwd_params;
int vt_mse_bwd(const vt_mse_bwd_params* p, void* stream);

/* =============================================================================================
 * Fused per-parameter gradient clipping + optimizer step (SURVEY §8f rank 1; reference model_trainer.py:155-170
 * clip_gradients + optimizer.py:33-38 SGD(momentum 0.9, nesterov) / AdamW(0.9, 0.999)).
 * Multi-tensor form: tensor i has parameter pptr[i], gradient gptr[i], state s1ptr[i] (momentum buffer / exp_avg) and
 * s2ptr[i] (exp_avg_sq), all fp32 device addresses stored as int64 in device arrays; `chunks` is a device table of
 * {int32 tensor, int32 len, int64 offset} (16 bytes each) covering every tensor, each tensor's chunks consecutive and in
 * offset order; lr / wd are per-tensor fp32 arrays.
 *   vt_opt_norm2 : norm2[i] = sum(grad_i^2)                          (the trainer's total norm = sqrt(sum_i norm2[i]))
 *                  one fp32 partial per chunk into `partials` (n_chunks floats), then each tensor's partials added in
 *                  chunk order: bitwise reproducible.  The update kernels do not read `partials`.
 *   vt_opt_sgd   : g = grad * min(1, clip / (sqrt(norm2) + 1e-6)) [clip > 0];  d = g + wd*p;  buf = first ? d : mom*buf + d;
 *                  p -= lr * (nesterov ? d + mom*buf : buf)           (torch.optim.SGD, dampening 0)
 *   vt_opt_adamw : p *= 1 - lr*wd;  m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;
 *                  p -= lr/bc1 * m / (sqrt(v)/sqrt(bc2) + eps)         (torch.optim.AdamW; bc_k = 1 - beta_k^step)
 * Gradients are read, never written back (the reference scales p.grad in place; nothing reads it afterwards).
 * hyper (optional): a device block of VT_OPT_HYPER_SIZE floats {clip, bc1, bc2, first_step (0 / 1), spare}.  When it is
 * given, vt_opt_sgd / vt_opt_adamw read those per-step scalars from it at run time and ignore the fields of the same
 * names (norm2 must then be given, and is read only where the block's clip is > 0), so a CUDA graph that recorded the
 * launch follows the values the host writes into the block between replays.  NULL: the fields are used, as always.
 * ============================================================================================= */
#define VT_OPT_HYPER_CLIP 0
#define VT_OPT_HYPER_BC1 1
#define VT_OPT_HYPER_BC2 2
#define VT_OPT_HYPER_FIRST_STEP 3
#define VT_OPT_HYPER_SIZE 5
typedef struct {
  const void* chunks; int32_t n_chunks; int32_t n_tensors;
  const int64_t* pptr; const int64_t* gptr; const int64_t* s1ptr; const int64_t* s2ptr;
  float* norm2; const float* lr; const float* wd;
  float clip, momentum, beta1, beta2, eps, bc1, bc2;
  int32_t nesterov, first_step;
  float* partials;          /* vt_opt_norm2 workspace: n_chunks floats */
  const float* hyper;       /* optional per-step scalars on the device, see above */
} vt_opt_params;
int vt_opt_norm2(const vt_opt_params* p, void* stream);
int vt_opt_sgd(const vt_opt_params* p, void* stream);
int vt_opt_adamw(const vt_opt_params* p, void* stream);

/* =============================================================================================
 * Classification head + loss, long-sequence attention maps, Mixup/CutMix operand (SURVEY §8 a18, f2, f4).
 * ============================================================================================= */

/* Skinny fp32 linear layer  y[M,N] = x[M,K] W[N,K]^T + b  (ClassificationHead.forward, transformer.py:78-80: 8 x 768 -> 400)
 * and its adjoints  dW = dy^T x, db = colsum(dy), dx = dy W  (dw / dx may be NULL to skip).  Warp-per-output GEMV on
 * the fp32 parameters themselves (no bf16 shadow); M <= 4096, K % 4 == 0, x / w / dw / dx 16-byte aligned (float4 rows). */
typedef struct { const float* x; const float* w; const float* b; float* y; int32_t M, N, K; } vt_linear_small_params;
int vt_linear_small_fwd(const vt_linear_small_params* p, void* stream);
typedef struct { const float* dy; const float* x; const float* w; float* dw; float* db; float* dx; int32_t M, N, K; } vt_linear_small_bwd_params;
int vt_linear_small_bwd(const vt_linear_small_bwd_params* p, void* stream);

/* Softmax cross-entropy, mean over rows: nn.CrossEntropyLoss (model_trainer.py:91, :208) with int64 `labels`, or timm's
 * SoftTargetCrossEntropy (:89) with fp32 `soft_targets` [M,N] (exactly one of the two).  One launch writes loss[0],
 * optional per-row losses and dlogits = d loss / d logits.  Row loss = sum_c t_c * log(sum_c e^(z_c - max z)) -
 * sum_c t_c (z_c - max z) over the classes with t_c != 0, so a -inf logit off the label gives torch's finite result.
 * Labels must lie in [0, N): any other label (torch's ignore_index -100 included) acts as a row of zero targets, whose
 * loss and dlogits are 0, and it still counts in the mean's 1/M. */
typedef struct {
  const float* logits; const int64_t* labels; const float* soft_targets;
  float* loss; float* row_loss; float* dlogits; int32_t M, N;
} vt_softmax_ce_params;
int vt_softmax_ce(const vt_softmax_ce_params* p, void* stream);
/* out[i] = in[i] * scalar[0] (device scalar: chain rule through the loss inside a captured graph) */
typedef struct { const float* in; const float* scalar; float* out; int64_t n; } vt_scale_params;
int vt_scale_by_scalar(const vt_scale_params* p, void* stream);

/* Top-k accuracy counters of an evaluation step (model_trainer.py validation_step / test_step):
 *   logits fp32 [B*V, C], row b*V + v = view v of clip b;  labels int64 [B]
 *   mean[b, :] = (sum_v logits[b*V + v, :]) * (1.0f / V)   (views summed in order, then scaled by the fp32 factor 1/V,
 *                which is how torch forms preds.view(-1, V, C).mean(1))
 *   probs fp32 [B, C] = softmax(mean[b, :])  (optional, NULL = not written)
 *   rank(b) = #{c : mean[b, c] > mean[b, label_b]};  hits[i] += #{b : rank(b) < k[i]} for i < n_k (n_k <= 4);  samples[0] += B
 * Counters are int64 device values accumulated with integer atomics (deterministic, graph-capturable).  A label outside
 * [0, C) or a NaN label score counts as a miss.  Against torch's test step (mean, softmax, topk on the probabilities) the
 * count can differ in two ways, both confined to near-ties: where two probabilities round to the same float, torch.topk
 * breaks the tie by index while this count ranks the label first among its equals; and where a reduction that sums the
 * views in another order gives a mean one ulp away, a class within that ulp of the label can change sides.  C <= 12000. */
typedef struct {
  const float* logits; const int64_t* labels; float* probs;
  int64_t* hits; int64_t* samples;
  int32_t B, V, C;
  int32_t n_k; int32_t k[4];
} vt_topk_hits_params;
int vt_topk_hits(const vt_topk_hits_params* p, void* stream);

/* vt_im2col_u8_bf16 with the batch-level Mixup / CutMix of mixup.py:102-114 folded in: sample b is blended with (mode 1,
 * lam*x + (1-lam)*x.flip(0)) or patched from (mode 2, box rows [yl,yh) x cols [xl,xh)) sample B-1-b after normalisation.
 * plan = device float[6] {mode, lam, yl, yh, xl, xh}. */
typedef struct {
  const uint8_t* x; const float* scale; const float* shift; const float* plan; void* cols;
  int32_t B, T, C, H, W, tube, ph, pw;
} vt_im2col_u8_mix_params;
int vt_im2col_u8_mix_bf16(const vt_im2col_u8_mix_params* p, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Bicubic resize of a positional-embedding grid (TimeSformer.interpolate_pos_encoding, video_transformer.py:171-191:
 * F.interpolate(mode='bicubic', align_corners=False, scale_factor=(scale_h, scale_w)) on the patch rows of pos_embed).
 * fp32 token-major rows, D contiguous: grid cell (y, x) of a gh x gw grid is row y * gw + x, read where it lies.
 *   vt_pos_resize_fwd: src = the gh x gw grid, dst = the oh x ow output (oh = floor(gh * scale_h), ow likewise).
 *   vt_pos_resize_bwd: src = the gradient of the oh x ow output, dst = the gradient of the gh x gw grid (every row
 *                      written; the exact adjoint, gathered per input cell: no atomics, deterministic).
 * Source coordinate (dst + 0.5) / scale - 0.5 (PyTorch's scale-factor form), cubic convolution A = -0.75, 4 x 4 taps
 * clamped to the grid, fp32 accumulation.  lds / ldd: row strides in elements.  oh + ow <= 8192.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  const float* src; int64_t lds;
  float* dst; int64_t ldd;
  int32_t gh, gw, oh, ow, D;
  double scale_h, scale_w;
} vt_pos_resize_params;
int vt_pos_resize_fwd(const vt_pos_resize_params* p, void* stream);
int vt_pos_resize_bwd(const vt_pos_resize_params* p, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Clip transforms on decode-resolution uint8 frames (the reference's DataLoader transforms, data_transform.py:495-615 and
 * data_trainer.py:75-115, as torchvision applies them to a uint8 T C H W clip).  Frames are HWC uint8.
 *
 * vt_resized_crop_u8: out [n, T, S, S, 3] uint8.  Output clip k reads the clip of desc[k]: frame t of it starts at byte
 * src + src_offset + t * H * pitch.  The crop box is resized to RH x RW with torchvision's antialiased filter (PIL's
 * formulation: bicubic a = -0.5 with support 2 * max(scale, 1), or bilinear with support max(scale, 1); weights computed
 * in fp32 and normalised by their sum, taps clamped at the crop box), width pass first with an fp32 intermediate, then
 * clamped and rounded half to even: what torchvision's resized_crop / resize give on uint8.  Only the S x S window at
 * (oy, ox) of the resized image is computed, mirrored left-right when flip is set.  An axis may need at most
 * VT_CROP_MAX_TAPS taps (2 * ceil(support) + 1 <= 32: bicubic downscale <= 7.5, bilinear <= 15).  A descriptor that
 * breaks a bound (taps, source bytes, window) makes its clip all zeros and sets *err (if given) to 1.
 * Launch: grid (n * T, ceil(S / 8)), 256 threads; S <= 512.
 *
 * vt_color_jitter_u8: torchvision ColorJitter on uint8, in place on frames [n, T, S, S, 3], one CTA per frame with the
 * frame resident in shared memory (S <= 256).  Clip k applies desc[k].op[0 .. n_ops) in order (0 brightness, 1 contrast,
 * 2 saturation), each _blend(x, y, r) = trunc(clamp(r * x + (1 - r) * y, 0, 255)) with the products and the sum rounded
 * separately in fp32; y is 0, the per-frame mean of the grayscale image (an exact integer sum, then one fp32 division),
 * or the grayscale image (0.2989 r + 0.587 g + 0.114 b, truncated).  one_minus[i] = fp32(1.0 - (double)factor[i]).
 *
 * vt_rand_augment_u8: torchvision RandAugment (NEAREST, fill None) on uint8, in place on frames [n, T, S, S, 3], one CTA
 * per frame with the frame resident in shared memory (S <= 256).  Clip k applies desc[k].op[0 .. n_ops) in order, with
 * torchvision's op index as the code: 0 Identity, 1 ShearX, 2 ShearY, 3 TranslateX, 4 TranslateY, 5 Rotate,
 * 6 Brightness, 7 Color, 8 Contrast, 9 Sharpness, 10 Posterize, 11 Solarize, 12 AutoContrast, 13 Equalize.
 *  - 1-5 sample the frame at nearest-rounded (half to even) source coordinates, zero outside: for the pixel centre
 *    (x, y) = (col - S/2 + 0.5, row - S/2 + 0.5), g = (x * theta[0] + y * theta[1]) + theta[2] (and theta[3..5] for
 *    the row), source = ((g + 1) * S - 1) / 2, every operation rounded separately in fp32.  theta is torchvision's
 *    inverse affine matrix rounded to fp32 and divided in fp32 by S / 2 (what _gen_affine_grid multiplies by).
 *  - 6-8 are ColorJitter's blends (above) with r = arg = fp32(1 + m), one_minus = fp32(1.0 - (1.0 + m)) in double.
 *  - 9 blends with the rounded [1 1 1; 1 5 1; 1 1 1] / 13 blur over interior pixels (each border pixel blends with
 *    itself); it is skipped when S <= 2.  The blur is computed exactly in integers: no blur of bytes lies within 1/26
 *    of a half-integer, so fp32 convolution rounds to the same value.
 *  - 10 keeps the bits of (int)arg, 11 inverts bytes >= arg (fp32 compare).
 *  - 12 and 13 work per frame and channel: 12 maps c to trunc((c - min) * s) with s = fp32(1 / (max - min)) * 255
 *    (torch's 255 / tensor is a reciprocal and a product), unless max == min;
 *    13 maps through torchvision's equalize table ((cumsum + step / 2) / step shifted right by one bin, lut[0] = 0,
 *    step = (pixels - count of the highest occupied bin) / 255) unless step == 0.
 * n_ops outside [0, VT_RANDAUG_MAX_OPS] or an op code outside [0, 13] makes the clip all zeros and sets *err (if given).
 * Launch: grid n * T, 512 threads, S * S * 3 bytes of dynamic shared memory.
 * ------------------------------------------------------------------------------------------- */
#define VT_CROP_MAX_TAPS 32
typedef struct {
  int64_t src_offset;                      /* bytes from vt_resized_crop_params.src to frame 0 of the clip */
  int32_t H, W, pitch;                     /* source frame size; row pitch in bytes (>= 3 W), frames H * pitch apart */
  int32_t crop_y, crop_x, crop_h, crop_w;  /* crop box inside the source frame */
  int32_t RH, RW;                          /* size the crop box is resized to */
  int32_t oy, ox;                          /* top-left of the S x S output window inside the RH x RW image */
  int32_t flip;                            /* 1: mirror the window left-right */
  int32_t filter;                          /* 0 bicubic, 1 bilinear */
  int32_t reserved;
} vt_crop_desc;
typedef struct {
  const uint8_t* src; int64_t src_bytes;   /* every byte a descriptor reads lies in [src, src + src_bytes) */
  const vt_crop_desc* desc;                /* device table, one per output clip */
  uint8_t* out;
  int32_t* err;                            /* optional device flag */
  int32_t n, T, S;
} vt_resized_crop_params;
int vt_resized_crop_u8(const vt_resized_crop_params* p, void* stream);

typedef struct {
  int32_t n_ops, op[3];
  float factor[3], one_minus[3];
} vt_jitter_desc;
typedef struct { uint8_t* frames; const vt_jitter_desc* desc; int32_t n, T, S; } vt_color_jitter_params;
int vt_color_jitter_u8(const vt_color_jitter_params* p, void* stream);

#define VT_RANDAUG_MAX_OPS 4
typedef struct {
  int32_t n_ops, op[VT_RANDAUG_MAX_OPS];
  float arg[VT_RANDAUG_MAX_OPS];           /* blend factor, posterize bit mask or solarize threshold */
  float one_minus[VT_RANDAUG_MAX_OPS];     /* blend ops: fp32(1.0 - (1.0 + m)) */
  float theta[VT_RANDAUG_MAX_OPS][6];      /* ops 1-5: the rescaled inverse affine matrix, row-major 2 x 3 */
} vt_randaug_desc;
typedef struct {
  uint8_t* frames;
  const vt_randaug_desc* desc;             /* device table, one per clip */
  int32_t* err;                            /* optional device flag */
  int32_t n, T, S;
} vt_rand_augment_params;
int vt_rand_augment_u8(const vt_rand_augment_params* p, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VT_B200_H */
