/*
 * vt_attn_maps.h — attention-map entry points of libvt_b200 (sm_90a): what visualize_attention.py consumes, computed on the
 * device without the [B', H, N, N] probability map.  Same conventions as vt_b200.h: a POD params struct per call, int
 * return code (0 = ok, message via vt_last_error), device pointers owned by the caller, enqueued on `stream`, no
 * allocation and no synchronisation (graph-capturable).
 */
#ifndef VT_ATTN_MAPS_H
#define VT_ATTN_MAPS_H

#include "vt_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Query row 0 (the cls token) of vt_attn_fwd's probs output alone (visualize_attention.py:71 keeps attentions[:, 0]):
 *   probs fp32 [Bp, H, N] = softmax_j(q_0 . k_j * scale), bit for bit row 0 of the [Bp, H, N, N] probs vt_attn_fwd writes
 *   for the same qkv (same device code as its route: the generic kernel's row function at N <= 256, the row-tile softmax
 *   kernel's score and softmax functions above).  qkv as in vt_attn_fwd (16-byte aligned), hd = 32, 64, 96 or 128.
 *   N >= 1; past 256 the CTA holds the score row and a 256-key tile in shared memory: N <= 24960 at hd 128 (joint
 *   attention at 16 x 448^2 is N = 12545).  One CTA per (batch', head). */
typedef struct {
  const void* qkv; float* probs;
  int32_t Bp, N, H, hd; float scale;
} vt_attn_cls_probs_params;
int vt_attn_cls_probs(const vt_attn_cls_probs_params* p, void* stream);

/* Threshold masks of show_attn (visualize_attention.py:73-82) per row of patch probabilities (finite, >= +0):
 *   row r = probs + r * ld, n entries; mask + r * ldm receives 1.0 where the entry is kept, else 0.0, in patch order.
 *   Kept: sorted ascending (ties by patch index), divided by the row sum, cumulative sum c_k > thresh.  thresh is
 *   show_attn's 1 - threshold rounded to fp32.  Equal to show_attn's torch arithmetic except where its cumulative mass
 *   lies within beta(n) = 1.01 (n + 5) 2^-24 of thresh, and up to the order of equal entries (bound derived in
 *   vt_attn_maps.cu).  1 <= n <= 16384, ld >= n, ldm >= n; one CTA per row. */
typedef struct {
  const float* probs; int64_t ld;
  float* mask; int64_t ldm;
  int32_t rows, n;
  float thresh;
} vt_attn_mass_mask_params;
int vt_attn_mass_mask(const vt_attn_mass_mask_params* p, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VT_ATTN_MAPS_H */
