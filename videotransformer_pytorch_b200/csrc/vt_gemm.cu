// Warp-specialised, persistent bf16 GEMM for sm_90a:
//   TMA (cp.async.bulk.tensor, 128B swizzle) -> shared-memory ring (mbarrier full / empty pairs) -> wgmma.mma_async
//   (fp32 accumulators in registers) -> epilogue fused with bias / forward-only GELU / residual / row maps.  The
//   bf16-output forms on plain rows stage the tile in shared memory and write it with TMA stores that run under the next
//   tile's MMAs.  The fp32 forms (residual adds through any row map, split-K partials) stage padded fp32 rows instead: two
//   otherwise idle warps of the producer warpgroup load each tile's residual rows with 1-D bulk copies while its MMAs run
//   and store the result rows the same way under the next tile's.  The bf16 forms with an output row map, and fp32 calls
//   at BN = 256 or with rows that are not 16-byte aligned, write straight from the accumulator registers to global memory.
// Persistent: one CTA per SM walks a static sequence of 128 x BN output tiles (x K split), BN in {128, 192, 256}.  384
// threads: warpgroup 0 = TMA producer (one thread), warpgroups 1-2 = consumers, each owning 64 rows of every tile.  The
// producer runs ahead across tile boundaries, so the next tile's first k-blocks load while the consumers run the epilogue.
// Both operands may be K-major or MN-major (wgmma transpose bits), so forward (X W^T), dgrad (dY W) and wgrad (dY^T X) all
// run without transposed copies.
// The same body also runs the fp8 inference form (gemm_e4m3_kernel, vt_gemm_e4m3): e4m3 K-major operands, BN = 128,
// per-k-block promotion into the fp32 accumulator and a per-row x per-column dequantisation scale before the epilogue.
#include <stdlib.h>
#include <string.h>

#include "vt_common.cuh"
#include "vt_sm90.cuh"

namespace vt {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int GEMM_THREADS = 384;        // producer warpgroup + 2 consumer warpgroups
constexpr int CHUNK_BYTES = 64 * BK * 2;  // one 64-wide MN chunk of an MN-major tile (8 KiB)

struct GemmDev {
  int M, N, K;
  int kblocks, splits;
  int num_m, num_n, tiles;   // tiles = num_m x num_n x splits
  int epi;
  const float* bias;
  const float* bias2;      // VT_EPI_F32 with aux only: second bias, added to the addend
  void* out;
  const void* aux;         // VT_EPI_F32 only: fp32 addend rows
  long long ldo, ldaux;
  const int* out_row;
  const int* aux_row;
  const float* row_scale;
  long long split_stride;  // elements between split partials (EPI_F32 only)
  // affine row map of the residual epilogue (vt_gemm_params::map_*), map_period = 0: none
  int map_period, map_skip, map_tcount;
  long long map_stride_t, map_stride_p, map_stride_b, map_base;
  float* special_out;      // special rows go to special_out + outer * special_ld, or are dropped
  long long special_ld;
  const float* a_scale;    // e4m3 forms only: per-row scale of A [M] and per-column scale of B [N]
  const float* b_scale;
};

// Epilogue kinds (kernel template parameter SE): 0 = from registers; 1 = one staged bf16 output (VT_EPI_BF16, VT_EPI_GELU_H);
// 3 = staged fp32 rows (VT_EPI_F32, BN = 128 / 192: residual rows loaded and result rows stored by 1-D bulk copies, see
// epi_f32_io).  The number 3 appears in the kernel names that profilers report and tests parse, so it stays.
constexpr int EPI_BOX_BYTES = 64 * 64 * 2;   // one 64-row x 64-column bf16 box, 128B-swizzled as TMA reads / writes it
constexpr int SE_F32 = 3;

template <int BN, int SE>
struct GemmCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int EPI_TILE_BYTES = BM * BN * 2;    // one staged 128 x BN bf16 tile (both consumer halves)
  // fp32 staging rows are padded by 32 bytes: the 8-byte accumulator pairs of a half-warp (4 rows x 32 contiguous bytes)
  // then fall in 4 different bank octets.  Unpadded, all 4 rows hit the same 8 banks.
  static constexpr int F32_PITCH = BN + 8;              // floats per staged fp32 row
  static constexpr int EPI_BYTES = SE == SE_F32 ? BM * F32_PITCH * 4 : SE == 1 ? EPI_TILE_BYTES : 0;
  static constexpr int SMEM_LIMIT = 232448, SMEM_EXTRA = 1024 /*align slack*/ + 256 /*barriers*/;
  // the ring gives up stages to the staging tiles: 6 / 5 / 4 stages at BN = 128 / 192 / 256 without staging, 4 / 3 at
  // BN = 128 / 192 with the fp32 staging tile
  static constexpr int STAGES_FIT = (SMEM_LIMIT - SMEM_EXTRA - EPI_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT < 6 ? STAGES_FIT : 6;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + SMEM_EXTRA;
  static_assert(STAGES >= 2 && SMEM_BYTES <= SMEM_LIMIT, "shared memory budget");
};

template <int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_tile(float (&acc)[BN / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (BN == 256) wgmma_m64n256k16<TA, TB>(acc, da, db, scale_d);
  else if constexpr (BN == 192) wgmma_m64n192k16<TA, TB>(acc, da, db, scale_d);
  else wgmma_m64n128k16<TA, TB>(acc, da, db, scale_d);
}

// Where one accumulator row goes: output row pointer (null = dropped), addend row (null = none).
struct EpiRow {
  char* out;
  const char* aux;
  float s;
};

__device__ __forceinline__ EpiRow epi_row(const GemmDev& p, int row, int split) {
  EpiRow r{nullptr, nullptr, 1.0f};
  if (row >= p.M) return r;
  if (p.row_scale) r.s = p.row_scale[row];
  if (p.epi == VT_EPI_F32) {
    float* out = static_cast<float*>(p.out);
    const float* aux = static_cast<const float*>(p.aux);
    if (p.map_period > 0) {
      const int outer = row / p.map_period, inner = row - outer * p.map_period;
      if (inner < p.map_skip) {
        if (p.special_out) r.out = reinterpret_cast<char*>(p.special_out + (long long)outer * p.special_ld);
        return r;
      }
      const long long off = p.map_base + (long long)(outer % p.map_tcount) * p.map_stride_t +
                            (long long)(inner - p.map_skip) * p.map_stride_p + (long long)(outer / p.map_tcount) * p.map_stride_b;
      r.out = reinterpret_cast<char*>(out + off);
      r.aux = reinterpret_cast<const char*>(aux + off);
      return r;
    }
    const int orow = p.out_row ? p.out_row[row] : row;
    if (orow >= 0) r.out = reinterpret_cast<char*>(out + (long long)split * p.split_stride + (long long)orow * p.ldo);
    if (aux) {
      const int arow = p.aux_row ? p.aux_row[row] : row;
      if (arow >= 0) r.aux = reinterpret_cast<const char*>(aux + (long long)arow * p.ldaux);
    }
    return r;
  }
  const int orow = p.out_row ? p.out_row[row] : row;
  if (orow < 0) return r;
  r.out = reinterpret_cast<char*>(static_cast<__nv_bfloat16*>(p.out) + (long long)orow * p.ldo);
  return r;
}

// The per-element arithmetic of the bf16 forms, shared by the register and the staged epilogue so that both give the
// same bits.
__device__ __forceinline__ void add_bias(const GemmDev& p, int n, float& v0, float& v1) {
  if (p.bias) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + n));
    v0 += b.x; v1 += b.y;
  }
}
// h from the bf16-rounded z: bit for bit what the stand-alone GELU kernel computes from the stored z
__device__ __forceinline__ uint32_t gelu_pair(uint32_t z) {
  const float2 zr = unpack_bf16x2(z);
  return pack_bf16x2(gelu_fast(zr.x), gelu_fast(zr.y));
}

// columns n, n + 1 of one row (n even, n + 1 < N since N % 8 == 0)
__device__ __forceinline__ void epi_pair(const GemmDev& p, const EpiRow& r, int n, float v0, float v1) {
  if (!r.out) return;
  add_bias(p, n, v0, v1);
  if (p.epi == VT_EPI_BF16) {
    *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(r.out) + n) = pack_bf16x2(r.s * v0, r.s * v1);
  } else if (p.epi == VT_EPI_F32) {
    float2 a = make_float2(0.f, 0.f);
    if (r.aux) a = *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(r.aux) + n);
    if (p.bias2) {
      const float2 b2 = __ldg(reinterpret_cast<const float2*>(p.bias2 + n));
      a.x += b2.x; a.y += b2.y;
    }
    *reinterpret_cast<float2*>(reinterpret_cast<float*>(r.out) + n) = make_float2(fmaf(r.s, v0, a.x), fmaf(r.s, v1, a.y));
  } else {  // VT_EPI_GELU_H
    *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(r.out) + n) = gelu_pair(pack_bf16x2(r.s * v0, r.s * v1));
  }
}

// Staged epilogue of one consumer warpgroup: its 64 x BN half of the tile goes to shared memory as BN / 64 boxes of
// 64 rows x 128 B in the SWIZZLE_128B layout (16-byte chunk c of row r at chunk c ^ (r % 8)).  A thread's column pair
// of 8 rows of one warp lands in 8 different chunks: the 32 lanes hit 32 different banks.  Rows >= M and columns >= N
// are left as they are; the TMA store clips them.  stage: this half's output tile.  EPI: VT_EPI_BF16 or VT_EPI_GELU_H.
template <int BN, int EPI>
__device__ __forceinline__ void epi_stage(const GemmDev& p, const float (&acc)[BN / 2], uint8_t* stage, int row0, int n0,
                                          int warp, int lane) {
  const int r = warp * 16 + (lane >> 2);          // rows r and r + 8 of the 64-row half; r % 8 == lane / 4
  float s[2] = {1.0f, 1.0f};
  if (p.row_scale) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (row0 + r + 8 * h < p.M) s[h] = p.row_scale[row0 + r + 8 * h];
  }
  // a1: this thread's word of chunk r % 8 (r % 8 in address bits [4, 7)); xor with j % 8 there gives chunk j ^ r
  const uint32_t a1 = smem_u32(stage) + r * 128 + 4 * (lane & 3) + ((lane >> 2) << 4);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n = n0 + 8 * j + 2 * (lane & 3);
    if (n >= p.N) break;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t off = (j >> 3) * EPI_BOX_BYTES + h * 8 * 128;
      const uint32_t o = (a1 ^ ((j & 7) << 4)) + off;
      float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      add_bias(p, n, v0, v1);
      if (EPI == VT_EPI_BF16) st_shared_u32(o, pack_bf16x2(s[h] * v0, s[h] * v1));
      else st_shared_u32(o, gelu_pair(pack_bf16x2(s[h] * v0, s[h] * v1)));
    }
  }
}

// Tile t of the persistent walk: n fastest, then m, then the K split, so the tiles the CTAs run at one time share A
// row-blocks in L2.
struct Tile {
  int m0, n0, split, kb0, kb1;
};

template <int BN>
__device__ __forceinline__ Tile tile_at(const GemmDev& p, int t) {
  Tile c;
  const int nt = t % p.num_n, rest = t / p.num_n;
  const int mt = rest % p.num_m;
  c.split = rest / p.num_m;
  c.m0 = mt * BM;
  c.n0 = nt * BN;
  c.kb0 = (int)(((long long)p.kblocks * c.split) / p.splits);
  c.kb1 = (int)(((long long)p.kblocks * (c.split + 1)) / p.splits);
  return c;
}

// Row mover of the staged fp32 epilogue: one warp of the producer warpgroup per consumer half; lane l owns rows l and
// l + 32 of the half's 64 x F32_PITCH staging tile `stage`, and the same lane loads and stores them, so its own bulk-group
// wait is what keeps a row from being refilled before its store has read it.  Per tile, under the tile's MMAs: each row
// with an addend is loaded (min(BN, N - n0) floats, one 1-D bulk copy, completing on `full`), a stored row without one is
// zero-filled; then, once the consumer half has written its results in place (`ready`), every row that has an output is
// stored through the same row mapping as the register epilogue (epi_row: plain rows, split-K partials, index arrays, the
// affine maps and their side rows).  Rows >= M, dropped rows and columns >= N are never written.
template <int BN>
__device__ __forceinline__ void epi_f32_io(const GemmDev& p, float* stage, uint64_t* full, uint64_t* ready, int half, int lane) {
  constexpr int PITCH = GemmCfg<BN, SE_F32>::F32_PITCH;
  uint32_t tj = 0;
  for (int t = blockIdx.x; t < p.tiles; t += gridDim.x, ++tj) {
    const Tile c = tile_at<BN>(p, t);
    const int cols = p.N - c.n0 < BN ? p.N - c.n0 : BN;
    const uint32_t bytes = (uint32_t)cols * 4;
    const int row0 = c.m0 + half * 64 + lane;
    const EpiRow e0 = epi_row(p, row0, c.split), e1 = epi_row(p, row0 + 32, c.split);
    float* s0 = stage + lane * PITCH;
    float* s1 = s0 + 32 * PITCH;
    tma_store_wait_read_all();        // this lane's stores of the previous tile have read its rows
    uint32_t tx = 0;
    if (p.aux) {
      if (e0.out && e0.aux) tx += bytes;
      if (e1.out && e1.aux) tx += bytes;
      for (int h = 0; h < 2; ++h) {
        const EpiRow& e = h ? e1 : e0;
        if (e.out && !e.aux)
          for (int i = 0; i < cols; i += 4) st_shared_zero16(smem_u32((h ? s1 : s0) + i));
      }
    }
    mbar_arrive_expect_tx(full, tx);  // also tells the consumers the rows are free when nothing is loaded
    if (tx) {
      if (e0.out && e0.aux) bulk_load_1d(s0, reinterpret_cast<const float*>(e0.aux) + c.n0, bytes, full);
      if (e1.out && e1.aux) bulk_load_1d(s1, reinterpret_cast<const float*>(e1.aux) + c.n0, bytes, full);
    }
    mbar_wait(ready, tj & 1);
    if (e0.out) bulk_store_1d(reinterpret_cast<float*>(e0.out) + c.n0, s0, bytes);
    if (e1.out) bulk_store_1d(reinterpret_cast<float*>(e1.out) + c.n0, s1, bytes);
    tma_store_commit();
  }
  tma_store_wait_read_all();          // shared memory stays valid until the last store has read it
}

// Consumer side of the staged fp32 epilogue: rows r, r + 8 of the half (r = 16 warp + lane / 4), column pairs
// 8j + 2 (lane % 4).  The arithmetic and its order are epi_pair's: v + bias, then fmaf(s, v, addend + bias2), with an
// addend of zero where the row has none (zero-filled, or no aux at all).
template <int BN>
__device__ __forceinline__ void epi_f32_stage(const GemmDev& p, const float (&acc)[BN / 2], const float* stage, int row0, int n0,
                                              int warp, int lane) {
  constexpr int PITCH = GemmCfg<BN, SE_F32>::F32_PITCH;
  const int r = warp * 16 + (lane >> 2);
  float s[2] = {1.0f, 1.0f};
  if (p.row_scale) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (row0 + r + 8 * h < p.M) s[h] = p.row_scale[row0 + r + 8 * h];
  }
  const uint32_t a0 = smem_u32(stage + r * PITCH + 2 * (lane & 3));
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n = n0 + 8 * j + 2 * (lane & 3);
    if (n >= p.N) break;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t o = a0 + (h * 8 * PITCH + 8 * j) * 4;
      float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      add_bias(p, n, v0, v1);
      float2 a = make_float2(0.f, 0.f);
      if (p.aux) a = ld_shared_f32x2(o);
      if (p.bias2) {
        const float2 b2 = __ldg(reinterpret_cast<const float2*>(p.bias2 + n));
        a.x += b2.x; a.y += b2.y;
      }
      st_shared_f32x2(o, fmaf(s[h], v0, a.x), fmaf(s[h], v1, a.y));
    }
  }
}

// min(tiles, SMs) CTAs; CTA b runs tiles b, b + gridDim.x, ...  The producer thread streams every tile's k-blocks
// through one shared-memory ring whose stage / phase count runs on across tiles, so barrier set-up, register hand-over and
// the tensor-map prefetch happen once per CTA and the ring refills during each epilogue.  The walk is static: a tile's
// result depends only on the tile, not on the grid size.
// SE = 1 (staged bf16 epilogue): each consumer warpgroup writes its half of the tile into its own staging boxes, and one
// of its threads stores them with TMA (tmC: out) and goes straight on to the next tile's MMAs; before the boxes are
// rewritten, that thread waits until the previous store has read them.
// F8 = 1: e4m3 operands (vt_gemm_e4m3), BN = 128, both K-major.  A k-block is then 128 elements (the same 128 bytes per
// row) and runs as 4 x wgmma k32 into a fresh register tile `part`, which the consumer adds to `acc` once the k-block's
// MMAs have retired (promotion every 128 K: FP8 wgmma's internal accumulation is not documented to be full fp32).  Before
// the epilogue acc is multiplied by a_scale[m] * b_scale[n].
// The body of both kernels below; the tensor maps are the kernels' __grid_constant__ parameters.
template <int BN, int TA, int TB, int SE, int F8>
__device__ __forceinline__ void gemm_wgmma_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC,
                                                const GemmDev& p) {
  using Cfg = GemmCfg<BN, SE>;
  static_assert(SE == 0 || SE == 1 || SE == SE_F32, "epilogue kinds: register, staged bf16, staged fp32");
  static_assert(!F8 || (BN == 128 && !TA && !TB), "e4m3 forms: BN = 128, K-major operands");
  static_assert(SE != SE_F32 || BN != 256, "the fp32 staging tile leaves too few ring stages at BN = 256");
  constexpr int STAGES = Cfg::STAGES;
  constexpr int KB_ELEMS = F8 ? 128 : BK;      // elements of one k-block (128 bytes per row either way)
  constexpr int HALF_BYTES = Cfg::EPI_TILE_BYTES / 2;   // one consumer warpgroup's 64 x BN part of a staged tile
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* epi_smem = smem + STAGES * Cfg::STAGE_BYTES;   // staging tile (1024-byte aligned), EPI_BYTES
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(epi_smem + Cfg::EPI_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* rows_full_bar = empty_bar + STAGES;   // SE_F32, per consumer half: residual rows loaded / staging rows free
  uint64_t* rows_ready_bar = rows_full_bar + 2;   // SE_F32, per consumer half: results written, rows may be stored

  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (SE == 1) tma_prefetch_desc(&tmC);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);   // one arrive per consumer warp
    }
    for (int h = 0; h < 2; ++h) {
      mbar_init(&rows_full_bar[h], 32);    // one arrive per lane of the row-moving warp
      mbar_init(&rows_ready_bar[h], 128);  // one arrive per consumer thread
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    const int pw = threadIdx.x >> 5;
    if constexpr (SE == SE_F32) {   // warps 1 and 2 move the fp32 rows of consumer halves 0 and 1
      if (pw == 1 || pw == 2) {
        float* rows = reinterpret_cast<float*>(epi_smem) + (pw - 1) * 64 * Cfg::F32_PITCH;
        epi_f32_io<BN>(p, rows, &rows_full_bar[pw - 1], &rows_ready_bar[pw - 1], pw - 1, threadIdx.x & 31);
      }
    }
    if (threadIdx.x == 0) {
      uint32_t it = 0;   // ring position: k-blocks loaded so far by this CTA
      uint32_t tj = 0;   // tiles of this CTA so far
      for (int t = blockIdx.x; t < p.tiles; t += gridDim.x, ++tj) {
        const Tile c = tile_at<BN>(p, t);
        for (int kb = c.kb0; kb < c.kb1; ++kb, ++it) {
          const int stage = (int)(it % STAGES);
          mbar_wait(&empty_bar[stage], ((it / STAGES) & 1) ^ 1);
          uint8_t* sA = smem + stage * Cfg::STAGE_BYTES;
          uint8_t* sB = sA + Cfg::A_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          if (!TA) {
            tma_load_2d(sA, &tmA, &full_bar[stage], kb * KB_ELEMS, c.m0);
          } else {
#pragma unroll
            for (int ch = 0; ch < BM / 64; ++ch) tma_load_2d(sA + ch * CHUNK_BYTES, &tmA, &full_bar[stage], c.m0 + ch * 64, kb * BK);
          }
          if (!TB) {
            tma_load_2d(sB, &tmB, &full_bar[stage], kb * KB_ELEMS, c.n0);
          } else {
#pragma unroll
            for (int ch = 0; ch < BN / 64; ++ch) tma_load_2d(sB + ch * CHUNK_BYTES, &tmB, &full_bar[stage], c.n0 + ch * 64, kb * BK);
          }
        }
      }
    }
    return;
  }

  setmaxnreg_inc<232>();
  const int cw = wg - 1;                       // consumer: rows [64 cw, 64 cw + 64) of every tile
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const bool leader = (threadIdx.x & 127) == 0;   // issues this warpgroup's TMA stores
  uint8_t* stage = epi_smem + cw * HALF_BYTES;
  uint32_t it = 0, tj = 0;
  float part[F8 ? BN / 2 : 1];
#pragma unroll
  for (int i = 0; i < (F8 ? BN / 2 : 1); ++i) part[i] = 0.f;
  for (int t = blockIdx.x; t < p.tiles; t += gridDim.x, ++tj) {
    const Tile c = tile_at<BN>(p, t);
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    if constexpr (F8) {
      for (int kb = c.kb0; kb < c.kb1; ++kb, ++it) {
        const int stage = (int)(it % STAGES);
        mbar_wait(&full_bar[stage], (it / STAGES) & 1);
        const uint32_t a_addr = smem_u32(smem + stage * Cfg::STAGE_BYTES) + cw * 64 * 128;
        const uint32_t b_addr = smem_u32(smem + stage * Cfg::STAGE_BYTES + Cfg::A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_m64n128k32_e4m3(part, sdesc_kmajor(a_addr + k * 32), sdesc_kmajor(b_addr + k * 32), k > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
      }
      // dequantise: acc * (a_scale[m] * b_scale[n]); rows >= M and columns >= N are never stored
      const int rr = c.m0 + cw * 64 + warp * 16 + (lane >> 2);
      const float sa0 = rr < p.M ? p.a_scale[rr] : 0.f, sa1 = rr + 8 < p.M ? p.a_scale[rr + 8] : 0.f;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = c.n0 + 8 * j + 2 * (lane & 3);
        if (n >= p.N) break;
        const float2 sb = __ldg(reinterpret_cast<const float2*>(p.b_scale + n));
        acc[4 * j] *= sa0 * sb.x;
        acc[4 * j + 1] *= sa0 * sb.y;
        acc[4 * j + 2] *= sa1 * sb.x;
        acc[4 * j + 3] *= sa1 * sb.y;
      }
    } else {
    int prev = -1;
    for (int kb = c.kb0; kb < c.kb1; ++kb, ++it) {
      const int stage = (int)(it % STAGES);
      mbar_wait(&full_bar[stage], (it / STAGES) & 1);
      const uint32_t a_addr = smem_u32(smem + stage * Cfg::STAGE_BYTES) + cw * (TA ? CHUNK_BYTES : 64 * 128);
      const uint32_t b_addr = smem_u32(smem + stage * Cfg::STAGE_BYTES + Cfg::A_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t da = TA ? sdesc_mnmajor(a_addr + k * 2048, CHUNK_BYTES) : sdesc_kmajor(a_addr + k * 32);
        const uint64_t db = TB ? sdesc_mnmajor(b_addr + k * 2048, CHUNK_BYTES) : sdesc_kmajor(b_addr + k * 32);
        wgmma_tile<BN, TA, TB>(acc, da, db, (kb > c.kb0 || k > 0) ? 1u : 0u);
      }
      wgmma_commit();
      // the previous k-block's MMAs have retired once at most this one is in flight: its stage is free
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
    }
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&empty_bar[prev]);   // the producer is already filling the ring for the next tile
    }

    if constexpr (SE == SE_F32) {
      const float* rows = reinterpret_cast<const float*>(epi_smem) + cw * 64 * Cfg::F32_PITCH;
      mbar_wait(&rows_full_bar[cw], tj & 1);
      epi_f32_stage<BN>(p, acc, rows, c.m0 + cw * 64, c.n0, warp, lane);
      fence_proxy_async_smem();
      mbar_arrive(&rows_ready_bar[cw]);
    } else if constexpr (SE == 1) {
      const int row0 = c.m0 + cw * 64;
      if (leader) tma_store_wait_read_all();       // the previous tile's store has read the staging boxes
      named_bar_sync(1 + cw, 128);
      if (p.epi == VT_EPI_GELU_H) epi_stage<BN, VT_EPI_GELU_H>(p, acc, stage, row0, c.n0, warp, lane);
      else epi_stage<BN, VT_EPI_BF16>(p, acc, stage, row0, c.n0, warp, lane);
      fence_proxy_async_smem();
      named_bar_sync(1 + cw, 128);
      if (leader) {
        if (row0 < p.M) {
#pragma unroll
          for (int b = 0; b < BN / 64; ++b) {
            if (c.n0 + 64 * b >= p.N) break;
            tma_store_2d(&tmC, stage + b * EPI_BOX_BYTES, c.n0 + 64 * b, row0);
          }
        }
        tma_store_commit();
      }
    } else {
      const int r0 = c.m0 + cw * 64 + warp * 16 + (lane >> 2);
      const EpiRow e0 = epi_row(p, r0, c.split), e1 = epi_row(p, r0 + 8, c.split);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = c.n0 + 8 * j + 2 * (lane & 3);
        if (n >= p.N) break;
        epi_pair(p, e0, n, acc[4 * j], acc[4 * j + 1]);
        epi_pair(p, e1, n, acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
  }
  if (SE == 1 && leader) tma_store_wait_read_all();   // shared memory stays valid until the last store has read it
}

template <int BN, int TA, int TB, int SE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmC, const GemmDev p) {
  gemm_wgmma_body<BN, TA, TB, SE, 0>(tmA, tmB, tmC, p);
}

// VT_EPI_F32 with the staged rows (SE_F32), BN = 128 or 192
template <int BN, int TA, int TB>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_f32_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmC, const GemmDev p) {
  gemm_wgmma_body<BN, TA, TB, SE_F32, 0>(tmA, tmB, tmC, p);
}

// vt_gemm_e4m3: 128-wide tiles, K-major e4m3 operands, SE = 0, 1 or SE_F32
template <int SE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_e4m3_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmC, const GemmDev p) {
  gemm_wgmma_body<128, 0, 0, SE, 1>(tmA, tmB, tmC, p);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !ptr) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// 2-D row-major [rows, cols] (leading dim ld) of 2-byte (bf16) or 1-byte (e4m3) elements, box {128 bytes of columns,
// box_rows}, 128B swizzle, OOB -> 0.
static int make_tmap_2d(CUtensorMap* map, int esize, const void* base, long long rows, long long cols, long long ld,
                        int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  VT_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled entry point unavailable");
  VT_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base pointer must be 16-byte aligned");
  VT_REQUIRE((ld * esize) % 16 == 0, "TMA leading dimension must be a multiple of %d elements (got %lld)", 16 / esize, ld);
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)(ld * esize)};
  cuuint32_t box[2] = {(cuuint32_t)(128 / esize), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = fn(map, esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base),
                  gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  VT_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld box_rows=%d", (int)r,
             rows, cols, ld, box_rows);
  return 0;
}

// 2-D bf16 row-major [rows, cols] (leading dim ld), box {64 cols, box_rows}, 128B swizzle, OOB -> 0.
int make_tmap_bf16_2d(CUtensorMap* map, const void* base, long long rows, long long cols, long long ld, int box_rows) {
  return make_tmap_2d(map, 2, base, rows, cols, ld, box_rows);
}

__global__ void reduce_rows_kernel(const float* __restrict__ in, float* __restrict__ out, long long stride, int S,
                                   long long n4, int accumulate, float scale) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < S; ++s) {
      const float4 v = *reinterpret_cast<const float4*>(in + (long long)s * stride + i * 4);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    acc.x *= scale; acc.y *= scale; acc.z *= scale; acc.w *= scale;
    float4* o = reinterpret_cast<float4*>(out + i * 4);
    if (accumulate) {
      const float4 p = *o;
      acc.x += p.x; acc.y += p.y; acc.z += p.z; acc.w += p.w;
    }
    *o = acc;
  }
}

// Tall reductions (many partial rows, few columns — LayerNorm dgamma/dbeta partials, the per-CTA column sums of the
// producer kernels): 4 column quads x 64 row lanes per CTA, rows strided over the row lanes, then a shared-memory sum in
// lane order.  Deterministic.  (16 quads x 16 lanes gave 12 CTAs walking 19 - 37 dependent rows each for n = 768.)
constexpr int RT_QUADS = 4, RT_LANES = 64;
__global__ void __launch_bounds__(RT_QUADS * RT_LANES)
reduce_rows_tall_kernel(const float* __restrict__ in, float* __restrict__ out, long long stride, int S, long long n4,
                        int accumulate, float scale) {
  const int cq = threadIdx.x % RT_QUADS, rl = threadIdx.x / RT_QUADS;
  const long long i = blockIdx.x * (long long)RT_QUADS + cq;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < n4) {
    for (int s = rl; s < S; s += RT_LANES) {
      const float4 v = *reinterpret_cast<const float4*>(in + (long long)s * stride + i * 4);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  __shared__ float4 sh[RT_LANES][RT_QUADS];
  sh[rl][cq] = acc;
  __syncthreads();
  // 16 threads per quad: thread j sums lanes j, j + 16, j + 32, j + 48; then lane 0 of the quad adds the 16 in order
  if (rl < 16) {
    float4 a = sh[rl][cq];
#pragma unroll
    for (int r = rl + 16; r < RT_LANES; r += 16) { a.x += sh[r][cq].x; a.y += sh[r][cq].y; a.z += sh[r][cq].z; a.w += sh[r][cq].w; }
    sh[rl][cq] = a;
  }
  __syncthreads();
  if (rl == 0 && i < n4) {
    float4 a = sh[0][cq];
#pragma unroll
    for (int r = 1; r < 16; ++r) { a.x += sh[r][cq].x; a.y += sh[r][cq].y; a.z += sh[r][cq].z; a.w += sh[r][cq].w; }
    a.x *= scale; a.y *= scale; a.z *= scale; a.w *= scale;
    float4* o = reinterpret_cast<float4*>(out + i * 4);
    if (accumulate) { const float4 p = *o; a.x += p.x; a.y += p.y; a.z += p.z; a.w += p.w; }
    *o = a;
  }
}

int launch_reduce_rows(const float* in, float* out, long long stride, int S, long long n, int accumulate, float scale,
                       cudaStream_t st) {
  VT_REQUIRE(n % 4 == 0 && stride % 4 == 0, "vt_reduce_rows: n and stride must be multiples of 4");
  const long long n4 = n / 4;
  if (S >= 32 && n4 <= 16 * 4096) {
    reduce_rows_tall_kernel<<<(int)((n4 + RT_QUADS - 1) / RT_QUADS), RT_QUADS * RT_LANES, 0, st>>>(in, out, stride, S, n4, accumulate, scale);
    return check_launch("reduce_rows_tall_kernel");
  }
  int blocks = (int)((n4 + 255) / 256);
  const int cap = sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  reduce_rows_kernel<<<blocks, 256, 0, st>>>(in, out, stride, S, n4, accumulate, scale);
  return check_launch("reduce_rows_kernel");
}

// tm: A, B, and for the staged bf16 epilogue the output
template <int BN, int TA, int TB, int SE, int F8 = 0>
static int launch_gemm_t(const CUtensorMap (&tm)[3], const GemmDev& d, cudaStream_t st) {
  using Cfg = GemmCfg<BN, SE>;
  void (*kernel)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const GemmDev);
  if constexpr (F8) kernel = gemm_e4m3_kernel<SE>;
  else if constexpr (SE == SE_F32) kernel = gemm_f32_kernel<BN, TA, TB>;
  else kernel = gemm_wgmma_kernel<BN, TA, TB, SE>;
  static bool attr_set = false;  // benign race: idempotent
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    VT_REQUIRE(e == cudaSuccess, "cudaFuncSetAttribute(smem=%d) failed: %s", Cfg::SMEM_BYTES, cudaGetErrorString(e));
    attr_set = true;
  }
  const int grid = d.tiles < persistent_sm_count() ? d.tiles : persistent_sm_count();
  kernel<<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, st>>>(tm[0], tm[1], tm[2], d);
  return check_launch(F8 ? "gemm_e4m3_kernel" : SE == SE_F32 ? "gemm_f32_kernel" : "gemm_wgmma_kernel");
}

template <int BN, int SE>
static int launch_layout(const vt_gemm_params* q, const CUtensorMap (&tm)[3], const GemmDev& d, cudaStream_t st) {
  if (!q->a_mn_major && !q->b_mn_major) return launch_gemm_t<BN, 0, 0, SE>(tm, d, st);
  if (!q->a_mn_major) return launch_gemm_t<BN, 0, 1, SE>(tm, d, st);
  if (!q->b_mn_major) return launch_gemm_t<BN, 1, 0, SE>(tm, d, st);
  return launch_gemm_t<BN, 1, 1, SE>(tm, d, st);
}

#ifndef VT_DEFAULT_STAGED_EPI
#define VT_DEFAULT_STAGED_EPI true
#endif
// Staged epilogue kind for this call (see GemmCfg): the bf16-output forms on plain rows, whose outputs TMA can address
// as [M, N] tensors, and the fp32 forms with any row mapping, whose rows move as 1-D bulk copies of
// 16-byte aligned segments.  gemm_dispatch checks out / aux and their pitches for that; the affine map only has to be
// even there, so a map with an offset or stride that is not a multiple of 4 elements stays on the register epilogue,
// as do BN = 256 and split-K partials at BN = 192 (launch_gemm).  VT_GEMM_STAGED_EPI=0 keeps every form on the register
// epilogue.
static int staged_kind(const vt_gemm_params* q) {
  if (!feature_on("VT_GEMM_STAGED_EPI", VT_DEFAULT_STAGED_EPI)) return 0;
  if (q->epilogue == VT_EPI_F32) {
    if (q->map_period > 0 &&
        (q->map_base % 4 || q->map_stride_t % 4 || q->map_stride_p % 4 || q->map_stride_b % 4 ||
         (q->map_special_base >= 0 && (q->map_special_base % 4 || q->map_special_stride % 4))))
      return 0;
    return SE_F32;
  }
  return q->out_row ? 0 : 1;   // VT_EPI_BF16, VT_EPI_GELU_H
}

template <int BN, int F8 = 0>
static int launch_gemm(const vt_gemm_params* q, GemmDev& d, cudaStream_t st) {
  CUtensorMap tm[3];
  memset(tm, 0, sizeof(tm));
  CUtensorMap &tmA = tm[0], &tmB = tm[1];
  int rc;
  if (F8) {   // K-major e4m3 operands (checked by gemm_dispatch)
    rc = make_tmap_2d(&tmA, 1, q->a, q->M, q->K, q->lda, BM);
    if (!rc) rc = make_tmap_2d(&tmB, 1, q->b, q->N, q->K, q->ldb, BN);
  } else if (!q->a_mn_major) rc = make_tmap_bf16_2d(&tmA, q->a, q->M, q->K, q->lda, BM);
  else rc = make_tmap_bf16_2d(&tmA, q->a, q->K, q->M, q->lda, BK);
  if (rc) return rc;
  if (!F8) {
    if (!q->b_mn_major) rc = make_tmap_bf16_2d(&tmB, q->b, q->N, q->K, q->ldb, BN);
    else rc = make_tmap_bf16_2d(&tmB, q->b, q->K, q->N, q->ldb, BK);
    if (rc) return rc;
  }
  d.num_m = (q->M + BM - 1) / BM;
  d.num_n = (q->N + BN - 1) / BN;
  const long long tiles = (long long)d.num_m * d.num_n * d.splits;
  VT_REQUIRE(tiles < (1LL << 31), "vt_gemm: M=%d N=%d gives too many tiles", q->M, q->N);
  d.tiles = (int)tiles;
  const long long tile_out = (long long)q->M * q->N;
  void* final_out = d.out;
  d.split_stride = 0;
  if (d.splits > 1) {            // partial tiles -> fp32 workspace [splits, M, N], summed below
    d.out = q->workspace;
    d.ldo = q->N;
    d.split_stride = tile_out;
  }
  // split-K partials take the staged rows at BN = 128 only: at 192 the 3 ring stages left cost more over the ~200
  // k-blocks of a weight gradient than the epilogue saves
  int se = staged_kind(q);
  if (se == SE_F32 && (BN == 256 || (d.splits > 1 && (BN != 128 || (reinterpret_cast<uintptr_t>(q->workspace) & 15))))) se = 0;
  if (se == 1) {
    rc = make_tmap_bf16_2d(&tm[2], q->out, q->M, q->N, q->ldo, 64);
    if (rc) return rc;
  }
  if constexpr (F8) {
    if (se == 1) rc = launch_gemm_t<BN, 0, 0, 1, 1>(tm, d, st);
    else if (se == SE_F32) rc = launch_gemm_t<BN, 0, 0, SE_F32, 1>(tm, d, st);
    else rc = launch_gemm_t<BN, 0, 0, 0, 1>(tm, d, st);
  } else {
    if (se == 1) rc = launch_layout<BN, 1>(q, tm, d, st);
    else if constexpr (BN != 256) {
      if (se == SE_F32) rc = launch_layout<BN, SE_F32>(q, tm, d, st);
      else rc = launch_layout<BN, 0>(q, tm, d, st);
    } else {
      rc = launch_layout<BN, 0>(q, tm, d, st);
    }
  }
  if (rc) return rc;
  if (d.splits > 1) {
    VT_REQUIRE(q->ldo == q->N, "vt_gemm: split-K requires ldo == N");
    return launch_reduce_rows(static_cast<const float*>(q->workspace), static_cast<float*>(final_out), tile_out, d.splits, tile_out,
                              0, 1.0f, st);
  }
  return 0;
}

}  // namespace vt

static int gemm_dispatch(const vt_gemm_params* q, const float* a_scale, const float* b_scale, void* stream);

extern "C" int vt_gemm(const vt_gemm_params* q, void* stream) {
  VT_REQUIRE(q != nullptr, "vt_gemm: null params");
  return gemm_dispatch(q, nullptr, nullptr, stream);
}

extern "C" int vt_gemm_e4m3(const vt_gemm_e4m3_params* p, void* stream) {
  using namespace vt;
  VT_REQUIRE(p != nullptr, "vt_gemm_e4m3: null params");
  const vt_gemm_params* q = &p->g;
  VT_REQUIRE(p->a_scale && p->b_scale && (reinterpret_cast<uintptr_t>(p->b_scale) & 15) == 0,
             "vt_gemm_e4m3: a_scale and b_scale are required (b_scale 16-byte aligned)");
  VT_REQUIRE(!q->a_mn_major && !q->b_mn_major, "vt_gemm_e4m3: both operands must be K-major");
  VT_REQUIRE(q->K > 0 && q->K % 16 == 0 && q->lda % 16 == 0 && q->ldb % 16 == 0,
             "vt_gemm_e4m3: K, lda and ldb must be multiples of 16 (got K=%d lda=%lld ldb=%lld)", q->K, (long long)q->lda,
             (long long)q->ldb);
  VT_REQUIRE(q->force_bn == 0 || q->force_bn == 128, "vt_gemm_e4m3: the e4m3 forms run 128-wide tiles only");
  int dev = 0, major = 0;
  VT_REQUIRE(cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) == cudaSuccess &&
                 major == 9, "vt_gemm_e4m3: needs an sm_90 device (compute capability %d.x found)", major);
  return gemm_dispatch(q, p->a_scale, p->b_scale, stream);
}

// a_scale / b_scale non-null: the e4m3 forms (vt_gemm_e4m3, arguments checked there)
static int gemm_dispatch(const vt_gemm_params* q, const float* a_scale, const float* b_scale, void* stream) {
  using namespace vt;
  VT_REQUIRE(q != nullptr, "vt_gemm: null params");
  const bool f8 = a_scale != nullptr;
  VT_REQUIRE(q->M > 0 && q->N > 0 && q->K > 0, "vt_gemm: bad shape M=%d N=%d K=%d", q->M, q->N, q->K);
  VT_REQUIRE(q->N % 8 == 0, "vt_gemm: N must be a multiple of 8 (got %d)", q->N);
  VT_REQUIRE(q->a && q->b && q->out, "vt_gemm: null operand");
  VT_REQUIRE(q->epilogue == VT_EPI_BF16 || q->epilogue == VT_EPI_F32 || q->epilogue == VT_EPI_GELU_H,
             "vt_gemm: bad epilogue %d (VT_EPI_BF16 = 0, VT_EPI_F32 = 1, VT_EPI_GELU_H = 4)", q->epilogue);
  const int esz = (q->epilogue == VT_EPI_F32) ? 4 : 2;
  VT_REQUIRE((q->ldo * esz) % 16 == 0 && (reinterpret_cast<uintptr_t>(q->out) & 15) == 0,
             "vt_gemm: out must be 16B aligned with 16B-multiple row pitch");
  // the bf16 epilogues have no addend: an aux pointer there would be silently ignored
  if (q->aux) VT_REQUIRE(q->epilogue == VT_EPI_F32, "vt_gemm: aux (the fp32 addend) needs VT_EPI_F32, got epilogue %d", q->epilogue);
  if (q->aux) VT_REQUIRE((reinterpret_cast<uintptr_t>(q->aux) & 15) == 0 && (q->ldaux * 4) % 16 == 0, "vt_gemm: aux misaligned");
  if (q->bias) VT_REQUIRE((reinterpret_cast<uintptr_t>(q->bias) & 15) == 0, "vt_gemm: bias misaligned");
  if (q->bias2) VT_REQUIRE(q->epilogue == VT_EPI_F32 && q->aux && (reinterpret_cast<uintptr_t>(q->bias2) & 15) == 0,
                           "vt_gemm: bias2 needs the fp32 epilogue with an addend, 16-byte aligned");
  VT_REQUIRE(q->force_bn == 0 || q->force_bn == 128 || q->force_bn == 192 || q->force_bn == 256,
             "vt_gemm: force_bn must be 128, 192 or 256");

  GemmDev d;
  d.M = q->M; d.N = q->N; d.K = q->K;
  d.epi = q->epilogue;
  d.bias = q->bias;
  d.bias2 = q->bias2;
  d.out = q->out; d.aux = q->aux;
  d.ldo = q->ldo; d.ldaux = q->ldaux;
  d.out_row = q->out_row; d.aux_row = q->aux_row; d.row_scale = q->row_scale;
  d.kblocks = f8 ? (q->K + 127) / 128 : (q->K + BK - 1) / BK;
  d.a_scale = a_scale; d.b_scale = b_scale;
  d.map_period = 0; d.map_skip = 0; d.map_tcount = 1;
  d.map_stride_t = d.map_stride_p = d.map_stride_b = d.map_base = 0;
  d.special_out = nullptr; d.special_ld = 0;
  if (q->map_period > 0) {
    VT_REQUIRE(q->epilogue == VT_EPI_F32 && q->aux, "vt_gemm: the affine row map applies to the fp32 residual epilogue only");
    VT_REQUIRE(q->M % q->map_period == 0 && q->map_tcount >= 1 && q->map_skip >= 0 && q->map_skip < q->map_period,
               "vt_gemm: bad affine row map (period %d, skip %d, tcount %d, M %d)", q->map_period, q->map_skip, q->map_tcount, q->M);
    // the epilogue moves column pairs as float2: every element offset of the map must be even
    VT_REQUIRE(q->map_base % 2 == 0 && q->map_stride_t % 2 == 0 && q->map_stride_p % 2 == 0 && q->map_stride_b % 2 == 0 &&
                   (q->map_special_base < 0 || (q->map_special_base % 2 == 0 && q->map_special_stride % 2 == 0)),
               "vt_gemm: affine row map offsets and strides must be even (8-byte aligned fp32 pairs)");
    d.map_period = q->map_period; d.map_skip = q->map_skip; d.map_tcount = q->map_tcount;
    d.map_stride_t = q->map_stride_t; d.map_stride_p = q->map_stride_p; d.map_stride_b = q->map_stride_b; d.map_base = q->map_base;
    d.special_out = q->map_special_base >= 0 ? static_cast<float*>(q->out) + q->map_special_base : nullptr;
    d.special_ld = q->map_special_stride;
  }

  // Cost ~ tiles per CTA of the persistent grid (ceil(tiles / SMs)) x per-tile time, where a tile (x K split) costs (its
  // k-blocks + a fixed epilogue overhead) x BN, with a small penalty for narrower tiles (they re-read A more often).
  // Splitting K is only possible for plain fp32 outputs with a workspace (weight gradients).
  // Short-K GEMMs without a split (K <= 1024: qkv, FC1 forward, FC2 data gradient, out-proj) take the 128-wide tile, which
  // the model undervalues: measured on an H100 at B = 8 it is 20-35 % faster than the 256-wide tile on the wide-output
  // ones with the register epilogue.  The staged bf16 form may also take the 192-wide tile (4 stages), which the model
  // picks for qkv (81 vs 92 us) and the projection's data gradient (29 vs 33 us); so may the staged fp32 form (3 stages),
  // which the model picks for the projections' forward with the residual add (56 vs 63 us, H100 at 700 W).
  if (f8) {   // two accumulator tiles per thread fit the register budget at BN = 128 only; no split-K
    d.splits = 1;
    return launch_gemm<128, 1>(q, d, static_cast<cudaStream_t>(stream));
  }
  const bool short_k = d.kblocks <= 16;
  const bool one_staged = staged_kind(q) == 1;
  const int sms = persistent_sm_count();
  const int num_m = (q->M + BM - 1) / BM;
  const bool can_split = q->epilogue == VT_EPI_F32 && q->workspace && !q->out_row && !q->aux && !q->row_scale && !q->bias &&
                         q->map_period == 0;
  // the staged fp32 rows exist at BN = 128 / 192 only; split-K calls keep the plan they had (a different split count
  // would change the sums) and take the register epilogue where it is 192 or 256 wide (launch_gemm)
  const bool f32_staged = staged_kind(q) == SE_F32 && !can_split;
  const int cand[3] = {256, 192, 128};
  const double penalty[3] = {1.0, 1.04, 1.10};
  double best = 1e30;
  int bn = 128, splits = 1;
  for (int i = 0; i < 3; ++i) {
    if (q->force_bn && cand[i] != q->force_bn) continue;
    if (!q->force_bn && !can_split && short_k && cand[i] != 128 && !((one_staged || f32_staged) && cand[i] == 192)) continue;
    if (!q->force_bn && f32_staged && cand[i] == 256) continue;
    const int num_n = (q->N + cand[i] - 1) / cand[i];
    const int smax = can_split ? 16 : 1;
    for (int sp = 1; sp <= smax; ++sp) {
      if (sp > 1 && (d.kblocks / sp < 4 || (long long)sp * q->M * q->N * 4 > q->workspace_bytes)) break;
      const long long tiles = (long long)num_m * num_n * sp;
      const double per_cta = (double)((tiles + sms - 1) / sms);
      const double cost = per_cta * ((double)d.kblocks / sp + 8.0) * cand[i] * penalty[i];
      if (cost < best - 1e-9) { best = cost; bn = cand[i]; splits = sp; }
    }
  }
  if (can_split && q->force_splits > 0) {
    splits = q->force_splits;
    const long long max_by_ws = q->workspace_bytes / ((long long)q->M * q->N * 4);
    if (splits > max_by_ws) splits = (int)max_by_ws;
    if (splits > d.kblocks) splits = d.kblocks;
    if (splits < 1) splits = 1;
  }
  d.splits = splits;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (bn == 256) return launch_gemm<256>(q, d, st);
  if (bn == 192) return launch_gemm<192>(q, d, st);
  return launch_gemm<128>(q, d, st);
}

extern "C" int vt_reduce_rows(const vt_reduce_params* p, void* stream) {
  using namespace vt;
  VT_REQUIRE(p && p->in && p->out && p->S >= 1, "vt_reduce_rows: bad params");
  return launch_reduce_rows(p->in, p->out, p->stride, p->S, p->n, p->accumulate, p->scale,
                            static_cast<cudaStream_t>(stream));
}
