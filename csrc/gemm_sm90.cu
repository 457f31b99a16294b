// wgmma / TMA grouped GEMM for sm_90a (H100).
//
// Replaces the reference's cuBLAS `torch.matmul` expert GEMMs (tutel/experts/ffn.py:114-118,
// tutel/experts/llama_ffn.py:38-41) and its host-synchronised per-expert loop
// `sparse_bmm_infer` (tutel/custom/custom_kernel.cpp:874-889) with ONE persistent, warp-specialised kernel
// (384 threads, 128 x 256 output tiles; 128 x 128 for the fused multi-GPU engine, the GLU epilogues, fp32 outputs and
// block_n=128, see Cfg and gemm_sm90_launch):
//
//   warp 0        TMA producer   cp.async.bulk.tensor (128B swizzle) -> smem ring, mbarrier complete_tx.
//   warp 1        store warp     (128 x 256 only) owns the output tile: TMA-stores each finished tile, then loads the next
//                                tile's aux operand (ReLU / activation gradient, add) into it; bulk-copies every tile's
//                                bias and fp8 column scales into shared memory while the main loop runs; adds up the
//                                consumer warps' bias-gradient partial rows and issues the global reductions.
//                                Warps 2, 3 (and warp 1 of the 128 x 128 configuration) only give their registers away
//                                (setmaxnreg).
//   warps 4..11   two consumer warpgroups, 64 rows of the tile each: wgmma.mma_async (m64n256 / m64n128, operands
//                                straight from the swizzled ring, fp32 accumulator fragment in registers), one stage in
//                                flight; a stage is handed back to the producer when the wgmma group that read it has retired.
//                                128 x 256 epilogue: scales / bias / activation / aux math on the fragment in registers,
//                                packed into the 16-bit output tile in the TMA box layout, bias-gradient column sums
//                                reduced per warp; the tile is handed to the store warp (out_full) and the consumers go
//                                straight on to the next tile's main loop (see wide_main and hand_over_tile).
//                                128 x 128 epilogue: every warp parks 16 x 128 of its fragment in its own shared-memory
//                                rows and reads it back with one lane per row and 32 consecutive columns per lane, applies
//                                the fused bias / activation / activation-grad / GLU / bias-grad math in fp32 and writes
//                                64 contiguous bytes per lane - locally or straight into PEER GPUs' memory plus a
//                                release.sys counter bump (GEMM -> combine all-to-all fusion) - while the producer
//                                already fills the ring for the next tile.
//
// The producer can also acquire system-scope "rows have arrived" counters before loading an A tile, which is
// how the dispatch all-to-all is overlapped tile-by-tile with the first expert GEMM.
#include "gemm_sm90.h"

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstdio>
#include <cstdlib>
#include <mutex>

#include "ptx.cuh"

namespace tb {

struct GemmArgs {
  int M, N, K, G;
  int b_group_div;
  int tiles_m, tiles_n;
  long long num_tiles;

  void* d;
  long long ldd, d_group_stride;
  const unsigned long long* d_ptr_table;
  int out_dtype;

  int epilogue;
  float alpha;
  const void* bias;
  long long bias_group_stride;
  int bias_is_fp32;
  int bias_is_bf16;
  const void* aux;
  long long ld_aux, aux_group_stride;
  const void* aux2;
  void* d2;
  void* d3;
  int dual;        // EPI_GLU: B tile = 64 columns of tmB + the same 64 columns of tmB2
  int act;
  const float* scale_b2;

  const int* row_counts;
  float* colsum;  // [G / b_group_div, N] fp32: += column sums of the epilogue result (bias gradient), may be null
  long long colsum_group_stride;
  const float* scale_a;  // [G, M] per-row dequantisation scales (fp8 operands), may be null
  long long scale_a_group_stride;
  const float* scale_b;  // [G / b_group_div, N] per-column scales, may be null
  long long scale_b_group_stride;

  const uint32_t* wait_flags;
  int wait_rows_per_flag, wait_flags_per_group;
  uint32_t wait_target;
  const unsigned long long* signal_ptr_table;
  int group_rot, group_mod;  // tile order visits group (g/mod)*mod + (g%mod + rot)%mod  (own-rank segment first)
  // Block-mapped B (packed expert layout): group g is one M tile whose B group (and bias / scale_b / colsum row) is
  // b_group_map[g]; rows of a tile past row_counts[g] are stored as zeros.  Tiles are banded across groups.
  const int* b_group_map;
  // Ragged K (weight gradients on the packed layout): A and B are single [K_total, *] tensors and group g reduces the
  // K range [k_offsets[g], k_offsets[g + 1]) (multiples of the 64-element K block).
  const int* k_offsets;
};

namespace {

constexpr int kThreads = 384;        // producer warpgroup + two consumer warpgroups
constexpr int kSwizzleBytes = 128;   // one swizzle row: 64 bf16 / 128 fp8
constexpr int kSmemLimit = 232448;   // 227 KB

// Two configurations of the same kernel (tiles of BM x BN):
//   BN 128  4 stages of 32 KB, 144 registers per thread.  The fused multi-GPU engine runs this one (see the resource
//           budget above gemm_sm90_kernel).
//   BN 256  m64n256 wgmma per consumer warpgroup (128 fp32 accumulators per thread): 48 KB of operands per 64-deep K
//           block for twice the FLOPs of a 128 x 128 tile's 32 KB, and each warpgroup's B reads from shared memory
//           serve 256 instead of 128 columns.  16-bit output only.  3 stages of 48 KB, the 64 KB output tile, barriers,
//           eight 1 KB bias-gradient partial rows (one per consumer warp) and two 2 KB side-input slots (bias and
//           column scales of two consecutive tiles): 221.5 KB.  168 registers per thread (producer warpgroup 40,
//           consumers 232), one CTA per SM.  The epilogue works on the accumulator fragment in registers and hands the
//           tile to the store warp, so the consumers start the next tile's main loop while the store drains.
template <int BN_>
struct Cfg {
  static constexpr int BM = 128;
  static constexpr int BN = BN_;
  static constexpr bool WIDE = BN_ == 256;
  static constexpr int A_BYTES = BM * kSwizzleBytes;
  static constexpr int B_BYTES = BN * kSwizzleBytes;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // 128 x 128 epilogue staging: per consumer warp 16 accumulator rows of 128 floats; 8 floats of padding per row keep
  // the fragment writes (float2, four rows per half-warp) free of bank conflicts.
  static constexpr int EPI_COLS = 128;
  static constexpr int EPI_PITCH = EPI_COLS + 8;
  static constexpr int EPI_WARP_BYTES = 16 * EPI_PITCH * 4;
  static constexpr int EPI_BYTES = WIDE ? 0 : 8 * EPI_WARP_BYTES;
  // 128 x 256 output tile in 16 bit, as the TMA boxes of the output tensor map: four boxes of 128 rows x 64 columns
  // (128 B per row, 128-byte swizzle).  It also receives the tile's aux operand.
  static constexpr int OUT_BOX_BYTES = BM * kSwizzleBytes;
  static constexpr int OUT_TILE_BYTES = WIDE ? BM * BN * 2 : 0;
  static constexpr int COLSUM_BYTES = WIDE ? 8 * BN * 4 : 0;      // per consumer warp one row of BN column sums
  static constexpr int SIDE_BIAS_BYTES = BN * 4;                  // bias of one tile (16-bit or fp32) ...
  static constexpr int SIDE_SLOT_BYTES = SIDE_BIAS_BYTES + BN * 4;   // ... and its fp32 column scales
  static constexpr int SIDE_BYTES = WIDE ? 2 * SIDE_SLOT_BYTES : 0;  // double-buffered: tile i+1's lands during tile i
  static constexpr int BAR_BYTES = 512;
  static constexpr int STAGES = WIDE ? 3 : 4;
  static constexpr int MAXNREG = WIDE ? 168 : 144;
  static constexpr int CONSUMER_REGS = WIDE ? 232 : 192;   // producer warpgroup: 40
  static constexpr int SMEM_BYTES =
      STAGES * STAGE_BYTES + 1024 + OUT_TILE_BYTES + BAR_BYTES + EPI_BYTES + COLSUM_BYTES + SIDE_BYTES;
  static_assert((STAGES * STAGE_BYTES) % 1024 == 0, "the output tile must stay 1024B aligned for the 128B swizzle");
  // 228 KB per SM, 1 KB reserved per resident block: a dispatch block (no shared memory of its own) must still fit
  static_assert(WIDE || SMEM_BYTES + 2 * 1024 <= 228 * 1024, "no room for the push kernel");
  static_assert(SMEM_BYTES <= kSmemLimit, "");
  static_assert(128 * 40 + 256 * CONSUMER_REGS <= 65536 && 384 * MAXNREG <= 65536, "register budget");
};

struct TileCoord {
  int g, m_blk, n_blk;
};

// Tiles are enumerated group-major; inside a group, bands of kBand row-blocks sweep all column blocks so that a
// wave of CTAs re-uses both its A band and its B columns out of L2.
template <int kBand>
__device__ __forceinline__ TileCoord decode_tile(long long t, int tiles_m, int tiles_n) {
  const int per_group = tiles_m * tiles_n;
  TileCoord c;
  c.g = static_cast<int>(t / per_group);
  int r = static_cast<int>(t - static_cast<long long>(c.g) * per_group);
  const int band_tiles = kBand * tiles_n;
  const int band = r / band_tiles;
  const int first_m = band * kBand;
  const int rows_in_band = min(kBand, tiles_m - first_m);
  r -= band * band_tiles;
  c.m_blk = first_m + r % rows_in_band;
  c.n_blk = r / rows_in_band;
  return c;
}

// mod > 1: ascending from `rot`;  mod < -1: descending from `rot` (matches a sender that walks destinations upwards).
__device__ __forceinline__ int rotate_group(int g, int rot, int mod) {
  if (mod > 1) {
    const int base = (g / mod) * mod;
    return base + (g - base + rot) % mod;
  }
  if (mod < -1) {
    const int m = -mod;
    const int base = (g / m) * m;
    return base + (rot + m - (g - base)) % m;
  }
  return g;
}

// The packed-layout launch modes (b_group_map, k_offsets) run in their own instantiations of the kernel (PK = true), so
// that every other launch compiles to code with none of their per-tile loads and branches.
//
// Tile t of a launch: group-major bands of row blocks (rotated groups for the fused engine), or - block-mapped B - one
// band sequence over all groups, which are single row blocks, so that a wave reuses B columns across neighbouring blocks.
template <int kBand, bool PK>
__device__ __forceinline__ TileCoord tile_of(long long t, const GemmArgs& args) {
  TileCoord tc;
  if (PK && args.b_group_map != nullptr) {
    tc = decode_tile<kBand>(t, args.G, args.tiles_n);
    tc.g = tc.m_blk;
    tc.m_blk = 0;
  } else {
    tc = decode_tile<kBand>(t, args.tiles_m, args.tiles_n);
    tc.g = rotate_group(tc.g, args.group_rot, args.group_mod);
  }
  return tc;
}

// B group of A group g, which is also the row of bias, scale_b and colsum.
template <bool PK>
__device__ __forceinline__ int b_group_of(int g, const GemmArgs& args) {
  return (PK && args.b_group_map != nullptr) ? args.b_group_map[g] : g / args.b_group_div;
}

// 64-deep K blocks of group g and the first K element: uniform, or the group's range of k_offsets.
template <bool PK>
__device__ __forceinline__ int2 k_range_of(int g, int num_kb, int bk_elems, const GemmArgs& args) {
  if (!PK || args.k_offsets == nullptr) return make_int2(num_kb, 0);
  const int k0 = args.k_offsets[g];
  const int len = args.k_offsets[g + 1] - k0;
  return make_int2(len > 0 ? (len + bk_elems - 1) / bk_elems : 0, k0);
}

// Block-mapped B: rows at or past the count are stored as zeros (r0 / r0 + 8 of wide_main's fragment layout).
__device__ __forceinline__ void wide_zero_rows(float (&acc)[128], bool ok0, bool ok1) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    if (!ok0) { acc[4 * j] = 0.0f; acc[4 * j + 1] = 0.0f; }
    if (!ok1) { acc[4 * j + 2] = 0.0f; acc[4 * j + 3] = 0.0f; }
  }
}

// Per-element epilogue formulas.  Both configurations call these, so that they produce the same bits per element.
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float silu(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
__device__ __forceinline__ float fast_sigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
// v = upstream gradient, x = forward activation output (ReLU) or pre-activation (GELU / SiLU)
__device__ __forceinline__ float relu_bwd(float v, float x) { return x > 0.0f ? v : 0.0f; }
__device__ __forceinline__ float gelu_bwd(float v, float x) {   // d/dx [x * Phi(x)] = Phi(x) + x * phi(x)
  const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752f));
  return v * (cdf + x * 0.3989422804014327f * __expf(-0.5f * x * x));
}
__device__ __forceinline__ float silu_bwd(float v, float x) {   // d/dx [x * s(x)] = s(x) * (1 + x * (1 - s(x)))
  const float sg = fast_sigmoid(x);
  return v * (sg * (1.0f + x * (1.0f - sg)));
}
// two floats <-> one word of two 16-bit values; both conversions are computed and one is selected, so a run-time dtype
// costs no branch inside an unrolled loop
__device__ __forceinline__ uint32_t pack2(float a, float b, bool bf16) {
  const __nv_bfloat162 hb = __floats2bfloat162_rn(a, b);
  const __half2 hh = __floats2half2_rn(a, b);
  return bf16 ? *reinterpret_cast<const uint32_t*>(&hb) : *reinterpret_cast<const uint32_t*>(&hh);
}
__device__ __forceinline__ float2 unpack2(uint32_t w, bool bf16) {
  const float2 h = __half22float2(*reinterpret_cast<const __half2*>(&w));
  return bf16 ? make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xFFFF0000u)) : h;
}

__device__ __forceinline__ void unpack8(const uint4& u, bool is_bf16, float* f) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (is_bf16) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
    } else {
      const __half2 h = *reinterpret_cast<const __half2*>(&w[i]);
      const float2 t = __half22float2(h);
      f[2 * i] = t.x;
      f[2 * i + 1] = t.y;
    }
  }
}
// 32 floats -> 16 packed words; the dtype branch is taken ONCE per segment (a per-element branch on a kernel argument
// serialises the unrolled loop and costs all its instruction-level parallelism).
template <bool BF16>
__device__ __forceinline__ void pack32_t(const float* v, uint32_t* w) {
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    if constexpr (BF16) {
      const __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
      w[i] = *reinterpret_cast<const uint32_t*>(&h);
    } else {
      const __half2 h = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
      w[i] = *reinterpret_cast<const uint32_t*>(&h);
    }
  }
}
__device__ __forceinline__ void pack32(const float* v, uint32_t* w, bool is_bf16) {
  if (is_bf16) pack32_t<true>(v, w); else pack32_t<false>(v, w);
}
template <bool BF16>
__device__ __forceinline__ void unpack32_t(const uint4* p, float* f) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint32_t w[4] = {p[q].x, p[q].y, p[q].z, p[q].w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if constexpr (BF16) {
        f[q * 8 + 2 * i] = __uint_as_float(w[i] << 16);
        f[q * 8 + 2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
      } else {
        const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
        f[q * 8 + 2 * i] = t.x;
        f[q * 8 + 2 * i + 1] = t.y;
      }
    }
  }
}
__device__ __forceinline__ void unpack32(const uint4* p, float* f, bool is_bf16) {
  if (is_bf16) unpack32_t<true>(p, f); else unpack32_t<false>(p, f);
}

// GLU math on one 32-column segment, activation fixed at compile time (branch-free, fully interleavable).
template <int ACT>
__device__ __forceinline__ void glu_fwd_seg(const float* g, const float* u, float* o) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    float a;
    if constexpr (ACT == ACT_RELU) a = fmaxf(g[j], 0.0f);
    else if constexpr (ACT == ACT_GELU) a = gelu_erf(g[j]);
    else a = g[j] * fast_sigmoid(g[j]);
    o[j] = a * u[j];
  }
}
// in: dh, g, u      out: o = d gate, u = d up
template <int ACT>
__device__ __forceinline__ void glu_bwd_seg(const float* r, const float* g, float* u, float* o) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float dh = r[j];
    float a, da;
    if constexpr (ACT == ACT_RELU) {
      a = fmaxf(g[j], 0.0f);
      da = g[j] > 0.0f ? 1.0f : 0.0f;
    } else if constexpr (ACT == ACT_GELU) {
      const float cdf = 0.5f * (1.0f + erff(g[j] * 0.70710678118654752f));
      a = g[j] * cdf;
      da = cdf + g[j] * 0.3989422804014327f * __expf(-0.5f * g[j] * g[j]);
    } else {
      const float sg = fast_sigmoid(g[j]);
      a = g[j] * sg;
      da = sg * (1.0f + g[j] * (1.0f - sg));
    }
    o[j] = dh * u[j] * da;
    u[j] = dh * a;
  }
}

// ---- 128 x 256 epilogue, on the accumulator fragment in registers ----
// A consumer thread (warp cw, lane l) holds tile rows r0 = 16 cw + l / 4 (acc[4j], acc[4j + 1]) and r0 + 8 (acc[4j + 2],
// acc[4j + 3]) at columns 8j + 2 (l % 4) + {0, 1}, j = 0..31.  In the 16-bit output tile, column block j lies in box
// j / 8 at 16-byte chunk j % 8 of its row, which the 128-byte swizzle moves to chunk (j % 8) ^ (row % 8), and row % 8 is
// l / 4 for both rows of a thread: each fragment word has one fixed shared-memory word, and the 32 lanes' words of one
// j cover 8 rows x 16 bytes in 32 distinct banks.
enum WideMain : int { WM_NONE, WM_BIAS, WM_RELU_BWD, WM_ADD, WM_GELU_BWD, WM_SILU_BWD };

__device__ __forceinline__ uint32_t out_tile_off(int j, int swz) {
  return static_cast<uint32_t>((j >> 3) * (128 * kSwizzleBytes) + (((j & 7) ^ swz) << 4));
}

// fp8 operands: acc *= scale_a[m] * scale_b[n]  (sb: this tile's column scales in shared memory, or null).  Columns are
// counted from the tile's first: n_lane = 2 (lane % 4), n_lim = N - n0.
__device__ __forceinline__ void wide_scale(float (&acc)[128], float sa0, float sa1, const float* sb, int n_lane, int n_lim) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int n = n_lane + 8 * j;
    if (sb != nullptr && n < n_lim) {
      const float2 s = *reinterpret_cast<const float2*>(sb + n);
      acc[4 * j] *= sa0 * s.x; acc[4 * j + 1] *= sa0 * s.y;
      acc[4 * j + 2] *= sa1 * s.x; acc[4 * j + 3] *= sa1 * s.y;
    } else {
      acc[4 * j] *= sa0; acc[4 * j + 1] *= sa0;
      acc[4 * j + 2] *= sa1; acc[4 * j + 3] *= sa1;
    }
  }
}

// alpha / bias / aux math.  The aux operand is read from the output tile (this thread's words at row0 and row0 + 8 rows),
// the bias from the tile's side-input slot (columns counted from the tile's first, as in wide_scale).
template <int WM>
__device__ __forceinline__ void wide_main(float (&acc)[128], const uint8_t* row0, int swz, const uint8_t* bias_s,
                                          bool bias_f32, bool bias_bf16, int n_lane, int n_lim, bool out_bf16, float alpha) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    if constexpr (WM == WM_NONE) {
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[4 * j + c] *= alpha;
    } else if constexpr (WM == WM_BIAS) {
      const int n = n_lane + 8 * j;
      float2 b = make_float2(0.0f, 0.0f);
      if (n < n_lim)
        b = bias_f32 ? *reinterpret_cast<const float2*>(bias_s + n * 4)
                     : unpack2(*reinterpret_cast<const uint32_t*>(bias_s + n * 2), bias_bf16);
      acc[4 * j] += b.x; acc[4 * j + 1] += b.y;
      acc[4 * j + 2] += b.x; acc[4 * j + 3] += b.y;
    } else {
      const uint32_t o = out_tile_off(j, swz);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float2 f = unpack2(*reinterpret_cast<const uint32_t*>(row0 + h * 8 * kSwizzleBytes + o), out_bf16);
        float& v0 = acc[4 * j + 2 * h];
        float& v1 = acc[4 * j + 2 * h + 1];
        if constexpr (WM == WM_RELU_BWD) { v0 = relu_bwd(v0, f.x); v1 = relu_bwd(v1, f.y); }
        else if constexpr (WM == WM_ADD) { v0 += f.x; v1 += f.y; }
        else if constexpr (WM == WM_GELU_BWD) { v0 = gelu_bwd(v0, f.x); v1 = gelu_bwd(v1, f.y); }
        else { v0 = silu_bwd(v0, f.x); v1 = silu_bwd(v1, f.y); }
      }
    }
  }
}

template <int ACT>
__device__ __forceinline__ void wide_act(float (&acc)[128]) {
#pragma unroll
  for (int i = 0; i < 128; ++i) {
    if constexpr (ACT == ACT_RELU) acc[i] = fmaxf(acc[i], 0.0f);
    else if constexpr (ACT == ACT_GELU) acc[i] = gelu_erf(acc[i]);
    else acc[i] = silu(acc[i]);
  }
}

__device__ __forceinline__ void wide_stage(const float (&acc)[128], uint8_t* row0, int swz, bool out_bf16) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const uint32_t o = out_tile_off(j, swz);
    *reinterpret_cast<uint32_t*>(row0 + o) = pack2(acc[4 * j], acc[4 * j + 1], out_bf16);
    *reinterpret_cast<uint32_t*>(row0 + 8 * kSwizzleBytes + o) = pack2(acc[4 * j + 2], acc[4 * j + 3], out_bf16);
  }
}

// One halving exchange of wide_colsum: lanes with bit OFF set keep the upper 2 OFF of the first 4 OFF sums, the others the
// lower ones, each adding its partner's.  OFF is a compile-time constant so that every index of s is one, and s stays in
// registers.
template <int OFF>
__device__ __forceinline__ void colsum_halve(float (&s)[64], int lane) {
  const bool upper = (lane & OFF) != 0;
#pragma unroll
  for (int i = 0; i < 2 * OFF; ++i) {
    const float lo = s[i], hi = s[i + 2 * OFF];
    const float recv = __shfl_xor_sync(0xffffffffu, upper ? lo : hi, OFF);
    s[i] = (upper ? hi : lo) + recv;
  }
}
// Bias gradient: this thread's two rows (those below the valid row count) summed per column, then reduced over the
// eight lanes that share its columns (lane bits 2..4) by halving exchanges, 32 + 16 + 8 shuffles: afterwards lane l
// holds the warp's sums of columns 32 (l / 4) + 8 i + 2 (l % 4) + {0, 1}, i = 0..3, which go into the warp's own row of
// the partial sums (the store warp adds up the eight rows).
__device__ __forceinline__ void wide_colsum(const float (&acc)[128], bool ok0, bool ok1, int lane, float* colrow) {
  float s[64];
#pragma unroll
  for (int j = 0; j < 32; ++j) {
#pragma unroll
    for (int c = 0; c < 2; ++c) s[2 * j + c] = (ok0 ? acc[4 * j + c] : 0.0f) + (ok1 ? acc[4 * j + 2 + c] : 0.0f);
  }
  colsum_halve<16>(s, lane);
  colsum_halve<8>(s, lane);
  colsum_halve<4>(s, lane);
  float* base = colrow + 32 * (lane >> 2) + 2 * (lane & 3);
#pragma unroll
  for (int q = 0; q < 4; ++q) *reinterpret_cast<float2*>(base + 8 * q) = make_float2(s[2 * q], s[2 * q + 1]);
}

// Consumers: hand the output tile of group g at rows m0.., columns n0.. to the store warp, called by all 256 consumer
// threads after writing their words of the tile.  A tile that straddles the group's row count (rows from m_valid on must
// stay untouched, which the output tensor map cannot express) is copied out here with row-guarded stores instead; the
// store warp then only releases it.  Every warp arrives on out_full once it no longer reads the tile.
__device__ __forceinline__ void hand_over_tile(const uint8_t* tile, bool straddle, int m0, int n0, int m_valid, int N, int g,
                                               long long group_stride, long long ld, uint8_t* dst, int ct, int lane,
                                               uint32_t out_full) {
  constexpr int kChunks = 256 / 8;   // 16-byte chunks per tile row
  ptx::fence_proxy_async_smem();     // this thread's tile writes -> visible to the async proxy (TMA)
  if (straddle) {
    ptx::named_bar_sync(1, 256);
    for (int i = ct; i < 128 * kChunks; i += 256) {
      const int r = i / kChunks, ch = i % kChunks;
      const int m = m0 + r, n = n0 + ch * 8;
      if (m < m_valid && n < N) {
        const uint4 v = *reinterpret_cast<const uint4*>(tile + (ch >> 3) * (128 * kSwizzleBytes) + r * kSwizzleBytes +
                                                        (((ch & 7) ^ (r & 7)) << 4));
        *reinterpret_cast<uint4*>(dst + (static_cast<long long>(g) * group_stride + static_cast<long long>(m) * ld + n) * 2) = v;
      }
    }
  }
  __syncwarp();
  if (lane == 0) ptx::mbar_arrive(out_full);
}

// Resource budget (deliberate): 384 threads x 144 registers = 55296 of the SM's 65536 registers (the producer warpgroup
// shrinks to 40 per thread, the two consumer warpgroups grow to 192: 128 x 40 + 256 x 192 = 54272) and 202 KB of its
// 228 KB shared memory, so ONE 128-thread x 64-register block of the dispatch kernel (encode_rows, which needs no
// shared memory) always fits next to a GEMM CTA.  That is what makes the dispatch+GEMM fusion deadlock-free: a GEMM
// whose producer spins on arrival flags can never starve the kernel that publishes them, whichever gets the SMs first.
// (This is the BN = 128 configuration; the BN = 256 one takes the whole SM and is never used by the fused engine.)
template <int BN_, bool A_MN, bool B_MN, int DT, bool PK>
__global__ void __maxnreg__(Cfg<BN_>::MAXNREG)
gemm_sm90_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmB2, const __grid_constant__ CUtensorMap tmD,
                 const __grid_constant__ CUtensorMap tmAux, const __grid_constant__ CUtensorMap tmD2,
                 const GemmArgs args) {
  using C = Cfg<BN_>;
  constexpr int BN = C::BN;
  extern __shared__ uint8_t smem_raw[];

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);  // warp-uniform role id
  const int lane = threadIdx.x & 31;

  // ---- shared memory carve-up (operand ring and output tile must be 1024B aligned for the 128B swizzle) ----
  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr int stages = C::STAGES;
  const uint32_t out_base = smem_base + static_cast<uint32_t>(stages) * C::STAGE_BYTES;   // 128 x 256 only
  const uint32_t bar_base = out_base + C::OUT_TILE_BYTES;
  auto smem_a = [&](int s) { return smem_base + s * C::STAGE_BYTES; };
  auto smem_b = [&](int s) { return smem_base + s * C::STAGE_BYTES + C::A_BYTES; };
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 64u + 8u * s; };
  // 128 x 256: the aux operand has landed in the output tile / the store warp has finished reading the output tile / the
  // consumers have handed the output tile to the store warp / a tile's side inputs have landed in slot 0 or 1
  const uint32_t aux_full = bar_base + 128u;
  const uint32_t out_empty = bar_base + 136u;
  const uint32_t out_full = bar_base + 144u;
  auto side_full = [&](uint32_t slot) { return bar_base + 152u + 8u * slot; };
  const uint32_t epi_base = bar_base + C::BAR_BYTES;
  float* epi_ptr = reinterpret_cast<float*>(smem_raw + (epi_base - ptx::smem_u32(smem_raw)));
  uint8_t* out_tile = smem_raw + (out_base - ptx::smem_u32(smem_raw));
  // 128 x 256 (EPI_BYTES is 0): eight rows of BN bias-gradient partial sums, then the two side-input slots
  float* colsum_part = epi_ptr;
  const uint32_t side_base = epi_base + C::COLSUM_BYTES;
  // The 128 x 256 epilogue reads the aux operand of RELU_BWD / ADD / ACT_BWD from the output tile; the store warp loads
  // it there with TMA while the main loop runs.
  const bool aux_tma = C::WIDE && (args.epilogue == EPI_RELU_BWD || args.epilogue == EPI_ADD || args.epilogue == EPI_ACT_BWD);
  // ... and the bias and column scales from the tile's side-input slot, which the store warp fills
  const bool side_bias = C::WIDE && args.bias != nullptr && !aux_tma && args.epilogue != EPI_NONE;
  const bool side_in = side_bias || (C::WIDE && args.scale_b != nullptr);
  // BIAS_GELU / BIAS_SILU with a pre-activation output: every tile goes through the output tile twice (d2, then d)
  const bool pre_act = C::WIDE && args.d2 != nullptr && (args.epilogue == EPI_BIAS_GELU || args.epilogue == EPI_BIAS_SILU);
  // block-mapped B: every row of a computed tile is stored, rows past the count as zeros
  const bool zero_pad = PK && args.b_group_map != nullptr;
  const bool ragged_k = PK && args.k_offsets != nullptr;

  if (warp == 0 && ptx::elect_one()) {
    ptx::prefetch_tensormap(&tmA);
    ptx::prefetch_tensormap(&tmB);
    if (args.dual) ptx::prefetch_tensormap(&tmB2);
    if (C::WIDE) ptx::prefetch_tensormap(&tmD);
    if (aux_tma) ptx::prefetch_tensormap(&tmAux);
    if (pre_act) ptx::prefetch_tensormap(&tmD2);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < stages; ++s) {
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), 2);   // one arrival per consumer warpgroup
    }
    ptx::mbar_init(aux_full, 1);
    ptx::mbar_init(out_empty, 1);
    ptx::mbar_init(out_full, 8);         // one arrival per consumer warp
    ptx::mbar_init(side_full(0), 1);
    ptx::mbar_init(side_full(1), 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();

  constexpr int kEltBytes = (DT == DT_E4M3 || DT == DT_E5M2) ? 1 : 2;   // 2: wgmma k16   1: wgmma k32
  static_assert(kEltBytes == 2 || (!A_MN && !B_MN), "8-bit operands are K-major only");
  const int num_kb = (args.K * kEltBytes + kSwizzleBytes - 1) / kSwizzleBytes;
  constexpr int bk_elems = kSwizzleBytes / kEltBytes;        // K elements per stage
  const long long tile_step = gridDim.x;
  const long long tile_first = blockIdx.x;
  constexpr int kBand = 16;
  // The GLU epilogues run on the 128 x 128 configuration only: with 64 accumulator columns still in registers, their
  // 32-column gate / up / gradient segments do not fit the consumers' 232 registers.
  const bool dual = !C::WIDE && args.dual != 0;
  const int tile_n = dual ? BN / 2 : BN;   // output columns per tile

  if (warp < 4) {
    ptx::setmaxnreg_dec<40>();
    if (warp == 0) {
      // =============================== TMA producer ===============================
      int s = 0;
      uint32_t ph = 0;
      int seen_group = -1;
      unsigned long long seen_mask = 0ull;
      for (long long t = tile_first; t < args.num_tiles; t += tile_step) {
        const TileCoord tc = tile_of<kBand, PK>(t, args);
        if (args.row_counts != nullptr && tc.m_blk * C::BM >= args.row_counts[tc.g]) continue;
        const int m0 = tc.m_blk * C::BM;
        const int n0 = tc.n_blk * BN;   // (non-dual) first B column of this tile
        // ragged K: A and B are single tensors, walked from the group's first K row
        const int2 kr = k_range_of<PK>(tc.g, num_kb, bk_elems, args);
        const int ga = ragged_k ? 0 : tc.g;
        const int gb = ragged_k ? 0 : b_group_of<PK>(tc.g, args);
        if (args.wait_flags != nullptr) {
          // Dispatch fusion: rows of this tile are pushed by peer GPUs; acquire their release flags - once per
          // (group, flag): consecutive tiles of a group share flags, so remember which ones were already seen.
          if (tc.g != seen_group) { seen_group = tc.g; seen_mask = 0ull; }
          const int f0 = (tc.m_blk * C::BM) / args.wait_rows_per_flag;
          const int f1 = (min(tc.m_blk * C::BM + C::BM, args.M) - 1) / args.wait_rows_per_flag;
          unsigned long long need = 0ull;
          for (int f = f0; f <= f1; ++f) need |= 1ull << (f & 63);
          if ((seen_mask & need) != need) {
            if (lane == 0) {
              for (int f = f0; f <= f1; ++f)
                if (!((seen_mask >> (f & 63)) & 1ull))
                  ptx::wait_flag_ge_sys_quiet(args.wait_flags + static_cast<long long>(tc.g) * args.wait_flags_per_group + f,
                                        args.wait_target);
              ptx::fence_proxy_async_global();  // order the upcoming async-proxy (TMA) reads after the acquire
            }
            __syncwarp();
            seen_mask |= need;
          }
        }
        for (int kb = 0; kb < kr.x; ++kb) {
          ptx::mbar_wait_quiet(empty_bar(s), ph ^ 1u);
          if (ptx::elect_one()) {
            const uint32_t fb = full_bar(s);
            ptx::mbar_expect_tx(fb, C::STAGE_BYTES);
            const int k0 = kr.y + kb * bk_elems;
            constexpr int chunk_elems = kSwizzleBytes / kEltBytes;    // MN-major: one 128-byte chunk of the MN axis ...
            constexpr int chunk_bytes = bk_elems * kSwizzleBytes;     // ... times the stage's K rows
            // ---- A ----
            if constexpr (!A_MN) {
              ptx::tma_load_3d(smem_a(s), &tmA, fb, k0, m0, ga);
            } else {
              for (int c = 0; c < C::BM / chunk_elems; ++c)
                ptx::tma_load_3d(smem_a(s) + c * chunk_bytes, &tmA, fb, m0 + c * chunk_elems, k0, ga);
            }
            // ---- B ----
            if (!dual) {
              if constexpr (!B_MN) {
                ptx::tma_load_3d(smem_b(s), &tmB, fb, k0, n0, gb);
              } else {
                for (int c = 0; c < BN / chunk_elems; ++c)
                  ptx::tma_load_3d(smem_b(s) + c * chunk_bytes, &tmB, fb, n0 + c * chunk_elems, k0, gb);
              }
            } else {
              // GLU: accumulator columns [0, BN/2) come from B, [BN/2, BN) from B2, both at weight columns nb0...
              const int nb0 = tc.n_blk * (BN / 2);
              if constexpr (!B_MN) {
                ptx::tma_load_3d(smem_b(s), &tmB, fb, k0, nb0, gb);
                ptx::tma_load_3d(smem_b(s) + (BN / 2) * kSwizzleBytes, &tmB2, fb, k0, nb0, gb);
              } else {
                constexpr int half_chunks = (BN / 2) / chunk_elems;
                for (int c = 0; c < 2 * half_chunks; ++c)
                  ptx::tma_load_3d(smem_b(s) + c * chunk_bytes, c < half_chunks ? &tmB : &tmB2, fb,
                                   nb0 + (c % half_chunks) * chunk_elems, k0, gb);
              }
            }
          }
          __syncwarp();
          if (++s == stages) { s = 0; ph ^= 1u; }
        }
      }
    } else if (C::WIDE && warp == 1) {
      // =============================== store warp (128 x 256) ===============================
      // Walks the consumers' tile sequence one tile behind them.  Each time the consumers hand over the output tile
      // (out_full), lane 0 TMA-stores it; the whole warp meanwhile adds up the bias-gradient partial rows; once the store
      // has read the tile, it is released to the consumers: with the next tile's aux operand (aux_full) for the aux
      // epilogues, by out_empty otherwise.  A tile's side inputs are copied into slot it % 2 when the consumers have handed
      // over tile it - 1, which they could only do after they had read slot it % 2 for tile it - 2.
      const int side_es = args.bias_is_fp32 ? 4 : 2;
      uint32_t it = 0;     // tiles seen
      uint32_t outs = 0;   // output tiles handed over so far (two per tile with pre_act)
      TileCoord prev{};
      int prev_m_valid = 0;
      // Stores the tile the consumers hand over next, through `map`; then releases it (with `next`'s aux operand when
      // has_next).
      auto drain = [&](const CUtensorMap* map, const TileCoord& tc, int m_valid, bool colsum, bool has_next, TileCoord next) {
        const int m0 = tc.m_blk * C::BM, n0 = tc.n_blk * BN;
        const bool straddle = zero_pad ? false : m0 + C::BM > m_valid && m_valid < args.M;   // the consumers copied it out row-guarded
        ptx::mbar_wait_quiet(out_full, outs & 1u);
        if (!straddle && lane == 0) {
          for (int b = 0; b < BN / 64; ++b)
            if (n0 + 64 * b < args.N) ptx::tma_store_3d(map, out_base + b * C::OUT_BOX_BYTES, n0 + 64 * b, m0, tc.g);
          ptx::bulk_commit_group();
        }
        if (colsum) {
          // the eight consumer warps' rows, added in warp order: lane l owns columns 4 l.. and 128 + 4 l..
#pragma unroll 1
          for (int h = 0; h < 2; ++h) {
            const int c = 128 * h + 4 * lane;
            float4 v = *reinterpret_cast<const float4*>(colsum_part + c);
#pragma unroll
            for (int w = 1; w < 8; ++w) {
              const float4 p = *reinterpret_cast<const float4*>(colsum_part + w * BN + c);
              v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
            }
            const int n = n0 + c;
            if (n < args.N) {   // N is a multiple of 8: all four columns are in range
              float* cs = args.colsum + static_cast<long long>(b_group_of<PK>(tc.g, args)) * args.colsum_group_stride + n;
              if ((reinterpret_cast<uintptr_t>(cs) & 15) == 0) {
                ptx::red_add_v4_f32(cs, v.x, v.y, v.z, v.w);
              } else {
                atomicAdd(cs, v.x); atomicAdd(cs + 1, v.y); atomicAdd(cs + 2, v.z); atomicAdd(cs + 3, v.w);
              }
            }
          }
        }
        __syncwarp();   // every lane has read the partial rows
        if (lane == 0) {
          ptx::bulk_wait_group_read<0>();   // the store has read the output tile
          if (has_next) {
            ptx::mbar_expect_tx(aux_full, C::OUT_TILE_BYTES);
            for (int b = 0; b < BN / 64; ++b)
              ptx::tma_load_3d(out_base + b * C::OUT_BOX_BYTES, &tmAux, aux_full, next.n_blk * BN + 64 * b,
                               next.m_blk * C::BM, next.g);
          } else if (!aux_tma) {
            ptx::mbar_arrive(out_empty);
          }
        }
        __syncwarp();
        ++outs;
      };
      for (long long t = tile_first; t < args.num_tiles; t += tile_step) {
        const TileCoord tc = tile_of<kBand, PK>(t, args);
        int m_valid = args.M;
        if (args.row_counts != nullptr) {
          m_valid = min(args.M, args.row_counts[tc.g]);
          if (tc.m_blk * C::BM >= m_valid) continue;
        }
        if (it > 0 && pre_act) drain(&tmD2, prev, prev_m_valid, false, false, prev);
        if (side_in) {
          // tile it's bias / column scales -> slot it % 2 (the consumers have finished tile it - 2 once out_full of
          // tile it - 1 has completed; with pre_act its first hand-over is enough)
          if (it > 0 && !pre_act) ptx::mbar_wait_quiet(out_full, outs & 1u);
          const int n0 = tc.n_blk * BN;
          const int gb = b_group_of<PK>(tc.g, args);
          const int cols = min(BN, args.N - n0);
          const uint32_t slot = side_base + (it & 1u) * C::SIDE_SLOT_BYTES;
          // (16-byte aligned: see gemm_sm90_launch)
          const uint8_t* bsrc = reinterpret_cast<const uint8_t*>(args.bias) +
                                (static_cast<long long>(gb) * args.bias_group_stride + n0) * side_es;
          const float* ssrc = args.scale_b + static_cast<long long>(gb) * args.scale_b_group_stride + n0;
          if (lane == 0) {
            const uint32_t bar = side_full(it & 1u);
            ptx::mbar_expect_tx(bar, (side_bias ? cols * side_es : 0) + (args.scale_b != nullptr ? cols * 4 : 0));
            if (side_bias) ptx::bulk_load(slot, bsrc, cols * side_es, bar);
            if (args.scale_b != nullptr) ptx::bulk_load(slot + C::SIDE_BIAS_BYTES, ssrc, cols * 4, bar);
          }
          __syncwarp();
        }
        if (it > 0) drain(&tmD, prev, prev_m_valid, args.colsum != nullptr, aux_tma, tc);
        else if (aux_tma && lane == 0) {   // the output tile is free: tile 0's aux operand
          ptx::mbar_expect_tx(aux_full, C::OUT_TILE_BYTES);
          for (int b = 0; b < BN / 64; ++b)
            ptx::tma_load_3d(out_base + b * C::OUT_BOX_BYTES, &tmAux, aux_full, tc.n_blk * BN + 64 * b, tc.m_blk * C::BM, tc.g);
        }
        __syncwarp();
        prev = tc;
        prev_m_valid = m_valid;
        ++it;
      }
      if (it > 0) {
        if (pre_act) drain(&tmD2, prev, prev_m_valid, false, false, prev);
        drain(&tmD, prev, prev_m_valid, args.colsum != nullptr, false, prev);
      }
      if (lane == 0) ptx::bulk_wait_group<0>();   // the last tile's store has completed
    }
  } else {
    ptx::setmaxnreg_inc<C::CONSUMER_REGS>();
    // =============================== consumers: wgmma main loop + epilogue ===============================
    const int cw = warp - 4;          // consumer warp 0..7 owns tile rows [16 cw, 16 cw + 16)
    const int wg = cw >> 2;           // consumer warpgroup: tile rows [64 wg, 64 wg + 64)
    const bool wg_leader = (threadIdx.x & 127) == 0;
    int s = 0;
    uint32_t ph = 0;
    // Descriptor = constant high word + low word {start>>4, lbo>>4}.  Advancing along K inside a stage and
    // from stage to stage only adds to the 14-bit start-address field (smem < 256 KB, so it never carries).
    constexpr uint32_t kMnChunkBytes = 64u * kSwizzleBytes;           // BK rows * 128 B (16-bit operands)
    constexpr uint32_t kMnKStep = 16u * kSwizzleBytes;                // 16 K rows * 128 B
    constexpr uint32_t a_lbo = A_MN ? kMnChunkBytes : 16u;
    constexpr uint32_t b_lbo = B_MN ? kMnChunkBytes : 16u;
    constexpr uint32_t a_kstep = (A_MN ? kMnKStep : 32u) >> 4;
    constexpr uint32_t b_kstep = (B_MN ? kMnKStep : 32u) >> 4;
    constexpr uint32_t desc_hi = (1024u >> 4) | (1u << 30);           // SBO | SWIZZLE_128B
    // this warpgroup's 64 rows of A: K-major 64 rows x 128 B, MN-major one 64-element chunk - 8 KB either way
    const uint32_t a_lo0 = (((smem_a(0) + static_cast<uint32_t>(wg) * 8192u) >> 4) & 0x3FFFu) | ((a_lbo >> 4) << 16);
    const uint32_t b_lo0 = ((smem_b(0) >> 4) & 0x3FFFu) | ((b_lbo >> 4) << 16);

    const bool out16 = (args.out_dtype != DT_FP32);
    const bool out_bf16 = (args.out_dtype == DT_BF16);
    const bool glu = !C::WIDE && (args.epilogue == EPI_GLU || args.epilogue == EPI_GLU_BWD);
    // Epilogue geometry: lane l works on accumulator row (l % 16) of this warp and on 32 consecutive columns, the
    // lower half-warp on the first and the upper half-warp on the second half of every 64-column chunk.
    float* epi_warp = epi_ptr + cw * 16 * C::EPI_PITCH;
    const float* epi_row = epi_warp + (lane & 15) * C::EPI_PITCH;
    const int col_half = (lane >> 4) * 32;
    auto load_acc = [&](int col, float* v) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 t4 = *reinterpret_cast<const float4*>(epi_row + col + q * 4);
        v[q * 4] = t4.x; v[q * 4 + 1] = t4.y; v[q * 4 + 2] = t4.z; v[q * 4 + 3] = t4.w;
      }
    };
    // 128 x 256 epilogue geometry (see wide_main): this thread's words of the output tile are at row0 + out_tile_off(j)
    // and 8 rows further down.
    const int ct = threadIdx.x - 128;       // consumer thread 0..255
    const int r0 = cw * 16 + (lane >> 2);
    const int swz = lane >> 2;              // = r0 % 8
    uint8_t* row0 = out_tile + r0 * kSwizzleBytes + (lane & 3) * 4;
    const int wmain = args.epilogue == EPI_NONE ? WM_NONE
                    : args.epilogue == EPI_ADD ? WM_ADD
                    : args.epilogue == EPI_RELU_BWD ? WM_RELU_BWD
                    : args.epilogue == EPI_ACT_BWD ? (args.act == ACT_GELU ? WM_GELU_BWD : args.act == ACT_SILU ? WM_SILU_BWD : WM_RELU_BWD)
                    : WM_BIAS;
    uint32_t it = 0;     // tiles processed
    uint32_t outs = 0;   // 128 x 256: output tiles handed to the store warp

    for (long long t = tile_first; t < args.num_tiles; t += tile_step) {
      const TileCoord tc = tile_of<kBand, PK>(t, args);
      int m_valid = args.M;
      if (args.row_counts != nullptr) {
        m_valid = min(args.M, args.row_counts[tc.g]);
        if (tc.m_blk * C::BM >= m_valid) continue;
      }
      const int tile_kb = ragged_k ? k_range_of<PK>(tc.g, num_kb, bk_elems, args).x : num_kb;
      // ------------------------------- main loop -------------------------------
      float acc[BN / 2];
      // (packed launches zero it too: an empty K range of a ragged-K tile runs no wgmma at all.  A definition that depends
      // on the tile, or a wgmma wait on a divergent path, would make ptxas serialise every wgmma of the main loop.)
      if (C::WIDE || PK) {
        // The first wgmma of a tile ignores the accumulator, but its register operands are read-write: without a fresh
        // definition the previous tile's 128 values would stay live through the whole epilogue.
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
      }
      int prev_s = 0;
      for (int kb = 0; kb < tile_kb; ++kb) {
        ptx::mbar_wait_quiet(full_bar(s), ph);
        const uint32_t a_lo = a_lo0 + static_cast<uint32_t>(s) * (C::STAGE_BYTES >> 4);
        const uint32_t b_lo = b_lo0 + static_cast<uint32_t>(s) * (C::STAGE_BYTES >> 4);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t ad = (static_cast<uint64_t>(desc_hi) << 32) | (a_lo + k * a_kstep);
          const uint64_t bd = (static_cast<uint64_t>(desc_hi) << 32) | (b_lo + k * b_kstep);
          if constexpr (BN == 256) ptx::wgmma_m64n256<DT, A_MN, B_MN>(acc, ad, bd, (kb | k) != 0);
          else ptx::wgmma_m64n128<DT, A_MN, B_MN>(acc, ad, bd, (kb | k) != 0);
        }
        ptx::wgmma_commit();
        if (kb > 0) {
          ptx::wgmma_wait<1>();                                   // the group that read the previous stage has retired
          if (wg_leader) ptx::mbar_arrive(empty_bar(prev_s));
        }
        prev_s = s;
        if (++s == stages) { s = 0; ph ^= 1u; }
      }
      ptx::wgmma_wait<0>();
      // (ragged K: an empty K range leaves the zeroed accumulator and consumes no stage)
      if (wg_leader && (!PK || tile_kb > 0)) ptx::mbar_arrive(empty_bar(prev_s));

      if constexpr (C::WIDE) {
        // ------------------------- 128 x 256 epilogue -------------------------
        const int m0 = tc.m_blk * C::BM, n0 = tc.n_blk * BN;
        const bool ok0 = m0 + r0 < m_valid, ok1 = m0 + r0 + 8 < m_valid;
        // block-mapped B stores rows past the count as zeros (branch-free: see the accumulator's definition above)
        const bool keep0 = !zero_pad || ok0, keep1 = !zero_pad || ok1;
        const int n_lane = 2 * (lane & 3);   // column in the tile
        const int n_lim = args.N - n0;
        // a row block that straddles the group's row count (at most one per group) must not write past the count,
        // which the output tensor map cannot express: it is copied out with row-guarded stores instead
        const bool straddle = zero_pad ? false : m0 + C::BM > m_valid && m_valid < args.M;
        // this tile's bias / column scales have landed in its side-input slot
        const uint8_t* side = reinterpret_cast<const uint8_t*>(colsum_part + 8 * BN) + (it & 1u) * C::SIDE_SLOT_BYTES;
        if (side_in) ptx::mbar_wait_quiet(side_full(it & 1u), (it >> 1) & 1u);
        if (args.scale_a != nullptr || args.scale_b != nullptr) {
          const float* sa = args.scale_a != nullptr ? args.scale_a + static_cast<long long>(tc.g) * args.scale_a_group_stride + m0 + r0 : nullptr;
          const float sa0 = (sa != nullptr && ok0) ? sa[0] : 1.0f;
          const float sa1 = (sa != nullptr && ok1) ? sa[8] : 1.0f;
          const float* sb = args.scale_b != nullptr ? reinterpret_cast<const float*>(side + C::SIDE_BIAS_BYTES) : nullptr;
          wide_scale(acc, sa0, sa1, sb, n_lane, n_lim);
        }
        // the output tile is free again: the store warp has read tile it - 1 (two hand-overs per tile with pre_act)
        auto wait_out_free = [&]() { ptx::mbar_wait_quiet(out_empty, (outs & 1u) ^ 1u); };
        auto hand_over = [&](uint8_t* dst) {
          hand_over_tile(out_tile, straddle, m0, n0, m_valid, args.N, tc.g, args.d_group_stride, args.ldd, dst, ct, lane, out_full);
          ++outs;
        };

        if (wmain == WM_BIAS) {
          if (side_bias)
            wide_main<WM_BIAS>(acc, row0, swz, side, args.bias_is_fp32 != 0, args.bias_is_bf16 != 0, n_lane, n_lim, out_bf16, 1.0f);
          if (pre_act) {
            // training: the backward pass needs the pre-activation (ReLU gets by with the sign of its output)
            wait_out_free();
            if constexpr (PK) wide_zero_rows(acc, keep0, keep1);
            wide_stage(acc, row0, swz, out_bf16);
            hand_over(reinterpret_cast<uint8_t*>(args.d2));
          }
          if (args.epilogue == EPI_BIAS_RELU) wide_act<ACT_RELU>(acc);
          else if (args.epilogue == EPI_BIAS_GELU) wide_act<ACT_GELU>(acc);
          else if (args.epilogue == EPI_BIAS_SILU) wide_act<ACT_SILU>(acc);
        } else if (wmain == WM_NONE) {
          if (args.alpha != 1.0f) wide_main<WM_NONE>(acc, row0, swz, nullptr, false, false, n_lane, n_lim, out_bf16, args.alpha);
        } else {
          ptx::mbar_wait_quiet(aux_full, it & 1u);   // this tile's aux operand is in the output tile
          if (wmain == WM_RELU_BWD) wide_main<WM_RELU_BWD>(acc, row0, swz, nullptr, false, false, n_lane, n_lim, out_bf16, 1.0f);
          else if (wmain == WM_ADD) wide_main<WM_ADD>(acc, row0, swz, nullptr, false, false, n_lane, n_lim, out_bf16, 1.0f);
          else if (wmain == WM_GELU_BWD) wide_main<WM_GELU_BWD>(acc, row0, swz, nullptr, false, false, n_lane, n_lim, out_bf16, 1.0f);
          else wide_main<WM_SILU_BWD>(acc, row0, swz, nullptr, false, false, n_lane, n_lim, out_bf16, 1.0f);
        }
        if (!aux_tma) wait_out_free();
        if constexpr (PK) wide_zero_rows(acc, keep0, keep1);
        wide_stage(acc, row0, swz, out_bf16);     // aux epilogues: each word overwrites the aux word it was computed from
        // the partial rows are free: the store warp read them before it released the output tile
        if (args.colsum != nullptr) wide_colsum(acc, ok0, ok1, lane, colsum_part + cw * BN);
        hand_over(reinterpret_cast<uint8_t*>(args.d));
        ++it;
        continue;
      }

      // ------------------------------- 128 x 128 epilogue -------------------------------
      {
        const int fr = lane >> 2, fc = (lane & 3) * 2;
#pragma unroll
        for (int j = 0; j < C::EPI_COLS / 8; ++j) {
          *reinterpret_cast<float2*>(epi_warp + fr * C::EPI_PITCH + j * 8 + fc) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(epi_warp + (fr + 8) * C::EPI_PITCH + j * 8 + fc) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
      __syncwarp();

      const int m = tc.m_blk * C::BM + cw * 16 + (lane & 15);
      const bool row_ok = m < m_valid;
      const int gb = b_group_of<PK>(tc.g, args);
      uint8_t* d_base = (args.d_ptr_table != nullptr)
                            ? reinterpret_cast<uint8_t*>(args.d_ptr_table[tc.g])
                            : reinterpret_cast<uint8_t*>(args.d) +
                                  static_cast<long long>(tc.g) * args.d_group_stride * (out16 ? 2 : 4);
      uint8_t* d_row = d_base + static_cast<long long>(m) * args.ldd * (out16 ? 2 : 4);
      const uint8_t* aux_row = nullptr;
      if (args.aux != nullptr)
        aux_row = reinterpret_cast<const uint8_t*>(args.aux) +
                  (static_cast<long long>(tc.g) * args.aux_group_stride + static_cast<long long>(m) * args.ld_aux) * 2;
      const uint8_t* aux2_row = nullptr;
      if (args.aux2 != nullptr)
        aux2_row = reinterpret_cast<const uint8_t*>(args.aux2) +
                   (static_cast<long long>(tc.g) * args.aux_group_stride + static_cast<long long>(m) * args.ld_aux) * 2;
      const uint8_t* bias_g = nullptr;
      if (args.bias != nullptr)
        bias_g = reinterpret_cast<const uint8_t*>(args.bias) +
                 static_cast<long long>(gb) * args.bias_group_stride * (args.bias_is_fp32 ? 4 : 2);

      // One 32-column segment of this lane's row -> global memory (local or a peer's): 64 contiguous bytes in 16 bit.
      // ncols (a multiple of 8) may be <= 0 for segments past the last column: nothing is touched then.
      // Block-mapped B stores rows past the count as zeros.
      auto store_seg = [&](uint8_t* row, int n, int ncols, const float* v) {
        if (!row_ok && !(zero_pad && m < args.M)) return;
        if (out16) {
          uint32_t w[16];
          pack32(v, w, out_bf16);
          if (zero_pad && !row_ok) {
#pragma unroll
            for (int q = 0; q < 16; ++q) w[q] = 0u;
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            if (q * 8 < ncols) {
              *reinterpret_cast<uint4*>(row + (n + q * 8) * 2) = make_uint4(w[q * 4], w[q * 4 + 1], w[q * 4 + 2], w[q * 4 + 3]);
            }
          }
        } else {
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            if (q * 4 < ncols) {
              float4 o = (!zero_pad || row_ok) ? make_float4(v[q * 4], v[q * 4 + 1], v[q * 4 + 2], v[q * 4 + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
              *reinterpret_cast<float4*>(row + (n + q * 4) * 4) = o;
            }
          }
        }
      };
      // 32 values of a 16-bit [.., ld] side input (zeros for rows / columns past the end)
      auto load_seg16 = [&](const uint8_t* row, int n, int ncols, float* f) {
        uint4 p[4];
#pragma unroll
        for (int q = 0; q < 4; ++q)
          p[q] = (row_ok && q * 8 < ncols) ? ptx::ld_nc_v4(row + (n + q * 8) * 2) : make_uint4(0u, 0u, 0u, 0u);
        unpack32(p, f, out_bf16);
      };

      if (glu) {
        // ---------------- gated-linear-unit epilogues ----------------
        const bool fwd = args.epilogue == EPI_GLU;
        const long long row_off = (static_cast<long long>(tc.g) * args.d_group_stride + static_cast<long long>(m) * args.ldd) * 2;
        uint8_t* d2_row = args.d2 != nullptr ? reinterpret_cast<uint8_t*>(args.d2) + row_off : nullptr;
        uint8_t* d3_row = args.d3 != nullptr ? reinterpret_cast<uint8_t*>(args.d3) + row_off : nullptr;
        const float sa = (args.scale_a != nullptr && row_ok)
                             ? args.scale_a[static_cast<long long>(tc.g) * args.scale_a_group_stride + m] : 1.0f;
#pragma unroll 1
        for (int c = 0; c < tile_n / 64; ++c) {
          const int col = c * 64 + col_half;
          const int n = tc.n_blk * tile_n + col;
          const int ncols = min(32, args.N - n);
          float g[32], u[32], o[32];
          if (fwd) {
            load_acc(col, g);
            load_acc(BN / 2 + col, u);
            if (args.scale_a != nullptr || args.scale_b != nullptr) {
              const float* sb = args.scale_b != nullptr ? args.scale_b + static_cast<long long>(gb) * args.scale_b_group_stride + n : nullptr;
              const float* sb2 = args.scale_b2 != nullptr ? args.scale_b2 + static_cast<long long>(gb) * args.scale_b_group_stride + n : nullptr;
#pragma unroll
              for (int j = 0; j < 32; ++j) {
                g[j] *= (sb != nullptr && j < ncols) ? sa * sb[j] : sa;
                u[j] *= (sb2 != nullptr && j < ncols) ? sa * sb2[j] : sa;
              }
            }
            if (d2_row != nullptr) {       // training: keep the pre-activations for the backward pass
              store_seg(d2_row, n, ncols, g);
              store_seg(d3_row, n, ncols, u);
            }
            if (args.act == ACT_RELU) glu_fwd_seg<ACT_RELU>(g, u, o);
            else if (args.act == ACT_GELU) glu_fwd_seg<ACT_GELU>(g, u, o);
            else glu_fwd_seg<ACT_SILU>(g, u, o);
            store_seg(d_row, n, ncols, o);
          } else {
            float dh[32];
            load_acc(col, dh);
            if (args.scale_a != nullptr || args.scale_b != nullptr) {     // fp8 operands: dh = acc * sa[m] * sb[n]
              const float* sb = args.scale_b != nullptr ? args.scale_b + static_cast<long long>(gb) * args.scale_b_group_stride + n : nullptr;
#pragma unroll
              for (int j = 0; j < 32; ++j) dh[j] *= (sb != nullptr && j < ncols) ? sa * sb[j] : sa;
            }
            load_seg16(aux_row, n, ncols, g);
            load_seg16(aux2_row, n, ncols, u);
            if (args.act == ACT_RELU) glu_bwd_seg<ACT_RELU>(dh, g, u, o);
            else if (args.act == ACT_GELU) glu_bwd_seg<ACT_GELU>(dh, g, u, o);
            else glu_bwd_seg<ACT_SILU>(dh, g, u, o);
            store_seg(d_row, n, ncols, o);
            store_seg(d2_row, n, ncols, u);
          }
        }
      } else {
#pragma unroll 1
      for (int c = 0; c < C::EPI_COLS / 64; ++c) {
        const int col = c * 64 + col_half;
        const int n = tc.n_blk * BN + col;
        float v[32];
        load_acc(col, v);
        const int ncols = min(32, args.N - n);  // multiple of 8, <= 0 past the last column
        if (args.scale_a != nullptr || args.scale_b != nullptr) {
          // fp8 operands were quantised with one scale per A row and per B column: D = acc * sa[m] * sb[n]
          const float sa = (args.scale_a != nullptr && row_ok)
                               ? args.scale_a[static_cast<long long>(tc.g) * args.scale_a_group_stride + m] : 1.0f;
          const float* sb = args.scale_b != nullptr ? args.scale_b + static_cast<long long>(gb) * args.scale_b_group_stride + n : nullptr;
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] *= (sb != nullptr && j < ncols) ? sa * sb[j] : sa;
        }

        if (args.epilogue == EPI_NONE) {
          if (args.alpha != 1.0f) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] *= args.alpha;
          }
        } else if (args.epilogue == EPI_RELU_BWD || args.epilogue == EPI_ADD || args.epilogue == EPI_ACT_BWD) {
          float f[32];
          load_seg16(aux_row, n, ncols, f);
          if (args.epilogue == EPI_RELU_BWD) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = relu_bwd(v[j], f[j]);
          } else if (args.epilogue == EPI_ADD) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] += f[j];
          } else if (args.act == ACT_GELU) {      // f = pre-activation
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = gelu_bwd(v[j], f[j]);
          } else if (args.act == ACT_SILU) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = silu_bwd(v[j], f[j]);
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = relu_bwd(v[j], f[j]);
          }
        } else {
          if (bias_g != nullptr) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              if (q * 8 < ncols) {
                float f[8];
                if (args.bias_is_fp32) {
                  const float4 b0 = *reinterpret_cast<const float4*>(bias_g + (n + q * 8) * 4);
                  const float4 b1 = *reinterpret_cast<const float4*>(bias_g + (n + q * 8 + 4) * 4);
                  f[0] = b0.x; f[1] = b0.y; f[2] = b0.z; f[3] = b0.w;
                  f[4] = b1.x; f[5] = b1.y; f[6] = b1.z; f[7] = b1.w;
                } else {
                  unpack8(*reinterpret_cast<const uint4*>(bias_g + (n + q * 8) * 2), args.bias_is_bf16 != 0, f);
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) v[q * 8 + j] += f[j];
              }
            }
          }
          if (args.d2 != nullptr && (args.epilogue == EPI_BIAS_GELU || args.epilogue == EPI_BIAS_SILU)) {
            // training: the backward pass needs the pre-activation (ReLU gets by with the sign of its output)
            uint8_t* d2_row = reinterpret_cast<uint8_t*>(args.d2) +
                              (static_cast<long long>(tc.g) * args.d_group_stride + static_cast<long long>(m) * args.ldd) * (out16 ? 2 : 4);
            store_seg(d2_row, n, ncols, v);
          }
          if (args.epilogue == EPI_BIAS_RELU) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.0f);
          } else if (args.epilogue == EPI_BIAS_GELU) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = gelu_erf(v[j]);
          } else if (args.epilogue == EPI_BIAS_SILU) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = silu(v[j]);
          }
        }

        if (args.colsum != nullptr) {
          // Bias gradient fused into the epilogue: transpose-reduce each half-warp's 16 rows x 32 columns with 30
          // shuffles (afterwards lane l holds the sums of columns 2 (l % 16) + {0, 1}) and add them to the fp32
          // accumulator in global memory.
          float s[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) s[j] = row_ok ? v[j] : 0.0f;
#pragma unroll
          for (int off = 8; off >= 1; off >>= 1) {
            const bool upper = (lane & off) != 0;
#pragma unroll
            for (int i = 0; i < 2 * off; ++i) {
              const float send = upper ? s[i] : s[i + 2 * off];
              const float recv = __shfl_xor_sync(0xffffffffu, send, off);
              s[i] = (upper ? s[i + 2 * off] : s[i]) + recv;
            }
          }
          const int cc = 2 * (lane & 15);
          float* cs = args.colsum + static_cast<long long>(gb) * args.colsum_group_stride + n + cc;
          if (cc < ncols) {
            atomicAdd(cs, s[0]);
            atomicAdd(cs + 1, s[1]);
          }
        }
        store_seg(d_row, n, ncols, v);
      }
      }
      __syncwarp();   // every lane has read its row before the next tile overwrites the staging rows
      if (args.signal_ptr_table != nullptr) {
        // Combine fusion: all 256 consumer threads' (possibly remote) stores -> one release.sys counter bump.
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (cw == 0 && lane == 0) {
          ptx::fence_acq_rel_sys();
          ptx::red_add_release_sys(reinterpret_cast<uint32_t*>(args.signal_ptr_table[tc.g]), 1u);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

bool make_operand_map(CUtensorMap* map, const void* base, int dtype, bool mn_major, long long rows_mn,
                      long long k, long long ld, long long group_stride, int groups, int box_mn_kmajor,
                      const char** why) {
  EncodeTiledFn enc = get_encode_fn();
  if (enc == nullptr) { *why = "cuTensorMapEncodeTiled unavailable"; return false; }
  const int eb = (dtype == DT_E4M3 || dtype == DT_E5M2) ? 1 : 2;
  CUtensorMapDataType dt = eb == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                   : (dtype == DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
  if ((reinterpret_cast<uintptr_t>(base) & 15) || ((ld * eb) & 15) || ((group_stride * eb) & 15)) {
    *why = "operand base/stride must be 16-byte aligned";
    return false;
  }
  cuuint64_t dims[3];
  cuuint64_t strides[2];
  cuuint32_t box[3];
  cuuint32_t estr[3] = {1, 1, 1};
  const cuuint32_t row_elems = kSwizzleBytes / eb;
  if (!mn_major) {
    dims[0] = static_cast<cuuint64_t>(k); dims[1] = static_cast<cuuint64_t>(rows_mn);
    box[0] = row_elems; box[1] = static_cast<cuuint32_t>(box_mn_kmajor);
  } else {
    dims[0] = static_cast<cuuint64_t>(rows_mn); dims[1] = static_cast<cuuint64_t>(k);
    box[0] = row_elems; box[1] = row_elems;  // BK k-rows x one 128-byte MN chunk
  }
  dims[2] = static_cast<cuuint64_t>(groups);
  box[2] = 1;
  strides[0] = static_cast<cuuint64_t>(ld) * eb;
  strides[1] = static_cast<cuuint64_t>(groups > 1 ? group_stride : (mn_major ? k : rows_mn) * ld) * eb;
  if (strides[1] == 0) strides[1] = strides[0];
  CUresult r = enc(map, dt, 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { *why = "cuTensorMapEncodeTiled failed"; return false; }
  return true;
}

// A 16-bit row-major [G][rows][cols] matrix (output, aux or pre-activation of the 128 x 256 epilogue) in boxes of
// 128 rows x 64 columns, 128-byte swizzle: the layout of the kernel's output tile.  Loads past the end read zeros,
// stores past the end are dropped.
bool make_tile_map(CUtensorMap* map, const void* base, int dtype, long long rows, long long cols, long long ld,
                   long long group_stride, int groups, const char** why) {
  EncodeTiledFn enc = get_encode_fn();
  if (enc == nullptr) { *why = "cuTensorMapEncodeTiled unavailable"; return false; }
  if ((reinterpret_cast<uintptr_t>(base) & 15) || ((ld * 2) & 15) || ((group_stride * 2) & 15)) {
    *why = "output / aux base and strides must be 16-byte aligned";
    return false;
  }
  const cuuint64_t dims[3] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(groups)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(ld) * 2,
                           static_cast<cuuint64_t>(groups > 1 ? group_stride : rows * ld) * 2};
  if (strides[1] == 0) strides[1] = strides[0];
  const cuuint32_t box[3] = {64, 128, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, dtype == DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3,
                   const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { *why = "cuTensorMapEncodeTiled failed"; return false; }
  return true;
}

template <int BN, bool A_MN, bool B_MN, int DT, bool PK = false>
cudaError_t launch_inst(const CUtensorMap& ta, const CUtensorMap& tb_, const CUtensorMap& tb2, const CUtensorMap& td,
                        const CUtensorMap& taux, const CUtensorMap& td2, const GemmArgs& args, int grid,
                        cudaStream_t stream) {
  auto* kern = gemm_sm90_kernel<BN, A_MN, B_MN, DT, PK>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::SMEM_BYTES);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  kern<<<grid, kThreads, Cfg<BN>::SMEM_BYTES, stream>>>(ta, tb_, tb2, td, taux, td2, args);
  return cudaGetLastError();
}

}  // namespace

cudaError_t gemm_sm90_launch(const GemmProblem& p, cudaStream_t stream, const char** why_out) {
  const char* why_local = nullptr;
  const char** why = why_out ? why_out : &why_local;
  *why = nullptr;
  if (p.M <= 0 || p.N <= 0 || p.K <= 0 || p.G <= 0) return cudaSuccess;
  const int eb = (p.in_dtype == DT_E4M3 || p.in_dtype == DT_E5M2) ? 1 : 2;
  if (p.N % 8 != 0) { *why = "N must be a multiple of 8"; return cudaErrorInvalidValue; }
  const int ob = p.out_dtype == DT_FP32 ? 4 : 2;
  if ((reinterpret_cast<uintptr_t>(p.d) & 15) || ((p.ldd * ob) & 15) || ((p.d_group_stride * ob) & 15)) {
    *why = "output base/stride must be 16-byte aligned";
    return cudaErrorInvalidValue;
  }

  int dev = 0;
  cudaGetDevice(&dev);
  static int sm_count_cache[64] = {0};
  if (sm_count_cache[dev & 63] == 0) cudaDeviceGetAttribute(&sm_count_cache[dev & 63], cudaDevAttrMultiProcessorCount, dev);
  int sms = sm_count_cache[dev & 63];
  if (p.max_ctas > 0) sms = p.max_ctas < sms ? p.max_ctas : sms;

  const bool dual = p.epilogue == EPI_GLU;
  if (dual && (p.b2 == nullptr || p.out_dtype == DT_FP32)) { *why = "EPI_GLU needs b2 and a 16-bit output"; return cudaErrorInvalidValue; }
  if (p.epilogue == EPI_GLU_BWD && (p.aux == nullptr || p.aux2 == nullptr || p.d2 == nullptr || p.out_dtype == DT_FP32)) {
    *why = "EPI_GLU_BWD needs aux, aux2, d2 and a 16-bit output";
    return cudaErrorInvalidValue;
  }
  if ((p.epilogue == EPI_GLU || p.epilogue == EPI_GLU_BWD) && p.d_ptr_table != nullptr) { *why = "GLU epilogues write local outputs only"; return cudaErrorInvalidValue; }
  const bool uses_aux = p.epilogue == EPI_RELU_BWD || p.epilogue == EPI_ADD || p.epilogue == EPI_GLU_BWD || p.epilogue == EPI_ACT_BWD;
  if (uses_aux && (p.aux == nullptr || p.out_dtype == DT_FP32 ||
                   ((reinterpret_cast<uintptr_t>(p.aux) | reinterpret_cast<uintptr_t>(p.aux2)) & 15) || ((p.ld_aux * 2) & 15) ||
                   ((p.aux_group_stride * 2) & 15))) {
    *why = "this epilogue needs a 16-byte aligned 16-bit aux operand";
    return cudaErrorInvalidValue;
  }
  // A zero group stride (an expanded tensor) would be taken for "one group" by the tensor maps, so group g would start g
  // rows into the matrix instead of at it: such operands must be materialised by the caller.
  // (block-mapped B: as many B groups as the map names, known to the caller only; ragged K: one A and one B group)
  const int groups_b = p.k_offsets != nullptr ? 1 : p.b_group_map != nullptr ? p.b_groups :
                       (p.G + (p.b_group_div > 0 ? p.b_group_div : 1) - 1) / (p.b_group_div > 0 ? p.b_group_div : 1);
  if ((p.G > 1 && ((p.k_offsets == nullptr && p.a_group_stride == 0) || (p.d_ptr_table == nullptr && p.d_group_stride == 0) ||
                   (uses_aux && p.aux_group_stride == 0))) ||
      (groups_b > 1 && p.b_group_stride == 0)) {
    *why = "group strides of A, B, aux and the output must be nonzero when there is more than one group";
    return cudaErrorInvalidValue;
  }
  // rotate_group permutes groups within blocks of |group_mod|; a partial block would map groups past G
  const int mod_abs = p.group_mod < 0 ? -p.group_mod : p.group_mod;
  if (mod_abs > 1 && (p.G % mod_abs != 0 || p.group_rot < 0)) {
    *why = "G must be a multiple of |group_mod|, and group_rot must not be negative";
    return cudaErrorInvalidValue;
  }
  if (p.alpha != 1.0f && p.epilogue != EPI_NONE) { *why = "alpha is applied by EPI_NONE only"; return cudaErrorInvalidValue; }
  if (p.cta_group < 0 || p.cta_group > 2) { *why = "cta_group must be 0, 1 or 2"; return cudaErrorInvalidValue; }
  if (p.block_n != 0 && p.block_n != 128 && p.block_n != 256) { *why = "block_n must be 0, 128 or 256"; return cudaErrorInvalidValue; }
  const bool fused_engine = p.wait_flags != nullptr || p.signal_ptr_table != nullptr || p.d_ptr_table != nullptr;
  if (p.b_group_map != nullptr && (eb != 2 || p.k_offsets != nullptr || p.M > 128 || fused_engine || p.group_mod != 1)) {
    *why = "b_group_map needs 16-bit operands and groups of at most 128 rows, and excludes k_offsets, group rotation and the "
           "fused engine";
    return cudaErrorInvalidValue;
  }
  if (p.k_offsets != nullptr && (eb != 2 || p.b_group_div != 1 || p.scale_a != nullptr || p.scale_b != nullptr ||
                                 fused_engine || p.group_mod != 1)) {
    *why = "k_offsets needs 16-bit operands and excludes b_group_div, scales, group rotation and the fused engine";
    return cudaErrorInvalidValue;
  }

  // 128 x 256 tiles unless the caller is the fused multi-GPU engine (flags, peer stores and per-128 x 128-tile
  // completion signals are built around the 128 x 128 configuration) or pins that configuration with block_n == 128.
  // The GLU epilogues (see gemm_sm90_kernel) and fp32 outputs (the 128 x 256 output tile is 16-bit) always take the
  // 128 x 128 configuration.
  // The 128 x 256 store warp bulk-copies each tile's bias and column scales into shared memory, which needs 16-byte
  // aligned rows; scale_b rows are only required to be 8-byte aligned, and such rows take the 128 x 128 configuration too.
  const bool side_aligned =
      ((reinterpret_cast<uintptr_t>(p.bias) | static_cast<uintptr_t>(p.bias_group_stride * 2)) & 15) == 0 &&
      ((reinterpret_cast<uintptr_t>(p.scale_b) | static_cast<uintptr_t>(p.scale_b_group_stride * 4)) & 15) == 0;
  const bool wide = p.block_n != 128 && p.wait_flags == nullptr && p.signal_ptr_table == nullptr && p.d_ptr_table == nullptr &&
                    p.epilogue != EPI_GLU && p.epilogue != EPI_GLU_BWD && p.out_dtype != DT_FP32 && side_aligned;
  constexpr int bm = 128;
  const int bn = wide ? 256 : 128;
  GemmArgs a{};
  a.M = p.M; a.N = p.N; a.K = p.K; a.G = p.G;
  a.b_group_div = p.b_group_div > 0 ? p.b_group_div : 1;
  a.tiles_m = (p.M + bm - 1) / bm;
  a.tiles_n = dual ? (p.N + bn / 2 - 1) / (bn / 2) : (p.N + bn - 1) / bn;
  a.num_tiles = static_cast<long long>(a.tiles_m) * a.tiles_n * p.G;
  a.d = p.d; a.ldd = p.ldd; a.d_group_stride = p.d_group_stride; a.d_ptr_table = p.d_ptr_table;
  a.out_dtype = p.out_dtype;
  a.epilogue = p.epilogue; a.alpha = p.alpha;
  a.bias = p.bias; a.bias_group_stride = p.bias_group_stride; a.bias_is_fp32 = 0;
  a.bias_is_bf16 = (eb == 2) ? (p.in_dtype == DT_BF16) : (p.out_dtype == DT_BF16);
  a.aux = p.aux; a.ld_aux = p.ld_aux; a.aux_group_stride = p.aux_group_stride;
  a.aux2 = p.aux2; a.d2 = p.d2; a.d3 = p.d3; a.dual = dual ? 1 : 0; a.act = p.act; a.scale_b2 = p.scale_b2;
  a.row_counts = p.row_counts;
  a.colsum = p.colsum; a.colsum_group_stride = p.colsum_group_stride;
  a.scale_a = p.scale_a; a.scale_a_group_stride = p.scale_a_group_stride;
  a.scale_b = p.scale_b; a.scale_b_group_stride = p.scale_b_group_stride;
  a.wait_flags = p.wait_flags; a.wait_rows_per_flag = p.wait_rows_per_flag > 0 ? p.wait_rows_per_flag : bm;
  a.wait_flags_per_group = p.wait_flags_per_group; a.wait_target = p.wait_target;
  a.signal_ptr_table = p.signal_ptr_table;
  a.group_rot = p.group_rot; a.group_mod = p.group_mod;
  a.b_group_map = p.b_group_map; a.k_offsets = p.k_offsets;

  CUtensorMap ta, tb_;
  const int gB = groups_b;
  const int gA = p.k_offsets != nullptr ? 1 : p.G;
  if (!make_operand_map(&ta, p.a, p.in_dtype, p.a_mn_major, p.M, p.K, p.lda, p.a_group_stride, gA, bm, why))
    return cudaErrorInvalidValue;
  const int b_box = dual ? bn / 2 : bn;
  if (!make_operand_map(&tb_, p.b, p.in_dtype, p.b_mn_major, p.N, p.K, p.ldb, p.b_group_stride, gB, b_box, why))
    return cudaErrorInvalidValue;
  CUtensorMap tb2 = tb_;
  if (dual && !make_operand_map(&tb2, p.b2, p.in_dtype, p.b_mn_major, p.N, p.K, p.ldb, p.b_group_stride, gB, b_box, why))
    return cudaErrorInvalidValue;
  // 128 x 256: the output (TMA store), the aux operand (TMA load) and the GELU / SiLU pre-activation (TMA store)
  CUtensorMap td = tb_, taux = tb_, td2 = tb_;
  if (wide) {
    if (!make_tile_map(&td, p.d, p.out_dtype, p.M, p.N, p.ldd, p.d_group_stride, p.G, why)) return cudaErrorInvalidValue;
    if (uses_aux && !make_tile_map(&taux, p.aux, p.out_dtype, p.M, p.N, p.ld_aux, p.aux_group_stride, p.G, why))
      return cudaErrorInvalidValue;
    if (p.d2 != nullptr && (p.epilogue == EPI_BIAS_GELU || p.epilogue == EPI_BIAS_SILU) &&
        !make_tile_map(&td2, p.d2, p.out_dtype, p.M, p.N, p.ldd, p.d_group_stride, p.G, why))
      return cudaErrorInvalidValue;
  }

  const int grid = static_cast<int>(a.num_tiles < sms ? a.num_tiles : sms);

  if (eb == 1) {
    if (p.a_mn_major || p.b_mn_major) { *why = "fp8 operands must be K-major"; return cudaErrorInvalidValue; }
    const bool xact = p.epilogue == EPI_BIAS_GELU || p.epilogue == EPI_BIAS_SILU || p.epilogue == EPI_ACT_BWD;
    if (xact) { *why = "GELU / SiLU epilogues need 16-bit operands"; return cudaErrorInvalidValue; }
    if (wide) {
      if (p.in_dtype == DT_E4M3) return launch_inst<256, false, false, DT_E4M3>(ta, tb_, tb2, td, taux, td2, a, grid, stream);
      return launch_inst<256, false, false, DT_E5M2>(ta, tb_, tb2, td, taux, td2, a, grid, stream);
    }
    if (p.in_dtype == DT_E4M3) return launch_inst<128, false, false, DT_E4M3>(ta, tb_, tb2, td, taux, td2, a, grid, stream);
    return launch_inst<128, false, false, DT_E5M2>(ta, tb_, tb2, td, taux, td2, a, grid, stream);
  }
#define TB_SWITCH_MAJOR(BNv, DTv, PKv)                                                                                         \
  do {                                                                                                                         \
    if (!p.a_mn_major && !p.b_mn_major) return launch_inst<BNv, false, false, DTv, PKv>(ta, tb_, tb2, td, taux, td2, a, grid, stream); \
    if (!p.a_mn_major && p.b_mn_major) return launch_inst<BNv, false, true, DTv, PKv>(ta, tb_, tb2, td, taux, td2, a, grid, stream);   \
    if (p.a_mn_major && !p.b_mn_major) return launch_inst<BNv, true, false, DTv, PKv>(ta, tb_, tb2, td, taux, td2, a, grid, stream);   \
    return launch_inst<BNv, true, true, DTv, PKv>(ta, tb_, tb2, td, taux, td2, a, grid, stream);                                      \
  } while (0)
  if (p.b_group_map != nullptr || p.k_offsets != nullptr) {
    if (p.in_dtype == DT_BF16) { if (wide) TB_SWITCH_MAJOR(256, DT_BF16, true); TB_SWITCH_MAJOR(128, DT_BF16, true); }
    if (p.in_dtype == DT_FP16) { if (wide) TB_SWITCH_MAJOR(256, DT_FP16, true); TB_SWITCH_MAJOR(128, DT_FP16, true); }
  }
  if (p.in_dtype == DT_BF16) { if (wide) TB_SWITCH_MAJOR(256, DT_BF16, false); TB_SWITCH_MAJOR(128, DT_BF16, false); }
  if (p.in_dtype == DT_FP16) { if (wide) TB_SWITCH_MAJOR(256, DT_FP16, false); TB_SWITCH_MAJOR(128, DT_FP16, false); }
#undef TB_SWITCH_MAJOR
  *why = "unsupported operand dtype";
  return cudaErrorInvalidValue;
}

// run-time spin-wait limit of this translation unit's kernels (ptx.cuh)
cudaError_t set_spin_timeout_gemm(unsigned long long ns) {
  return cudaMemcpyToSymbol(tb_spin_timeout_ns, &ns, sizeof(ns));
}

}  // namespace tb

