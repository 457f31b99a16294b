// Block-scaled fp8 GEMM for sm_90a, the DeepSeek-V3 recipe:  D[g] = epilogue(A[g] * B[g]^T)  with e4m3 operands, one
// fp32 scale per 1 x 128 tile of A (a token's 128 channels) and one per 128 x 128 block of B (a weight block).
// Hopper's tensor cores know no block scales, so every 128-deep K step is
//     4 x wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3      (one scratch fragment, a fresh sum per K step)
// followed by one promotion into the fp32 accumulator:  acc[m, n] += scratch[m, n] * (sa[m, kb] * sb[n / 128, kb]).
// That is a quarter of the fold work of the MX kernel (gemm_mx.cu), which promotes once per 32 K elements, and a 128-wide
// N tile needs one weight scale per K step (two in the GLU layout, one per 64 columns).
//
// Layout of one CTA (384 threads, 128 x 128 tiles; K walked in 128-element = 128-byte steps, 6 stages):
//   warp 0        TMA producer: A and B tiles [128 x 128 B] (SWIZZLE_128B) plus the A tile's 512 bytes of scales
//                 (one bulk copy) per stage, all completing on the stage's "full" mbarrier
//   warps 4..11   two consumer warpgroups, 64 rows of the tile each.  The B scales of a K step (one or two floats per
//                 tile) are read straight from global memory, one step ahead; they are the same for every thread of
//                 the CTA and stay in L1.  Epilogue straight from the accumulator fragment.
// Persistent: CTA b works on tiles b, b + grid, ...; the producer runs ahead into the next tile during the epilogue.
//
// Weight gradients (WGRAD instantiation): K is the token dimension and B, like A, has one scale per row and K step
// ([G, K / 128, N], MN-major).  The producer bulk-copies the B tile's 512 bytes of scales next to A's; each consumer
// thread reads the 32 of its fragment's columns from shared memory and promotes with acc = fmaf(part, sa[m] * sb[n], acc).
//
// Quantisers: block_fp8_quantize_act_kernel (activations, 1 x 128 tiles), block_fp8_quantize_dual_kernel (activations,
// 1 x 128 and, transposed, 128 x 1 tiles from one read, for the weight-gradient GEMM) and block_fp8_quantize_weight_kernel
// (weights, 128 x 128 blocks; both orientations from one read, optionally in the SwiGLU gate / up layout).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>

#include <cfloat>
#include <algorithm>
#include <mutex>

#include "gemm_block_fp8.h"
#include "gemm_sm90.h"
#include "moe_kernels.h"
#include "ptx.cuh"

namespace tb {
namespace {

constexpr int kBM = 128;
constexpr int kBN = 128;
constexpr int kBK = 128;                 // e4m3 elements = bytes per K step (one 128-byte swizzle row)
constexpr int kSaBytes = kBM * 4;        // fp32 scales of 128 rows for one K step
constexpr int kThreads = 384;            // producer warpgroup + two consumer warpgroups

struct Cfg {
  static constexpr int STAGES = 6;
  static constexpr uint32_t A_BYTES = kBM * kBK;
  static constexpr uint32_t B_BYTES = kBN * kBK;
  static constexpr uint32_t OP_BYTES = A_BYTES + B_BYTES;
  static constexpr uint32_t BAR_BYTES = 128;
  static constexpr uint32_t SMEM_BYTES = 1024 + STAGES * (OP_BYTES + kSaBytes) + BAR_BYTES;
  static_assert(SMEM_BYTES <= 232448, "227 KB of shared memory per block");
};

struct Args {
  const float* sa;
  const float* sb;
  __nv_bfloat16 *d, *d2, *d3;
  long long ldd, d_group_stride;
  int M, N, K, G;
  int tiles_m, tiles_n;
  int sa_rows;                         // roundup(M, 128)
  int sb_rows;                         // N / 128, or N / 64 for the GLU forward
  const __nv_bfloat16* bias;
  long long bias_group_stride;
  const __nv_bfloat16 *aux, *aux2;
  long long ld_aux, aux_group_stride;
  long long num_tiles;
  int epi, act;
  const int* row_counts;               // COUNTS: live rows of each group (device); PACKED: of each row tile
  int split;                           // WGRAD: columns >= split go to d2 (at column n - split); 0: all to d
  const int* b_group_map;              // PACKED forward: B group of each row tile of the packed A (device)
  const int* k_offsets;                // PACKED WGRAD: K range [k_offsets[g], k_offsets[g + 1]) of group g (device)
};

// WGRAD: B's per-column scales of each stage, 512 bytes after the barriers
constexpr uint32_t kWgradSmemBytes = Cfg::SMEM_BYTES + Cfg::STAGES * kSaBytes;
static_assert(kWgradSmemBytes <= 232448, "227 KB of shared memory per block");

__device__ __forceinline__ float2 lds_f2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
  return v;
}

__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}

// Output tiles are walked in bands of 8 row tiles so that co-resident CTAs share A and B tiles in L2.
__device__ __forceinline__ void decode_tile(long long t, int tiles_m, int tiles_n, int& g, int& m_blk, int& n_blk) {
  const long long per_group = static_cast<long long>(tiles_m) * tiles_n;
  g = static_cast<int>(t / per_group);
  const int r = static_cast<int>(t % per_group);
  constexpr int kBand = 8;
  const int band = r / (kBand * tiles_n);
  const int in_band = r % (kBand * tiles_n);
  const int rows = min(kBand, tiles_m - band * kBand);
  m_blk = band * kBand + in_band % rows;
  n_blk = in_band / rows;
}

// Activation formulas of the 16-bit GLU epilogues (gemm_sm90.cu), so that the two paths agree on what act(g) means.
__device__ __forceinline__ float fast_sigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ void act_and_grad(int act, float g, float& a, float& da) {
  if (act == ACT_RELU) {
    a = fmaxf(g, 0.0f);
    da = g > 0.0f ? 1.0f : 0.0f;
  } else if (act == ACT_GELU) {
    const float cdf = 0.5f * (1.0f + erff(g * 0.70710678118654752f));
    a = g * cdf;
    da = cdf + g * 0.3989422804014327f * __expf(-0.5f * g * g);
  } else {
    const float sg = fast_sigmoid(g);
    a = g * sg;
    da = sg * (1.0f + g * (1.0f - sg));
  }
}

// Live rows of group g: all M, or min(row_counts[g], M) with device row counts (dropless prefill).  The producer and the
// consumers both derive a tile's skip from this one value, so they walk the same stages of the mbarrier ring.
template <bool COUNTS>
__device__ __forceinline__ int live_rows(const Args& args, int g) {
  return COUNTS ? max(0, min(args.row_counts[g], args.M)) : args.M;
}

// Ragged K (weight gradients on the expert-packed layout): group g reduces over the 128-deep K steps [kb0, kb0 + steps)
// of the one packed operand pair.  The producer and the consumers both derive the step count from here.
__device__ __forceinline__ void k_range(const Args& args, int g, int num_kb, int& kb0, int& steps) {
  const int lo = min(max(args.k_offsets[g], 0) / kBK, num_kb);
  const int hi = min(max(args.k_offsets[g + 1], 0) / kBK, num_kb);
  kb0 = lo;
  steps = max(hi - lo, 0);
}

// PACKED selects the expert-packed launch modes (csrc/gemm_block_fp8.h): with COUNTS, the block-mapped forward (A is one
// [R, K] buffer; row tile m takes B, its scales and bias from group b_group_map[m], row_counts[m] of its rows are live;
// a tile with none is skipped entirely); with WGRAD, ragged K (A and B are single operands, group g reduces over its
// K range).
template <bool COUNTS, bool WGRAD, bool PACKED = false>
__global__ void __launch_bounds__(kThreads, 1)
block_fp8_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const Args args) {
  static_assert(!(COUNTS && WGRAD), "row counts are for the forward GEMMs");
  static_assert(!PACKED || COUNTS || WGRAD, "the block-mapped forward takes per-tile row counts");
  constexpr bool MAPPED = PACKED && !WGRAD, RAGGED = PACKED && WGRAD;
  using C = Cfg;
  extern __shared__ uint8_t smem_raw[];
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;

  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sa_base = smem_base + C::STAGES * C::OP_BYTES;
  const uint32_t bar_base = sa_base + C::STAGES * kSaBytes;
  auto smem_a = [&](int s) { return smem_base + s * C::OP_BYTES; };
  auto smem_b = [&](int s) { return smem_base + s * C::OP_BYTES + C::A_BYTES; };
  auto smem_sa = [&](int s) { return sa_base + s * kSaBytes; };
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 64u + 8u * s; };
  auto smem_sb = [&](int s) { return bar_base + C::BAR_BYTES + s * kSaBytes; };   // WGRAD only

  if (warp == 0 && ptx::elect_one()) {
    ptx::prefetch_tensormap(&tmA);
    ptx::prefetch_tensormap(&tmB);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), 8);      // one arrival per consumer warp: each reads the stage's scales itself
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  const int num_kb = args.K / kBK;
  const long long tile_first = blockIdx.x, tile_step = gridDim.x;

  if (warp < 4) {
    ptx::setmaxnreg_dec<40>();
    if (warp == 0) {
      // =============================== TMA producer ===============================
      int s = 0;
      uint32_t ph = 0;
      for (long long t = tile_first; t < args.num_tiles; t += tile_step) {
        int g, m_blk, n_blk;
        decode_tile(t, args.tiles_m, args.tiles_n, g, m_blk, n_blk);
        const int m0 = m_blk * kBM, n0 = n_blk * kBN;
        if constexpr (MAPPED) {
          if (args.row_counts[m_blk] <= 0) continue;                    // a tile with no live rows: no stage
        } else {
          if (COUNTS && m0 >= live_rows<COUNTS>(args, g)) continue;    // no stage is filled for a tile past the count
        }
        const int gb = MAPPED ? args.b_group_map[m_blk] : g;           // B group
        const int ga = RAGGED ? 0 : g;                                 // operand group of A (and of B, ragged)
        int kb0 = 0, steps = num_kb;
        if constexpr (RAGGED) k_range(args, g, num_kb, kb0, steps);
        const float* sa_g = args.sa + static_cast<long long>(ga) * num_kb * args.sa_rows + m0;
        for (int kb = kb0; kb < kb0 + steps; ++kb) {
          ptx::mbar_wait_quiet(empty_bar(s), ph ^ 1u);
          if (ptx::elect_one()) {
            const uint32_t fb = full_bar(s);
            ptx::mbar_expect_tx(fb, C::OP_BYTES + (WGRAD ? 2 : 1) * kSaBytes);
            ptx::tma_load_3d(smem_a(s), &tmA, fb, kb * kBK, m0, ga);
            ptx::tma_load_3d(smem_b(s), &tmB, fb, kb * kBK, n0, RAGGED ? 0 : gb);
            ptx::bulk_load(smem_sa(s), sa_g + static_cast<long long>(kb) * args.sa_rows, kSaBytes, fb);
            if constexpr (WGRAD)
              ptx::bulk_load(smem_sb(s), args.sb + (static_cast<long long>(ga) * num_kb + kb) * args.N + n0, kSaBytes, fb);
          }
          __syncwarp();
          if (++s == C::STAGES) { s = 0; ph ^= 1u; }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<232>();
    // =============================== consumers ===============================
    const int cw = warp - 4;                       // consumer warp 0..7
    const int wg = cw >> 2;                        // warpgroup: tile rows [64 wg, 64 wg + 64)
    const int r0 = cw * 16 + (lane >> 2);          // this thread's accumulator rows in the tile: r0 and r0 + 8
    const int c0 = (lane & 3) * 2;                 // ... and columns 8 j + c0 + {0, 1}, j = 0..15
    // Operand descriptors: K-major, SWIZZLE_128B, 8-row groups 1024 B apart; a K=32 step advances the start by 32 B.
    constexpr uint32_t desc_hi = (1024u >> 4) | (1u << 30);
    const bool glu = args.epi == BF8_EPI_GLU;
    int s = 0;
    uint32_t ph = 0;
    for (long long t = tile_first; t < args.num_tiles; t += tile_step) {
      int g, m_blk, n_blk;
      decode_tile(t, args.tiles_m, args.tiles_n, g, m_blk, n_blk);
      int gb = g;                                  // B group (B scales, bias)
      if constexpr (MAPPED) {
        if (args.row_counts[m_blk] <= 0) continue;  // as in the producer: no stage, and nothing is stored
        gb = args.b_group_map[m_blk];
      }
      // B scales of this tile: columns 0..63 and 64..127 (the same row unless the tile holds 64 gate + 64 up columns)
      const float* sb_lo = args.sb + (static_cast<long long>(gb) * args.sb_rows + (glu ? 2 * n_blk : n_blk)) * num_kb;
      const float* sb_hi = glu ? sb_lo + num_kb : sb_lo;
      float sbl = 0.f, sbh = 0.f;
      if constexpr (!WGRAD) { sbl = __ldg(sb_lo); sbh = __ldg(sb_hi); }
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      // MAPPED: row_counts[m_blk] of this tile's rows are live (absolute bound m_blk * 128 + count)
      const int live = MAPPED ? m_blk * kBM + min(args.row_counts[m_blk], kBM) : live_rows<COUNTS>(args, g);
      // a tile past the count takes no stage (as in the producer) and stores zeros
      int steps = COUNTS && m_blk * kBM >= live ? 0 : num_kb;
      if constexpr (RAGGED) {
        int kb0;
        k_range(args, g, num_kb, kb0, steps);     // an empty group runs no step and stores zeros
      }
      for (int kb = 0; kb < steps; ++kb) {
        ptx::mbar_wait_quiet(full_bar(s), ph);
        const uint32_t a_lo = (((smem_a(s) + static_cast<uint32_t>(wg) * 8192u) >> 4) & 0x3FFFu) | (1u << 16);
        const uint32_t b_lo = ((smem_b(s) >> 4) & 0x3FFFu) | (1u << 16);
        float part[64];
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          ptx::wgmma_m64n128<DT_E4M3, false, false>(part, (static_cast<uint64_t>(desc_hi) << 32) | (a_lo + 2u * k),
                                                    (static_cast<uint64_t>(desc_hi) << 32) | (b_lo + 2u * k), k > 0 ? 1u : 0u);
        ptx::wgmma_commit();
        const float sa0 = __uint_as_float(lds_u32(smem_sa(s) + 4u * r0));
        const float sa1 = __uint_as_float(lds_u32(smem_sa(s) + 4u * (r0 + 8)));
        if constexpr (WGRAD) {
          // this thread's columns 8 j + c0 + {0, 1}: read before the stage is released
          float2 sbv[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) sbv[j] = lds_f2(smem_sb(s) + 4u * (8 * j + c0));
          ptx::wgmma_wait<0>();
          __syncwarp();
          if (lane == 0) ptx::mbar_arrive(empty_bar(s));
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            acc[4 * j] = fmaf(part[4 * j], sa0 * sbv[j].x, acc[4 * j]);
            acc[4 * j + 1] = fmaf(part[4 * j + 1], sa0 * sbv[j].y, acc[4 * j + 1]);
            acc[4 * j + 2] = fmaf(part[4 * j + 2], sa1 * sbv[j].x, acc[4 * j + 2]);
            acc[4 * j + 3] = fmaf(part[4 * j + 3], sa1 * sbv[j].y, acc[4 * j + 3]);
          }
          if (++s == C::STAGES) { s = 0; ph ^= 1u; }
          continue;
        }
        const float s00 = sa0 * sbl, s01 = sa0 * sbh, s10 = sa1 * sbl, s11 = sa1 * sbh;
        if (kb + 1 < steps) { sbl = __ldg(sb_lo + kb + 1); sbh = __ldg(sb_hi + kb + 1); }
        ptx::wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(empty_bar(s));
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            acc[4 * j + e] = fmaf(part[4 * j + e], j < 8 ? s00 : s01, acc[4 * j + e]);
            acc[4 * j + 2 + e] = fmaf(part[4 * j + 2 + e], j < 8 ? s10 : s11, acc[4 * j + 2 + e]);
          }
        }
        if (++s == C::STAGES) { s = 0; ph ^= 1u; }
      }

      // ------------------------------- epilogue -------------------------------
      if constexpr (WGRAD) {
        // bf16 D; with a split, tiles at or past column `split` store into the second output
        __nv_bfloat16* dst = args.d;
        int ncol = n_blk * kBN;
        if (args.split > 0 && ncol >= args.split) { dst = args.d2; ncol -= args.split; }
        dst += static_cast<long long>(g) * args.d_group_stride + ncol + c0;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = m_blk * kBM + r0 + 8 * h;
          if (row >= args.M) continue;
          __nv_bfloat16* o = dst + static_cast<long long>(row) * args.ldd;
#pragma unroll
          for (int j = 0; j < 16; ++j)
            *reinterpret_cast<__nv_bfloat162*>(o + 8 * j) = __floats2bfloat162_rn(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
        continue;
      }
      const int epi = args.epi;
      const long long goff = static_cast<long long>(g) * args.d_group_stride;
      const long long aoff = static_cast<long long>(g) * args.aux_group_stride;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = m_blk * kBM + r0 + 8 * h;
        if (row >= args.M) continue;
        const long long drow = goff + static_cast<long long>(row) * args.ldd;
        if (COUNTS && row >= live) {
          // rows past the count are zero in every output (their A rows are never read into the result)
          const __nv_bfloat162 z = __floats2bfloat162_rn(0.f, 0.f);
          const int w = epi == BF8_EPI_GLU ? 8 : 16;
          const long long o = drow + (epi == BF8_EPI_GLU ? n_blk * 64 : n_blk * kBN) + c0;
          for (int j = 0; j < w; ++j) {
            *reinterpret_cast<__nv_bfloat162*>(args.d + o + 8 * j) = z;
            if (epi == BF8_EPI_GLU || epi == BF8_EPI_GLU_BWD) *reinterpret_cast<__nv_bfloat162*>(args.d2 + o + 8 * j) = z;
            if (epi == BF8_EPI_GLU) *reinterpret_cast<__nv_bfloat162*>(args.d3 + o + 8 * j) = z;
          }
          continue;
        }
        if (epi == BF8_EPI_GLU) {
          // column 8 j + c0 (j < 8) is gate column n_blk * 64 + 8 j + c0; its up partner sits 64 columns on, at j + 8
          const long long o = drow + n_blk * 64 + c0;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            float hv[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float a, da;
              act_and_grad(args.act, acc[4 * j + 2 * h + e], a, da);
              hv[e] = a * acc[4 * (j + 8) + 2 * h + e];
            }
            *reinterpret_cast<__nv_bfloat162*>(args.d + o + 8 * j) = __floats2bfloat162_rn(hv[0], hv[1]);
            *reinterpret_cast<__nv_bfloat162*>(args.d2 + o + 8 * j) =
                __floats2bfloat162_rn(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            *reinterpret_cast<__nv_bfloat162*>(args.d3 + o + 8 * j) =
                __floats2bfloat162_rn(acc[4 * (j + 8) + 2 * h], acc[4 * (j + 8) + 2 * h + 1]);
          }
          continue;
        }
        const int n0 = n_blk * kBN + c0;
        const long long o = drow + n0;
        const long long ao = aoff + static_cast<long long>(row) * args.ld_aux + n0;
        const __nv_bfloat16* bias = args.bias == nullptr ? nullptr : args.bias + static_cast<long long>(gb) * args.bias_group_stride + n0;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          float lo = acc[4 * j + 2 * h], hi = acc[4 * j + 2 * h + 1];
          if (epi == BF8_EPI_GLU_BWD) {
            const float2 gv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(args.aux + ao + 8 * j));
            const float2 uv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(args.aux2 + ao + 8 * j));
            float a0, da0, a1, da1;
            act_and_grad(args.act, gv.x, a0, da0);
            act_and_grad(args.act, gv.y, a1, da1);
            *reinterpret_cast<__nv_bfloat162*>(args.d + o + 8 * j) = __floats2bfloat162_rn(lo * uv.x * da0, hi * uv.y * da1);
            *reinterpret_cast<__nv_bfloat162*>(args.d2 + o + 8 * j) = __floats2bfloat162_rn(lo * a0, hi * a1);
            continue;
          }
          if (bias != nullptr) {
            const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(bias + 8 * j));
            lo += b.x; hi += b.y;
          }
          if (epi == BF8_EPI_RELU) { lo = fmaxf(lo, 0.f); hi = fmaxf(hi, 0.f); }
          if (epi == BF8_EPI_RELU_BWD) {
            // keep the gradient where the forward activation was positive
            const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(args.aux + ao + 8 * j));
            lo = a.x > 0.f ? lo : 0.f; hi = a.y > 0.f ? hi : 0.f;
          }
          *reinterpret_cast<__nv_bfloat162*>(args.d + o + 8 * j) = __floats2bfloat162_rn(lo, hi);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// quantisers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_scale(float amax) {
  // (at least FLT_MIN: below it 1 / s overflows, and a block of tiny values would turn its zeros into 0 * inf = NaN)
  return amax > 0.0f ? fmaxf(amax * (1.0f / 448.0f), FLT_MIN) : 1.0f;
}

__device__ __forceinline__ uint2 quantize8(const float* f, float inv) {
  const __nv_fp8x4_e4m3 lo(make_float4(f[0] * inv, f[1] * inv, f[2] * inv, f[3] * inv));
  const __nv_fp8x4_e4m3 hi(make_float4(f[4] * inv, f[5] * inv, f[6] * inv, f[7] * inv));
  return make_uint2(*reinterpret_cast<const uint32_t*>(&lo), *reinterpret_cast<const uint32_t*>(&hi));
}

__device__ __forceinline__ void unpack8(const uint4& raw, float* f) {
  const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 v = __bfloat1622float2(p[i]);
    f[2 * i] = v.x; f[2 * i + 1] = v.y;
  }
}

// 16 consecutive threads own one 1 x 128 tile (8 elements = one 16-byte load each); tiles are walked K-fastest so a
// warp reads 512 contiguous bytes.  Pad rows (R <= r < Rp) only write their scale, 0.  The loop runs per warp (two
// tiles), so that every lane reaches the shuffles.
// BOUND (G == 1): only rows below *bound are walked; the units past it read and write nothing, and the ones below are
// exactly those of the unbounded launch.
template <bool BOUND>
__global__ void __launch_bounds__(256)
block_fp8_quantize_act_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q, float* __restrict__ s, int G,
                              int R, int Rp, int K, const int* __restrict__ bound) {
  const int KT = K / kBK;
  long long units = static_cast<long long>(G) * Rp * KT;
  if constexpr (BOUND) units = min(units, static_cast<long long>(max(0, __ldg(bound))) * KT);
  const int sub = threadIdx.x & 15, half = (threadIdx.x >> 4) & 1;
  const long long warps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  for (long long wi = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; wi * 2 < units; wi += warps) {
    const long long u = wi * 2 + half;
    const bool in = u < units;
    const int kt = static_cast<int>(u % KT);
    const long long gr = u / KT;
    const int g = static_cast<int>(gr / Rp), r = static_cast<int>(gr % Rp);
    const bool live = in && r < R;
    const long long off = (static_cast<long long>(g) * R + r) * K + kt * kBK + sub * 8;
    float f[8];
    float amax = 0.0f;
    if (live) {
      unpack8(ptx::ld_nc_v4(x + off), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(f[i]));
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float sc = block_scale(amax);
    if (live) *reinterpret_cast<uint2*>(q + off) = quantize8(f, 1.0f / sc);
    if (in && sub == 0) s[(static_cast<long long>(g) * KT + kt) * Rp + r] = live ? sc : 0.0f;
  }
}

constexpr int kTilePitch = 132;          // bytes: a column read by 8 threads 16 rows apart spreads over 8 banks

// Transposed write of a 128 x 128 byte tile: thread (c, part) writes 16 bytes of row c of the output (tile column c),
// 8 threads cover one 128-byte row segment.  `row_ptr(c)` is where output row c's 128 bytes go.
template <typename RowPtr>
__device__ __forceinline__ void store_tile_transposed(const uint8_t* tile, int t, RowPtr row_ptr) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int task = t + 256 * i;
    const int c = task >> 3, part = task & 7;
    uint32_t w4[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      uint32_t v = 0;
#pragma unroll
      for (int b = 0; b < 4; ++b) v |= static_cast<uint32_t>(tile[(part * 16 + 4 * k + b) * kTilePitch + c]) << (8 * b);
      w4[k] = v;
    }
    *reinterpret_cast<uint4*>(row_ptr(c) + part * 16) = make_uint4(w4[0], w4[1], w4[2], w4[3]);
  }
}

// Both orientations of an activation x [G, R, K] from one read, for the weight-gradient GEMM.  One block of 256 threads
// per 128 x 128 tile (rows rb, K columns kt); thread t holds columns 8 (t % 16) + 0..7 of rows t / 16 + 16 i, i < 8.
//   row-wise   (q != null): q [G, R, K] and s [G, K / 128, Rp], the 1 x 128 tiles of block_fp8_quantize_act_kernel with
//              the same arithmetic (one half warp per row), so the bytes and scales are that kernel's
//   column-wise: qT [G, K, Rp] and sT [G, Rp / 128, K], one scale per column and 128-row block; rows past R are not read,
//              they are zero bytes and take no part in the scale
// BOUND (G == 1): the tiles of 128 rows that start at or past *bound (a multiple of 128) read and write nothing.
template <bool BOUND>
__global__ void __launch_bounds__(256)
block_fp8_quantize_dual_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q, float* __restrict__ s,
                               uint8_t* __restrict__ qT, float* __restrict__ sT, int R, int Rp, int K, const int* __restrict__ bound) {
  __shared__ __align__(16) uint8_t tile[kBM * kTilePitch];
  __shared__ float red[8][kBK];
  __shared__ float csc[kBK];
  const int kt = blockIdx.x, rb = blockIdx.y, g = blockIdx.z;
  if constexpr (BOUND) {
    if (rb * kBM >= __ldg(bound)) return;              // the whole block: no thread reaches a barrier
  }
  const int t = threadIdx.x, c8 = (t & 15) * 8;
  const int KT = K / kBK;
  float f[8][8];
  float cmax[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) cmax[j] = 0.0f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = rb * kBM + (t >> 4) + 16 * i;
    if (r < R) {
      unpack8(ptx::ld_nc_v4(x + (static_cast<long long>(g) * R + r) * K + kt * kBK + c8), f[i]);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[i][j] = 0.0f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) cmax[j] = fmaxf(cmax[j], fabsf(f[i][j]));
  }
  if (q != nullptr) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = rb * kBM + (t >> 4) + 16 * i;
      float amax = 0.0f;
#pragma unroll
      for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(f[i][j]));
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
      const float sc = block_scale(amax);
      if (r < R) *reinterpret_cast<uint2*>(q + (static_cast<long long>(g) * R + r) * K + kt * kBK + c8) = quantize8(f[i], 1.0f / sc);
      if ((t & 15) == 0) s[(static_cast<long long>(g) * KT + kt) * Rp + r] = r < R ? sc : 0.0f;
    }
  }
  // column maxima: the two half warps, then the 8 warps through shared memory
#pragma unroll
  for (int j = 0; j < 8; ++j) cmax[j] = fmaxf(cmax[j], __shfl_xor_sync(0xffffffffu, cmax[j], 16));
  if ((t & 31) < 16) {
#pragma unroll
    for (int j = 0; j < 8; ++j) red[t >> 5][c8 + j] = cmax[j];
  }
  __syncthreads();
  if (t < kBK) {
    float m = red[0][t];
#pragma unroll
    for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w][t]);
    const float sc = block_scale(m);
    csc[t] = sc;
    sT[(static_cast<long long>(g) * (Rp / kBM) + rb) * K + kt * kBK + t] = sc;
  }
  __syncthreads();
  float inv[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) inv[j] = 1.0f / csc[c8 + j];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const __nv_fp8x4_e4m3 lo(make_float4(f[i][0] * inv[0], f[i][1] * inv[1], f[i][2] * inv[2], f[i][3] * inv[3]));
    const __nv_fp8x4_e4m3 hi(make_float4(f[i][4] * inv[4], f[i][5] * inv[5], f[i][6] * inv[6], f[i][7] * inv[7]));
    uint32_t* dst = reinterpret_cast<uint32_t*>(tile + ((t >> 4) + 16 * i) * kTilePitch + c8);
    dst[0] = *reinterpret_cast<const uint32_t*>(&lo);
    dst[1] = *reinterpret_cast<const uint32_t*>(&hi);
  }
  __syncthreads();
  uint8_t* qTg = qT + (static_cast<long long>(g) * K + kt * kBK) * Rp + rb * kBM;
  store_tile_transposed(tile, t, [&](int c) { return qTg + static_cast<long long>(c) * Rp; });
}

// One block of 256 threads per 128 x 128 weight block: a reduction for the scale, the row-major e4m3 copy written
// straight from registers, the transposed copy through a shared byte tile.  GLU: blockIdx.z = 2 g + (0 gate | 1 up),
// rows are M, columns H, and the outputs go to the concatenated [G, M, 2H] and the interleaved [G, 2H, M] layouts.

template <bool GLU>
__global__ void __launch_bounds__(256)
block_fp8_quantize_weight_kernel(const __nv_bfloat16* __restrict__ w, const __nv_bfloat16* __restrict__ w2,
                                 uint8_t* __restrict__ q, float* __restrict__ s, uint8_t* __restrict__ qT,
                                 float* __restrict__ sT, int R, int Cn) {
  __shared__ __align__(16) uint8_t tile[kBM * kTilePitch];
  __shared__ float red[8];
  const int cb = blockIdx.x, rb = blockIdx.y;
  const int g = GLU ? blockIdx.z >> 1 : blockIdx.z;
  const int which = GLU ? blockIdx.z & 1 : 0;
  const __nv_bfloat16* src = (which ? w2 : w) + (static_cast<long long>(g) * R + rb * kBM) * Cn + cb * kBK;
  const int t = threadIdx.x;
  const int c8 = (t & 15) * 8;
  float f[8][8];
  float amax = 0.0f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = (t >> 4) + 16 * i;
    unpack8(ptx::ld_nc_v4(src + static_cast<long long>(r) * Cn + c8), f[i]);
#pragma unroll
    for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(f[i][j]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if ((t & 31) == 0) red[t >> 5] = amax;
  __syncthreads();
  amax = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) amax = fmaxf(amax, red[i]);
  const float sc = block_scale(amax);
  const float inv = 1.0f / sc;
  const int RB = R / kBM, CB = Cn / kBK;
  // row-major copy: [G, R, Cn] (or the gate / up half of [G, M, 2H])
  const long long ldq = GLU ? 2LL * Cn : Cn;
  uint8_t* qg = q + static_cast<long long>(g) * R * ldq + which * Cn + cb * kBK;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = (t >> 4) + 16 * i;
    const uint2 v = quantize8(f[i], inv);
    *reinterpret_cast<uint2*>(qg + static_cast<long long>(rb * kBM + r) * ldq + c8) = v;
    const uint8_t* b = reinterpret_cast<const uint8_t*>(&v);
#pragma unroll
    for (int j = 0; j < 8; ++j) tile[r * kTilePitch + c8 + j] = b[j];
  }
  if (t == 0) {
    if (GLU) {
      s[(static_cast<long long>(g) * RB + rb) * (2 * CB) + which * CB + cb] = sc;
      // rows 64 n of the interleaved copy: gate / up column blocks 2 cb and 2 cb + 1 of 64
      float* sg = sT + (static_cast<long long>(g) * 4 * CB + 4 * cb + which) * RB + rb;
      sg[0] = sc;
      sg[2 * RB] = sc;
    } else {
      s[(static_cast<long long>(g) * RB + rb) * CB + cb] = sc;
      sT[(static_cast<long long>(g) * CB + cb) * RB + rb] = sc;
    }
  }
  __syncthreads();
  // transposed copy
  const long long NT = GLU ? 2LL * Cn : Cn;
  store_tile_transposed(tile, t, [&](int c) {
    const int col = cb * kBK + c;
    const long long n = GLU ? (static_cast<long long>(col / 64) * 128 + which * 64 + col % 64) : col;
    return qT + (static_cast<long long>(g) * NT + n) * R + rb * kBM;
  });
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess &&
        qr == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// e4m3 [groups, rows, k] row-major -> boxes of 128 rows x 128 bytes, 128-byte swizzle; rows past `rows` read as zero
bool operand_map(CUtensorMap* map, const void* base, long long rows, long long k, int groups) {
  EncodeTiledFn enc = encode_fn();
  if (enc == nullptr) return false;
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(k), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(groups)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(k), static_cast<cuuint64_t>(rows) * static_cast<cuuint64_t>(k)};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(kBK), 128u, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

bool misaligned(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

// persistent grid: one resident CTA per SM (at most max_ctas if > 0), never more than there are tiles
unsigned grid_size(long long num_tiles, int max_ctas) {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  long long ctas = sms;
  if (max_ctas > 0) ctas = std::max<long long>(1, std::min<long long>(ctas, max_ctas));
  return static_cast<unsigned>(std::min<long long>(num_tiles, ctas));
}

}  // namespace

cudaError_t block_fp8_gemm_launch(const BlockFp8GemmProblem& p, cudaStream_t stream, const char** why) {
  using C = Cfg;
  auto fail = [&](const char* msg) { if (why) *why = msg; return cudaErrorInvalidValue; };
  if (p.M <= 0 || p.N <= 0 || p.K <= 0 || p.G <= 0) return fail("empty block fp8 GEMM");
  if (p.K % kBK != 0) return fail("block fp8 GEMM: K must be a multiple of 128");
  if (p.N % kBN != 0) return fail("block fp8 GEMM: N must be a multiple of 128");
  if (p.epilogue < BF8_EPI_NONE || p.epilogue > BF8_EPI_GLU_BWD) return fail("block fp8 GEMM: unknown epilogue");
  if (misaligned(p.a) || misaligned(p.b) || misaligned(p.sa) || (reinterpret_cast<uintptr_t>(p.sb) & 3) || misaligned(p.d))
    return fail("block fp8 GEMM: operands must be 16-byte aligned (B scales 4-byte aligned)");
  if (p.ldd % 8 != 0 || p.d_group_stride % 8 != 0) return fail("block fp8 GEMM: output strides must be multiples of 8 elements");
  const bool glu = p.epilogue == BF8_EPI_GLU, glu_bwd = p.epilogue == BF8_EPI_GLU_BWD;
  if ((glu || glu_bwd) && (p.act < ACT_RELU || p.act > ACT_SILU)) return fail("block fp8 GEMM: act must be 1 (relu), 2 (gelu) or 3 (silu)");
  if (glu && (p.d2 == nullptr || p.d3 == nullptr || misaligned(p.d2) || misaligned(p.d3)))
    return fail("block fp8 GEMM: the GLU epilogue needs 16-byte aligned g and u outputs");
  if (glu_bwd && (p.d2 == nullptr || misaligned(p.d2))) return fail("block fp8 GEMM: the GLU-backward epilogue needs a 16-byte aligned du output");
  const bool reads_aux = p.epilogue == BF8_EPI_RELU_BWD || glu_bwd;
  if (reads_aux && (p.aux == nullptr || misaligned(p.aux) || p.ld_aux % 8 || p.aux_group_stride % 8))
    return fail("block fp8 GEMM: this epilogue needs a 16-byte aligned aux operand");
  if (glu_bwd && (p.aux2 == nullptr || misaligned(p.aux2))) return fail("block fp8 GEMM: the GLU-backward epilogue needs a 16-byte aligned aux2 (u)");
  if (p.bias != nullptr && (glu || reads_aux)) return fail("block fp8 GEMM: bias is for the NONE and RELU epilogues");
  if (p.bias != nullptr && (misaligned(p.bias) || p.bias_group_stride % 8)) return fail("block fp8 GEMM: bias must be 16-byte aligned");

  const bool mapped = p.b_group_map != nullptr;
  if (mapped && (p.row_counts == nullptr || p.M % kBM != 0))
    return fail("block fp8 GEMM: a block-mapped launch needs per-tile row counts and M (packed rows) % 128 == 0");
  CUtensorMap ta, tb_;
  if (!operand_map(&ta, p.a, p.M, p.K, mapped ? 1 : p.G) || !operand_map(&tb_, p.b, p.N, p.K, p.G))
    return fail("cuTensorMapEncodeTiled failed for a block fp8 operand");
  Args a{};
  a.sa = p.sa;
  a.sb = p.sb;
  a.d = static_cast<__nv_bfloat16*>(p.d);
  a.d2 = static_cast<__nv_bfloat16*>(p.d2);
  a.d3 = static_cast<__nv_bfloat16*>(p.d3);
  a.ldd = p.ldd;
  a.d_group_stride = p.d_group_stride;
  a.M = p.M; a.N = p.N; a.K = p.K; a.G = p.G;
  a.tiles_m = (p.M + kBM - 1) / kBM;
  a.tiles_n = p.N / kBN;
  a.sa_rows = a.tiles_m * kBM;
  a.sb_rows = glu ? p.N / 64 : p.N / 128;
  a.bias = static_cast<const __nv_bfloat16*>(p.bias);
  a.bias_group_stride = p.bias_group_stride;
  a.aux = static_cast<const __nv_bfloat16*>(p.aux);
  a.aux2 = static_cast<const __nv_bfloat16*>(p.aux2);
  a.ld_aux = p.ld_aux;
  a.aux_group_stride = p.aux_group_stride;
  a.epi = p.epilogue;
  a.act = p.act;
  a.row_counts = p.row_counts;
  a.split = 0;
  a.b_group_map = p.b_group_map;
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [] {
    attr_err = cudaFuncSetAttribute(block_fp8_gemm_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (attr_err == cudaSuccess)
      attr_err = cudaFuncSetAttribute(block_fp8_gemm_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (attr_err == cudaSuccess)
      attr_err = cudaFuncSetAttribute(block_fp8_gemm_kernel<true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
  });
  if (attr_err != cudaSuccess) return attr_err;
  // block-mapped: one A group of R / 128 row tiles, walked in the same 8-tile bands (neighbouring tiles mostly share B)
  a.num_tiles = static_cast<long long>(a.tiles_m) * a.tiles_n * (mapped ? 1 : p.G);
  const unsigned grid = grid_size(a.num_tiles, p.max_ctas);
  if (mapped)
    block_fp8_gemm_kernel<true, false, true><<<grid, kThreads, C::SMEM_BYTES, stream>>>(ta, tb_, a);
  else if (p.row_counts != nullptr)
    block_fp8_gemm_kernel<true, false><<<grid, kThreads, C::SMEM_BYTES, stream>>>(ta, tb_, a);
  else
    block_fp8_gemm_kernel<false, false><<<grid, kThreads, C::SMEM_BYTES, stream>>>(ta, tb_, a);
  return cudaGetLastError();
}

cudaError_t block_fp8_wgrad_gemm_launch(const BlockFp8WgradProblem& p, cudaStream_t stream, const char** why) {
  auto fail = [&](const char* msg) { if (why) *why = msg; return cudaErrorInvalidValue; };
  if (p.M <= 0 || p.N <= 0 || p.K <= 0 || p.G <= 0) return fail("empty block fp8 weight-gradient GEMM");
  if (p.M % kBM != 0 || p.N % kBN != 0 || p.K % kBK != 0)
    return fail("block fp8 weight-gradient GEMM: M, N and K must be multiples of 128");
  if (p.split != 0 && (p.split % kBN != 0 || p.N != 2 * p.split || p.d2 == nullptr))
    return fail("block fp8 weight-gradient GEMM: a split output needs N == 2 * split, split % 128 == 0 and a second output");
  if (misaligned(p.a) || misaligned(p.b) || misaligned(p.sa) || misaligned(p.sb) || misaligned(p.d) ||
      (p.split != 0 && misaligned(p.d2)))
    return fail("block fp8 weight-gradient GEMM: operands, scales and outputs must be 16-byte aligned");
  const bool ragged = p.k_offsets != nullptr;
  CUtensorMap ta, tb_;
  if (!operand_map(&ta, p.a, p.M, p.K, ragged ? 1 : p.G) || !operand_map(&tb_, p.b, p.N, p.K, ragged ? 1 : p.G))
    return fail("cuTensorMapEncodeTiled failed for a block fp8 operand");
  Args a{};
  a.sa = p.sa;
  a.sb = p.sb;
  a.k_offsets = p.k_offsets;
  a.d = static_cast<__nv_bfloat16*>(p.d);
  a.d2 = static_cast<__nv_bfloat16*>(p.d2);
  a.split = p.split;
  a.ldd = p.split != 0 ? p.split : p.N;
  a.d_group_stride = static_cast<long long>(p.M) * a.ldd;
  a.M = p.M; a.N = p.N; a.K = p.K; a.G = p.G;
  a.tiles_m = p.M / kBM;
  a.tiles_n = p.N / kBN;
  a.sa_rows = p.M;
  a.sb_rows = p.N;
  a.epi = BF8_EPI_NONE;
  a.num_tiles = static_cast<long long>(a.tiles_m) * a.tiles_n * p.G;
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [] {
    attr_err = cudaFuncSetAttribute(block_fp8_gemm_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgradSmemBytes);
    if (attr_err == cudaSuccess)
      attr_err = cudaFuncSetAttribute(block_fp8_gemm_kernel<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgradSmemBytes);
  });
  if (attr_err != cudaSuccess) return attr_err;
  const unsigned grid = grid_size(a.num_tiles, p.max_ctas);
  if (ragged)
    block_fp8_gemm_kernel<false, true, true><<<grid, kThreads, kWgradSmemBytes, stream>>>(ta, tb_, a);
  else
    block_fp8_gemm_kernel<false, true><<<grid, kThreads, kWgradSmemBytes, stream>>>(ta, tb_, a);
  return cudaGetLastError();
}

cudaError_t block_fp8_quantize_act_dual(const void* x, void* q, float* s, void* qT, float* sT, int groups, int rows, int k,
                                        cudaStream_t stream, const int* live_rows) {
  if (k % kBK != 0 || groups < 0 || rows < 0 || groups > 65535 || (q == nullptr) != (s == nullptr)) return cudaErrorInvalidValue;
  if (live_rows != nullptr && groups > 1) return cudaErrorInvalidValue;
  const int Rp = (rows + kBM - 1) / kBM * kBM;
  if (groups == 0 || Rp == 0 || k == 0) return cudaSuccess;
  const dim3 grid(k / kBK, Rp / kBM, groups);
  const auto* xb = static_cast<const __nv_bfloat16*>(x);
  if (live_rows != nullptr)
    block_fp8_quantize_dual_kernel<true><<<grid, 256, 0, stream>>>(xb, static_cast<uint8_t*>(q), s, static_cast<uint8_t*>(qT), sT,
                                                                  rows, Rp, k, live_rows);
  else
    block_fp8_quantize_dual_kernel<false><<<grid, 256, 0, stream>>>(xb, static_cast<uint8_t*>(q), s, static_cast<uint8_t*>(qT), sT,
                                                                   rows, Rp, k, nullptr);
  return cudaGetLastError();
}

cudaError_t block_fp8_quantize_act(const void* x, void* q, float* s, int groups, int rows, int k, cudaStream_t stream,
                                   const int* live_rows) {
  if (k % kBK != 0 || groups < 0 || rows < 0) return cudaErrorInvalidValue;
  if (live_rows != nullptr && groups > 1) return cudaErrorInvalidValue;
  const int Rp = (rows + kBM - 1) / kBM * kBM;
  const long long units = static_cast<long long>(groups) * Rp * (k / kBK);
  if (units == 0) return cudaSuccess;
  const int blocks = static_cast<int>(std::min<long long>((units * 16 + 255) / 256, 132LL * 16));
  const auto* xb = static_cast<const __nv_bfloat16*>(x);
  if (live_rows != nullptr)
    block_fp8_quantize_act_kernel<true><<<blocks, 256, 0, stream>>>(xb, static_cast<uint8_t*>(q), s, groups, rows, Rp, k, live_rows);
  else
    block_fp8_quantize_act_kernel<false><<<blocks, 256, 0, stream>>>(xb, static_cast<uint8_t*>(q), s, groups, rows, Rp, k, nullptr);
  return cudaGetLastError();
}

cudaError_t block_fp8_quantize_weight(const void* w, void* q, float* s, void* qT, float* sT, int groups, int rows, int cols,
                                      cudaStream_t stream) {
  if (rows % kBM != 0 || cols % kBK != 0 || groups < 0) return cudaErrorInvalidValue;
  if (groups == 0 || rows == 0 || cols == 0) return cudaSuccess;
  const dim3 grid(cols / kBK, rows / kBM, groups);
  block_fp8_quantize_weight_kernel<false><<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(w), nullptr,
                                                                    static_cast<uint8_t*>(q), s, static_cast<uint8_t*>(qT), sT,
                                                                    rows, cols);
  return cudaGetLastError();
}

cudaError_t block_fp8_quantize_glu_weight(const void* w1, const void* w2, void* qcat, float* scat, void* qglu, float* sglu,
                                          int groups, int m, int h, cudaStream_t stream) {
  if (m % kBM != 0 || h % kBK != 0 || groups < 0) return cudaErrorInvalidValue;
  if (groups == 0 || m == 0 || h == 0) return cudaSuccess;
  const dim3 grid(h / kBK, m / kBM, 2 * groups);
  block_fp8_quantize_weight_kernel<true><<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(w1),
                                                                   static_cast<const __nv_bfloat16*>(w2),
                                                                   static_cast<uint8_t*>(qcat), scat,
                                                                   static_cast<uint8_t*>(qglu), sglu, m, h);
  return cudaGetLastError();
}

cudaError_t set_spin_timeout_block_fp8(unsigned long long ns) {
  return cudaMemcpyToSymbol(tb_spin_timeout_ns, &ns, sizeof(ns));
}

}  // namespace tb
