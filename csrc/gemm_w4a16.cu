// Mixed-input grouped GEMM for group-32 int4 weights (W4A16) on sm_90a:  D[g] = epilogue(A[g] * B[g]^T)  with bf16
// activations and int4 weights expanded on chip.  The tensor cores see bf16 operands: every weight becomes
// bf16_rn(q * s) in shared memory (q * s is exact, so this is one rounding), the MMA is
//     4 x wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 per 64-deep K step
// into one fp32 accumulator, and the output is bf16.  Epilogues: NONE, and GLU for the interleaved gate / up operand of
// LlamaFFNNetwork(weight_format='int4'): a 128-wide N tile holds 64 gate rows and their 64 up partners, and only
// h = act(g) * u is stored (inference has no use for g and u).
//
// Layout of one CTA (384 threads, 128 x 128 output tiles, K walked in 64-element steps, 8 stages):
//   warp 0        TMA producer: per stage the A tile [128 rows x 64 bf16] (SWIZZLE_128B, 16 KB) and the B tile's packed
//                 nibbles [128 rows x 32 bytes] (no swizzle, 4 KB), both completing on the stage's "full" mbarrier.
//                 setmaxnreg 40.
//   warps 4..11   two consumer warpgroups, 64 rows of the tile each (setmaxnreg 232).  They also expand B: thread t of
//                 the 256 takes row t / 2 and 32-element group t % 2 of a stage's nibbles (one 16-byte shared load) and
//                 its bf16 scale (one 2-byte global load; the scales are 1/16 of the nibble bytes and stay in L2), and
//                 writes 64 bytes of bf16 into the swizzled [128 x 64] tile wgmma reads.  Two such tiles alternate:
//                 while the wgmma of step k runs on one, the consumers expand step k + 1 into the other; a named barrier
//                 over the 256 consumer threads after each step orders both the expansion before its wgmma and the
//                 wgmma before the tile is overwritten.  A separate expansion warpgroup would need registers the split
//                 leaves no room for: 128 x 40 + 256 x 232 = 64,512 of the SM's 65,536.
// Nibble to bf16: (0x43004300 | u0 | u1 << 16) is the bf16 pair (128 + u0, 128 + u1) exactly; subtracting 136 gives q
// exactly, and one bf16x2 multiply by the scale pair rounds q * s once.
// Persistent: CTA b works on tiles b, b + grid, ...; the producer runs ahead into the next tile during the epilogue.
// Device row counts (dropless prefill): tiles whose first row is at or past the count load nothing, and rows past the
// count are stored as zero.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <mutex>

#include "gemm_sm90.h"
#include "gemm_w4a16.h"
#include "ptx.cuh"

namespace tb {
namespace {

constexpr int kBM = 128;
constexpr int kBN = 128;
constexpr int kBK = 64;                         // bf16 elements per K step: one 128-byte swizzle row of A
constexpr int kThreads = 384;
constexpr int kStages = 8;
constexpr uint32_t kABytes = kBM * kBK * 2;     // 16 KB
constexpr uint32_t kBpBytes = kBN * kBK / 2;    // 4 KB of nibbles
constexpr uint32_t kStageBytes = kABytes + kBpBytes;
constexpr uint32_t kBfBytes = kBN * kBK * 2;    // one expanded B tile, 16 KB
constexpr uint32_t kSmemBytes = 1024 + kStages * kStageBytes + 2 * kBfBytes + 256;
static_assert(kStageBytes % 1024 == 0, "stages keep the 1024-byte alignment of the swizzled tiles");
static_assert(kSmemBytes <= 232448, "227 KB of shared memory per block");

struct Args {
  const uint16_t* sb;
  __nv_bfloat16* d;
  long long ldd;
  int M, N, K, G;
  int tiles_m, tiles_n;
  long long num_tiles;
  int epi, act;
  const int* row_counts;
};

__device__ __forceinline__ void decode_tile(long long t, int tiles_m, int tiles_n, int& g, int& m_blk, int& n_blk) {
  const long long per_group = static_cast<long long>(tiles_m) * tiles_n;
  g = static_cast<int>(t / per_group);
  const int r = static_cast<int>(t % per_group);
  constexpr int kBand = 8;                      // bands of 8 row tiles: co-resident CTAs share A and B tiles in L2
  const int band = r / (kBand * tiles_n);
  const int in_band = r % (kBand * tiles_n);
  const int rows = min(kBand, tiles_m - band * kBand);
  m_blk = band * kBand + in_band % rows;
  n_blk = in_band / rows;
}

// act(g) of the 16-bit GLU epilogues (gemm_sm90.cu, gemm_block_fp8.cu)
__device__ __forceinline__ float glu_act(int act, float g) {
  if (act == ACT_RELU) return fmaxf(g, 0.0f);
  if (act == ACT_GELU) return g * (0.5f * (1.0f + erff(g * 0.70710678118654752f)));
  return g * __fdividef(1.0f, 1.0f + __expf(-g));
}

__device__ __forceinline__ int live_rows(const Args& args, int g) {
  return args.row_counts != nullptr ? max(0, min(args.row_counts[g], args.M)) : args.M;
}

// Expand this thread's 32 weights of K step kb (stage nibbles at bp) into the swizzled bf16 tile at bf.
__device__ __forceinline__ void expand_b(uint32_t bp, uint32_t bf, const uint16_t* __restrict__ srow, int kb, int ct) {
  const int n = ct >> 1, h = ct & 1;
  uint32_t w[4];
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "r"(bp + n * 32 + h * 16) : "memory");
  const uint16_t sbits = __ldg(srow + 2 * kb + h);
  const __nv_bfloat162 s2 = __halves2bfloat162(__ushort_as_bfloat16(sbits), __ushort_as_bfloat16(sbits));
  const __nv_bfloat162 off = __floats2bfloat162_rn(136.0f, 136.0f);
#pragma unroll
  for (int p = 0; p < 4; ++p) {                 // word p: elements 8p .. 8p + 7 of the group, 16 bytes of bf16
    uint32_t out[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t t = w[p] >> (8 * i);
      const uint32_t v = (t & 0xFu) | ((t & 0xF0u) << 12) | 0x43004300u;
      __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(&v);
      b = __hmul2(__hsub2(b, off), s2);
      out[i] = *reinterpret_cast<const uint32_t*>(&b);
    }
    const int c = 4 * h + p;                    // 16-byte chunk of the 128-byte row, swizzled by the row's low 3 bits
    const uint32_t dst = bf + n * 128 + ((c ^ (n & 7)) << 4);
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "r"(out[0]), "r"(out[1]), "r"(out[2]), "r"(out[3])
                 : "memory");
  }
}

__global__ void __launch_bounds__(kThreads, 1)
w4a16_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const Args args) {
  extern __shared__ uint8_t smem_raw[];
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;

  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bf_base = smem_base + kStages * kStageBytes;
  const uint32_t bar_base = bf_base + 2 * kBfBytes;
  auto smem_a = [&](int s) { return smem_base + s * kStageBytes; };
  auto smem_bp = [&](int s) { return smem_base + s * kStageBytes + kABytes; };
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 64u + 8u * s; };

  if (warp == 0 && ptx::elect_one()) {
    ptx::prefetch_tensormap(&tmA);
    ptx::prefetch_tensormap(&tmB);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), 8);          // one arrival per consumer warp
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
        if (m0 >= live_rows(args, g)) continue;   // no stage is filled for a tile past the count
        for (int kb = 0; kb < num_kb; ++kb) {
          ptx::mbar_wait_quiet(empty_bar(s), ph ^ 1u);
          if (ptx::elect_one()) {
            const uint32_t fb = full_bar(s);
            ptx::mbar_expect_tx(fb, kStageBytes);
            ptx::tma_load_3d(smem_a(s), &tmA, fb, kb * kBK, m0, g);
            ptx::tma_load_3d(smem_bp(s), &tmB, fb, kb * (kBK / 2), n0, g);
          }
          __syncwarp();
          if (++s == kStages) { s = 0; ph ^= 1u; }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<232>();
    // =============================== consumers ===============================
    const int ct = threadIdx.x - 128;              // 0..255: expansion row ct / 2, group ct % 2
    const int cw = warp - 4;
    const int wg = cw >> 2;                        // warpgroup: tile rows [64 wg, 64 wg + 64)
    const int r0 = cw * 16 + (lane >> 2);          // accumulator rows r0, r0 + 8 of the tile
    const int c0 = (lane & 3) * 2;                 // ... columns 8 j + c0 + {0, 1}
    constexpr uint32_t desc_hi = (1024u >> 4) | (1u << 30);   // K-major, SWIZZLE_128B, 8-row groups 1024 B apart
    const bool glu = args.epi == W4A16_EPI_GLU;
    const int K32 = args.K / 32;
    int s = 0;
    uint32_t ph = 0;
    for (long long t = tile_first; t < args.num_tiles; t += tile_step) {
      int g, m_blk, n_blk;
      decode_tile(t, args.tiles_m, args.tiles_n, g, m_blk, n_blk);
      const int live = live_rows(args, g);
      const int steps = m_blk * kBM >= live ? 0 : num_kb;   // as in the producer
      const uint16_t* srow = args.sb + (static_cast<long long>(g) * args.N + n_blk * kBN + (ct >> 1)) * K32;
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      if (steps > 0) {
        ptx::mbar_wait_quiet(full_bar(s), ph);
        expand_b(smem_bp(s), bf_base, srow, 0, ct);
        ptx::fence_proxy_async_smem();
        ptx::named_bar_sync(1, 256);
      }
      for (int kb = 0; kb < steps; ++kb) {
        const uint32_t a_lo = (((smem_a(s) + static_cast<uint32_t>(wg) * 8192u) >> 4) & 0x3FFFu) | (1u << 16);
        const uint32_t b_lo = (((bf_base + (kb & 1) * kBfBytes) >> 4) & 0x3FFFu) | (1u << 16);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          ptx::wgmma_m64n128<ptx::WG_BF16, false, false>(acc, (static_cast<uint64_t>(desc_hi) << 32) | (a_lo + 2u * k),
                                                         (static_cast<uint64_t>(desc_hi) << 32) | (b_lo + 2u * k), 1u);
        ptx::wgmma_commit();
        int ns = s + 1;
        uint32_t nph = ph;
        if (ns == kStages) { ns = 0; nph ^= 1u; }
        if (kb + 1 < steps) {                      // expand the next step while this one's MMAs run
          ptx::mbar_wait_quiet(full_bar(ns), nph);
          expand_b(smem_bp(ns), bf_base + ((kb + 1) & 1) * kBfBytes, srow, kb + 1, ct);
          ptx::fence_proxy_async_smem();
        }
        ptx::wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(empty_bar(s));
        ptx::named_bar_sync(1, 256);
        s = ns;
        ph = nph;
      }

      // ------------------------------- epilogue -------------------------------
      const long long goff = static_cast<long long>(g) * args.M * args.ldd;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = m_blk * kBM + r0 + 8 * h;
        if (row >= args.M) continue;
        const long long drow = goff + static_cast<long long>(row) * args.ldd;
        const bool dead = row >= live;           // rows past the count are zero (their A rows take no part)
        if (glu) {
          // column 8 j + c0 (j < 8) is gate column n_blk * 64 + 8 j + c0; its up partner sits 64 columns on, at j + 8
          const long long o = drow + n_blk * 64 + c0;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            float hv[2];
#pragma unroll
            for (int e = 0; e < 2; ++e)
              hv[e] = dead ? 0.f : glu_act(args.act, acc[4 * j + 2 * h + e]) * acc[4 * (j + 8) + 2 * h + e];
            *reinterpret_cast<__nv_bfloat162*>(args.d + o + 8 * j) = __floats2bfloat162_rn(hv[0], hv[1]);
          }
        } else {
          const long long o = drow + n_blk * kBN + c0;
#pragma unroll
          for (int j = 0; j < 16; ++j)
            *reinterpret_cast<__nv_bfloat162*>(args.d + o + 8 * j) =
                dead ? __floats2bfloat162_rn(0.f, 0.f) : __floats2bfloat162_rn(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
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

// [groups, rows, row_bytes] -> boxes of 128 rows x box_bytes; rows past `rows` read as zero
bool tile_map(CUtensorMap* map, const void* base, CUtensorMapDataType dt, int elem_bytes, long long rows, long long cols,
              int groups, uint32_t box_cols, CUtensorMapSwizzle swz) {
  EncodeTiledFn enc = encode_fn();
  if (enc == nullptr) return false;
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(groups)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(cols * elem_bytes), static_cast<cuuint64_t>(rows * cols * elem_bytes)};
  cuuint32_t box[3] = {box_cols, 128u, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  return enc(map, dt, 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

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

bool misaligned(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

}  // namespace

cudaError_t w4a16_gemm_launch(const W4A16GemmProblem& p, cudaStream_t stream, const char** why) {
  auto fail = [&](const char* msg) { if (why) *why = msg; return cudaErrorInvalidValue; };
  if (p.M <= 0 || p.N <= 0 || p.K <= 0 || p.G <= 0) return fail("empty w4a16 GEMM");
  if (p.K % kBK != 0) return fail("w4a16 GEMM: K must be a multiple of 64");
  if (p.N % kBN != 0) return fail("w4a16 GEMM: N must be a multiple of 128");
  if (p.epilogue != W4A16_EPI_NONE && p.epilogue != W4A16_EPI_GLU) return fail("w4a16 GEMM: unknown epilogue");
  if (p.epilogue == W4A16_EPI_GLU && (p.act < ACT_RELU || p.act > ACT_SILU))
    return fail("w4a16 GEMM: act must be 1 (relu), 2 (gelu) or 3 (silu)");
  if (misaligned(p.a) || misaligned(p.b) || misaligned(p.d) || (reinterpret_cast<uintptr_t>(p.sb) & 1))
    return fail("w4a16 GEMM: operands must be 16-byte aligned (scales 2-byte aligned)");
  CUtensorMap ta, tb_;
  if (!tile_map(&ta, p.a, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, p.M, p.K, p.G, kBK, CU_TENSOR_MAP_SWIZZLE_128B) ||
      !tile_map(&tb_, p.b, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, p.N, p.K / 2, p.G, kBK / 2, CU_TENSOR_MAP_SWIZZLE_NONE))
    return fail("cuTensorMapEncodeTiled failed for a w4a16 operand");
  Args a{};
  a.sb = static_cast<const uint16_t*>(p.sb);
  a.d = static_cast<__nv_bfloat16*>(p.d);
  a.ldd = p.epilogue == W4A16_EPI_GLU ? p.N / 2 : p.N;
  a.M = p.M; a.N = p.N; a.K = p.K; a.G = p.G;
  a.tiles_m = (p.M + kBM - 1) / kBM;
  a.tiles_n = p.N / kBN;
  a.num_tiles = static_cast<long long>(a.tiles_m) * a.tiles_n * p.G;
  a.epi = p.epilogue;
  a.act = p.act;
  a.row_counts = p.row_counts;
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [] {
    attr_err = cudaFuncSetAttribute(w4a16_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
  });
  if (attr_err != cudaSuccess) return attr_err;
  w4a16_gemm_kernel<<<grid_size(a.num_tiles, p.max_ctas), kThreads, kSmemBytes, stream>>>(ta, tb_, a);
  return cudaGetLastError();
}

}  // namespace tb
