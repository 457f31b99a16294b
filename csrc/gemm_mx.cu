// MX block-scaled fp8 GEMM for sm_90a:  D[g] = A[g] * B[g]^T  with e4m3 operands that carry one UE8M0 scale per
// 32 consecutive K elements (OCP MX).  Hopper's tensor cores know no block scales, so every 32-element K block is one
//     wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3
// into a scratch fragment that the issuing threads then fold into the fp32 accumulator with the block's two scales:
//     acc[m, n] += scratch[m, n] * 2^(sfa[m, kb] - 127) * 2^(sfb[n, kb] - 127).
// The reference has no reduced-precision expert path at all (tutel/experts/ffn.py runs torch.matmul in the model
// dtype); the row-scaled e4m3 path of gemm_sm90.cu is what the fused engine uses, this kernel is the finer-grained
// alternative (outliers only cost the 32 elements next to them their precision, not the whole row).
//
// Layout of one CTA (384 threads, 128 x 128 tiles; K walked in 128-element = 128-byte steps, 6 stages):
//   warp 0        TMA producer: A and B tiles [128 x 128 B] (SWIZZLE_128B) plus the two scale atoms (512 B per 128 rows)
//                 per stage, all completing on the stage's "full" mbarrier
//   warps 4..11   two consumer warpgroups, 64 rows of the tile each: per stage the scale words of the thread's 2 rows
//                 and 32 columns are read once, then four times {wgmma k32 -> scratch, scale-and-add}; while one
//                 warpgroup scales, the other one's wgmma keeps the tensor cores busy.  Epilogue straight from the
//                 accumulator fragment: bias / ReLU / ReLU-backward mask in fp32, packed bf16 pairs to global memory.
// Persistent: CTA b works on tiles b, b + grid, ...; the producer runs ahead into the next tile during the epilogue.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <mutex>

#include "gemm_mx.h"
#include "gemm_sm90.h"
#include "moe_kernels.h"
#include "ptx.cuh"

namespace tb {
namespace {

constexpr int kBM = 128;
constexpr int kBN = 128;
constexpr int kBK = 128;                 // e4m3 elements = bytes per K step (one 128-byte swizzle row)
constexpr int kSfAtomBytes = 512;        // scales of 128 rows x 128 K elements
constexpr int kMxThreads = 384;          // producer warpgroup + two consumer warpgroups

struct MxCfg {
  static constexpr int STAGES = 6;
  static constexpr uint32_t A_BYTES = kBM * kBK;
  static constexpr uint32_t B_BYTES = kBN * kBK;
  static constexpr uint32_t OP_BYTES = A_BYTES + B_BYTES;
  static constexpr uint32_t SF_BYTES = 2 * kSfAtomBytes;            // A rows' and B columns' scales of one K step
  static constexpr uint32_t BAR_BYTES = 128;
  static constexpr uint32_t SMEM_BYTES = 1024 + STAGES * (OP_BYTES + SF_BYTES) + BAR_BYTES;
  static_assert(SMEM_BYTES <= 232448, "227 KB of shared memory per block");
};

struct MxArgs {
  const uint8_t* sfa;
  const uint8_t* sfb;
  __nv_bfloat16* d;
  long long ldd, d_group_stride;
  int M, N, K, G;
  int tiles_m, tiles_n;
  int sfa_row_tiles, sfb_row_tiles;   // 128-row tiles of the scale arrays
  const __nv_bfloat16* bias;          // [G, N] or null
  long long bias_group_stride;
  const __nv_bfloat16* aux;           // MX_EPI_RELU_BWD: forward activation [G, M, N]
  long long ld_aux, aux_group_stride;
  long long num_tiles;
  int epi;
};

__device__ __forceinline__ void bulk_load(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_dst),
               "l"(gsrc), "r"(bytes), "r"(bar)
               : "memory");
}

__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}

// byte k of a word of four UE8M0 scales -> 2^(byte - 127) as a float (byte 0, which only all-zero blocks get, -> 0)
__device__ __forceinline__ float ue8m0_to_float(uint32_t w, int k) { return __uint_as_float(((w >> (8 * k)) & 0xFFu) << 23); }

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

__global__ void __launch_bounds__(kMxThreads, 1)
mx_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const MxArgs args) {
  using C = MxCfg;
  extern __shared__ uint8_t smem_raw[];
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;

  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sf_base = smem_base + C::STAGES * C::OP_BYTES;
  const uint32_t bar_base = sf_base + C::STAGES * C::SF_BYTES;
  auto smem_a = [&](int s) { return smem_base + s * C::OP_BYTES; };
  auto smem_b = [&](int s) { return smem_base + s * C::OP_BYTES + C::A_BYTES; };
  auto smem_sfa = [&](int s) { return sf_base + s * C::SF_BYTES; };
  auto smem_sfb = [&](int s) { return sf_base + s * C::SF_BYTES + kSfAtomBytes; };
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 64u + 8u * s; };

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
        const uint8_t* sfa_g = args.sfa + static_cast<long long>(g) * num_kb * args.sfa_row_tiles * kSfAtomBytes;
        const uint8_t* sfb_g = args.sfb + static_cast<long long>(g) * num_kb * args.sfb_row_tiles * kSfAtomBytes;
        for (int kb = 0; kb < num_kb; ++kb) {
          ptx::mbar_wait_quiet(empty_bar(s), ph ^ 1u);
          if (ptx::elect_one()) {
            const uint32_t fb = full_bar(s);
            ptx::mbar_expect_tx(fb, C::OP_BYTES + C::SF_BYTES);
            ptx::tma_load_3d(smem_a(s), &tmA, fb, kb * kBK, m0, g);
            ptx::tma_load_3d(smem_b(s), &tmB, fb, kb * kBK, n0, g);
            bulk_load(smem_sfa(s), sfa_g + (static_cast<long long>(kb) * args.sfa_row_tiles + m_blk) * kSfAtomBytes,
                      kSfAtomBytes, fb);
            bulk_load(smem_sfb(s), sfb_g + (static_cast<long long>(kb) * args.sfb_row_tiles + n_blk) * kSfAtomBytes,
                      kSfAtomBytes, fb);
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
    // position of row / column i's four scale bytes inside a 512-byte atom (gemm_mx.h)
    auto sf_off = [](int i) { return static_cast<uint32_t>((i % 32) * 16 + (i / 32) * 4); };
    const uint32_t sa_off0 = sf_off(r0), sa_off1 = sf_off(r0 + 8);
    // Operand descriptors: K-major, SWIZZLE_128B, 8-row groups 1024 B apart; a K=32 step advances the start by 32 B.
    constexpr uint32_t desc_hi = (1024u >> 4) | (1u << 30);
    int s = 0;
    uint32_t ph = 0;
    const int epi = args.epi;
    for (long long t = tile_first; t < args.num_tiles; t += tile_step) {
      int g, m_blk, n_blk;
      decode_tile(t, args.tiles_m, args.tiles_n, g, m_blk, n_blk);
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < num_kb; ++kb) {
        ptx::mbar_wait_quiet(full_bar(s), ph);
        const uint32_t a_lo = (((smem_a(s) + static_cast<uint32_t>(wg) * 8192u) >> 4) & 0x3FFFu) | (1u << 16);
        const uint32_t b_lo = ((smem_b(s) >> 4) & 0x3FFFu) | (1u << 16);
        const uint32_t saw0 = lds_u32(smem_sfa(s) + sa_off0), saw1 = lds_u32(smem_sfa(s) + sa_off1);
        uint32_t sbw[32];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          sbw[2 * j] = lds_u32(smem_sfb(s) + sf_off(8 * j + c0));
          sbw[2 * j + 1] = lds_u32(smem_sfb(s) + sf_off(8 * j + c0 + 1));
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float part[64];
          ptx::wgmma_fence();
          ptx::wgmma_m64n128<DT_E4M3, false, false>(part, (static_cast<uint64_t>(desc_hi) << 32) | (a_lo + 2u * k),
                                                    (static_cast<uint64_t>(desc_hi) << 32) | (b_lo + 2u * k), 0u);
          ptx::wgmma_commit();
          const float sa0 = ue8m0_to_float(saw0, k), sa1 = ue8m0_to_float(saw1, k);
          ptx::wgmma_wait<0>();
#pragma unroll
          for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float sb = ue8m0_to_float(sbw[2 * j + e], k);
              acc[4 * j + e] = fmaf(part[4 * j + e], sa0 * sb, acc[4 * j + e]);
              acc[4 * j + 2 + e] = fmaf(part[4 * j + 2 + e], sa1 * sb, acc[4 * j + 2 + e]);
            }
          }
        }
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(empty_bar(s));
        if (++s == C::STAGES) { s = 0; ph ^= 1u; }
      }

      // ------------------------------- epilogue -------------------------------
      const int n0 = n_blk * kBN + c0;
      const __nv_bfloat16* bias = args.bias == nullptr ? nullptr : args.bias + static_cast<long long>(g) * args.bias_group_stride + n0;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = m_blk * kBM + r0 + 8 * h;
        if (row >= args.M) continue;
        __nv_bfloat16* drow = args.d + static_cast<long long>(g) * args.d_group_stride + static_cast<long long>(row) * args.ldd + n0;
        const __nv_bfloat16* arow = (epi == MX_EPI_RELU_BWD)
            ? args.aux + static_cast<long long>(g) * args.aux_group_stride + static_cast<long long>(row) * args.ld_aux + n0 : nullptr;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          float lo = acc[4 * j + 2 * h], hi = acc[4 * j + 2 * h + 1];
          if (bias != nullptr) {
            const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(bias + 8 * j));
            lo += b.x; hi += b.y;
          }
          if (epi == MX_EPI_RELU) { lo = fmaxf(lo, 0.f); hi = fmaxf(hi, 0.f); }
          if (epi == MX_EPI_RELU_BWD) {
            // keep the gradient where the forward activation was positive
            const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(arow + 8 * j));
            lo = a.x > 0.f ? lo : 0.f; hi = a.y > 0.f ? hi : 0.f;
          }
          *reinterpret_cast<__nv_bfloat162*>(drow + 8 * j) = __floats2bfloat162_rn(lo, hi);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// quantiser: 16-bit rows -> e4m3 + UE8M0 block scales in the atom layout of gemm_mx.h
// ------------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

// Four consecutive threads own one 32-element block (8 elements = one 16-byte load each).  The shared exponent is the
// smallest power of two that brings the block's largest magnitude inside e4m3's finite range (448):
//     e = ceil(log2(amax / 448)),   q = rn_satfinite(x * 2^-e),   scale byte = e + 127.
template <typename T>
__global__ void __launch_bounds__(256)
mx_quantize_kernel(const T* __restrict__ x, uint8_t* __restrict__ q, uint8_t* __restrict__ sf, long long total, int R, int K,
                   int row_tiles) {
  const int k8 = K / 8;
  const int num_kb = K / kBK;
  for (long long i0 = static_cast<long long>(blockIdx.x) * blockDim.x; i0 < total; i0 += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long i = i0 + threadIdx.x;
    const bool valid = i < total;
    float f[8];
    float amax = 0.f;
    if (valid) {
      const uint4 raw = ptx::ld_nc_v4(x + i * 8);
      const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        f[j] = to_f32<T>(e[j]);
        amax = fmaxf(amax, fabsf(f[j]));
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = 0.f;
    }
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
    const uint32_t bits = __float_as_uint(amax * (1.0f / 448.0f));
    int e = static_cast<int>((bits >> 23) & 0xFFu) - 127 + ((bits & 0x7FFFFFu) != 0u ? 1 : 0);
    e = max(-127, min(126, e));
    const float inv = __uint_as_float(static_cast<uint32_t>(127 - e) << 23);   // 2^-e
    if (valid) {
      const __nv_fp8x4_e4m3 lo(make_float4(f[0] * inv, f[1] * inv, f[2] * inv, f[3] * inv));
      const __nv_fp8x4_e4m3 hi(make_float4(f[4] * inv, f[5] * inv, f[6] * inv, f[7] * inv));
      uint2 w;
      w.x = *reinterpret_cast<const uint32_t*>(&lo);
      w.y = *reinterpret_cast<const uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(q + i * 8) = w;
      if ((threadIdx.x & 3) == 0) {
        const long long grow = i / k8;
        const int k = static_cast<int>(i % k8) * 8;
        const int g = static_cast<int>(grow / R);
        const int r = static_cast<int>(grow % R);
        const long long atom = (static_cast<long long>(g) * num_kb + k / kBK) * row_tiles + r / 128;
        sf[atom * kSfAtomBytes + (r % 32) * 16 + ((r % 128) / 32) * 4 + (k % kBK) / 32] = static_cast<uint8_t>(e + 127);
      }
    }
  }
}

// Transposing variant for weights: x [G, R, K] -> qT [G, K, R] quantised along R (the operand of a GEMM that reduces over
// R), without materialising the 16-bit transpose.  One block = 128 (R) x 64 (K) tile through shared memory; thread
// (k, rb) owns the 32 values x[r0 + 32 rb .. +32, k0 + k]: one scale, 32 output bytes (one full sector).
constexpr int kTrR = 128, kTrK = 64, kTrPitch = kTrK + 2;   // pitch in elements: 33 words -> conflict-free both ways

template <typename T>
__global__ void __launch_bounds__(256)
mx_quantize_transpose_kernel(const T* __restrict__ x, uint8_t* __restrict__ qT, uint8_t* __restrict__ sf, int R, int K,
                             int row_tiles) {
  __shared__ __align__(16) T tile[kTrR * kTrPitch];
  const int k0 = blockIdx.x * kTrK, r0 = blockIdx.y * kTrR, g = blockIdx.z;
  const T* src = x + (static_cast<long long>(g) * R + r0) * K + k0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int idx = threadIdx.x + j * 256;
    const int row = idx >> 3, c = idx & 7;
    const uint4 raw = ptx::ld_nc_v4(src + static_cast<long long>(row) * K + c * 8);
    uint32_t* dst = reinterpret_cast<uint32_t*>(tile + row * kTrPitch + c * 8);
    dst[0] = raw.x; dst[1] = raw.y; dst[2] = raw.z; dst[3] = raw.w;
  }
  __syncthreads();
  const int k = threadIdx.x & 63, rb = threadIdx.x >> 6;
  float f[32];
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    f[i] = to_f32<T>(tile[(rb * 32 + i) * kTrPitch + k]);
    amax = fmaxf(amax, fabsf(f[i]));
  }
  const uint32_t bits = __float_as_uint(amax * (1.0f / 448.0f));
  int e = static_cast<int>((bits >> 23) & 0xFFu) - 127 + ((bits & 0x7FFFFFu) != 0u ? 1 : 0);
  e = max(-127, min(126, e));
  const float inv = __uint_as_float(static_cast<uint32_t>(127 - e) << 23);
  uint32_t w[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const __nv_fp8x4_e4m3 p4(make_float4(f[4 * i] * inv, f[4 * i + 1] * inv, f[4 * i + 2] * inv, f[4 * i + 3] * inv));
    w[i] = *reinterpret_cast<const uint32_t*>(&p4);
  }
  const int krow = k0 + k;
  uint8_t* dst = qT + (static_cast<long long>(g) * K + krow) * R + r0 + rb * 32;
  *reinterpret_cast<uint4*>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
  *reinterpret_cast<uint4*>(dst + 16) = make_uint4(w[4], w[5], w[6], w[7]);
  const long long atom = (static_cast<long long>(g) * (R / 128) + r0 / 128) * row_tiles + krow / 128;
  sf[atom * kSfAtomBytes + (krow % 32) * 16 + ((krow % 128) / 32) * 4 + rb] = static_cast<uint8_t>(e + 127);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn mx_encode_fn() {
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

// e4m3 [groups, rows, k] row-major -> boxes of `box_rows` rows x 128 bytes, 128-byte swizzle
bool mx_operand_map(CUtensorMap* map, const void* base, long long rows, long long k, int groups, int box_rows) {
  EncodeTiledFn enc = mx_encode_fn();
  if (enc == nullptr) return false;
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(k), static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(groups)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(k), static_cast<cuuint64_t>(rows) * static_cast<cuuint64_t>(k)};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(kBK), static_cast<cuuint32_t>(box_rows), 1};
  cuuint32_t estr[3] = {1, 1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

cudaError_t mx_launch(const MxGemmProblem& p, cudaStream_t stream, const char** why) {
  using C = MxCfg;
  CUtensorMap ta, tb_;
  if (!mx_operand_map(&ta, p.a, p.M, p.K, p.G, kBM) || !mx_operand_map(&tb_, p.b, p.N, p.K, p.G, kBN)) {
    if (why) *why = "cuTensorMapEncodeTiled failed for an MX operand";
    return cudaErrorInvalidValue;
  }
  MxArgs a;
  a.sfa = static_cast<const uint8_t*>(p.sfa);
  a.sfb = static_cast<const uint8_t*>(p.sfb);
  a.d = static_cast<__nv_bfloat16*>(p.d);
  a.ldd = p.ldd;
  a.d_group_stride = p.d_group_stride;
  a.M = p.M; a.N = p.N; a.K = p.K; a.G = p.G;
  a.tiles_m = (p.M + kBM - 1) / kBM;
  a.tiles_n = p.N / kBN;
  a.sfa_row_tiles = (p.M + 127) / 128;
  a.sfb_row_tiles = (p.N + 127) / 128;
  a.bias = static_cast<const __nv_bfloat16*>(p.bias);
  a.bias_group_stride = p.bias_group_stride;
  a.aux = static_cast<const __nv_bfloat16*>(p.aux);
  a.ld_aux = p.ld_aux;
  a.aux_group_stride = p.aux_group_stride;
  a.epi = p.epilogue;
  static std::once_flag once;
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [] {
    attr_err = cudaFuncSetAttribute(mx_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
  });
  if (attr_err != cudaSuccess) return attr_err;
  a.num_tiles = static_cast<long long>(a.tiles_m) * a.tiles_n * p.G;
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  long long ctas = sms;                                                    // one resident CTA per SM
  if (p.max_ctas > 0) ctas = std::max<long long>(1, std::min<long long>(ctas, p.max_ctas));
  const unsigned grid = static_cast<unsigned>(std::min<long long>(a.num_tiles, ctas));
  mx_gemm_kernel<<<grid, kMxThreads, C::SMEM_BYTES, stream>>>(ta, tb_, a);
  return cudaGetLastError();
}

}  // namespace

cudaError_t mx_gemm_launch(const MxGemmProblem& p, cudaStream_t stream, const char** why) {
  auto fail = [&](const char* msg) { if (why) *why = msg; return cudaErrorInvalidValue; };
  if (p.M <= 0 || p.N <= 0 || p.K <= 0 || p.G <= 0) return fail("empty MX GEMM");
  if (p.K % kBK != 0) return fail("MX GEMM: K must be a multiple of 128");
  if (p.N % 128 != 0) return fail("MX GEMM: N must be a multiple of 128");
  if ((reinterpret_cast<uintptr_t>(p.a) | reinterpret_cast<uintptr_t>(p.b) | reinterpret_cast<uintptr_t>(p.sfa) |
       reinterpret_cast<uintptr_t>(p.sfb) | reinterpret_cast<uintptr_t>(p.d)) & 15)
    return fail("MX GEMM: operands must be 16-byte aligned");
  if (p.ldd % 8 != 0 || p.d_group_stride % 8 != 0) return fail("MX GEMM: output strides must be multiples of 8 elements");
  if (p.epilogue == MX_EPI_RELU_BWD && (p.aux == nullptr || (reinterpret_cast<uintptr_t>(p.aux) & 15) || p.ld_aux % 8 || p.aux_group_stride % 8))
    return fail("MX GEMM: the ReLU-backward epilogue needs a 16-byte aligned aux operand");
  if (p.bias != nullptr && ((reinterpret_cast<uintptr_t>(p.bias) & 15) || p.bias_group_stride % 8))
    return fail("MX GEMM: bias must be 16-byte aligned");
  // block_n / cta_group are the tile-shape hints of callers written for wider tiles and CTA pairs: validated, but this
  // kernel has ONE tile shape (128 x 128, one CTA), so they do not change what runs.
  if (p.block_n != 0 && p.block_n != 128 && p.block_n != 256) return fail("MX GEMM: block_n must be 0, 128 or 256");
  if (p.block_n == 256 && p.N % 256 != 0) return fail("MX GEMM: block_n 256 needs N % 256 == 0");
  if (p.cta_group < 0 || p.cta_group > 2) return fail("MX GEMM: cta_group must be 0, 1 or 2");
  if (p.cta_group == 2 && p.block_n != 0 && p.block_n != 256) return fail("MX GEMM: CTA pairs need block_n 256");
  return mx_launch(p, stream, why);
}

cudaError_t mx_quantize(const void* x, void* q, void* sf, int groups, int rows, int k, int elem_type, cudaStream_t stream) {
  if (k % kBK != 0 || (elem_type != ET_F16 && elem_type != ET_BF16)) return cudaErrorInvalidValue;
  const long long total = static_cast<long long>(groups) * rows * (k / 8);
  if (total == 0) return cudaSuccess;
  const int row_tiles = (rows + 127) / 128;
  const int blocks = static_cast<int>(std::min<long long>((total + 255) / 256, 132LL * 16));
  if (elem_type == ET_BF16)
    mx_quantize_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), static_cast<uint8_t*>(q),
                                                                  static_cast<uint8_t*>(sf), total, rows, k, row_tiles);
  else
    mx_quantize_kernel<__half><<<blocks, 256, 0, stream>>>(static_cast<const __half*>(x), static_cast<uint8_t*>(q),
                                                           static_cast<uint8_t*>(sf), total, rows, k, row_tiles);
  return cudaGetLastError();
}

cudaError_t mx_quantize_transpose(const void* x, void* qT, void* sf, int groups, int rows, int k, int elem_type,
                                  cudaStream_t stream) {
  if (rows % kTrR != 0 || k % kTrK != 0 || (elem_type != ET_F16 && elem_type != ET_BF16)) return cudaErrorInvalidValue;
  if (groups == 0 || rows == 0 || k == 0) return cudaSuccess;
  const dim3 grid(k / kTrK, rows / kTrR, groups);
  const int row_tiles = (k + 127) / 128;
  if (elem_type == ET_BF16)
    mx_quantize_transpose_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), static_cast<uint8_t*>(qT),
                                                                            static_cast<uint8_t*>(sf), rows, k, row_tiles);
  else
    mx_quantize_transpose_kernel<__half><<<grid, 256, 0, stream>>>(static_cast<const __half*>(x), static_cast<uint8_t*>(qT),
                                                                     static_cast<uint8_t*>(sf), rows, k, row_tiles);
  return cudaGetLastError();
}

cudaError_t set_spin_timeout_mx(unsigned long long ns) {
  return cudaMemcpyToSymbol(tb_spin_timeout_ns, &ns, sizeof(ns));
}

}  // namespace tb
