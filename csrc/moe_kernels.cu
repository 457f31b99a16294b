// Routing and sparse dispatch/combine kernels for sm_90a.
//
// Functional counterpart of the reference's SIMT JIT kernels (tutel/jit_kernels/sparse.py:17-134), its
// `tutel_ops.cumsum` Blelloch scan (tutel/custom/custom_kernel.cpp:822-872) and the ~15 small torch kernels of
// `extract_critical` (tutel/impls/fast_dispatch.py:143-204), re-designed slot-centrically:
//
//   * routing produces, besides idx/loc, an INVERSE map slot -> (token, choice).  Encode then becomes a fully
//     coalesced row gather that also writes the zero padding (no separate zero-fill pass, one launch for all k,
//     native bf16/fp16 - the reference up-casts bf16 to fp32 and launches k scatters);
//   * encode can push rows straight into PEER GPUs' receive buffers (16-byte NVLink stores) and publish
//     release.sys counters per row block - the dispatch all-to-all is fused into the scatter;
//   * decode sums all k choices in one pass with fp32 accumulation and can acquire per-expert arrival counters
//     (combine all-to-all fused into the GEMM epilogue on the producer side).
#include "moe_kernels.h"

#include <cfloat>

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include "ptx.cuh"

namespace tb {
namespace {

constexpr int kRouteBlock = 1024;
constexpr int kInvalidLoc = 0x3fffffff;

// ------------------------------------------------------------------------------------------------
// routing
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRouteBlock) route_hist_kernel(const int* __restrict__ idx, int* __restrict__ ws,
                                                                int S, int E, int k) {
  extern __shared__ int hist[];
  const int b = blockIdx.x;
  const int s = b * kRouteBlock + threadIdx.x;
  for (int j = 0; j < k; ++j) {
    for (int e = threadIdx.x; e < E; e += kRouteBlock) hist[e] = 0;
    __syncthreads();
    if (s < S) {
      const int e = idx[static_cast<long long>(j) * S + s];
      if (e >= 0 && e < E) atomicAdd(&hist[e], 1);
    }
    __syncthreads();
    for (int e = threadIdx.x; e < E; e += kRouteBlock) ws[(static_cast<long long>(b) * k + j) * E + e] = hist[e];
    __syncthreads();
  }
}

// One thread per expert: exclusive prefix over (choice, block) in that order -> every block learns where its
// tokens start in each expert's queue.
__global__ void route_scan_kernel(int* __restrict__ ws, int* __restrict__ counts, int nblocks, int E, int k) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  int running = 0;
  for (int j = 0; j < k; ++j) {
    for (int b = 0; b < nblocks; ++b) {
      const long long o = (static_cast<long long>(b) * k + j) * E + e;
      const int v = ws[o];
      ws[o] = running;
      running += v;
    }
  }
  counts[e] = running;
}

__global__ void __launch_bounds__(kRouteBlock) route_rank_kernel(const int* __restrict__ idx,
                                                                const int* __restrict__ ws, int* __restrict__ loc,
                                                                int* __restrict__ slot_src, int S, int E, int k,
                                                                int C) {
  extern __shared__ int cnt[];
  const int b = blockIdx.x;
  const int s = b * kRouteBlock + threadIdx.x;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  for (int j = 0; j < k; ++j) {
    for (int e = threadIdx.x; e < E; e += kRouteBlock) cnt[e] = 0;
    __syncthreads();
    int e = -1;
    if (s < S) {
      e = idx[static_cast<long long>(j) * S + s];
      if (e >= E) e = -1;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, e);
    const int rank_in_warp = __popc(peers & ((1u << lane) - 1u));
    const int leader = __ffs(peers) - 1;
    int base = 0;
    for (int w = 0; w < kRouteBlock / 32; ++w) {
      if (warp == w && e >= 0 && lane == leader) {
        base = cnt[e];
        cnt[e] = base + __popc(peers);
      }
      __syncthreads();
    }
    base = __shfl_sync(0xffffffffu, base, leader);
    if (s < S) {
      int l = kInvalidLoc;
      if (e >= 0) {
        l = ws[(static_cast<long long>(b) * k + j) * E + e] + base + rank_in_warp;
        if (slot_src != nullptr && l < C) slot_src[static_cast<long long>(e) * C + l] = s * k + j;
      }
      loc[static_cast<long long>(j) * S + s] = l;
    }
    __syncthreads();
  }
}

__global__ void slot_map_kernel(const int* __restrict__ idx, const int* __restrict__ loc, int* __restrict__ slot_src,
                                int S, int E, int k, int C) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(S) * k) return;
  const int j = static_cast<int>(i / S);
  const int s = static_cast<int>(i - static_cast<long long>(j) * S);
  const int e = idx[i];
  const int l = loc[i];
  if (e >= 0 && e < E && l >= 0 && l < C) slot_src[static_cast<long long>(e) * C + l] = s * k + j;
}

// ------------------------------------------------------------------------------------------------
// expert-packed layout: expert e's rows are [seg_off[e], seg_off[e] + counts[e]), segments start on 128-row blocks
// ------------------------------------------------------------------------------------------------
constexpr int kPackBlock = 128;

// One block of 1024 threads: warp 0 scans the rounded counts 32 experts at a time, then every thread describes blocks.
__global__ void __launch_bounds__(1024)
packed_layout_kernel(const int* __restrict__ counts, int* __restrict__ seg_off, int* __restrict__ block_expert,
                     int* __restrict__ block_rows, int E, int nblocks) {
  extern __shared__ int sh_off[];   // [E + 1]
  if (threadIdx.x < 32) {
    int carry = 0;
    for (int e0 = 0; e0 < E; e0 += 32) {
      const int e = e0 + static_cast<int>(threadIdx.x);
      const int c = e < E ? max(counts[e], 0) : 0;
      const int v = (c + kPackBlock - 1) / kPackBlock * kPackBlock;
      int incl = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (static_cast<int>(threadIdx.x) >= o) incl += t;
      }
      if (e < E) sh_off[e] = carry + incl - v;
      carry += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (threadIdx.x == 0) sh_off[E] = carry;
  }
  __syncthreads();
  for (int e = threadIdx.x; e <= E; e += blockDim.x) seg_off[e] = sh_off[e];
  const int total = sh_off[E];
  for (int b = threadIdx.x; b < nblocks; b += blockDim.x) {
    const int r0 = b * kPackBlock;
    int e = 0, rows = 0;
    if (r0 < total) {
      int lo = 0, hi = E - 1;       // the last e with sh_off[e] <= r0 (empty experts share their successor's offset)
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (sh_off[mid] <= r0) lo = mid; else hi = mid - 1;
      }
      e = lo;
      rows = min(kPackBlock, sh_off[e] + max(counts[e], 0) - r0);
    }
    block_expert[b] = e;
    block_rows[b] = rows;
  }
}

__global__ void packed_slot_kernel(const int* __restrict__ idx, const int* __restrict__ loc, const int* __restrict__ seg_off,
                                   int* __restrict__ slot_src, int S, int E, int k, int R) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(S) * k) return;
  const int j = static_cast<int>(i / S);
  const int s = static_cast<int>(i - static_cast<long long>(j) * S);
  const int e = idx[i];
  const int l = loc[i];
  if (e >= 0 && e < E && l >= 0) {
    const int r = seg_off[e] + l;
    if (r < R) slot_src[r] = s * k + j;
  }
}

// ------------------------------------------------------------------------------------------------
// 16-byte vector helpers
// ------------------------------------------------------------------------------------------------
template <typename T>
struct Vec;  // 16 bytes of T
template <>
struct Vec<float> {
  static constexpr int N = 4;
  static __device__ __forceinline__ void unpack(const uint4& u, float* f) {
    f[0] = __uint_as_float(u.x); f[1] = __uint_as_float(u.y); f[2] = __uint_as_float(u.z); f[3] = __uint_as_float(u.w);
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
  }
};
template <>
struct Vec<__half> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void unpack(const uint4& u, float* f) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
      f[2 * i] = t.x; f[2 * i + 1] = t.y;
    }
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<const uint32_t*>(&h);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
};
template <>
struct Vec<__nv_bfloat16> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void unpack(const uint4& u, float* f) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
    }
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<const uint32_t*>(&h);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
};

template <typename T>
__device__ __forceinline__ float to_f(T v);
template <>
__device__ __forceinline__ float to_f<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <>
__device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T>
__device__ __forceinline__ T from_f(float v);
template <>
__device__ __forceinline__ float from_f<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// ------------------------------------------------------------------------------------------------
// encode: slot-centric row gather (+ optional remote push and release counters)
// ------------------------------------------------------------------------------------------------
constexpr int kEncThreads = 256;      // local gather
constexpr int kEncPushThreads = 128;  // remote push: 128 x 64 registers fit next to a resident GEMM CTA (gemm_sm90.cu)

template <typename T, bool VEC, int THREADS>
__global__ void __launch_bounds__(THREADS, 65536 / (THREADS * 64))
encode_rows_kernel(const T* __restrict__ x, const float* __restrict__ gates, const int* __restrict__ slot_src,
                   T* __restrict__ out, const unsigned long long* __restrict__ dst_ptr_table,
                   const unsigned long long* __restrict__ signal_ptr_table, unsigned int* __restrict__ chunk_counters,
                   int chunk_rows, int unit_rows, int S, int E, int k, int C, int M, int rot_units,
                   uint32_t signal_value, const int* __restrict__ valid_rows) {
  // Work unit = `unit_rows` consecutive slots of one expert (one warp per row).  Many blocks cooperate on one flag
  // chunk (`chunk_rows` rows); the block that finishes the chunk's last unit publishes the flag.
  constexpr int kEncWarps = THREADS / 32;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int units_per_expert = (C + unit_rows - 1) / unit_rows;
  const int chunks_per_expert = (C + chunk_rows - 1) / chunk_rows;
  const long long total_units = static_cast<long long>(E) * units_per_expert;
  for (long long ui = blockIdx.x; ui < total_units; ui += gridDim.x) {
    const long long u = (ui + rot_units) % total_units;
    const int e = static_cast<int>(u / units_per_expert);
    const int r0 = static_cast<int>(u - static_cast<long long>(e) * units_per_expert) * unit_rows;
    int r1 = min(r0 + unit_rows, C);
    if (valid_rows != nullptr) r1 = min(r1, valid_rows[e]);   // dropless bound buffers: rows past the count are never read
    T* dst_e = dst_ptr_table != nullptr ? reinterpret_cast<T*>(dst_ptr_table[e])
                                        : out + static_cast<long long>(e) * C * M;
    for (int r = r0 + warp; r < r1; r += kEncWarps) {
      const int src = slot_src[static_cast<long long>(e) * C + r];
      T* drow = dst_e + static_cast<long long>(r) * M;
      if (src < 0) {
        if constexpr (VEC) {
          const uint4 z = make_uint4(0, 0, 0, 0);
          for (int v = lane; v < M / Vec<T>::N; v += 32) ptx::st_na_v4(reinterpret_cast<uint4*>(drow) + v, z);
        } else {
          for (int m = lane; m < M; m += 32) drow[m] = from_f<T>(0.0f);
        }
        continue;
      }
      const int tok = src / k;
      const int j = src - tok * k;
      const float g = gates != nullptr ? gates[static_cast<long long>(j) * S + tok] : 1.0f;
      const T* srow = x + static_cast<long long>(tok) * M;
      if constexpr (VEC) {
        const int nv = M / Vec<T>::N;
        const uint4* sv = reinterpret_cast<const uint4*>(srow);
        uint4* dv = reinterpret_cast<uint4*>(drow);
        int v = lane;
        for (; v + 224 < nv; v += 256) {   // 8 x 16 B in flight per lane
          uint4 a[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) a[q] = ptx::ld_nc_v4(sv + v + 32 * q);
          if (gates != nullptr) {
#pragma unroll
            for (int q = 0; q < 8; ++q) {
              float f[Vec<T>::N];
              Vec<T>::unpack(a[q], f);
#pragma unroll
              for (int i = 0; i < Vec<T>::N; ++i) f[i] *= g;
              a[q] = Vec<T>::pack(f);
            }
          }
#pragma unroll
          for (int q = 0; q < 8; ++q) ptx::st_na_v4(dv + v + 32 * q, a[q]);
        }
        for (; v < nv; v += 32) {
          uint4 a = ptx::ld_nc_v4(sv + v);
          if (gates != nullptr) {
            float f[Vec<T>::N];
            Vec<T>::unpack(a, f);
#pragma unroll
            for (int i = 0; i < Vec<T>::N; ++i) f[i] *= g;
            a = Vec<T>::pack(f);
          }
          ptx::st_na_v4(dv + v, a);
        }
      } else {
        for (int m = lane; m < M; m += 32) drow[m] = from_f<T>(to_f<T>(srow[m]) * g);
      }
    }
    if (signal_ptr_table != nullptr) {
      __syncthreads();  // every warp's stores of this unit are issued and ordered before the counter update below
      if (threadIdx.x == 0) {
        const int ci = r0 / chunk_rows;
        const int chunk_begin = ci * chunk_rows;
        const int chunk_end = min(chunk_begin + chunk_rows, C);
        const unsigned units_in_chunk = static_cast<unsigned>((chunk_end - chunk_begin + unit_rows - 1) / unit_rows);
        unsigned int* cnt = chunk_counters + static_cast<long long>(e) * chunks_per_expert + ci;
        unsigned prev;
        asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(prev) : "l"(cnt) : "memory");
        if (prev == units_in_chunk - 1u) {
          *cnt = 0u;  // re-arm for the next launch (stream ordered)
          uint32_t* flag = reinterpret_cast<uint32_t*>(signal_ptr_table[e]) + ci;
          ptx::fence_acq_rel_sys();
          if (signal_value != 0u) ptx::st_release_sys(flag, signal_value);
          else ptx::red_add_release_sys(flag, 1u);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// decode: token-centric weighted gather of k rows
// ------------------------------------------------------------------------------------------------
constexpr int kMaxK = 16;

// Weight of the shared experts' output in the combine: sigmoid(logit) in fp32 (IEEE division and expf, no fast-math
// intrinsics; a logit below about -88 gives exp = inf and weight 0).
__device__ __forceinline__ float shared_weight(float logit) { return 1.0f / (1.0f + expf(-logit)); }

// SH: shared experts.  After the routed fmaf chain (unchanged, choice order) one more fmaf adds w_s * base[s] with
// w_s = 1 or shared_weight(shared_logit[s]); the sum is rounded to T once.  A token whose choices were all dropped gets
// the shared term alone.
template <typename T, bool VEC, bool SEG, bool SH>
__global__ void __launch_bounds__(256)
decode_rows_kernel(const T* __restrict__ buf, const float* __restrict__ gates, const int* __restrict__ idx,
                   const int* __restrict__ loc, T* __restrict__ out, const uint32_t* __restrict__ wait_flags,
                   uint32_t wait_target, int S, int E, int k, int C, int M, const int* __restrict__ seg_off,
                   const T* __restrict__ base, const float* __restrict__ shared_logit) {
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  for (long long s = static_cast<long long>(blockIdx.x) * 8 + warp; s < S; s += static_cast<long long>(gridDim.x) * 8) {
    const T* rows[kMaxK];
    float w[kMaxK];
    int nsel = 0;
    const T* brow = nullptr;
    float ws = 1.0f;
    if constexpr (SH) {
      brow = base + s * M;
      if (shared_logit != nullptr) ws = shared_weight(shared_logit[s]);
    }
    for (int j = 0; j < k; ++j) {
      const int e = idx[static_cast<long long>(j) * S + s];
      const int l = loc[static_cast<long long>(j) * S + s];
      if (e >= 0 && e < E && l >= 0 && l < C) {
        if (wait_flags != nullptr) {
          if (lane == 0) ptx::wait_flag_ge_sys(wait_flags + e, wait_target);
          __syncwarp();
        }
        rows[nsel] = buf + ((SEG ? static_cast<long long>(seg_off[e]) : static_cast<long long>(e) * C) + l) * M;
        w[nsel] = gates != nullptr ? gates[static_cast<long long>(j) * S + s] : 1.0f;
        ++nsel;
      }
    }
    T* orow = out + s * M;
    if constexpr (VEC) {
      const int nv = M / Vec<T>::N;
      for (int v0 = lane; v0 < nv; v0 += 64) {
        float acc[2][Vec<T>::N];
#pragma unroll
        for (int u = 0; u < 2; ++u)
#pragma unroll
          for (int q = 0; q < Vec<T>::N; ++q) acc[u][q] = 0.0f;
        for (int t = 0; t < nsel; ++t) {
          uint4 a[2];
#pragma unroll
          for (int u = 0; u < 2; ++u)
            if (v0 + 32 * u < nv) a[u] = ptx::ld_v4(reinterpret_cast<const uint4*>(rows[t]) + v0 + 32 * u);
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            if (v0 + 32 * u < nv) {
              float f[Vec<T>::N];
              Vec<T>::unpack(a[u], f);
#pragma unroll
              for (int q = 0; q < Vec<T>::N; ++q) acc[u][q] = fmaf(w[t], f[q], acc[u][q]);
            }
          }
        }
        if constexpr (SH) {
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            if (v0 + 32 * u < nv) {
              float f[Vec<T>::N];
              Vec<T>::unpack(ptx::ld_v4(reinterpret_cast<const uint4*>(brow) + v0 + 32 * u), f);
#pragma unroll
              for (int q = 0; q < Vec<T>::N; ++q) acc[u][q] = fmaf(ws, f[q], acc[u][q]);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < 2; ++u)
          if (v0 + 32 * u < nv) ptx::st_na_v4(reinterpret_cast<uint4*>(orow) + v0 + 32 * u, Vec<T>::pack(acc[u]));
      }
    } else {
      for (int m = lane; m < M; m += 32) {
        float acc = 0.0f;
        for (int t = 0; t < nsel; ++t) acc = fmaf(w[t], to_f<T>(rows[t][m]), acc);
        if constexpr (SH) acc = fmaf(ws, to_f<T>(brow[m]), acc);
        orow[m] = from_f<T>(acc);
      }
    }
  }
}

// SH: gated shared experts.  In the same pass over the tokens: d_base[s] = w_s * a[s] (rounded to T) and
// d_shared_logit[s] = w_s (1 - w_s) <a[s], base[s]>, w_s = shared_weight(shared_logit[s]).  k may be 0 (pre-scored
// routing, whose combine has no gate gradient): then only the shared terms are computed.
template <typename T, bool VEC, bool SEG, bool SH>
__global__ void __launch_bounds__(256)
gate_grad_kernel(const T* __restrict__ a, const T* __restrict__ buf, const int* __restrict__ idx,
                 const int* __restrict__ loc, float* __restrict__ dgate, int S, int E, int k, int C, int M,
                 const int* __restrict__ seg_off, const T* __restrict__ base, const float* __restrict__ shared_logit,
                 T* __restrict__ d_base, float* __restrict__ d_shared_logit) {
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  for (long long s = static_cast<long long>(blockIdx.x) * 8 + warp; s < S; s += static_cast<long long>(gridDim.x) * 8) {
    const T* arow = a + s * M;
    for (int j = 0; j < k; ++j) {
      const int e = idx[static_cast<long long>(j) * S + s];
      const int l = loc[static_cast<long long>(j) * S + s];
      float acc = 0.0f;
      if (e >= 0 && e < E && l >= 0 && l < C) {
        const T* brow = buf + ((SEG ? static_cast<long long>(seg_off[e]) : static_cast<long long>(e) * C) + l) * M;
        if constexpr (VEC) {
          const int nv = M / Vec<T>::N;
          for (int v = lane; v < nv; v += 32) {
            float fa[Vec<T>::N], fb[Vec<T>::N];
            Vec<T>::unpack(ptx::ld_v4(reinterpret_cast<const uint4*>(arow) + v), fa);
            Vec<T>::unpack(ptx::ld_v4(reinterpret_cast<const uint4*>(brow) + v), fb);
#pragma unroll
            for (int q = 0; q < Vec<T>::N; ++q) acc = fmaf(fa[q], fb[q], acc);
          }
        } else {
          for (int m = lane; m < M; m += 32) acc = fmaf(to_f<T>(arow[m]), to_f<T>(brow[m]), acc);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      }
      if (lane == 0) dgate[static_cast<long long>(j) * S + s] = acc;
    }
    if constexpr (SH) {
      const float ws = shared_weight(shared_logit[s]);
      const T* brow = base + s * M;
      T* drow = d_base + s * M;
      float acc = 0.0f;
      if constexpr (VEC) {
        const int nv = M / Vec<T>::N;
        for (int v = lane; v < nv; v += 32) {
          float fa[Vec<T>::N], fb[Vec<T>::N];
          Vec<T>::unpack(ptx::ld_v4(reinterpret_cast<const uint4*>(arow) + v), fa);
          Vec<T>::unpack(ptx::ld_v4(reinterpret_cast<const uint4*>(brow) + v), fb);
#pragma unroll
          for (int q = 0; q < Vec<T>::N; ++q) {
            acc = fmaf(fa[q], fb[q], acc);
            fa[q] *= ws;
          }
          ptx::st_na_v4(reinterpret_cast<uint4*>(drow) + v, Vec<T>::pack(fa));
        }
      } else {
        for (int m = lane; m < M; m += 32) {
          const float fa = to_f<T>(arow[m]);
          acc = fmaf(fa, to_f<T>(brow[m]), acc);
          drow[m] = from_f<T>(fa * ws);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) d_shared_logit[s] = ws * (1.0f - ws) * acc;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// per-row e4m3 quantisation (activations / K-major weights for the fp8 wgmma GEMM): one warp per row
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
quantize_rows_kernel(const T* __restrict__ x, uint8_t* __restrict__ q, float* __restrict__ scale, long long R, int K) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int VN = Vec<T>::N;
  for (long long r = static_cast<long long>(blockIdx.x) * 8 + warp; r < R; r += static_cast<long long>(gridDim.x) * 8) {
    const T* row = x + r * K;
    float amax = 0.0f;
    const int nv = K / VN;
    for (int v = lane; v < nv; v += 32) {
      float f[VN];
      Vec<T>::unpack(ptx::ld_v4(reinterpret_cast<const uint4*>(row) + v), f);
#pragma unroll
      for (int i = 0; i < VN; ++i) amax = fmaxf(amax, fabsf(f[i]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    // (at least FLT_MIN: below it 1 / s overflows, and a row of tiny values would turn its zeros into 0 * inf = NaN)
    const float s = amax > 0.0f ? fmaxf(amax * (1.0f / 448.0f), FLT_MIN) : 1.0f;
    const float inv = 1.0f / s;
    if (lane == 0) scale[r] = s;
    uint8_t* qrow = q + r * K;
    for (int v = lane; v < nv; v += 32) {
      float f[VN];
      Vec<T>::unpack(ptx::ld_v4(reinterpret_cast<const uint4*>(row) + v), f);
      uint32_t packed[VN / 4];
#pragma unroll
      for (int i = 0; i < VN / 4; ++i) {
        const __nv_fp8x4_e4m3 p4(make_float4(f[4 * i] * inv, f[4 * i + 1] * inv, f[4 * i + 2] * inv, f[4 * i + 3] * inv));
        packed[i] = *reinterpret_cast<const uint32_t*>(&p4);
      }
      if constexpr (VN == 8) {
        *reinterpret_cast<uint2*>(qrow + static_cast<long long>(v) * 8) = make_uint2(packed[0], packed[1]);
      } else {
        *reinterpret_cast<uint32_t*>(qrow + static_cast<long long>(v) * 4) = packed[0];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// fp8 dispatch: encode (slot-centric gather) + per-row e4m3 quantisation + optional remote push, one warp per row.
// Destination row = M bytes of e4m3 and one fp32 scale (max|row| / 448) in a separate [E, C] array; the scale factors out
// of the expert GEMM's dot product and is applied in its epilogue (scale_a).  Half the NVLink bytes of a 16-bit push.
// ------------------------------------------------------------------------------------------------
template <typename T, int THREADS>
__global__ void __launch_bounds__(THREADS, 65536 / (THREADS * 64))
encode_rows_fp8_kernel(const T* __restrict__ x, const float* __restrict__ gates, const int* __restrict__ slot_src,
                       uint8_t* __restrict__ out, float* __restrict__ scale_out,
                       const unsigned long long* __restrict__ dst_ptr_table,
                       const unsigned long long* __restrict__ scale_ptr_table,
                       const unsigned long long* __restrict__ signal_ptr_table, unsigned int* __restrict__ chunk_counters,
                       int chunk_rows, int unit_rows, int S, int E, int k, int C, int M, int rot_units,
                       uint32_t signal_value) {
  static_assert(Vec<T>::N == 8, "16-bit sources only");
  constexpr int kWarps = THREADS / 32;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int units_per_expert = (C + unit_rows - 1) / unit_rows;
  const int chunks_per_expert = (C + chunk_rows - 1) / chunk_rows;
  const long long total_units = static_cast<long long>(E) * units_per_expert;
  const int n16 = M / 16;                                    // 16-element groups per row (M % 16 == 0)
  for (long long ui = blockIdx.x; ui < total_units; ui += gridDim.x) {
    const long long u = (ui + rot_units) % total_units;
    const int e = static_cast<int>(u / units_per_expert);
    const int r0 = static_cast<int>(u - static_cast<long long>(e) * units_per_expert) * unit_rows;
    const int r1 = min(r0 + unit_rows, C);
    uint8_t* dst_e = dst_ptr_table != nullptr ? reinterpret_cast<uint8_t*>(dst_ptr_table[e])
                                              : out + static_cast<long long>(e) * C * M;
    float* sc_e = scale_ptr_table != nullptr ? reinterpret_cast<float*>(scale_ptr_table[e])
                                             : scale_out + static_cast<long long>(e) * C;
    for (int r = r0 + warp; r < r1; r += kWarps) {
      const int src = slot_src[static_cast<long long>(e) * C + r];
      uint4* drow = reinterpret_cast<uint4*>(dst_e + static_cast<long long>(r) * M);
      if (src < 0) {
        const uint4 z = make_uint4(0, 0, 0, 0);
        for (int v = lane; v < n16; v += 32) ptx::st_na_v4(drow + v, z);
        if (lane == 0) sc_e[r] = 1.0f;
        continue;
      }
      const int tok = src / k;
      const int j = src - tok * k;
      const float g = gates != nullptr ? gates[static_cast<long long>(j) * S + tok] : 1.0f;
      const uint4* sv = reinterpret_cast<const uint4*>(x + static_cast<long long>(tok) * M);
      float amax = 0.0f;
      for (int v = lane; v < 2 * n16; v += 32) {
        float f[8];
        Vec<T>::unpack(ptx::ld_v4(sv + v), f);
#pragma unroll
        for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(f[i]));
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
      amax *= fabsf(g);
      const float sc = amax > 0.0f ? fmaxf(amax * (1.0f / 448.0f), FLT_MIN) : 1.0f;     // (FLT_MIN: see quantize_rows)
      const float inv = g / sc;
      if (lane == 0) sc_e[r] = sc;
      for (int v = lane; v < n16; v += 32) {                 // second pass hits L1/L2: 2 x 16 B in, 16 B out
        float f[16];
        Vec<T>::unpack(ptx::ld_v4(sv + 2 * v), f);
        Vec<T>::unpack(ptx::ld_v4(sv + 2 * v + 1), f + 8);
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const __nv_fp8x4_e4m3 p4(make_float4(f[4 * i] * inv, f[4 * i + 1] * inv, f[4 * i + 2] * inv, f[4 * i + 3] * inv));
          w[i] = *reinterpret_cast<const uint32_t*>(&p4);
        }
        ptx::st_na_v4(drow + v, make_uint4(w[0], w[1], w[2], w[3]));
      }
    }
    if (signal_ptr_table != nullptr) {
      __syncthreads();
      if (threadIdx.x == 0) {
        const int ci = r0 / chunk_rows;
        const int chunk_begin = ci * chunk_rows;
        const int chunk_end = min(chunk_begin + chunk_rows, C);
        const unsigned units_in_chunk = static_cast<unsigned>((chunk_end - chunk_begin + unit_rows - 1) / unit_rows);
        unsigned int* cnt = chunk_counters + static_cast<long long>(e) * chunks_per_expert + ci;
        unsigned prev;
        asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(prev) : "l"(cnt) : "memory");
        if (prev == units_in_chunk - 1u) {
          *cnt = 0u;
          uint32_t* flag = reinterpret_cast<uint32_t*>(signal_ptr_table[e]) + ci;
          ptx::fence_acq_rel_sys();
          if (signal_value != 0u) ptx::st_release_sys(flag, signal_value);
          else ptx::red_add_release_sys(flag, 1u);
        }
      }
    }
  }
}

// y[r, :] = float(q[r, :]) * scale[r]   (e4m3 rows back to 16 bit: received fp8 activations feed 16-bit weight-gradient GEMMs)
template <typename T>
__global__ void __launch_bounds__(256)
dequant_rows_kernel(const uint8_t* __restrict__ q, const float* __restrict__ scale, T* __restrict__ y, long long R, int K) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (long long r = static_cast<long long>(blockIdx.x) * 8 + warp; r < R; r += static_cast<long long>(gridDim.x) * 8) {
    const float sc = scale[r];
    const uint4* qrow = reinterpret_cast<const uint4*>(q + r * K);
    uint4* yrow = reinterpret_cast<uint4*>(y + r * K);
    for (int v = lane; v < K / 16; v += 32) {
      const uint4 u = ptx::ld_nc_v4(qrow + v);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
      float f[16];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const __nv_fp8x4_e4m3 p4 = *reinterpret_cast<const __nv_fp8x4_e4m3*>(&w[i]);
        const float4 t = static_cast<float4>(p4);
        f[4 * i] = t.x * sc; f[4 * i + 1] = t.y * sc; f[4 * i + 2] = t.z * sc; f[4 * i + 3] = t.w * sc;
      }
      ptx::st_na_v4(yrow + 2 * v, Vec<T>::pack(f));
      ptx::st_na_v4(yrow + 2 * v + 1, Vec<T>::pack(f + 8));
    }
  }
}

// ------------------------------------------------------------------------------------------------
// transposing e4m3 quantisation of a weight: x [G, R, K] (16 bit) -> qT [G, K, R] with one scale per OUTPUT row k
// (= per column of x).  Two passes over x and half-size writes, instead of a 16-bit transpose copy followed by a row
// quantisation: (1) column |max| with 16-byte loads, (2) 128 x 64 tiles through shared memory, coalesced on both sides.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
col_amax_kernel(const T* __restrict__ x, float* __restrict__ amax, int R, int K, int rows_per_split) {
  __shared__ float sm[16][16 * 8 + 1];
  const int cl = threadIdx.x & 15, rl = threadIdx.x >> 4;
  const int col = (blockIdx.x * 16 + cl) * 8;
  const int g = blockIdx.z;
  const int r_begin = blockIdx.y * rows_per_split;
  const int r_end = min(R, r_begin + rows_per_split);
  float a[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = 0.0f;
  if (col < K) {
    const T* base = x + static_cast<long long>(g) * R * K + col;
    for (int r = r_begin + rl; r < r_end; r += 16) {
      float f[8];
      Vec<T>::unpack(ptx::ld_nc_v4(base + static_cast<long long>(r) * K), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = fmaxf(a[i], fabsf(f[i]));
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) sm[rl][cl * 8 + i] = a[i];
  __syncthreads();
  for (int c = threadIdx.x; c < 128; c += 256) {
    float t = 0.0f;
#pragma unroll
    for (int q = 0; q < 16; ++q) t = fmaxf(t, sm[q][c]);
    const int n = blockIdx.x * 128 + c;
    if (n < K) atomicMax(reinterpret_cast<int*>(amax) + static_cast<long long>(g) * K + n, __float_as_int(t));   // t >= 0
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
quantize_transpose_kernel(const T* __restrict__ x, const float* __restrict__ amax, uint8_t* __restrict__ qT,
                          float* __restrict__ scale, int R, int K) {
  // tile: rows [r0, r0+128) x columns [k0, k0+64)
  __shared__ __align__(16) uint8_t sm_in[128 * 144];       // 16-bit tile, row stride 144 B
  __shared__ uint32_t sm_out[64 * 33];                     // e4m3 tile transposed: [k][r/4] words, row stride 33 words
  const int g = blockIdx.z;
  const int r0 = blockIdx.y * 128, k0 = blockIdx.x * 64;
  const T* xg = x + static_cast<long long>(g) * R * K;
  for (int i = threadIdx.x; i < 128 * 8; i += 256) {
    const int r = i >> 3, v = i & 7;
    const uint4 u = ptx::ld_nc_v4(xg + static_cast<long long>(r0 + r) * K + k0 + v * 8);
    *reinterpret_cast<uint4*>(sm_in + r * 144 + v * 16) = u;
  }
  const int k = threadIdx.x & 63;
  const float am = amax[static_cast<long long>(g) * K + k0 + k];
  const float sc = am > 0.0f ? fmaxf(am * (1.0f / 448.0f), FLT_MIN) : 1.0f;      // (FLT_MIN: see quantize_rows)
  const float inv = 1.0f / sc;
  if (blockIdx.y == 0 && threadIdx.x < 64) scale[static_cast<long long>(g) * K + k0 + k] = sc;
  __syncthreads();
  for (int r4 = threadIdx.x >> 6; r4 < 32; r4 += 4) {
    float f[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) f[j] = to_f<T>(*reinterpret_cast<const T*>(sm_in + (r4 * 4 + j) * 144 + k * 2)) * inv;
    const __nv_fp8x4_e4m3 p4(make_float4(f[0], f[1], f[2], f[3]));
    sm_out[k * 33 + r4] = *reinterpret_cast<const uint32_t*>(&p4);
  }
  __syncthreads();
  uint8_t* og = qT + static_cast<long long>(g) * K * R;
  for (int i = threadIdx.x; i < 64 * 32; i += 256) {
    const int kk = i >> 5, w = i & 31;
    *reinterpret_cast<uint32_t*>(og + static_cast<long long>(k0 + kk) * R + r0 + w * 4) = sm_out[kk * 33 + w];
  }
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

}  // namespace

size_t route_workspace_ints(int S, int E, int k) {
  const size_t nblocks = (static_cast<size_t>(S) + kRouteBlock - 1) / kRouteBlock;
  return (nblocks + 1) * static_cast<size_t>(k) * E;
}

cudaError_t route_locations(const int* idx, int* loc, int* counts, int* workspace, int S, int E, int k,
                            cudaStream_t stream) {
  if (S <= 0) return cudaMemsetAsync(counts, 0, sizeof(int) * E, stream);
  const int nblocks = (S + kRouteBlock - 1) / kRouteBlock;
  const size_t smem = sizeof(int) * E;
  route_hist_kernel<<<nblocks, kRouteBlock, smem, stream>>>(idx, workspace, S, E, k);
  route_scan_kernel<<<(E + 127) / 128, 128, 0, stream>>>(workspace, counts, nblocks, E, k);
  route_rank_kernel<<<nblocks, kRouteBlock, smem, stream>>>(idx, workspace, loc, nullptr, S, E, k, 0);
  return cudaGetLastError();
}

cudaError_t packed_layout(const int* idx, const int* loc, const int* counts, int* seg_off, int* block_expert,
                          int* block_rows, int* slot_src, int S, int E, int k, int R, cudaStream_t stream) {
  if (E <= 0 || R <= 0 || R % kPackBlock != 0) return cudaErrorInvalidValue;
  const int nblocks = R / kPackBlock;
  packed_layout_kernel<<<1, 1024, sizeof(int) * (E + 1), stream>>>(counts, seg_off, block_expert, block_rows, E, nblocks);
  cudaError_t e = cudaMemsetAsync(slot_src, 0xFF, sizeof(int) * static_cast<size_t>(R), stream);
  if (e != cudaSuccess) return e;
  const long long n = static_cast<long long>(S) * k;
  if (n > 0) packed_slot_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(idx, loc, seg_off, slot_src, S, E, k, R);
  return cudaGetLastError();
}

cudaError_t build_slot_map(const int* idx, const int* loc, int* slot_src, int S, int E, int k, int C,
                           cudaStream_t stream) {
  cudaError_t e = cudaMemsetAsync(slot_src, 0xFF, sizeof(int) * static_cast<size_t>(E) * C, stream);
  if (e != cudaSuccess) return e;
  const long long n = static_cast<long long>(S) * k;
  if (n > 0) slot_map_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(idx, loc, slot_src, S, E, k, C);
  return cudaGetLastError();
}

template <typename T>
static cudaError_t encode_rows_t(const void* x, const void* gates, const int* slot_src, void* out,
                                 const unsigned long long* dst_ptr_table, const unsigned long long* signal_ptr_table,
                                 unsigned int* chunk_counters, int signal_rows, int S, int E, int k, int C, int M,
                                 int rot_chunks, int signal_value, const int* valid_rows, cudaStream_t stream) {
  if (E <= 0 || C <= 0 || M <= 0) return cudaSuccess;
  const int unit_rows = 16;
  int chunk_rows = signal_rows > 0 ? signal_rows : unit_rows;
  chunk_rows = (chunk_rows + unit_rows - 1) / unit_rows * unit_rows;
  if (signal_ptr_table != nullptr && chunk_counters == nullptr) return cudaErrorInvalidValue;
  const long long units = static_cast<long long>(E) * ((C + unit_rows - 1) / unit_rows);
  // remote pushes share the SMs with the concurrently running expert GEMM: 2 blocks per SM are plenty for NVLink
  const long long cap = (dst_ptr_table != nullptr ? 2LL : 4LL) * num_sms();
  const int grid = static_cast<int>(units < cap ? units : cap);
  const int rot_units = rot_chunks * (chunk_rows / unit_rows);
  const bool vec = (M % Vec<T>::N == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) &&
                   (dst_ptr_table != nullptr || (reinterpret_cast<uintptr_t>(out) & 15) == 0);
#define TB_ENC_LAUNCH(VECv, THRv)                                                                                   \
  encode_rows_kernel<T, VECv, THRv><<<grid, THRv, 0, stream>>>(                                                      \
      static_cast<const T*>(x), static_cast<const float*>(gates), slot_src, static_cast<T*>(out), dst_ptr_table,     \
      signal_ptr_table, chunk_counters, chunk_rows, unit_rows, S, E, k, C, M, rot_units,                             \
      static_cast<uint32_t>(signal_value), valid_rows)
  if (dst_ptr_table != nullptr) {
    if (vec) TB_ENC_LAUNCH(true, kEncPushThreads); else TB_ENC_LAUNCH(false, kEncPushThreads);
  } else {
    if (vec) TB_ENC_LAUNCH(true, kEncThreads); else TB_ENC_LAUNCH(false, kEncThreads);
  }
#undef TB_ENC_LAUNCH
  return cudaGetLastError();
}

cudaError_t encode_rows(const void* x, const void* gates, const int* slot_src, void* out,
                        const unsigned long long* dst_ptr_table, const unsigned long long* signal_ptr_table,
                        unsigned int* chunk_counters, int signal_rows, int S, int E, int k, int C, int M, int elem_type,
                        int rot_chunks, int signal_value, const int* valid_rows, cudaStream_t stream) {
  switch (elem_type) {
    case ET_F32: return encode_rows_t<float>(x, gates, slot_src, out, dst_ptr_table, signal_ptr_table, chunk_counters, signal_rows, S, E, k, C, M, rot_chunks, signal_value, valid_rows, stream);
    case ET_F16: return encode_rows_t<__half>(x, gates, slot_src, out, dst_ptr_table, signal_ptr_table, chunk_counters, signal_rows, S, E, k, C, M, rot_chunks, signal_value, valid_rows, stream);
    case ET_BF16: return encode_rows_t<__nv_bfloat16>(x, gates, slot_src, out, dst_ptr_table, signal_ptr_table, chunk_counters, signal_rows, S, E, k, C, M, rot_chunks, signal_value, valid_rows, stream);
  }
  return cudaErrorInvalidValue;
}

cudaError_t encode_rows_fp8(const void* x, const void* gates, const int* slot_src, void* out, float* scale_out,
                            const unsigned long long* dst_ptr_table, const unsigned long long* scale_ptr_table,
                            const unsigned long long* signal_ptr_table, unsigned int* chunk_counters, int signal_rows, int S,
                            int E, int k, int C, int M, int elem_type, int rot_chunks, int signal_value, cudaStream_t stream) {
  if (E <= 0 || C <= 0 || M <= 0) return cudaSuccess;
  if (M % 16 || (reinterpret_cast<uintptr_t>(x) & 15) || (elem_type != ET_F16 && elem_type != ET_BF16)) return cudaErrorInvalidValue;
  if (signal_ptr_table != nullptr && chunk_counters == nullptr) return cudaErrorInvalidValue;
  const int unit_rows = 16;
  int chunk_rows = signal_rows > 0 ? signal_rows : unit_rows;
  chunk_rows = (chunk_rows + unit_rows - 1) / unit_rows * unit_rows;
  const long long units = static_cast<long long>(E) * ((C + unit_rows - 1) / unit_rows);
  const bool remote = dst_ptr_table != nullptr;
  const long long cap = (remote ? 2LL : 4LL) * num_sms();
  const int grid = static_cast<int>(units < cap ? units : cap);
  const int rot_units = rot_chunks * (chunk_rows / unit_rows);
#define TB_ENC8(Tv, THRv)                                                                                              \
  encode_rows_fp8_kernel<Tv, THRv><<<grid, THRv, 0, stream>>>(                                                          \
      static_cast<const Tv*>(x), static_cast<const float*>(gates), slot_src, static_cast<uint8_t*>(out), scale_out,    \
      dst_ptr_table, scale_ptr_table, signal_ptr_table, chunk_counters, chunk_rows, unit_rows, S, E, k, C, M, rot_units, \
      static_cast<uint32_t>(signal_value))
  if (elem_type == ET_BF16) { if (remote) TB_ENC8(__nv_bfloat16, kEncPushThreads); else TB_ENC8(__nv_bfloat16, kEncThreads); }
  else { if (remote) TB_ENC8(__half, kEncPushThreads); else TB_ENC8(__half, kEncThreads); }
#undef TB_ENC8
  return cudaGetLastError();
}

cudaError_t dequant_rows_e4m3(const void* q, const float* scale, void* y, long long R, int K, int elem_type,
                              cudaStream_t stream) {
  if (R <= 0 || K <= 0) return cudaSuccess;
  if (K % 16 || (reinterpret_cast<uintptr_t>(q) & 15) || (reinterpret_cast<uintptr_t>(y) & 15)) return cudaErrorInvalidValue;
  const long long want = (R + 7) / 8;
  const int grid = static_cast<int>(want < 16LL * num_sms() ? want : 16LL * num_sms());
  if (elem_type == ET_BF16)
    dequant_rows_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(static_cast<const uint8_t*>(q), scale, static_cast<__nv_bfloat16*>(y), R, K);
  else if (elem_type == ET_F16)
    dequant_rows_kernel<__half><<<grid, 256, 0, stream>>>(static_cast<const uint8_t*>(q), scale, static_cast<__half*>(y), R, K);
  else
    return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t quantize_transpose_e4m3(const void* x, void* qT, float* scale, float* amax_ws, int G, int R, int K, int elem_type,
                                    cudaStream_t stream) {
  if (G <= 0 || R <= 0 || K <= 0) return cudaSuccess;
  if (R % 128 || K % 64 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(qT) & 3)) return cudaErrorInvalidValue;
  cudaError_t e = cudaMemsetAsync(amax_ws, 0, sizeof(float) * static_cast<size_t>(G) * K, stream);
  if (e != cudaSuccess) return e;
  const int strips = (K + 127) / 128;
  int splits = 1;
  while (static_cast<long long>(strips) * G * splits < 2LL * num_sms() && R / (splits * 2) >= 64) splits *= 2;
  const int rps = (R + splits - 1) / splits;
  dim3 g1(strips, splits, G), g2(K / 64, R / 128, G);
  if (elem_type == ET_BF16) {
    col_amax_kernel<__nv_bfloat16><<<g1, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), amax_ws, R, K, rps);
    quantize_transpose_kernel<__nv_bfloat16><<<g2, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), amax_ws,
                                                                     static_cast<uint8_t*>(qT), scale, R, K);
  } else if (elem_type == ET_F16) {
    col_amax_kernel<__half><<<g1, 256, 0, stream>>>(static_cast<const __half*>(x), amax_ws, R, K, rps);
    quantize_transpose_kernel<__half><<<g2, 256, 0, stream>>>(static_cast<const __half*>(x), amax_ws, static_cast<uint8_t*>(qT),
                                                              scale, R, K);
  } else {
    return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <typename T>
static cudaError_t decode_rows_t(const void* buf, const void* gates, const int* idx, const int* loc, void* out,
                                 const uint32_t* wait_flags, uint32_t wait_target, int S, int E, int k, int C, int M,
                                 const int* seg_off, const void* base, const float* shared_logit, cudaStream_t stream) {
  if (S <= 0 || M <= 0) return cudaSuccess;
  if (k > kMaxK) return cudaErrorInvalidValue;
  if (base == nullptr && shared_logit != nullptr) return cudaErrorInvalidValue;
  const long long want = (static_cast<long long>(S) + 7) / 8;
  const int grid = static_cast<int>(want < 8LL * num_sms() ? want : 8LL * num_sms());
  const bool vec = (M % Vec<T>::N == 0) && aligned16(buf) && aligned16(out) && (base == nullptr || aligned16(base));
  // (expert-packed buffers and the shared-expert term run their own instantiations: the padded combine without shared
  // experts keeps its code)
#define TB_DEC(VECv, SEGv, SHv)                                                                                         \
  decode_rows_kernel<T, VECv, SEGv, SHv><<<grid, 256, 0, stream>>>(                                                     \
      static_cast<const T*>(buf), static_cast<const float*>(gates), idx, loc, static_cast<T*>(out), wait_flags,          \
      wait_target, S, E, k, C, M, seg_off, static_cast<const T*>(base), shared_logit)
#define TB_DEC_SEG(VECv, SHv) \
  if (seg_off != nullptr) TB_DEC(VECv, true, SHv); else TB_DEC(VECv, false, SHv)
  if (base != nullptr) { if (vec) TB_DEC_SEG(true, true); else TB_DEC_SEG(false, true); }
  else { if (vec) TB_DEC_SEG(true, false); else TB_DEC_SEG(false, false); }
#undef TB_DEC_SEG
#undef TB_DEC
  return cudaGetLastError();
}

cudaError_t decode_rows(const void* buf, const void* gates, const int* idx, const int* loc, void* out,
                        const uint32_t* wait_flags, uint32_t wait_target, int S, int E, int k, int C, int M,
                        int elem_type, cudaStream_t stream, const int* seg_off, const void* base,
                        const float* shared_logit) {
  switch (elem_type) {
    case ET_F32: return decode_rows_t<float>(buf, gates, idx, loc, out, wait_flags, wait_target, S, E, k, C, M, seg_off, base, shared_logit, stream);
    case ET_F16: return decode_rows_t<__half>(buf, gates, idx, loc, out, wait_flags, wait_target, S, E, k, C, M, seg_off, base, shared_logit, stream);
    case ET_BF16: return decode_rows_t<__nv_bfloat16>(buf, gates, idx, loc, out, wait_flags, wait_target, S, E, k, C, M, seg_off, base, shared_logit, stream);
  }
  return cudaErrorInvalidValue;
}

template <typename T>
static cudaError_t gate_grad_t(const void* a, const void* buf, const int* idx, const int* loc, void* dgate, int S, int E,
                               int k, int C, int M, const int* seg_off, const void* base, const float* shared_logit,
                               void* d_base, float* d_shared_logit, cudaStream_t stream) {
  if (S <= 0) return cudaSuccess;
  const bool sh = shared_logit != nullptr;
  if (sh && (base == nullptr || d_base == nullptr || d_shared_logit == nullptr)) return cudaErrorInvalidValue;
  if (k > 0 && (buf == nullptr || dgate == nullptr)) return cudaErrorInvalidValue;
  const long long want = (static_cast<long long>(S) + 7) / 8;
  const int grid = static_cast<int>(want < 8LL * num_sms() ? want : 8LL * num_sms());
  const bool vec = (M % Vec<T>::N == 0) && aligned16(a) && aligned16(buf) &&
                   (!sh || (aligned16(base) && aligned16(d_base)));
#define TB_GG(VECv, SEGv, SHv)                                                                                          \
  gate_grad_kernel<T, VECv, SEGv, SHv><<<grid, 256, 0, stream>>>(                                                       \
      static_cast<const T*>(a), static_cast<const T*>(buf), idx, loc, static_cast<float*>(dgate), S, E, k, C, M,         \
      seg_off, static_cast<const T*>(base), shared_logit, static_cast<T*>(d_base), d_shared_logit)
#define TB_GG_SEG(VECv, SHv) \
  if (seg_off != nullptr) TB_GG(VECv, true, SHv); else TB_GG(VECv, false, SHv)
  if (sh) { if (vec) TB_GG_SEG(true, true); else TB_GG_SEG(false, true); }
  else { if (vec) TB_GG_SEG(true, false); else TB_GG_SEG(false, false); }
#undef TB_GG_SEG
#undef TB_GG
  return cudaGetLastError();
}

cudaError_t gate_grad(const void* a, const void* buf, const int* idx, const int* loc, void* dgate, int S, int E, int k,
                      int C, int M, int elem_type, cudaStream_t stream, const int* seg_off, const void* base,
                      const float* shared_logit, void* d_base, float* d_shared_logit) {
  switch (elem_type) {
    case ET_F32: return gate_grad_t<float>(a, buf, idx, loc, dgate, S, E, k, C, M, seg_off, base, shared_logit, d_base, d_shared_logit, stream);
    case ET_F16: return gate_grad_t<__half>(a, buf, idx, loc, dgate, S, E, k, C, M, seg_off, base, shared_logit, d_base, d_shared_logit, stream);
    case ET_BF16: return gate_grad_t<__nv_bfloat16>(a, buf, idx, loc, dgate, S, E, k, C, M, seg_off, base, shared_logit, d_base, d_shared_logit, stream);
  }
  return cudaErrorInvalidValue;
}

cudaError_t quantize_rows_e4m3(const void* x, void* q, float* scale, long long R, int K, int elem_type,
                               cudaStream_t stream) {
  if (R <= 0 || K <= 0) return cudaSuccess;
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(q) & 7)) return cudaErrorInvalidValue;
  const long long want = (R + 7) / 8;
  const int grid = static_cast<int>(want < 16LL * num_sms() ? want : 16LL * num_sms());
  switch (elem_type) {
    case ET_F32:
      if (K % 4) return cudaErrorInvalidValue;
      quantize_rows_kernel<float><<<grid, 256, 0, stream>>>(static_cast<const float*>(x), static_cast<uint8_t*>(q), scale, R, K);
      break;
    case ET_F16:
      if (K % 8) return cudaErrorInvalidValue;
      quantize_rows_kernel<__half><<<grid, 256, 0, stream>>>(static_cast<const __half*>(x), static_cast<uint8_t*>(q), scale, R, K);
      break;
    case ET_BF16:
      if (K % 8) return cudaErrorInvalidValue;
      quantize_rows_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), static_cast<uint8_t*>(q), scale, R, K);
      break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

// run-time spin-wait limit of this translation unit's kernels (ptx.cuh)
cudaError_t set_spin_timeout_moe(unsigned long long ns) {
  return cudaMemcpyToSymbol(tb_spin_timeout_ns, &ns, sizeof(ns));
}

}  // namespace tb
