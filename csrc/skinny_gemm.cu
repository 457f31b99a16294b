// Skinny grouped GEMM for dropless / decoder-inference routing: a handful of tokens per expert, many experts.
//
// The reference's "Megablocks" path (tutel/custom/custom_kernel.cpp:874-889) copies the per-expert counts to the host,
// synchronises, and loops over experts with one cuBLAS call each.  With <= a few rows per expert the problem is purely
// bound by streaming the weights of the ACTIVE experts once; this kernel does exactly that, driven by the device-side
// counts (experts with zero tokens cost nothing), in fp32 / fp16 / bf16 with fp32 accumulation:
//
//      y[g, r, :] = act( x[g, r, :] @ W[g] (+ bias[g]) )     for r < counts[g]
//
// W is [G, N, K] ("nk", one warp per output column, lanes stride K) or [G, K, N] ("kn", lanes stride N).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include "moe_kernels.h"

namespace tb {
namespace {

constexpr int kRows = 8;       // rows (tokens) handled per pass
constexpr int kKChunk = 1024;  // K elements of x staged in smem per pass

template <typename T> __device__ __forceinline__ float ldf(const T* p);
template <> __device__ __forceinline__ float ldf<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ldf<__half>(const __half* p) { return __half2float(*p); }
template <> __device__ __forceinline__ float ldf<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <typename T> __device__ __forceinline__ void stf(T* p, float v);
template <> __device__ __forceinline__ void stf<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void stf<__half>(__half* p, float v) { *p = __float2half_rn(v); }
template <> __device__ __forceinline__ void stf<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

// grid: (ceil(N / cols_per_block), G); block: 256 threads
template <typename T, bool KN>
__global__ void __launch_bounds__(256)
skinny_kernel(const T* __restrict__ x, const T* __restrict__ w, const T* __restrict__ bias, T* __restrict__ y,
              const int* __restrict__ counts, int rows_cap, int N, int K, int relu) {
  __shared__ float xs[kRows][kKChunk];
  const int g = blockIdx.y;
  int count = counts != nullptr ? min(counts[g], rows_cap) : rows_cap;
  if (count <= 0) return;
  const T* xg = x + static_cast<long long>(g) * rows_cap * K;
  const T* wg = w + static_cast<long long>(g) * N * K;
  T* yg = y + static_cast<long long>(g) * rows_cap * N;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  for (int r0 = 0; r0 < count; r0 += kRows) {
    const int nr = min(kRows, count - r0);
    if constexpr (KN) {
      // one output column per thread; W rows (fixed k) are read coalesced across the block
      const int n = blockIdx.x * 256 + threadIdx.x;
      float acc[kRows];
#pragma unroll
      for (int r = 0; r < kRows; ++r) acc[r] = 0.0f;
      for (int k0 = 0; k0 < K; k0 += kKChunk) {
        const int kc = min(kKChunk, K - k0);
        __syncthreads();
        for (int i = threadIdx.x; i < nr * kc; i += 256) xs[i / kc][i % kc] = ldf<T>(xg + static_cast<long long>(r0 + i / kc) * K + k0 + i % kc);
        __syncthreads();
        if (n < N) {
          for (int k = 0; k < kc; ++k) {
            const float wv = ldf<T>(wg + static_cast<long long>(k0 + k) * N + n);
#pragma unroll
            for (int r = 0; r < kRows; ++r) acc[r] = fmaf(xs[r][k], wv, acc[r]);
          }
        }
      }
      if (n < N) {
        const float b = bias != nullptr ? ldf<T>(bias + static_cast<long long>(g) * N + n) : 0.0f;
        for (int r = 0; r < nr; ++r) {
          float v = acc[r] + b;
          if (relu) v = fmaxf(v, 0.0f);
          stf<T>(yg + static_cast<long long>(r0 + r) * N + n, v);
        }
      }
    } else {
      // one output column per warp (8 per block-iteration); lanes stride K, warp-reduce at the end
      for (int nb = blockIdx.x * 64; nb < min(N, blockIdx.x * 64 + 64); nb += 8) {
        const int n = nb + warp;
        float acc[kRows];
#pragma unroll
        for (int r = 0; r < kRows; ++r) acc[r] = 0.0f;
        for (int k0 = 0; k0 < K; k0 += kKChunk) {
          const int kc = min(kKChunk, K - k0);
          __syncthreads();
          for (int i = threadIdx.x; i < nr * kc; i += 256) xs[i / kc][i % kc] = ldf<T>(xg + static_cast<long long>(r0 + i / kc) * K + k0 + i % kc);
          __syncthreads();
          if (n < N) {
            const T* wrow = wg + static_cast<long long>(n) * K + k0;
            for (int k = lane; k < kc; k += 32) {
              const float wv = ldf<T>(wrow + k);
#pragma unroll
              for (int r = 0; r < kRows; ++r) acc[r] = fmaf(xs[r][k], wv, acc[r]);
            }
          }
        }
        if (n < N) {
#pragma unroll
          for (int r = 0; r < kRows; ++r)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
          if (lane == 0) {
            const float b = bias != nullptr ? ldf<T>(bias + static_cast<long long>(g) * N + n) : 0.0f;
            for (int r = 0; r < nr; ++r) {
              float v = acc[r] + b;
              if (relu) v = fmaxf(v, 0.0f);
              stf<T>(yg + static_cast<long long>(r0 + r) * N + n, v);
            }
          }
        }
      }
    }
  }
}

template <typename T>
cudaError_t launch(const void* x, const void* w, const void* bias, void* y, const int* counts, int G, int rows_cap, int N,
                   int K, bool kn, bool relu, cudaStream_t stream) {
  if (G <= 0 || rows_cap <= 0 || N <= 0 || K <= 0) return cudaSuccess;
  if (kn) {
    dim3 grid((N + 255) / 256, G);
    skinny_kernel<T, true><<<grid, 256, 0, stream>>>(static_cast<const T*>(x), static_cast<const T*>(w),
                                                     static_cast<const T*>(bias), static_cast<T*>(y), counts, rows_cap, N,
                                                     K, relu ? 1 : 0);
  } else {
    dim3 grid((N + 63) / 64, G);
    skinny_kernel<T, false><<<grid, 256, 0, stream>>>(static_cast<const T*>(x), static_cast<const T*>(w),
                                                      static_cast<const T*>(bias), static_cast<T*>(y), counts, rows_cap, N,
                                                      K, relu ? 1 : 0);
  }
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Whole expert FFN for a few rows per expert in ONE launch:  y[g] (+)= act(x[g] @ W1[g]^T + b1[g]) @ W2[g] (+ b2[g])
// ------------------------------------------------------------------------------------------------
// Block (g, s) owns hidden units [s*kHS, s*kHS + kHS) of expert g: it streams the kHS rows of W1[g] ([H, K], K
// contiguous) to form its slice of the hidden activations in shared memory, then streams the matching kHS rows of W2[g]
// ([H, N], N contiguous) and adds its partial outputs to y with fp32 atomics (y is zero-initialised, block s == 0 adds the
// bias).  Every byte of an ACTIVE expert's weights is read exactly once with 16-byte loads and several loads in flight
// per lane; experts without tokens cost one block exit.  No host synchronisation: counts are read on the device.
constexpr int kHS = 64;         // hidden units per block
constexpr int kFfnRows = 4;     // rows per pass (more rows re-stream the slice); keeps the kernel at <= 128 registers, 2 blocks / SM
constexpr size_t kFfnSmemLimit = 200 * 1024;   // dynamic shared memory (staged x rows + slice buffers) per block

template <typename T> struct WVec;
template <> struct WVec<float> {
  static constexpr int N = 4;
  static __device__ __forceinline__ void load(const float* p, float* f) {
    const float4 v = __ldcs(reinterpret_cast<const float4*>(p));     // streaming: every weight byte is touched once
    f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
  }
};
template <> struct WVec<__half> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void load(const __half* p, float* f) {
    const uint4 u = __ldcs(reinterpret_cast<const uint4*>(p));
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
      f[2 * i] = t.x; f[2 * i + 1] = t.y;
    }
  }
};
template <> struct WVec<__nv_bfloat16> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void load(const __nv_bfloat16* p, float* f) {
    const uint4 u = __ldcs(reinterpret_cast<const uint4*>(p));
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
    }
  }
};

// act: 0 none, 1 relu, 2 gelu (erf), 3 silu
__device__ __forceinline__ float ffn_act(float v, int act) {
  if (act == 1) return fmaxf(v, 0.0f);
  if (act == 2) return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));
  if (act == 3) return v / (1.0f + __expf(-v));
  return v;
}

// Stage rows [r0, r0 + nr) of x[g] ([rows, K], fp32 in shared memory) for one pass.  Passes of 3-4 rows run the
// kFfnRows specialisation, so its missing rows are zeroed (they then contribute zeros and are never stored).
template <typename T>
__device__ __forceinline__ void stage_rows(float* __restrict__ xs, const T* __restrict__ xrow0, int nr, int K) {
  constexpr int V = WVec<T>::N;
  __syncthreads();
  for (int i = threadIdx.x * V; i < nr * K; i += 256 * V) {
    float f[V];
    WVec<T>::load(xrow0 + i, f);
#pragma unroll
    for (int q = 0; q < V; ++q) xs[i + q] = f[q];
  }
  if (nr > 2)
    for (int i = threadIdx.x + nr * K; i < kFfnRows * K; i += 256) xs[i] = 0.0f;
  __syncthreads();
}

// Second layer of a pass: yrow0[r, :] += hsm[r, :hs] @ w2g[:hs, :] (+ b2g) for r < nr, with fp32 atomics.  w2g points at
// the block's hs rows of the [H, N] weight (N contiguous); each thread owns V output columns per pass and walks the rows.
template <typename T, int ROWS>
__device__ __forceinline__ void ffn_layer2(const float* __restrict__ hsm, const T* __restrict__ w2g, const T* __restrict__ b2g,
                                           float* __restrict__ yrow0, int nr, int hs, int N, bool add_bias) {
  constexpr int V = WVec<T>::N;
  for (int n = threadIdx.x * V; n < N; n += 256 * V) {
    float acc[ROWS][V];
#pragma unroll
    for (int r = 0; r < ROWS; ++r)
#pragma unroll
      for (int q = 0; q < V; ++q) acc[r][q] = 0.0f;
    for (int j = 0; j < hs; j += 8) {
      float wv[8][V];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        if (j + u < hs) WVec<T>::load(w2g + static_cast<long long>(j + u) * N + n, wv[u]);
        else {
#pragma unroll
          for (int q = 0; q < V; ++q) wv[u][q] = 0.0f;
        }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        if (j + u < hs) {
#pragma unroll
          for (int r = 0; r < ROWS; ++r) {
            const float hv = hsm[r * kHS + j + u];
#pragma unroll
            for (int q = 0; q < V; ++q) acc[r][q] = fmaf(hv, wv[u][q], acc[r][q]);
          }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      if (r < nr) {
#pragma unroll
        for (int q = 0; q < V; ++q) {
          float v = acc[r][q];
          if (add_bias) v += ldf<T>(b2g + n + q);
          atomicAdd(yrow0 + static_cast<long long>(r) * N + n + q, v);
        }
      }
    }
  }
}

// One pass over this block's weight slices for ROWS (compile-time) rows: the inner products cost ROWS shared-memory reads
// and 4*ROWS FMAs per 16 bytes of weights, so the common 1-2 rows per expert stay far below the issue limits.
template <typename T, int ROWS>
__device__ __forceinline__ void ffn_pass(const float* __restrict__ xs, float* __restrict__ hsm, const T* __restrict__ w1g,
                                         const T* __restrict__ b1g, const T* __restrict__ w2g, const T* __restrict__ b2g,
                                         float* __restrict__ yrow0, int nr, int K, int hs, int N, int act, bool add_bias) {
  constexpr int V = WVec<T>::N;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // ---- layer 1: one hidden unit per warp and pass, lanes stride K with 16-byte loads ----
  for (int j = warp; j < hs; j += 8) {
    const T* wrow = w1g + static_cast<long long>(j) * K;
    float acc[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) acc[r] = 0.0f;
    for (int k = lane * V; k < K; k += 32 * V * 4) {
      float wv[4][V];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int kk = k + u * 32 * V;
        if (kk < K) WVec<T>::load(wrow + kk, wv[u]);
        else {
#pragma unroll
          for (int q = 0; q < V; ++q) wv[u][q] = 0.0f;
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int kk = k + u * 32 * V;
        if (kk < K) {
#pragma unroll
          for (int r = 0; r < ROWS; ++r) {
            const float* xr = xs + r * K + kk;
#pragma unroll
            for (int q = 0; q < V; ++q) acc[r] = fmaf(xr[q], wv[u][q], acc[r]);
          }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
    if (lane == 0) {
      const float b = b1g != nullptr ? ldf<T>(b1g + j) : 0.0f;
#pragma unroll
      for (int r = 0; r < ROWS; ++r) hsm[r * kHS + j] = ffn_act(acc[r] + b, act);
    }
  }
  __syncthreads();
  ffn_layer2<T, ROWS>(hsm, w2g, b2g, yrow0, nr, hs, N, add_bias);
}

template <typename T>
__global__ void __launch_bounds__(256, 2)
skinny_ffn_kernel(const T* __restrict__ x, const T* __restrict__ w1, const T* __restrict__ b1, const T* __restrict__ w2,
                  const T* __restrict__ b2, float* __restrict__ y, const int* __restrict__ counts, int rows_cap, int K,
                  int H, int N, int act) {
  extern __shared__ float sm[];                 // x rows [kFfnRows][K] | hidden slice [kFfnRows][kHS]
  const int g = blockIdx.y;
  const int count = counts != nullptr ? min(counts[g], rows_cap) : rows_cap;
  if (count <= 0) return;
  const int h0 = blockIdx.x * kHS;
  const int hs = min(kHS, H - h0);
  float* xs = sm;
  float* hsm = sm + kFfnRows * K;
  const T* xg = x + static_cast<long long>(g) * rows_cap * K;
  const T* w1g = w1 + (static_cast<long long>(g) * H + h0) * K;
  const T* w2g = w2 + (static_cast<long long>(g) * H + h0) * N;
  const T* b1g = b1 != nullptr ? b1 + static_cast<long long>(g) * H + h0 : nullptr;
  const T* b2g = b2 != nullptr ? b2 + static_cast<long long>(g) * N : nullptr;
  float* yg = y + static_cast<long long>(g) * rows_cap * N;
  const bool add_bias = blockIdx.x == 0 && b2 != nullptr;

  for (int r0 = 0; r0 < count; r0 += kFfnRows) {
    const int nr = min(kFfnRows, count - r0);
    stage_rows<T>(xs, xg + static_cast<long long>(r0) * K, nr, K);
    float* yrow0 = yg + static_cast<long long>(r0) * N;
    if (nr == 1) ffn_pass<T, 1>(xs, hsm, w1g, b1g, w2g, b2g, yrow0, nr, K, hs, N, act, add_bias);
    else if (nr == 2) ffn_pass<T, 2>(xs, hsm, w1g, b1g, w2g, b2g, yrow0, nr, K, hs, N, act, add_bias);
    else ffn_pass<T, kFfnRows>(xs, hsm, w1g, b1g, w2g, b2g, yrow0, nr, K, hs, N, act, add_bias);
  }
}

template <typename T>
cudaError_t launch_ffn(const void* x, const void* w1, const void* b1, const void* w2, const void* b2, float* y,
                       const int* counts, int G, int rows_cap, int K, int H, int N, int act, cudaStream_t stream) {
  constexpr int V = WVec<T>::N;
  if (K % V || N % V) return cudaErrorInvalidValue;
  const size_t smem = sizeof(float) * (static_cast<size_t>(kFfnRows) * K + kFfnRows * kHS);
  if (smem > kFfnSmemLimit) return cudaErrorInvalidValue;
  auto* kern = skinny_ffn_kernel<T>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
  }
  dim3 grid((H + kHS - 1) / kHS, G);
  kern<<<grid, 256, smem, stream>>>(static_cast<const T*>(x), static_cast<const T*>(w1), static_cast<const T*>(b1),
                                    static_cast<const T*>(w2), static_cast<const T*>(b2), y, counts, rows_cap, K, H, N, act);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// SwiGLU expert for a few rows per expert in ONE launch:  y[g] += (act(x[g] @ W1[g]) * (x[g] @ W2[g])) @ W3[g]
// ------------------------------------------------------------------------------------------------
// W1, W2 are [G, M, H] and W3 [G, H, N], all with the last dim contiguous (LlamaFFNNetwork's parameters).  Block (g, s)
// owns hidden units [s*kHS, s*kHS + kHS): in layer 1 it reads the kHS-wide column strip of every one of the M rows of
// both W1 and W2 (64 contiguous elements: 256 bytes in fp32, 128 bytes in 16 bit, so every segment is whole 128-byte
// lines).  Warps 0-3 stream W1 and warps 4-7 stream W2 over the same staged rows of x: kHS / V lanes cover one row
// segment with 16-byte loads, the other lanes and warps stride M.  The gate and up partial sums are reduced across the
// lanes of a warp with shuffles and across the four warps of each matrix in shared memory, where they become
// act(gate) * up.  Layer 2 is the FFN kernel's W2 pass over the slice's kHS rows of W3.
constexpr int kGluWarps = 8;                    // 4 warps per layer-1 matrix

template <typename T, int ROWS>
__device__ __forceinline__ void glu_pass(const float* __restrict__ xs, float* __restrict__ part, float* __restrict__ hsm,
                                         const T* __restrict__ w1g, const T* __restrict__ w2g, const T* __restrict__ w3g,
                                         float* __restrict__ yrow0, int nr, int M, int H, int hs, int N, int act) {
  constexpr int V = WVec<T>::N;
  constexpr int LPR = kHS / V;                  // lanes per row segment: 8 (16 bit) or 16 (fp32)
  constexpr int KLW = 32 / LPR;                 // rows of one matrix per warp and load
  constexpr int KL = 4 * KLW;                   // rows of one matrix per load over its four warps
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = (lane % LPR) * V;               // first hidden unit of this lane inside the slice
  const int kl = (warp & 3) * KLW + lane / LPR;
  const T* wg = (warp < 4 ? w1g : w2g) + c;
  float acc[ROWS][V];
#pragma unroll
  for (int r = 0; r < ROWS; ++r)
#pragma unroll
    for (int q = 0; q < V; ++q) acc[r][q] = 0.0f;
  if (c < hs) {
    for (int k = kl; k < M; k += KL * 4) {
      float wv[4][V];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int kk = k + u * KL;
        if (kk < M) WVec<T>::load(wg + static_cast<long long>(kk) * H, wv[u]);
        else {
#pragma unroll
          for (int q = 0; q < V; ++q) wv[u][q] = 0.0f;
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int kk = k + u * KL;
        if (kk < M) {
#pragma unroll
          for (int r = 0; r < ROWS; ++r) {
            const float xv = xs[r * M + kk];
#pragma unroll
            for (int q = 0; q < V; ++q) acc[r][q] = fmaf(xv, wv[u][q], acc[r][q]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < ROWS; ++r)
#pragma unroll
    for (int q = 0; q < V; ++q)
#pragma unroll
      for (int o = LPR; o < 32; o <<= 1) acc[r][q] += __shfl_xor_sync(0xffffffffu, acc[r][q], o);
  if (lane < LPR) {
#pragma unroll
    for (int r = 0; r < ROWS; ++r)
#pragma unroll
      for (int q = 0; q < V; ++q) part[(warp * kFfnRows + r) * kHS + c + q] = acc[r][q];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < ROWS * kHS; i += 256) {
    float gs = 0.0f, us = 0.0f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      gs += part[w * kFfnRows * kHS + i];
      us += part[(w + 4) * kFfnRows * kHS + i];
    }
    hsm[i] = ffn_act(gs, act) * us;
  }
  __syncthreads();
  ffn_layer2<T, ROWS>(hsm, w3g, nullptr, yrow0, nr, hs, N, false);
}

template <typename T>
__global__ void __launch_bounds__(256, 2)
skinny_glu_ffn_kernel(const T* __restrict__ x, const T* __restrict__ w1, const T* __restrict__ w2, const T* __restrict__ w3,
                      float* __restrict__ y, const int* __restrict__ counts, int rows_cap, int M, int H, int N, int act) {
  extern __shared__ float sm[];                 // x rows [kFfnRows][M] | hidden slice [kFfnRows][kHS] | partial sums
  const int g = blockIdx.y;
  const int count = counts != nullptr ? min(counts[g], rows_cap) : rows_cap;
  if (count <= 0) return;
  const int h0 = blockIdx.x * kHS;
  const int hs = min(kHS, H - h0);
  float* xs = sm;
  float* hsm = xs + kFfnRows * M;
  float* part = hsm + kFfnRows * kHS;           // [kGluWarps][kFfnRows][kHS]
  const T* xg = x + static_cast<long long>(g) * rows_cap * M;
  const T* w1g = w1 + static_cast<long long>(g) * M * H + h0;
  const T* w2g = w2 + static_cast<long long>(g) * M * H + h0;
  const T* w3g = w3 + (static_cast<long long>(g) * H + h0) * N;
  float* yg = y + static_cast<long long>(g) * rows_cap * N;

  for (int r0 = 0; r0 < count; r0 += kFfnRows) {
    const int nr = min(kFfnRows, count - r0);
    stage_rows<T>(xs, xg + static_cast<long long>(r0) * M, nr, M);
    float* yrow0 = yg + static_cast<long long>(r0) * N;
    if (nr == 1) glu_pass<T, 1>(xs, part, hsm, w1g, w2g, w3g, yrow0, nr, M, H, hs, N, act);
    else if (nr == 2) glu_pass<T, 2>(xs, part, hsm, w1g, w2g, w3g, yrow0, nr, M, H, hs, N, act);
    else glu_pass<T, kFfnRows>(xs, part, hsm, w1g, w2g, w3g, yrow0, nr, M, H, hs, N, act);
  }
}

template <typename T>
cudaError_t launch_glu_ffn(const void* x, const void* w1, const void* w2, const void* w3, float* y, const int* counts, int G,
                           int rows_cap, int M, int H, int N, int act, cudaStream_t stream) {
  constexpr int V = WVec<T>::N;
  if (M % V || H % V || N % V) return cudaErrorInvalidValue;
  const size_t smem = sizeof(float) * (static_cast<size_t>(kFfnRows) * M + (1 + kGluWarps) * kFfnRows * kHS);
  if (smem > kFfnSmemLimit) return cudaErrorInvalidValue;
  auto* kern = skinny_glu_ffn_kernel<T>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
  }
  dim3 grid((H + kHS - 1) / kHS, G);
  kern<<<grid, 256, smem, stream>>>(static_cast<const T*>(x), static_cast<const T*>(w1), static_cast<const T*>(w2),
                                    static_cast<const T*>(w3), y, counts, rows_cap, M, H, N, act);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Weight-only fp8: the two expert kernels above with e4m3 weights and one fp32 scale per weight row (W8A16)
// ------------------------------------------------------------------------------------------------
// The operands are the cached copies the e4m3 wgmma forward reads (ops/gemm.py: fp8_weight), so prefill and decode share
// one e4m3 copy per weight.  Both kernels have the same two layers:
//   layer 1: rows of an [H, K] matrix (K contiguous), one hidden unit per warp, lanes stride K with 16-byte loads;
//            h = act(s1[j] * dot + b1[j])  (FFN)  or  act(s1[j] * dot1) * (s2[j] * dot2)  (SwiGLU, both rows in one loop);
//   layer 2: rows of an [N, H] matrix (H contiguous): the block's kHS8-unit slice of output n's row is one 128-byte line,
//            spread over 8 lanes and reduced with three shuffles; y[r, n] += s[n] * partial (+ bias[n]) with fp32 atomics.
// x stays 16 bit on the way in (staged as fp32), accumulation is fp32 and each scale multiplies a finished dot product.
constexpr int kHS8 = 128;       // hidden units per block: 128 e4m3 bytes per layer-2 row, the bytes of the 16-bit kHS slice

// 16 e4m3 values (one 16-byte load) -> fp32 with the hardware unpack (F2FP.F16.E4M3.UNPACK, then f16 -> f32); e4m3 is
// exact in f16.  Byte i of the load is element i.
__device__ __forceinline__ void e4m3x16(const uint4 u, float* f) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w[i] >> (16 * p)), __NV_E4M3);
      const float2 t = __half22float2(__half2(h));
      f[4 * i + 2 * p] = t.x;
      f[4 * i + 2 * p + 1] = t.y;
    }
  }
}

// Index of element k of a staged row of length K (K % 16 == 0) in the "chunk-split" layout: the four float4s of 16-element
// chunk c lie K/16 float4s apart, so a lane that owns the 16 weights of chunk c reads its four float4s of x at
// consecutive addresses across consecutive lanes (no bank conflicts), instead of 64 contiguous bytes per lane.
__device__ __forceinline__ int split_index(int k, int K) { return ((((k & 15) >> 2) * (K >> 4) + (k >> 4)) << 2) + (k & 3); }

template <typename T>
__device__ __forceinline__ void stage_rows_split(float* __restrict__ xs, const T* __restrict__ xrow0, int nr, int K) {
  __syncthreads();
  for (int i = threadIdx.x * 8; i < nr * K; i += 256 * 8) {
    float f[8];
    WVec<T>::load(xrow0 + i, f);          // 8 elements of one row (K % 16 == 0): two float4s of one chunk
    const int r = i / K, k = i - r * K;
    float* row = xs + r * K;
    *reinterpret_cast<float4*>(row + split_index(k, K)) = make_float4(f[0], f[1], f[2], f[3]);
    *reinterpret_cast<float4*>(row + split_index(k + 4, K)) = make_float4(f[4], f[5], f[6], f[7]);
  }
  if (nr > 2)
    for (int i = threadIdx.x + nr * K; i < kFfnRows * K; i += 256) xs[i] = 0.0f;
  __syncthreads();
}

// Warp-wide dot products of ROWS staged rows of x with row q[0] (and q[1] when NMAT == 2) of K e4m3 weights; every lane
// gets the full sums.  Four 16-byte loads per matrix in flight per lane; each weight is converted once for all rows.
template <int ROWS, int NMAT>
__device__ __forceinline__ void fp8_row_dots(const float* __restrict__ xs, const uint8_t* const (&q)[NMAT], int K,
                                             float (&acc)[NMAT][ROWS]) {
  const int lane = threadIdx.x & 31;
  const int K16 = K >> 4;
#pragma unroll
  for (int m = 0; m < NMAT; ++m)
#pragma unroll
    for (int r = 0; r < ROWS; ++r) acc[m][r] = 0.0f;
  for (int c = lane; c < K16; c += 32 * 4) {
    uint4 raw[4][NMAT];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int m = 0; m < NMAT; ++m)
        raw[u][m] = c + 32 * u < K16 ? __ldcs(reinterpret_cast<const uint4*>(q[m]) + c + 32 * u) : make_uint4(0, 0, 0, 0);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int cc = c + 32 * u;
      if (cc < K16) {
        float wv[NMAT][16];
#pragma unroll
        for (int m = 0; m < NMAT; ++m) e4m3x16(raw[u][m], wv[m]);
#pragma unroll
        for (int r = 0; r < ROWS; ++r) {
          const float4* xr = reinterpret_cast<const float4*>(xs + r * K) + cc;
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            const float4 xv = xr[p * K16];
#pragma unroll
            for (int m = 0; m < NMAT; ++m) {
              acc[m][r] = fmaf(xv.x, wv[m][4 * p], acc[m][r]);
              acc[m][r] = fmaf(xv.y, wv[m][4 * p + 1], acc[m][r]);
              acc[m][r] = fmaf(xv.z, wv[m][4 * p + 2], acc[m][r]);
              acc[m][r] = fmaf(xv.w, wv[m][4 * p + 3], acc[m][r]);
            }
          }
        }
      }
    }
  }
#pragma unroll
  for (int m = 0; m < NMAT; ++m)
#pragma unroll
    for (int r = 0; r < ROWS; ++r)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[m][r] += __shfl_xor_sync(0xffffffffu, acc[m][r], o);
}

// Layer 2 of a pass (shared by both kernels): yrow0[r, n] += s[n] * sum_{j < hs} h[r, j] * q[n, j] (+ bias[n]) for r < nr.
// q points at the slice's first column of the [N, H] matrix; hsm holds h [ROWS][kHS8] in the chunk-split layout.  Lane
// (sub, c) of a warp takes hidden units [16c, 16c + 16) of output sub (4 outputs per warp and load, each a whole line); its
// 16 h values per row stay in registers for the whole pass.  After the 8-lane reduction lane c adds row c.
// BLOCK: q is block-scaled (128 x 128) and the slice is one 128-deep K block of it, so output n's reduced partial takes the
// single scale s[(n / 128) * s_ld] (s points at the slice's block column, s_ld = H / 128); otherwise the row scale s[n].
template <typename T, int ROWS, bool BLOCK = false>
__device__ __forceinline__ void fp8_layer2(const float* __restrict__ hsm, const uint8_t* __restrict__ q,
                                           const float* __restrict__ s, const T* __restrict__ bias,
                                           float* __restrict__ yrow0, int nr, int hs, int H, int N, int s_ld = 0) {
  constexpr int U = ROWS <= 2 ? 8 : 4;          // loads in flight per lane
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = lane & 7, sub = lane >> 3;
  const bool live = c * 16 < hs;                // hs % 16 == 0: a chunk is wholly inside the slice or wholly outside
  float hv[ROWS][16];
#pragma unroll
  for (int r = 0; r < ROWS; ++r)
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const float4 t = live ? reinterpret_cast<const float4*>(hsm + r * kHS8)[p * (kHS8 / 16) + c] : make_float4(0.f, 0.f, 0.f, 0.f);
      hv[r][4 * p] = t.x; hv[r][4 * p + 1] = t.y; hv[r][4 * p + 2] = t.z; hv[r][4 * p + 3] = t.w;
    }
  for (int nb = warp * 4; nb < N; nb += 32 * U) {   // warp-uniform bound: all lanes reach the shuffles
    uint4 raw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int n = nb + sub + 32 * u;
      raw[u] = live && n < N ? __ldcs(reinterpret_cast<const uint4*>(q + static_cast<long long>(n) * H) + c) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float wv[16];
      e4m3x16(raw[u], wv);
      float acc[ROWS];
#pragma unroll
      for (int r = 0; r < ROWS; ++r) {
        acc[r] = 0.0f;
#pragma unroll
        for (int e = 0; e < 16; ++e) acc[r] = fmaf(hv[r][e], wv[e], acc[r]);
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
      }
      const int n = nb + sub + 32 * u;
      if (c < nr && n < N) {
        float v = acc[0];
#pragma unroll
        for (int r = 1; r < ROWS; ++r) if (c == r) v = acc[r];
        v *= s[BLOCK ? (n >> 7) * s_ld : n];
        if (bias != nullptr) v += ldf<T>(bias + n);
        atomicAdd(yrow0 + static_cast<long long>(c) * N + n, v);
      }
    }
  }
}

template <typename T, int ROWS>
__device__ __forceinline__ void ffn_fp8_pass(const float* __restrict__ xs, float* __restrict__ hsm, const uint8_t* __restrict__ q1g,
                                             const float* __restrict__ s1g, const T* __restrict__ b1g,
                                             const uint8_t* __restrict__ q2g, const float* __restrict__ s2g,
                                             const T* __restrict__ b2g, float* __restrict__ yrow0, int nr, int K, int hs,
                                             int H, int N, int act) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = warp; j < hs; j += 8) {
    const uint8_t* const rows[1] = {q1g + static_cast<long long>(j) * K};
    float acc[1][ROWS];
    fp8_row_dots<ROWS, 1>(xs, rows, K, acc);
    if (lane < ROWS) {
      float v = acc[0][0];
#pragma unroll
      for (int r = 1; r < ROWS; ++r) if (lane == r) v = acc[0][r];
      const float b = b1g != nullptr ? ldf<T>(b1g + j) : 0.0f;
      hsm[lane * kHS8 + split_index(j, kHS8)] = ffn_act(fmaf(s1g[j], v, b), act);
    }
  }
  __syncthreads();
  fp8_layer2<T, ROWS>(hsm, q2g, s2g, b2g, yrow0, nr, hs, H, N);
}

template <typename T>
__global__ void __launch_bounds__(256, 2)
skinny_ffn_fp8_kernel(const T* __restrict__ x, const uint8_t* __restrict__ q1, const float* __restrict__ s1,
                      const T* __restrict__ b1, const uint8_t* __restrict__ q2t, const float* __restrict__ s2,
                      const T* __restrict__ b2, float* __restrict__ y, const int* __restrict__ counts, int rows_cap, int K,
                      int H, int N, int act) {
  extern __shared__ __align__(16) float sm8[];  // x rows [kFfnRows][K] | hidden slice [kFfnRows][kHS8], both chunk-split
  const int g = blockIdx.y;
  const int count = counts != nullptr ? min(counts[g], rows_cap) : rows_cap;
  if (count <= 0) return;
  const int h0 = blockIdx.x * kHS8;
  const int hs = min(kHS8, H - h0);
  float* xs = sm8;
  float* hsm = sm8 + kFfnRows * K;
  const T* xg = x + static_cast<long long>(g) * rows_cap * K;
  const uint8_t* q1g = q1 + (static_cast<long long>(g) * H + h0) * K;
  const float* s1g = s1 + static_cast<long long>(g) * H + h0;
  const T* b1g = b1 != nullptr ? b1 + static_cast<long long>(g) * H + h0 : nullptr;
  const uint8_t* q2g = q2t + static_cast<long long>(g) * N * H + h0;
  const float* s2g = s2 + static_cast<long long>(g) * N;
  const T* b2g = b2 != nullptr && blockIdx.x == 0 ? b2 + static_cast<long long>(g) * N : nullptr;
  float* yg = y + static_cast<long long>(g) * rows_cap * N;

  for (int r0 = 0; r0 < count; r0 += kFfnRows) {
    const int nr = min(kFfnRows, count - r0);
    stage_rows_split<T>(xs, xg + static_cast<long long>(r0) * K, nr, K);
    float* yrow0 = yg + static_cast<long long>(r0) * N;
    if (nr == 1) ffn_fp8_pass<T, 1>(xs, hsm, q1g, s1g, b1g, q2g, s2g, b2g, yrow0, nr, K, hs, H, N, act);
    else if (nr == 2) ffn_fp8_pass<T, 2>(xs, hsm, q1g, s1g, b1g, q2g, s2g, b2g, yrow0, nr, K, hs, H, N, act);
    else ffn_fp8_pass<T, kFfnRows>(xs, hsm, q1g, s1g, b1g, q2g, s2g, b2g, yrow0, nr, K, hs, H, N, act);
  }
}

template <typename T, int ROWS>
__device__ __forceinline__ void glu_fp8_pass(const float* __restrict__ xs, float* __restrict__ hsm, const uint8_t* __restrict__ q1g,
                                             const float* __restrict__ s1g, const uint8_t* __restrict__ q2g,
                                             const float* __restrict__ s2g, const uint8_t* __restrict__ q3g,
                                             const float* __restrict__ s3g, float* __restrict__ yrow0, int nr, int M, int hs,
                                             int H, int N, int act) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = warp; j < hs; j += 8) {
    const uint8_t* const rows[2] = {q1g + static_cast<long long>(j) * M, q2g + static_cast<long long>(j) * M};
    float acc[2][ROWS];
    fp8_row_dots<ROWS, 2>(xs, rows, M, acc);
    if (lane < ROWS) {
      float gv = acc[0][0], uv = acc[1][0];
#pragma unroll
      for (int r = 1; r < ROWS; ++r)
        if (lane == r) { gv = acc[0][r]; uv = acc[1][r]; }
      hsm[lane * kHS8 + split_index(j, kHS8)] = ffn_act(s1g[j] * gv, act) * (s2g[j] * uv);
    }
  }
  __syncthreads();
  fp8_layer2<T, ROWS>(hsm, q3g, s3g, nullptr, yrow0, nr, hs, H, N);
}

template <typename T>
__global__ void __launch_bounds__(256, 2)
skinny_glu_ffn_fp8_kernel(const T* __restrict__ x, const uint8_t* __restrict__ q1t, const float* __restrict__ s1,
                          const uint8_t* __restrict__ q2t, const float* __restrict__ s2, const uint8_t* __restrict__ q3t,
                          const float* __restrict__ s3, float* __restrict__ y, const int* __restrict__ counts, int rows_cap,
                          int M, int H, int N, int act) {
  extern __shared__ __align__(16) float sm8[];  // x rows [kFfnRows][M] | hidden slice [kFfnRows][kHS8], both chunk-split
  const int g = blockIdx.y;
  const int count = counts != nullptr ? min(counts[g], rows_cap) : rows_cap;
  if (count <= 0) return;
  const int h0 = blockIdx.x * kHS8;
  const int hs = min(kHS8, H - h0);
  float* xs = sm8;
  float* hsm = sm8 + kFfnRows * M;
  const T* xg = x + static_cast<long long>(g) * rows_cap * M;
  const uint8_t* q1g = q1t + (static_cast<long long>(g) * H + h0) * M;
  const uint8_t* q2g = q2t + (static_cast<long long>(g) * H + h0) * M;
  const float* s1g = s1 + static_cast<long long>(g) * H + h0;
  const float* s2g = s2 + static_cast<long long>(g) * H + h0;
  const uint8_t* q3g = q3t + static_cast<long long>(g) * N * H + h0;
  const float* s3g = s3 + static_cast<long long>(g) * N;
  float* yg = y + static_cast<long long>(g) * rows_cap * N;

  for (int r0 = 0; r0 < count; r0 += kFfnRows) {
    const int nr = min(kFfnRows, count - r0);
    stage_rows_split<T>(xs, xg + static_cast<long long>(r0) * M, nr, M);
    float* yrow0 = yg + static_cast<long long>(r0) * N;
    if (nr == 1) glu_fp8_pass<T, 1>(xs, hsm, q1g, s1g, q2g, s2g, q3g, s3g, yrow0, nr, M, hs, H, N, act);
    else if (nr == 2) glu_fp8_pass<T, 2>(xs, hsm, q1g, s1g, q2g, s2g, q3g, s3g, yrow0, nr, M, hs, H, N, act);
    else glu_fp8_pass<T, kFfnRows>(xs, hsm, q1g, s1g, q2g, s2g, q3g, s3g, yrow0, nr, M, hs, H, N, act);
  }
}

// ------------------------------------------------------------------------------------------------
// Block-scaled fp8 SwiGLU expert (the DeepSeek-V3 checkpoint format), W8A16, one launch
// ------------------------------------------------------------------------------------------------
// Operands are the stored weights of LlamaFFNNetwork(weight_format='fp8_block'), which are also the B operands of the
// block GEMM's forward (ops/block_fp8.py):
//   qglu [G, 2H, M] e4m3: W1^T and W2^T interleaved every 64 rows (row 128 t + j = gate unit 64 t + j, row 128 t + 64 + j
//        = its up partner), sglu [G, 2H / 64, M / 128] fp32, one scale per 64 rows and 128-deep K block;
//   q3t  [G, N, H] e4m3 (the down projection, K = H contiguous), s3t [G, N / 128, H / 128] fp32.
// Block (g, s) owns hidden units [128 s, 128 s + 128): rows [256 s, 256 s + 256) of qglu, two whole interleave groups, so
// a gate row and its up partner are read by the same warp in one loop.
//   layer 1: one hidden unit per warp and pass; lanes stride M in 16-byte (16-element) chunks.  A chunk lies inside one
//            128-deep K block (chunk c in block c / 8): its 16-term fp32 partial sum is multiplied once by that block's
//            scale and added to the lane's sum, the per-block promotion of the GEMM, never a per-element dequantisation;
//   layer 2: fp8_layer2<BLOCK>: the block's 128-unit slice of q3t row n is one 128-byte line and one 128-deep K block, so
//            the 8-lane reduced partial takes the one scale s3t[n / 128, s] before its fp32 atomic add.
// x stays bf16 in shared memory (two 16-byte halves of a chunk K/16 uint4s apart, so lanes read consecutive 16 bytes):
// 8 M + 2 KB bytes per block, 58 KB at M = 7168 (DeepSeek-V3, Kimi-K2), under the 100 KB of two resident blocks of 256
// threads per SM (<= 128 registers: __launch_bounds__(256, 2)); fp32 staging (16 M + 2 KB) would not fit M = 7168.
// Every active expert's bytes are read once per kFfnRows rows; an expert without rows costs one block exit.
__device__ __forceinline__ void bf16x8(const uint4 u, float* f) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
  }
}

// Rows [0, nr) of x (bf16 [nr, K], K % 16 == 0) into xs [kFfnRows][K]; half p of chunk c of a row at uint4 p * K/16 + c.
// Passes of 3 rows run the kFfnRows specialisation, so the missing row is zeroed.
__device__ __forceinline__ void stage_rows_bf16(uint4* __restrict__ xs, const __nv_bfloat16* __restrict__ xrow0, int nr, int K) {
  const int K8 = K >> 3, K16 = K >> 4;
  __syncthreads();
  for (int i = threadIdx.x; i < nr * K8; i += 256) {
    const int r = i / K8, h = i - r * K8;              // h: 8-element half-chunk of row r
    xs[r * K8 + (h & 1) * K16 + (h >> 1)] = __ldg(reinterpret_cast<const uint4*>(xrow0) + i);
  }
  if (nr > 2)
    for (int i = threadIdx.x + nr * K8; i < kFfnRows * K8; i += 256) xs[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
}

// Warp-wide gate and up dot products of ROWS staged rows with one gate row and one up row of K e4m3 weights whose K-block
// scales are sg[K / 128] and su[K / 128]; every lane gets the full sums.
template <int ROWS>
__device__ __forceinline__ void block_glu_dots(const uint4* __restrict__ xs, const uint8_t* __restrict__ qg,
                                               const uint8_t* __restrict__ qu, const float* __restrict__ sg,
                                               const float* __restrict__ su, int K, float (&acc)[2][ROWS]) {
  const int lane = threadIdx.x & 31;
  const int K16 = K >> 4, K8 = K >> 3;
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int r = 0; r < ROWS; ++r) acc[m][r] = 0.0f;
  for (int c = lane; c < K16; c += 32 * 4) {
    uint4 raw[4][2];
    float sc[4][2];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int cc = c + 32 * u;
      const bool in = cc < K16;
      raw[u][0] = in ? __ldcs(reinterpret_cast<const uint4*>(qg) + cc) : make_uint4(0, 0, 0, 0);
      raw[u][1] = in ? __ldcs(reinterpret_cast<const uint4*>(qu) + cc) : make_uint4(0, 0, 0, 0);
      sc[u][0] = in ? __ldg(sg + (cc >> 3)) : 0.0f;
      sc[u][1] = in ? __ldg(su + (cc >> 3)) : 0.0f;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int cc = c + 32 * u;
      if (cc < K16) {
        float wv[2][16];
        e4m3x16(raw[u][0], wv[0]);
        e4m3x16(raw[u][1], wv[1]);
#pragma unroll
        for (int r = 0; r < ROWS; ++r) {
          float xf[16];
          bf16x8(xs[r * K8 + cc], xf);
          bf16x8(xs[r * K8 + K16 + cc], xf + 8);
#pragma unroll
          for (int m = 0; m < 2; ++m) {
            float part = 0.0f;
#pragma unroll
            for (int e = 0; e < 16; ++e) part = fmaf(xf[e], wv[m][e], part);
            acc[m][r] = fmaf(part, sc[u][m], acc[m][r]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int r = 0; r < ROWS; ++r)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[m][r] += __shfl_xor_sync(0xffffffffu, acc[m][r], o);
}

template <int ROWS>
__device__ __forceinline__ void glu_block_fp8_pass(const uint4* __restrict__ xs, float* __restrict__ hsm,
                                                   const uint8_t* __restrict__ qglu_s, const float* __restrict__ sglu_s,
                                                   const uint8_t* __restrict__ q3g, const float* __restrict__ s3g,
                                                   float* __restrict__ yrow0, int nr, int M, int H, int N, int act) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int KB = M >> 7;
  for (int j = warp; j < kHS8; j += 8) {
    const int t = j >> 6, jj = j & 63;                 // interleave group of the slice, unit inside it
    const uint8_t* qg = qglu_s + static_cast<long long>(128 * t + jj) * M;
    float acc[2][ROWS];
    block_glu_dots<ROWS>(xs, qg, qg + 64LL * M, sglu_s + (2 * t) * KB, sglu_s + (2 * t + 1) * KB, M, acc);
    if (lane < ROWS) {
      float gv = acc[0][0], uv = acc[1][0];
#pragma unroll
      for (int r = 1; r < ROWS; ++r)
        if (lane == r) { gv = acc[0][r]; uv = acc[1][r]; }
      hsm[lane * kHS8 + split_index(j, kHS8)] = ffn_act(gv, act) * uv;
    }
  }
  __syncthreads();
  fp8_layer2<__nv_bfloat16, ROWS, true>(hsm, q3g, s3g, nullptr, yrow0, nr, kHS8, H, N, H >> 7);
}

__global__ void __launch_bounds__(256, 2)
skinny_glu_ffn_block_fp8_kernel(const __nv_bfloat16* __restrict__ x, const uint8_t* __restrict__ qglu,
                                const float* __restrict__ sglu, const uint8_t* __restrict__ q3t,
                                const float* __restrict__ s3t, float* __restrict__ y, const int* __restrict__ counts,
                                int rows_cap, int M, int H, int N, int act) {
  extern __shared__ __align__(16) uint4 smb[];   // x rows [kFfnRows][M] bf16, chunk-split | hidden slice [kFfnRows][kHS8] fp32
  const int g = blockIdx.y;
  const int count = counts != nullptr ? min(counts[g], rows_cap) : rows_cap;
  if (count <= 0) return;
  const int s = blockIdx.x, h0 = s * kHS8;
  uint4* xs = smb;
  float* hsm = reinterpret_cast<float*>(smb + kFfnRows * (M >> 3));
  const __nv_bfloat16* xg = x + static_cast<long long>(g) * rows_cap * M;
  const uint8_t* qglu_s = qglu + (static_cast<long long>(g) * 2 * H + 2 * h0) * M;
  const float* sglu_s = sglu + (static_cast<long long>(g) * (H >> 5) + (h0 >> 5)) * (M >> 7);
  const uint8_t* q3g = q3t + static_cast<long long>(g) * N * H + h0;
  const float* s3g = s3t + static_cast<long long>(g) * (N >> 7) * (H >> 7) + s;
  float* yg = y + static_cast<long long>(g) * rows_cap * N;

  for (int r0 = 0; r0 < count; r0 += kFfnRows) {
    const int nr = min(kFfnRows, count - r0);
    stage_rows_bf16(xs, xg + static_cast<long long>(r0) * M, nr, M);
    float* yrow0 = yg + static_cast<long long>(r0) * N;
    if (nr == 1) glu_block_fp8_pass<1>(xs, hsm, qglu_s, sglu_s, q3g, s3g, yrow0, nr, M, H, N, act);
    else if (nr == 2) glu_block_fp8_pass<2>(xs, hsm, qglu_s, sglu_s, q3g, s3g, yrow0, nr, M, H, N, act);
    else glu_block_fp8_pass<kFfnRows>(xs, hsm, qglu_s, sglu_s, q3g, s3g, yrow0, nr, M, H, N, act);
  }
}

// ------------------------------------------------------------------------------------------------
// Group-32 int4 SwiGLU expert (W4A16, the compressed-tensors pack-quantized format), one launch
// ------------------------------------------------------------------------------------------------
// Operands are the stored weights of LlamaFFNNetwork(weight_format='int4') (ops/int4.py):
//   qglu [G, 2H, M / 2] bytes: W1^T and W2^T rows interleaved every 64 (as for fp8_block), byte j of a row holds element
//        2j in bits 0-3 and 2j + 1 in bits 4-7, each as u = q + 8; sglu [G, 2H, M / 32] bf16, one scale per 32 elements;
//   q3t  [G, N, H / 2] bytes (the down projection, K = H), s3t [G, N, H / 32] bf16.
// A 16-byte load of a row is exactly one 32-element group: its word i holds elements 8i .. 8i + 7, element 8i + e in bits
// 4e .. 4e + 3.  Block (g, s) owns hidden units [128 s, 128 s + 128), two whole interleave groups:
//   layer 1: one hidden unit per warp and pass; lane c takes groups c, c + 32, ... of the gate row and its up partner.  A
//            group's 32 products q * x are exact in fp32 (4 + 8 significant bits); their fp32 sum is multiplied by the
//            group's scale inside one fma into the lane's sum (acc = fma(part, s, acc)), then a 5-step shuffle tree;
//   layer 2: the block's 128-unit slice of q3t row n is 64 bytes, four groups: lane (sub, c) takes group c of output
//            sub + 8 i, sums its 32 products h * q, multiplies by the group's scale, and the four lanes of an output are
//            reduced with two shuffles before one fp32 atomic add.
// x stays bf16 in shared memory with the four 8-element quarters of group c at uint4 p * M/32 + c (lanes read consecutive
// 16 bytes): 8 M + 2 KB per block, as for fp8_block.  Every active expert's bytes are read once per kFfnRows rows.
__device__ __forceinline__ float int4_value(uint32_t w, int e) {
  return __uint_as_float(0x4B000000u | ((w >> (4 * e)) & 0xFu)) - 8388616.0f;   // (2^23 + u) - (2^23 + 8) = u - 8, exact
}

__device__ __forceinline__ float bf16_value(uint16_t b) { return __uint_as_float(static_cast<uint32_t>(b) << 16); }

// Rows [0, nr) of x (bf16 [nr, K], K % 32 == 0) into xs [kFfnRows][K]: quarter p of group c of a row at uint4 p * K/32 + c.
__device__ __forceinline__ void stage_rows_int4(uint4* __restrict__ xs, const __nv_bfloat16* __restrict__ xrow0, int nr, int K) {
  const int K8 = K >> 3, K32 = K >> 5;
  __syncthreads();
  for (int i = threadIdx.x; i < nr * K8; i += 256) {
    const int r = i / K8, h = i - r * K8;
    xs[r * K8 + (h & 3) * K32 + (h >> 2)] = __ldg(reinterpret_cast<const uint4*>(xrow0) + i);
  }
  if (nr > 2)
    for (int i = threadIdx.x + nr * K8; i < kFfnRows * K8; i += 256) xs[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
}

// Warp-wide gate and up dot products of ROWS staged rows with one gate row and one up row of K int4 weights whose group
// scales are sg[K / 32] and su[K / 32]; every lane gets the full sums.
template <int ROWS>
__device__ __forceinline__ void int4_glu_dots(const uint4* __restrict__ xs, const uint8_t* __restrict__ qg,
                                              const uint8_t* __restrict__ qu, const __nv_bfloat16* __restrict__ sg,
                                              const __nv_bfloat16* __restrict__ su, int K, float (&acc)[2][ROWS]) {
  const int lane = threadIdx.x & 31;
  const int K32 = K >> 5, K8 = K >> 3;
  const uint16_t* sgb = reinterpret_cast<const uint16_t*>(sg);
  const uint16_t* sub = reinterpret_cast<const uint16_t*>(su);
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int r = 0; r < ROWS; ++r) acc[m][r] = 0.0f;
  for (int c = lane; c < K32; c += 32 * 2) {
    uint4 raw[2][2];
    float sc[2][2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int cc = c + 32 * u;
      const bool in = cc < K32;
      raw[u][0] = in ? __ldcs(reinterpret_cast<const uint4*>(qg) + cc) : make_uint4(0, 0, 0, 0);
      raw[u][1] = in ? __ldcs(reinterpret_cast<const uint4*>(qu) + cc) : make_uint4(0, 0, 0, 0);
      sc[u][0] = in ? bf16_value(__ldg(sgb + cc)) : 0.0f;
      sc[u][1] = in ? bf16_value(__ldg(sub + cc)) : 0.0f;
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int cc = c + 32 * u;
      if (cc < K32) {
        const uint32_t w[2][4] = {{raw[u][0].x, raw[u][0].y, raw[u][0].z, raw[u][0].w},
                                  {raw[u][1].x, raw[u][1].y, raw[u][1].z, raw[u][1].w}};
        float part[2][ROWS];
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
          for (int r = 0; r < ROWS; ++r) part[m][r] = 0.0f;
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          float wv[2][8];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            wv[0][e] = int4_value(w[0][p], e);
            wv[1][e] = int4_value(w[1][p], e);
          }
#pragma unroll
          for (int r = 0; r < ROWS; ++r) {
            float xf[8];
            bf16x8(xs[r * K8 + p * K32 + cc], xf);
#pragma unroll
            for (int m = 0; m < 2; ++m)
#pragma unroll
              for (int e = 0; e < 8; ++e) part[m][r] = fmaf(xf[e], wv[m][e], part[m][r]);
          }
        }
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
          for (int r = 0; r < ROWS; ++r) acc[m][r] = fmaf(part[m][r], sc[u][m], acc[m][r]);
      }
    }
  }
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int r = 0; r < ROWS; ++r)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[m][r] += __shfl_xor_sync(0xffffffffu, acc[m][r], o);
}

// Layer 2: yrow0[r, n] += sum over the slice's four groups of s3[n, group] * sum_{32 units} h[r, j] * q3[n, j], r < nr.
// hsm holds h [ROWS][kHS8] with unit 32 c + e at index (e >> 2) * 16 + 4 c + (e & 3), so the four lanes of an output
// read four consecutive float4s.
template <int ROWS>
__device__ __forceinline__ void int4_layer2(const float* __restrict__ hsm, const uint8_t* __restrict__ q,
                                            const __nv_bfloat16* __restrict__ s, float* __restrict__ yrow0, int nr, int H,
                                            int N) {
  constexpr int U = 4;                          // loads in flight per lane
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = lane & 3, sub = lane >> 2;
  const uint16_t* sb = reinterpret_cast<const uint16_t*>(s);
  const long long qld = H >> 1, sld = H >> 5;
  for (int nb = warp * 8; nb < N; nb += 64 * U) {   // warp-uniform bound: all lanes reach the shuffles
    uint4 raw[U];
    float sc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int n = nb + sub + 64 * u;
      raw[u] = n < N ? __ldcs(reinterpret_cast<const uint4*>(q + n * qld) + c) : make_uint4(0, 0, 0, 0);
      sc[u] = n < N ? bf16_value(__ldg(sb + n * sld + c)) : 0.0f;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint32_t w[4] = {raw[u].x, raw[u].y, raw[u].z, raw[u].w};
      float acc[ROWS];
#pragma unroll
      for (int r = 0; r < ROWS; ++r) acc[r] = 0.0f;
#pragma unroll 1
      for (int p = 0; p < 4; ++p) {
        float wv[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) wv[e] = int4_value(w[p], e);
#pragma unroll
        for (int r = 0; r < ROWS; ++r) {
          const float4* hr = reinterpret_cast<const float4*>(hsm + r * kHS8);
          const float4 h0 = hr[(2 * p) * 4 + c], h1 = hr[(2 * p + 1) * 4 + c];
          acc[r] = fmaf(h0.x, wv[0], acc[r]);
          acc[r] = fmaf(h0.y, wv[1], acc[r]);
          acc[r] = fmaf(h0.z, wv[2], acc[r]);
          acc[r] = fmaf(h0.w, wv[3], acc[r]);
          acc[r] = fmaf(h1.x, wv[4], acc[r]);
          acc[r] = fmaf(h1.y, wv[5], acc[r]);
          acc[r] = fmaf(h1.z, wv[6], acc[r]);
          acc[r] = fmaf(h1.w, wv[7], acc[r]);
        }
      }
#pragma unroll
      for (int r = 0; r < ROWS; ++r) {
        acc[r] *= sc[u];
        acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], 1);
        acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], 2);
      }
      const int n = nb + sub + 64 * u;
      if (c < nr && n < N) {
        float v = acc[0];
#pragma unroll
        for (int r = 1; r < ROWS; ++r) if (c == r) v = acc[r];
        atomicAdd(yrow0 + static_cast<long long>(c) * N + n, v);
      }
    }
  }
}

template <int ROWS>
__device__ __forceinline__ void glu_int4_pass(const uint4* __restrict__ xs, float* __restrict__ hsm,
                                              const uint8_t* __restrict__ qglu_s, const __nv_bfloat16* __restrict__ sglu_s,
                                              const uint8_t* __restrict__ q3g, const __nv_bfloat16* __restrict__ s3g,
                                              float* __restrict__ yrow0, int nr, int M, int H, int N, int act) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long qld = M >> 1, sld = M >> 5;
  for (int j = warp; j < kHS8; j += 8) {
    const int t = j >> 6, jj = j & 63;                 // interleave group of the slice, unit inside it
    const long long row = 128 * t + jj;
    float acc[2][ROWS];
    int4_glu_dots<ROWS>(xs, qglu_s + row * qld, qglu_s + (row + 64) * qld, sglu_s + row * sld, sglu_s + (row + 64) * sld,
                        M, acc);
    if (lane < ROWS) {
      float gv = acc[0][0], uv = acc[1][0];
#pragma unroll
      for (int r = 1; r < ROWS; ++r)
        if (lane == r) { gv = acc[0][r]; uv = acc[1][r]; }
      const int c = j >> 5, e = j & 31;
      hsm[lane * kHS8 + (e >> 2) * 16 + 4 * c + (e & 3)] = ffn_act(gv, act) * uv;
    }
  }
  __syncthreads();
  int4_layer2<ROWS>(hsm, q3g, s3g, yrow0, nr, H, N);
}

__global__ void __launch_bounds__(256, 2)
skinny_glu_ffn_int4_kernel(const __nv_bfloat16* __restrict__ x, const uint8_t* __restrict__ qglu,
                           const __nv_bfloat16* __restrict__ sglu, const uint8_t* __restrict__ q3t,
                           const __nv_bfloat16* __restrict__ s3t, float* __restrict__ y, const int* __restrict__ counts,
                           int rows_cap, int M, int H, int N, int act) {
  extern __shared__ __align__(16) uint4 smb[];   // x rows [kFfnRows][M] bf16, group-split | hidden slice [kFfnRows][kHS8] fp32
  const int g = blockIdx.y;
  const int count = counts != nullptr ? min(counts[g], rows_cap) : rows_cap;
  if (count <= 0) return;
  const int s = blockIdx.x, h0 = s * kHS8;
  uint4* xs = smb;
  float* hsm = reinterpret_cast<float*>(smb + kFfnRows * (M >> 3));
  const __nv_bfloat16* xg = x + static_cast<long long>(g) * rows_cap * M;
  const uint8_t* qglu_s = qglu + (static_cast<long long>(g) * 2 * H + 2 * h0) * (M >> 1);
  const __nv_bfloat16* sglu_s = sglu + (static_cast<long long>(g) * 2 * H + 2 * h0) * (M >> 5);
  const uint8_t* q3g = q3t + static_cast<long long>(g) * N * (H >> 1) + (h0 >> 1);
  const __nv_bfloat16* s3g = s3t + static_cast<long long>(g) * N * (H >> 5) + (h0 >> 5);
  float* yg = y + static_cast<long long>(g) * rows_cap * N;

  for (int r0 = 0; r0 < count; r0 += kFfnRows) {
    const int nr = min(kFfnRows, count - r0);
    stage_rows_int4(xs, xg + static_cast<long long>(r0) * M, nr, M);
    float* yrow0 = yg + static_cast<long long>(r0) * N;
    if (nr == 1) glu_int4_pass<1>(xs, hsm, qglu_s, sglu_s, q3g, s3g, yrow0, nr, M, H, N, act);
    else if (nr == 2) glu_int4_pass<2>(xs, hsm, qglu_s, sglu_s, q3g, s3g, yrow0, nr, M, H, N, act);
    else glu_int4_pass<kFfnRows>(xs, hsm, qglu_s, sglu_s, q3g, s3g, yrow0, nr, M, H, N, act);
  }
}


// Dynamic shared memory of both fp8 kernels: the staged x rows and the hidden slice (K % 16 == 0 keeps both 16-byte aligned).
size_t fp8_smem_bytes(int K) { return sizeof(float) * (static_cast<size_t>(kFfnRows) * K + kFfnRows * kHS8); }

template <typename Kern>
cudaError_t fp8_opt_in(Kern* kern, size_t smem) {
  if (smem > kFfnSmemLimit) return cudaErrorInvalidValue;
  if (smem > 48 * 1024) return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  return cudaSuccess;
}

template <typename T>
cudaError_t launch_ffn_fp8(const void* x, const void* q1, const float* s1, const void* b1, const void* q2t, const float* s2,
                           const void* b2, float* y, const int* counts, int G, int rows_cap, int K, int H, int N, int act,
                           cudaStream_t stream) {
  const size_t smem = fp8_smem_bytes(K);
  auto* kern = skinny_ffn_fp8_kernel<T>;
  cudaError_t e = fp8_opt_in(kern, smem);
  if (e != cudaSuccess) return e;
  dim3 grid((H + kHS8 - 1) / kHS8, G);
  kern<<<grid, 256, smem, stream>>>(static_cast<const T*>(x), static_cast<const uint8_t*>(q1), s1, static_cast<const T*>(b1),
                                    static_cast<const uint8_t*>(q2t), s2, static_cast<const T*>(b2), y, counts, rows_cap, K,
                                    H, N, act);
  return cudaGetLastError();
}

template <typename T>
cudaError_t launch_glu_ffn_fp8(const void* x, const void* q1t, const float* s1, const void* q2t, const float* s2,
                               const void* q3t, const float* s3, float* y, const int* counts, int G, int rows_cap, int M,
                               int H, int N, int act, cudaStream_t stream) {
  const size_t smem = fp8_smem_bytes(M);
  auto* kern = skinny_glu_ffn_fp8_kernel<T>;
  cudaError_t e = fp8_opt_in(kern, smem);
  if (e != cudaSuccess) return e;
  dim3 grid((H + kHS8 - 1) / kHS8, G);
  kern<<<grid, 256, smem, stream>>>(static_cast<const T*>(x), static_cast<const uint8_t*>(q1t), s1,
                                    static_cast<const uint8_t*>(q2t), s2, static_cast<const uint8_t*>(q3t), s3, y, counts,
                                    rows_cap, M, H, N, act);
  return cudaGetLastError();
}

// Dynamic shared memory of the block-scaled kernel: bf16 x rows and the fp32 hidden slice.
size_t block_fp8_smem_bytes(int M) { return 2 * static_cast<size_t>(kFfnRows) * M + sizeof(float) * kFfnRows * kHS8; }

}  // namespace

cudaError_t skinny_grouped_gemm(const void* x, const void* w, const void* bias, void* y, const int* counts, int G,
                                int rows_cap, int N, int K, bool w_is_kn, bool relu, int elem_type, cudaStream_t stream) {
  switch (elem_type) {
    case ET_F32: return launch<float>(x, w, bias, y, counts, G, rows_cap, N, K, w_is_kn, relu, stream);
    case ET_F16: return launch<__half>(x, w, bias, y, counts, G, rows_cap, N, K, w_is_kn, relu, stream);
    case ET_BF16: return launch<__nv_bfloat16>(x, w, bias, y, counts, G, rows_cap, N, K, w_is_kn, relu, stream);
  }
  return cudaErrorInvalidValue;
}

cudaError_t skinny_grouped_ffn(const void* x, const void* w1, const void* b1, const void* w2, const void* b2, float* y,
                               const int* counts, int G, int rows_cap, int K, int H, int N, int act, int elem_type,
                               cudaStream_t stream) {
  if (G <= 0 || rows_cap <= 0 || K <= 0 || H <= 0 || N <= 0) return cudaSuccess;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w1) | reinterpret_cast<uintptr_t>(w2)) & 15) return cudaErrorInvalidValue;
  switch (elem_type) {
    case ET_F32: return launch_ffn<float>(x, w1, b1, w2, b2, y, counts, G, rows_cap, K, H, N, act, stream);
    case ET_F16: return launch_ffn<__half>(x, w1, b1, w2, b2, y, counts, G, rows_cap, K, H, N, act, stream);
    case ET_BF16: return launch_ffn<__nv_bfloat16>(x, w1, b1, w2, b2, y, counts, G, rows_cap, K, H, N, act, stream);
  }
  return cudaErrorInvalidValue;
}

cudaError_t skinny_grouped_glu_ffn(const void* x, const void* w1, const void* w2, const void* w3, float* y, const int* counts,
                                   int G, int rows_cap, int M, int H, int N, int act, int elem_type, cudaStream_t stream) {
  if (G <= 0 || rows_cap <= 0 || M <= 0 || H <= 0 || N <= 0) return cudaSuccess;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w1) | reinterpret_cast<uintptr_t>(w2) |
       reinterpret_cast<uintptr_t>(w3)) & 15) return cudaErrorInvalidValue;
  switch (elem_type) {
    case ET_F32: return launch_glu_ffn<float>(x, w1, w2, w3, y, counts, G, rows_cap, M, H, N, act, stream);
    case ET_F16: return launch_glu_ffn<__half>(x, w1, w2, w3, y, counts, G, rows_cap, M, H, N, act, stream);
    case ET_BF16: return launch_glu_ffn<__nv_bfloat16>(x, w1, w2, w3, y, counts, G, rows_cap, M, H, N, act, stream);
  }
  return cudaErrorInvalidValue;
}

cudaError_t skinny_grouped_ffn_fp8(const void* x, const void* q1, const float* s1, const void* b1, const void* q2t,
                                   const float* s2, const void* b2, float* y, const int* counts, int G, int rows_cap, int K,
                                   int H, int N, int act, int elem_type, cudaStream_t stream) {
  if (G <= 0 || rows_cap <= 0 || K <= 0 || H <= 0 || N <= 0) return cudaSuccess;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(q1) | reinterpret_cast<uintptr_t>(q2t)) & 15) return cudaErrorInvalidValue;
  if (K % 16 || H % 16 || N % 16) return cudaErrorInvalidValue;
  switch (elem_type) {
    case ET_F16: return launch_ffn_fp8<__half>(x, q1, s1, b1, q2t, s2, b2, y, counts, G, rows_cap, K, H, N, act, stream);
    case ET_BF16: return launch_ffn_fp8<__nv_bfloat16>(x, q1, s1, b1, q2t, s2, b2, y, counts, G, rows_cap, K, H, N, act, stream);
  }
  return cudaErrorInvalidValue;
}

cudaError_t skinny_grouped_glu_ffn_fp8(const void* x, const void* q1t, const float* s1, const void* q2t, const float* s2,
                                       const void* q3t, const float* s3, float* y, const int* counts, int G, int rows_cap,
                                       int M, int H, int N, int act, int elem_type, cudaStream_t stream) {
  if (G <= 0 || rows_cap <= 0 || M <= 0 || H <= 0 || N <= 0) return cudaSuccess;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(q1t) | reinterpret_cast<uintptr_t>(q2t) |
       reinterpret_cast<uintptr_t>(q3t)) & 15) return cudaErrorInvalidValue;
  if (M % 16 || H % 16 || N % 16) return cudaErrorInvalidValue;
  switch (elem_type) {
    case ET_F16: return launch_glu_ffn_fp8<__half>(x, q1t, s1, q2t, s2, q3t, s3, y, counts, G, rows_cap, M, H, N, act, stream);
    case ET_BF16:
      return launch_glu_ffn_fp8<__nv_bfloat16>(x, q1t, s1, q2t, s2, q3t, s3, y, counts, G, rows_cap, M, H, N, act, stream);
  }
  return cudaErrorInvalidValue;
}

cudaError_t skinny_grouped_glu_ffn_block_fp8(const void* x, const void* qglu, const float* sglu, const void* q3t,
                                             const float* s3t, float* y, const int* counts, int G, int rows_cap, int M, int H,
                                             int N, int act, cudaStream_t stream) {
  if (G <= 0 || rows_cap <= 0 || M <= 0 || H <= 0 || N <= 0) return cudaSuccess;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(qglu) | reinterpret_cast<uintptr_t>(q3t)) & 15)
    return cudaErrorInvalidValue;
  if (M % 128 || H % 128 || N % 128 || act < 1 || act > 3) return cudaErrorInvalidValue;
  const size_t smem = block_fp8_smem_bytes(M);
  auto* kern = skinny_glu_ffn_block_fp8_kernel;
  cudaError_t e = fp8_opt_in(kern, smem);
  if (e != cudaSuccess) return e;
  dim3 grid(H / kHS8, G);
  kern<<<grid, 256, smem, stream>>>(static_cast<const __nv_bfloat16*>(x), static_cast<const uint8_t*>(qglu), sglu,
                                    static_cast<const uint8_t*>(q3t), s3t, y, counts, rows_cap, M, H, N, act);
  return cudaGetLastError();
}

cudaError_t skinny_grouped_glu_ffn_int4(const void* x, const void* qglu, const void* sglu, const void* q3t, const void* s3t,
                                        float* y, const int* counts, int G, int rows_cap, int M, int H, int N, int act,
                                        cudaStream_t stream) {
  if (G <= 0 || rows_cap <= 0 || M <= 0 || H <= 0 || N <= 0) return cudaSuccess;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(qglu) | reinterpret_cast<uintptr_t>(q3t)) & 15)
    return cudaErrorInvalidValue;
  if ((reinterpret_cast<uintptr_t>(sglu) | reinterpret_cast<uintptr_t>(s3t)) & 1) return cudaErrorInvalidValue;
  if (M % 128 || H % 128 || N % 128 || act < 1 || act > 3) return cudaErrorInvalidValue;
  const size_t smem = block_fp8_smem_bytes(M);     // the same bf16 x rows and fp32 hidden slice
  auto* kern = skinny_glu_ffn_int4_kernel;
  cudaError_t e = fp8_opt_in(kern, smem);
  if (e != cudaSuccess) return e;
  dim3 grid(H / kHS8, G);
  kern<<<grid, 256, smem, stream>>>(static_cast<const __nv_bfloat16*>(x), static_cast<const uint8_t*>(qglu),
                                    static_cast<const __nv_bfloat16*>(sglu), static_cast<const uint8_t*>(q3t),
                                    static_cast<const __nv_bfloat16*>(s3t), y, counts, rows_cap, M, H, N, act);
  return cudaGetLastError();
}

}  // namespace tb
