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

}  // namespace tb
