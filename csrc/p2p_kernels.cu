// Peer-to-peer collectives written as plain CUDA kernels over NVLink-mapped memory: the H100-native replacement
// for the reference's grouped ncclSend/ncclRecv all-to-alls (tutel/custom/custom_kernel.cpp:463-518, 520-654)
// and c10d all_to_all_single (tutel/impls/communicate.py:181-192).  One launch = handshake + payload + completion:
//
//   1. every rank posts, in each peer's mailbox, WHERE in its arena this call's data must land (epoch | offset/256,
//      one st.release.sys.u64) - receive buffers are therefore chosen per call and per rank (zero-copy results)
//   2. CTAs push their share of the payload with 16-byte stores into the destination GPU's heap
//   3. each CTA publishes completion with fence.acq_rel.sys + red.release.sys on the peer's done[] counter
//   4. the kernel does not exit before all of its own inbound pushes are complete (ld.acquire.sys polling with a
//      bounded spin), so plain stream order makes the received data visible to the next kernel.
#include "p2p_kernels.h"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "moe_kernels.h"
#include "ptx.cuh"

namespace tb {
namespace {

constexpr int kPushThreadsBig = 512;
constexpr int kPushThreadsSmall = 128;   // 128 threads x <= 64 registers: fits next to a resident persistent GEMM CTA (gemm_sm90.cu)

template <int kPushThreads>
__global__ void __launch_bounds__(kPushThreads, kPushThreads == 128 ? 8 : 1)
p2p_push_kernel(const uint8_t* __restrict__ src, const PushPlan plan, const unsigned long long* __restrict__ peer_table,
                long long recv_heap_off, long long mail_off, long long done_off, long long scratch_off, int rank,
                int world, uint32_t epoch, int blocks_per_peer) {
  const int pi = blockIdx.x / blocks_per_peer;           // which peer (rotated so that traffic is spread)
  const int sub = blockIdx.x - pi * blocks_per_peer;     // which slice of that peer's payload
  const int peer = (rank + pi) % world;
  uint8_t* peer_base = reinterpret_cast<uint8_t*>(peer_table[peer]);
  uint8_t* my_base = reinterpret_cast<uint8_t*>(peer_table[rank]);

  // (1) mailboxes: tell every peer where this rank receives this call's data (also the "buffer is free" credit)
  if (blockIdx.x == 0 && threadIdx.x < world) {
    uint8_t* pb = reinterpret_cast<uint8_t*>(peer_table[threadIdx.x]);
    const unsigned long long word = (static_cast<unsigned long long>(epoch) << 32) |
                                    static_cast<unsigned long long>(recv_heap_off >> 8);
    ptx::st_release_sys_u64(reinterpret_cast<unsigned long long*>(pb + mail_off) + rank, word);
  }
  // (2) wait for the destination's mailbox entry, then push
  __shared__ unsigned long long dst_heap_off_s;
  if (threadIdx.x == 0)
    dst_heap_off_s = static_cast<unsigned long long>(ptx::wait_mailbox_sys(
                         reinterpret_cast<const unsigned long long*>(my_base + mail_off) + peer, epoch)) << 8;
  __syncthreads();
  const long long dst_heap_off = static_cast<long long>(dst_heap_off_s);

  const long long total = plan.bytes[peer];
  const uint8_t* s = src + plan.src_off[peer];
  uint8_t* d = peer_base + dst_heap_off + plan.dst_off[peer];
  const bool aligned = (((reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(d)) & 15) == 0);
  if (aligned) {
    const long long nvec = total >> 4;
    const long long per = (nvec + blocks_per_peer - 1) / blocks_per_peer;
    const long long v0 = per * sub;
    const long long v1 = min(nvec, v0 + per);
    const uint4* sv = reinterpret_cast<const uint4*>(s);
    uint4* dv = reinterpret_cast<uint4*>(d);
    long long v = v0 + threadIdx.x;
    for (; v + 3LL * kPushThreads < v1; v += 4LL * kPushThreads) {
      uint4 a[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) a[u] = ptx::ld_nc_v4(sv + v + u * kPushThreads);
#pragma unroll
      for (int u = 0; u < 4; ++u) ptx::st_na_v4(dv + v + u * kPushThreads, a[u]);
    }
    for (; v < v1; v += kPushThreads) ptx::st_na_v4(dv + v, ptx::ld_nc_v4(sv + v));
    if (sub == blocks_per_peer - 1)
      for (long long b = (nvec << 4) + threadIdx.x; b < total; b += kPushThreads) d[b] = s[b];
  } else {
    const long long per = (total + blocks_per_peer - 1) / blocks_per_peer;
    const long long b0 = per * sub, b1 = min(total, b0 + per);
    for (long long b = b0 + threadIdx.x; b < b1; b += kPushThreads) d[b] = s[b];
  }
  // (3) completion: the LAST block working for this peer publishes one release.sys increment, so the receiver's
  //     target is simply the call number (it does not need to know how many blocks the sender used)
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t* local_cnt = reinterpret_cast<uint32_t*>(my_base + scratch_off) + peer;
    uint32_t prev;
    asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(prev) : "l"(local_cnt) : "memory");
    if (prev == static_cast<uint32_t>(blocks_per_peer) - 1u) {
      *local_cnt = 0u;  // every block of this call has arrived; re-arm for the next call (stream-ordered)
      ptx::fence_acq_rel_sys();
      ptx::red_add_release_sys(reinterpret_cast<uint32_t*>(peer_base + done_off) + rank, 1u);
    }
  }
  // (4) inbound completion: block i (< world) watches source i
  if (blockIdx.x < world && threadIdx.x == 0)
    ptx::wait_flag_ge_sys(reinterpret_cast<const uint32_t*>(my_base + done_off) + blockIdx.x, epoch);
}

template <typename T>
__device__ __forceinline__ float ldf(const T* p);
template <> __device__ __forceinline__ float ldf<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ldf<__half>(const __half* p) { return __half2float(*p); }
template <> __device__ __forceinline__ float ldf<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <typename T>
__device__ __forceinline__ void stf(T* p, float v);
template <> __device__ __forceinline__ void stf<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void stf<__half>(__half* p, float v) { *p = __float2half_rn(v); }
template <> __device__ __forceinline__ void stf<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

template <typename T>
__global__ void __launch_bounds__(256)
p2p_reduce_slice_kernel(T* __restrict__ out, const unsigned long long* __restrict__ peer_table, long long stage_off,
                        long long slice_off_bytes, long long n, int rank, int world, bool is_max) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    float acc = is_max ? -INFINITY : 0.0f;
    for (int q = 0; q < world; ++q) {
      const int p = (rank + q) % world;
      const T* pp = reinterpret_cast<const T*>(reinterpret_cast<const uint8_t*>(peer_table[p]) + stage_off + slice_off_bytes);
      const float v = ldf<T>(pp + i);
      acc = is_max ? fmaxf(acc, v) : acc + v;
    }
    stf<T>(out + i, acc);
  }
}

// ---- one-shot all-reduce ---------------------------------------------------------------------------------
template <typename T> struct RedT;
template <> struct RedT<float> { using Acc = float; static __device__ float up(float v) { return v; } static __device__ float down(float v) { return v; } };
template <> struct RedT<__half> { using Acc = float; static __device__ float up(__half v) { return __half2float(v); } static __device__ __half down(float v) { return __float2half_rn(v); } };
template <> struct RedT<__nv_bfloat16> { using Acc = float; static __device__ float up(__nv_bfloat16 v) { return __bfloat162float(v); } static __device__ __nv_bfloat16 down(float v) { return __float2bfloat16_rn(v); } };
template <> struct RedT<int> { using Acc = int; static __device__ int up(int v) { return v; } static __device__ int down(int v) { return v; } };
template <> struct RedT<long long> { using Acc = long long; static __device__ long long up(long long v) { return v; } static __device__ long long down(long long v) { return v; } };

template <typename T>
__global__ void __launch_bounds__(256)
p2p_allreduce_oneshot_kernel(const T* __restrict__ in, T* __restrict__ out,
                             const unsigned long long* __restrict__ peer_table, long long inbox_off, long long slot_bytes,
                             long long flag_off, long long n, int rank, int world, uint32_t epoch, bool is_max) {
  using Acc = typename RedT<T>::Acc;
  const int parity = static_cast<int>(epoch & 1u);
  const long long per = (n + gridDim.x - 1) / gridDim.x;
  const long long per_al = (per * static_cast<long long>(sizeof(T)) + 15) / 16 * 16 / static_cast<long long>(sizeof(T));
  const long long i0 = per_al * blockIdx.x;
  const long long i1 = min(n, i0 + per_al);
  // (1) my chunk -> slot [parity][rank] of every peer's inbox (own inbox included: the reduction reads W uniform slots)
  if (i0 < i1) {
    const long long nb = (i1 - i0) * static_cast<long long>(sizeof(T));
    const uint8_t* s = reinterpret_cast<const uint8_t*>(in + i0);
    const bool vec = ((reinterpret_cast<uintptr_t>(s) & 15) == 0);
    for (int q = 0; q < world; ++q) {
      const int p = (rank + q) % world;
      uint8_t* d = reinterpret_cast<uint8_t*>(peer_table[p]) + inbox_off +
                   (static_cast<long long>(parity) * world + rank) * slot_bytes + i0 * static_cast<long long>(sizeof(T));
      if (vec) {
        const long long nv = nb >> 4;
        for (long long v = threadIdx.x; v < nv; v += blockDim.x)
          ptx::st_na_v4(reinterpret_cast<uint4*>(d) + v, ptx::ld_nc_v4(reinterpret_cast<const uint4*>(s) + v));
        for (long long b = (nv << 4) + threadIdx.x; b < nb; b += blockDim.x) d[b] = s[b];
      } else {
        for (long long b = threadIdx.x; b < nb; b += blockDim.x) d[b] = s[b];
      }
    }
  }
  __syncthreads();
  // (2) publish: one flag per (source rank, block) on every peer;  (3) wait for the W flags of this block
  if (threadIdx.x < world) {
    const int p = threadIdx.x;
    uint32_t* f = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(peer_table[p]) + flag_off) +
                  (static_cast<long long>(parity) * world + rank) * kOneShotMaxBlocks + blockIdx.x;
    ptx::fence_acq_rel_sys();
    ptx::st_release_sys(f, epoch);
    const uint32_t* mine = reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(peer_table[rank]) + flag_off) +
                           (static_cast<long long>(parity) * world + p) * kOneShotMaxBlocks + blockIdx.x;
    ptx::wait_flag_ge_sys(mine, epoch);
  }
  __syncthreads();
  // (4) reduce the W copies in rank order
  const uint8_t* inbox = reinterpret_cast<const uint8_t*>(peer_table[rank]) + inbox_off +
                         static_cast<long long>(parity) * world * slot_bytes;
  for (long long i = i0 + threadIdx.x; i < i1; i += blockDim.x) {
    Acc acc = RedT<T>::up(*reinterpret_cast<const volatile T*>(inbox + i * static_cast<long long>(sizeof(T))));
    for (int p = 1; p < world; ++p) {
      const Acc v = RedT<T>::up(*reinterpret_cast<const volatile T*>(inbox + p * slot_bytes + i * static_cast<long long>(sizeof(T))));
      acc = is_max ? (v > acc ? v : acc) : acc + v;
    }
    out[i] = RedT<T>::down(acc);
  }
}

// ---- 2-D hierarchical all-to-all: record transpose between the two phases ---------------------------------------
__global__ void __launch_bounds__(256)
p2p_stride_copy_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int rows, int cols, long long width) {
  const long long records = static_cast<long long>(rows) * cols;
  const bool vec = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst) | static_cast<uintptr_t>(width)) & 15) == 0;
  for (long long i = blockIdx.y; i < records; i += gridDim.y) {
    const long long r = i / cols, c = i - r * cols;
    const uint8_t* s = src + i * width;
    uint8_t* d = dst + (c * rows + r) * width;
    if (vec) {
      const long long nv = width >> 4;
      for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < nv;
           v += static_cast<long long>(gridDim.x) * blockDim.x)
        ptx::st_na_v4(reinterpret_cast<uint4*>(d) + v, ptx::ld_nc_v4(reinterpret_cast<const uint4*>(s) + v));
    } else {
      for (long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; b < width;
           b += static_cast<long long>(gridDim.x) * blockDim.x)
        d[b] = s[b];
    }
  }
}

__global__ void p2p_barrier_kernel(const unsigned long long* __restrict__ peer_table, long long bar_off, int rank,
                                   int world, uint32_t epoch) {
  const int p = threadIdx.x;
  if (p < world) {
    uint8_t* pb = reinterpret_cast<uint8_t*>(peer_table[p]);
    ptx::fence_acq_rel_sys();
    ptx::red_add_release_sys(reinterpret_cast<uint32_t*>(pb + bar_off) + rank, 1u);
    const uint8_t* mb = reinterpret_cast<const uint8_t*>(peer_table[rank]);
    ptx::wait_flag_ge_sys(reinterpret_cast<const uint32_t*>(mb + bar_off) + p, epoch);
  }
}

}  // namespace

cudaError_t p2p_push(const void* src, const PushPlan& plan, const unsigned long long* peer_table,
                     long long recv_heap_off, long long mail_off, long long done_off, long long scratch_off, int rank,
                     int world, uint32_t epoch, int blocks_per_peer, bool small_blocks, cudaStream_t stream) {
  if (world > kMaxPeers) return cudaErrorInvalidValue;
  if (blocks_per_peer < 1) blocks_per_peer = 1;
  const int grid = world * blocks_per_peer;
  if (small_blocks)     // overlap with a running expert GEMM: blocks that can co-reside with its CTAs
    p2p_push_kernel<kPushThreadsSmall><<<grid, kPushThreadsSmall, 0, stream>>>(
        static_cast<const uint8_t*>(src), plan, peer_table, recv_heap_off, mail_off, done_off, scratch_off, rank, world, epoch,
        blocks_per_peer);
  else
    p2p_push_kernel<kPushThreadsBig><<<grid, kPushThreadsBig, 0, stream>>>(
        static_cast<const uint8_t*>(src), plan, peer_table, recv_heap_off, mail_off, done_off, scratch_off, rank, world, epoch,
        blocks_per_peer);
  return cudaGetLastError();
}

cudaError_t p2p_reduce_slice(void* out, const unsigned long long* peer_table, long long stage_off,
                             long long slice_off_bytes, long long n_elems, int elem_type, int rank, int world,
                             bool is_max, cudaStream_t stream) {
  if (n_elems <= 0) return cudaSuccess;
  long long want = (n_elems + 255) / 256;
  const int grid = static_cast<int>(want < 592 ? want : 592);
  switch (elem_type) {
    case ET_F32:
      p2p_reduce_slice_kernel<float><<<grid, 256, 0, stream>>>(static_cast<float*>(out), peer_table, stage_off,
                                                               slice_off_bytes, n_elems, rank, world, is_max);
      break;
    case ET_F16:
      p2p_reduce_slice_kernel<__half><<<grid, 256, 0, stream>>>(static_cast<__half*>(out), peer_table, stage_off,
                                                                slice_off_bytes, n_elems, rank, world, is_max);
      break;
    case ET_BF16:
      p2p_reduce_slice_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(static_cast<__nv_bfloat16*>(out), peer_table,
                                                                       stage_off, slice_off_bytes, n_elems, rank,
                                                                       world, is_max);
      break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

cudaError_t p2p_allreduce_oneshot(const void* in, void* out, const unsigned long long* peer_table, long long inbox_off,
                                  long long slot_bytes, long long flag_off, long long n_elems, int elem_type, int rank,
                                  int world, uint32_t epoch, bool is_max, cudaStream_t stream) {
  if (n_elems <= 0) return cudaSuccess;
  if (world > kMaxPeers) return cudaErrorInvalidValue;
  const int es = elem_type == ET_F32 || elem_type == ET_I32 ? 4 : (elem_type == ET_I64 ? 8 : 2);
  const long long bytes = n_elems * es;
  if (bytes > slot_bytes) return cudaErrorInvalidValue;
  long long want = (bytes + 4095) / 4096;            // 256 threads x 16 B per block and pass
  const int grid = static_cast<int>(want < 1 ? 1 : (want > kOneShotMaxBlocks ? kOneShotMaxBlocks : want));
#define TB_ONESHOT(T)                                                                                                   \
  p2p_allreduce_oneshot_kernel<T><<<grid, 256, 0, stream>>>(static_cast<const T*>(in), static_cast<T*>(out), peer_table, \
                                                            inbox_off, slot_bytes, flag_off, n_elems, rank, world, epoch, \
                                                            is_max)
  switch (elem_type) {
    case ET_F32: TB_ONESHOT(float); break;
    case ET_F16: TB_ONESHOT(__half); break;
    case ET_BF16: TB_ONESHOT(__nv_bfloat16); break;
    case ET_I32: TB_ONESHOT(int); break;
    case ET_I64: TB_ONESHOT(long long); break;
    default: return cudaErrorInvalidValue;
  }
#undef TB_ONESHOT
  return cudaGetLastError();
}

cudaError_t p2p_stride_copy(const void* src, void* dst, int rows, int cols, long long width_bytes, cudaStream_t stream) {
  if (rows <= 0 || cols <= 0 || width_bytes <= 0) return cudaSuccess;
  const long long records = static_cast<long long>(rows) * cols;
  const long long per = (width_bytes / 16 + 255) / 256;
  dim3 grid(static_cast<unsigned>(per < 1 ? 1 : (per > 64 ? 64 : per)), static_cast<unsigned>(records < 4096 ? records : 4096));
  p2p_stride_copy_kernel<<<grid, 256, 0, stream>>>(static_cast<const uint8_t*>(src), static_cast<uint8_t*>(dst), rows, cols,
                                                   width_bytes);
  return cudaGetLastError();
}


cudaError_t p2p_barrier(const unsigned long long* peer_table, long long bar_off, int rank, int world, uint32_t epoch,
                        cudaStream_t stream) {
  p2p_barrier_kernel<<<1, 32, 0, stream>>>(peer_table, bar_off, rank, world, epoch);
  return cudaGetLastError();
}

// run-time spin-wait limit of this translation unit's kernels (ptx.cuh)
cudaError_t set_spin_timeout_p2p(unsigned long long ns) {
  return cudaMemcpyToSymbol(tb_spin_timeout_ns, &ns, sizeof(ns));
}

}  // namespace tb
