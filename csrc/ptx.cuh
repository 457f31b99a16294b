// Thin inline-PTX layer for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma,
// cluster helpers and system-scope acquire/release primitives used by the cross-GPU protocols.
// Everything here is written against the PTX ISA for CUDA 12.9; nothing is borrowed from CUTLASS.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cuda.h>
#include <cuda_runtime.h>

#ifndef TB_SPIN_TIMEOUT_NS
#define TB_SPIN_TIMEOUT_NS 300000000000ull   // default 300 s; set at run time with TUTEL_B200_SPIN_TIMEOUT_SEC
#endif

// Every spin-wait (mbarrier pipelines and cross-GPU flags alike: a GEMM whose producer waits for a late peer stalls its
// MMA and epilogue warps on their mbarriers for just as long) is bounded by this run-time value.  It lives in constant
// memory and is only read on the slow path, after a first poll has failed.  One copy per translation unit; the host
// setters (set_spin_timeout_*) keep them in sync.
static __constant__ unsigned long long tb_spin_timeout_ns = TB_SPIN_TIMEOUT_NS;

namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ uint32_t elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred;
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}

__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Arrive on the barrier living at the same smem offset in CTA `cta` of this cluster.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}\n" ::"r"(bar),
      "r"(cta)
      : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done;
}
// Bounded wait: a dead pipeline traps (visible as a CUDA error on the host) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = globaltimer_ns();
  while (!mbar_try_wait(bar, parity)) {
    if (globaltimer_ns() - t0 > tb_spin_timeout_ns) {
      printf("[tutel_b200] mbarrier wait timeout: block %d thread %d bar 0x%x parity %u\n", blockIdx.x,
             threadIdx.x, bar, parity);
      __trap();
    }
  }
}

// Same bound, no message: for kernels that issue wgmma (ptxas serialises the MMAs of a kernel that contains a call,
// and printf is one).
__device__ __forceinline__ void mbar_wait_quiet(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = globaltimer_ns();
  while (!mbar_try_wait(bar, parity)) {
    if (globaltimer_ns() - t0 > tb_spin_timeout_ns) __trap();
  }
}

// ----------------------------------------------------------------------------------------------
// proxies / fences
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_global() {
  asm volatile("fence.proxy.async.global;" ::: "memory");
}
__device__ __forceinline__ void fence_acq_rel_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// system-scope flag primitives (cross-GPU, peer-mapped memory)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_add_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// Mailbox word = (epoch << 32) | payload.  Spin until the epoch field reaches `epoch`; returns the payload.
__device__ __forceinline__ uint32_t wait_mailbox_sys(const unsigned long long* p, uint32_t epoch) {
  unsigned long long v = ld_acquire_sys_u64(p);
  if (static_cast<int32_t>(static_cast<uint32_t>(v >> 32) - epoch) >= 0) return static_cast<uint32_t>(v);
  const uint64_t t0 = globaltimer_ns();
  for (;;) {
    __nanosleep(64);
    v = ld_acquire_sys_u64(p);
    if (static_cast<int32_t>(static_cast<uint32_t>(v >> 32) - epoch) >= 0) return static_cast<uint32_t>(v);
    if (globaltimer_ns() - t0 > tb_spin_timeout_ns) {
      printf("[tutel_b200] peer mailbox wait timeout: block %d mailbox %p have epoch %u want %u\n", blockIdx.x, p,
             static_cast<uint32_t>(v >> 32), epoch);
      __trap();
    }
  }
}

// Spin until *p >= target (monotonic epoch counters; wrap-safe signed compare). Traps on timeout.
__device__ __forceinline__ void wait_flag_ge_sys(const uint32_t* p, uint32_t target) {
  if (static_cast<int32_t>(ld_acquire_sys(p) - target) >= 0) return;
  const uint64_t t0 = globaltimer_ns();
  while (static_cast<int32_t>(ld_acquire_sys(p) - target) < 0) {
    __nanosleep(64);
    if (globaltimer_ns() - t0 > tb_spin_timeout_ns) {
      printf("[tutel_b200] peer flag wait timeout: block %d thread %d flag %p have %u want %u\n", blockIdx.x,
             threadIdx.x, p, ld_relaxed_sys(p), target);
      __trap();
    }
  }
}

// Same without the message (see mbar_wait_quiet), for kernels that issue wgmma.
__device__ __forceinline__ void wait_flag_ge_sys_quiet(const uint32_t* p, uint32_t target) {
  if (static_cast<int32_t>(ld_acquire_sys(p) - target) >= 0) return;
  const uint64_t t0 = globaltimer_ns();
  while (static_cast<int32_t>(ld_acquire_sys(p) - target) < 0) {
    __nanosleep(64);
    if (globaltimer_ns() - t0 > tb_spin_timeout_ns) __trap();
  }
}

// 16-byte streaming global access (peer or local); keeps L1 clean for one-touch data.
__device__ __forceinline__ uint4 ld_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint4 ld_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_na_v4(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tensormap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}

// 3-D tiled load into this CTA's smem, completing on this CTA's mbarrier.
__device__ __forceinline__ void tma_load_3d(uint32_t smem_dst, const void* tmap, uint32_t bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// Plain (non-tensor) bulk copy global -> this CTA's smem, completing on this CTA's mbarrier: `bytes` a multiple of 16,
// both addresses 16-byte aligned.
__device__ __forceinline__ void bulk_load(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_dst),
               "l"(gsrc), "r"(bytes), "r"(bar)
               : "memory");
}
// Ask the L2 to fetch `bytes` (multiple of 16) starting at a 16-byte aligned global address.
__device__ __forceinline__ void prefetch_l2_bulk(const void* gptr, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gptr), "r"(bytes) : "memory");
}

// Tensor store smem -> global (bulk async group of the issuing thread); out-of-range rows / columns are clipped.
__device__ __forceinline__ void tma_store_3d(const void* tmap, uint32_t smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(tmap),
               "r"(smem_src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// Wait until at most N of this thread's bulk groups are still reading their shared-memory source ...
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// ... or are still in flight at all.
template <int N>
__device__ __forceinline__ void bulk_wait_group() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// Named barrier over `count` threads (a multiple of 32), id 1..15 (0 is __syncthreads).
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// Four fp32 adds to consecutive, 16-byte aligned global words, result unused.
__device__ __forceinline__ void red_add_v4_f32(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma: warpgroup-wide asynchronous MMA, operands in shared memory, fp32 accumulator fragment in registers.
// One m64n128 instruction leaves 64 floats per thread: d[4j + {0,1}] = row (warp % 4) * 16 + lane / 4, columns
// 8j + 2 * (lane % 4) + {0,1};  d[4j + {2,3}] = the same columns eight rows further down.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

enum WgmmaType : int { WG_BF16 = 0, WG_FP16 = 1, WG_E4M3 = 3, WG_E5M2 = 4 };   // values of tb::GemmDtype

#define TB_ACC8(d, o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
#define TB_ACC64(d) TB_ACC8(d, 0), TB_ACC8(d, 8), TB_ACC8(d, 16), TB_ACC8(d, 24), TB_ACC8(d, 32), TB_ACC8(d, 40), TB_ACC8(d, 48), TB_ACC8(d, 56)
#define TB_D64 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define TB_WGMMA16(TYPES)                                                                                       \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                               \
               "wgmma.mma_async.sync.aligned.m64n128k16.f32." TYPES " " TB_D64 ", %64, %65, p, 1, 1, %67, %68;\n\t}\n" \
               : TB_ACC64(d)                                                                                    \
               : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA ? 1 : 0), "n"(TB ? 1 : 0))
#define TB_WGMMA8(TYPES)                                                                                        \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                               \
               "wgmma.mma_async.sync.aligned.m64n128k32.f32." TYPES " " TB_D64 ", %64, %65, p, 1, 1;\n\t}\n"      \
               : TB_ACC64(d)                                                                                    \
               : "l"(adesc), "l"(bdesc), "r"(accumulate))

// d (+)= A[64 x K] * B[K x 128], K = 16 (16-bit types) or 32 (8-bit types, K-major only).  TA / TB: the operand is
// MN-major in shared memory (16-bit types only).
template <int T, bool TA, bool TB>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  static_assert(T == WG_BF16 || T == WG_FP16 || (!TA && !TB), "8-bit operands are K-major only");
  if constexpr (T == WG_BF16) TB_WGMMA16("bf16.bf16");
  else if constexpr (T == WG_FP16) TB_WGMMA16("f16.f16");
  else if constexpr (T == WG_E4M3) TB_WGMMA8("e4m3.e4m3");
  else TB_WGMMA8("e5m2.e5m2");
}
#undef TB_WGMMA16
#undef TB_WGMMA8

// m64n256: 128 floats per thread, same fragment layout with j = 0..31.
#define TB_ACC64O(d, o) TB_ACC8(d, o), TB_ACC8(d, o + 8), TB_ACC8(d, o + 16), TB_ACC8(d, o + 24), TB_ACC8(d, o + 32), TB_ACC8(d, o + 40), TB_ACC8(d, o + 48), TB_ACC8(d, o + 56)
#define TB_D128 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
#define TB_WGMMA16(TYPES)                                                                                        \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"                                               \
               "wgmma.mma_async.sync.aligned.m64n256k16.f32." TYPES " " TB_D128 ", %128, %129, p, 1, 1, %131, %132;\n\t}\n" \
               : TB_ACC64O(d, 0), TB_ACC64O(d, 64)                                                               \
               : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA ? 1 : 0), "n"(TB ? 1 : 0))
#define TB_WGMMA8(TYPES)                                                                                         \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"                                               \
               "wgmma.mma_async.sync.aligned.m64n256k32.f32." TYPES " " TB_D128 ", %128, %129, p, 1, 1;\n\t}\n"      \
               : TB_ACC64O(d, 0), TB_ACC64O(d, 64)                                                               \
               : "l"(adesc), "l"(bdesc), "r"(accumulate))

// d (+)= A[64 x K] * B[K x 256]; operand rules of wgmma_m64n128.
template <int T, bool TA, bool TB>
__device__ __forceinline__ void wgmma_m64n256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  static_assert(T == WG_BF16 || T == WG_FP16 || (!TA && !TB), "8-bit operands are K-major only");
  if constexpr (T == WG_BF16) TB_WGMMA16("bf16.bf16");
  else if constexpr (T == WG_FP16) TB_WGMMA16("f16.f16");
  else if constexpr (T == WG_E4M3) TB_WGMMA8("e4m3.e4m3");
  else TB_WGMMA8("e5m2.e5m2");
}
#undef TB_WGMMA16
#undef TB_WGMMA8
#undef TB_D128
#undef TB_ACC64O
#undef TB_D64
#undef TB_ACC64
#undef TB_ACC8

template <int NREG> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(NREG)); }
template <int NREG> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(NREG)); }

// ----------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor, 128-byte swizzle.
//   bits [0,14)  start address >> 4      bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4 bits [62,64) layout (1 = SWIZZLE_128B)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes,
                                                         uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

}  // namespace ptx
