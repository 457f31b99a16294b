// Fused gating + routing for sm_90a: TWO launches take the gate logits to everything the dispatch needs.
//
// The reference spends ~15 PyTorch kernels on softmax / top-k / one-hot masks / GShard loss / gate normalisation
// (tutel/impls/moe_layer.py:283-305, tutel/impls/losses.py:12-19) and k cumsum passes + k compares on the locations
// (tutel/impls/fast_dispatch.py:143-204, `tutel_ops.cumsum` tutel/custom/custom_kernel.cpp:822-872).  Here:
//
//   gate_route_kernel    one warp per token: softmax in registers, iterative arg-max top-k, gate normalisation, the
//                        per-block histogram of every choice (the routing scan's input), per-block importance sums
//                        for the loss; the grid also pre-fills the slot map with -1.
//   route_finish_kernel  one thread per token: every block derives its own queue offsets from the block histograms
//                        (no separate scan launch), ranks its tokens (match.any), writes locations and the inverse
//                        slot -> (token, choice) map; block 0 also emits the per-expert counts and the auxiliary loss.
//
// Backward of the whole gate is ONE kernel (closed form through normalisation, top-k selection and softmax).
//
// Both gate kernels and route_finish_kernel also have a sigmoid instantiation (SIGMOID = true, DeepSeek-V3 routing):
// scores sigmoid(z), selection on score + per-expert bias, optionally limited to the best `topk_group` of `n_group`
// expert groups, gates from the unbiased scores times `routed_scaling_factor`, and the balance loss
// E / (k S^2) sum_e n_e sum_s s_se / T_s on all-choice counts n_e.  expert_bias_update_kernel applies the
// auxiliary-loss-free balancing step to the bias.
// Also here: grouped column sums (bias gradients at copy bandwidth) and the public `fast_cumsum_sub_one` scan.
#include "moe_kernels.h"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "ptx.cuh"

namespace tb {
namespace {

constexpr int kTileTokens = 256;      // tokens per routing tile (histogram granularity)
constexpr int kGateThreads = 1024;    // gate kernel: 32 warps, 8 tokens per warp
constexpr int kInvalidLoc = 0x3fffffff;

template <typename T> __device__ __forceinline__ float ldf(const T* p);
template <> __device__ __forceinline__ float ldf<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ldf<__half>(const __half* p) { return __half2float(*p); }
template <> __device__ __forceinline__ float ldf<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <typename T> __device__ __forceinline__ void stf(T* p, float v);
template <> __device__ __forceinline__ void stf<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void stf<__half>(__half* p, float v) { *p = __float2half_rn(v); }
template <> __device__ __forceinline__ void stf<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

// Parameters of the sigmoid instantiations (ignored by the softmax ones).
struct SigmoidArgs {
  const float* bias;     // [E] selection bias (e_score_correction_bias)
  float* load;           // [E] += all-choice counts of this call, or null
  int n_group;           // expert groups; 1 = no group limit
  int topk_group;        // groups a token may choose from
  float scale;           // routed_scaling_factor
};

// Group-limited selection, one warp per token: the score of group g (experts [g*E/n_group, (g+1)*E/n_group)) is the
// sum of its top min(2, E/n_group) keys, lane g computes it from the warp's key row in shared memory; the best
// `topk_group` groups are picked by iterative arg-max (ties -> lower group id; NaN / -inf keys and group scores never
// win against the -inf sentinel).  Returns the lane's experts outside the kept groups as a bit mask over i
// (bit i: expert lane + 32 i), ready to be OR-ed into the top-k loop's `taken` mask.
template <int VPT>
__device__ __forceinline__ unsigned excluded_by_groups(const float* sm_key, int E, int n_group, int topk_group,
                                                       int lane) {
  const int gsz = E / n_group;
  float gs = -INFINITY;
  if (lane < n_group) {
    float b1 = -INFINITY, b2 = -INFINITY;
#pragma unroll 1                    // (unrolled, the group loops push the 16-value instantiations into spills)
    for (int e = lane * gsz; e < (lane + 1) * gsz; ++e) {
      const float key = sm_key[e];
      if (key > b1) { b2 = b1; b1 = key; }
      else if (key > b2) b2 = key;
    }
    gs = gsz > 1 ? b1 + b2 : b1;
  }
  unsigned kept = 0;
#pragma unroll 1
  for (int t = 0; t < topk_group; ++t) {
    float best = ((kept >> lane) & 1u) ? -INFINITY : gs;
    int best_g = best > -INFINITY ? lane : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int og = __shfl_xor_sync(0xffffffffu, best_g, o);
      if (ob > best || (ob == best && og < best_g)) { best = ob; best_g = og; }
    }
    if (best_g >= 32) break;
    kept |= 1u << best_g;
  }
  unsigned excluded = 0;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int e = lane + 32 * i;
    if (e < E && !((kept >> (e / gsz)) & 1u)) excluded |= 1u << i;
  }
  return excluded;
}

// ------------------------------------------------------------------------------------------------
// launch 1: softmax + top-k + normalised gates + per-tile histograms / importance sums (+ slot map pre-fill)
// ------------------------------------------------------------------------------------------------
template <typename T, int VPT, bool SIGMOID>
__global__ void __launch_bounds__(kGateThreads)
gate_route_kernel(const T* __restrict__ logits, float* __restrict__ scores, int* __restrict__ idx,
                  float* __restrict__ top, float* __restrict__ gates, float* __restrict__ me_partial,
                  int* __restrict__ hist, int* __restrict__ slot_src, long long slot_n, int S, int E, int k,
                  int normalize, float eps, SigmoidArgs sg) {
  // [k * E] histogram, then [E] floats of importance sums; sigmoid: then [E] bias and a [32][E] key row per warp
  extern __shared__ int sm_dyn[];
  int* sm_hist = sm_dyn;
  float* sm_me = reinterpret_cast<float*>(sm_dyn + k * E);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  float* sm_bias = sm_me + E;
  float* sm_s = sm_bias + E + warp * E;
  for (int i = threadIdx.x; i < k * E; i += kGateThreads) sm_hist[i] = 0;
  for (int i = threadIdx.x; i < E; i += kGateThreads) sm_me[i] = 0.0f;
  if constexpr (SIGMOID)
    for (int i = threadIdx.x; i < E; i += kGateThreads) sm_bias[i] = sg.bias[i];
  for (long long i = static_cast<long long>(blockIdx.x) * kGateThreads + threadIdx.x; i < slot_n;
       i += static_cast<long long>(gridDim.x) * kGateThreads)
    slot_src[i] = -1;
  __syncthreads();

  float me[VPT];
#pragma unroll
  for (int i = 0; i < VPT; ++i) me[i] = 0.0f;
  const long long s_begin = static_cast<long long>(blockIdx.x) * kTileTokens;
  const long long s_end = min(s_begin + kTileTokens, static_cast<long long>(S));
  for (long long s = s_begin + warp; s < s_end; s += kGateThreads / 32) {
    float v[VPT];
    if constexpr (!SIGMOID) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < VPT; ++i) {
        const int e = lane + 32 * i;
        v[i] = e < E ? ldf<T>(logits + s * E + e) : -INFINITY;
        mx = fmaxf(mx, v[i]);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float sum = 0.0f;
#pragma unroll
      for (int i = 0; i < VPT; ++i) {
        v[i] = (lane + 32 * i < E) ? expf(v[i] - mx) : 0.0f;
        sum += v[i];
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      const float inv = 1.0f / sum;
#pragma unroll
      for (int i = 0; i < VPT; ++i) {
        const int e = lane + 32 * i;
        v[i] *= inv;
        if (e < E) {
          scores[s * E + e] = v[i];
          me[i] += v[i];
        }
      }
    } else {
      // v = sigmoid(z); me += v / T_s; the selection keys v + bias go to the warp's shared row (read by the group
      // scores and the top-k loop: at 16 values per lane, registers for both v and me would spill)
      float tsum = 0.0f;
#pragma unroll
      for (int i = 0; i < VPT; ++i) {
        const int e = lane + 32 * i;
        v[i] = 0.0f;
        if (e < E) {
          v[i] = 1.0f / (1.0f + expf(-ldf<T>(logits + s * E + e)));
          scores[s * E + e] = v[i];
        }
        tsum += v[i];
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) tsum += __shfl_xor_sync(0xffffffffu, tsum, o);
      const float inv = 1.0f / tsum;
#pragma unroll
      for (int i = 0; i < VPT; ++i) {
        const int e = lane + 32 * i;
        if (e < E) {
          me[i] += v[i] * inv;
          sm_s[e] = v[i] + sm_bias[e];
        }
      }
      __syncwarp();
    }
    // iterative arg-max (ties -> lower expert id); lane j keeps the j-th choice
    unsigned taken = 0;
    if constexpr (SIGMOID)
      if (sg.n_group > 1) taken = excluded_by_groups<VPT>(sm_s, E, sg.n_group, sg.topk_group, lane);
    float mine = 0.0f;
    int mine_e = -1;
    for (int j = 0; j < k; ++j) {
      float best = SIGMOID ? -INFINITY : -1.0f;     // sigmoid keys can be negative (the bias can be)
      int best_e = 0x7fffffff;
#pragma unroll
      for (int i = 0; i < VPT; ++i) {
        const int e = lane + 32 * i;
        const float key = SIGMOID ? (e < E ? sm_s[e] : 0.0f) : v[i];
        if (e < E && !((taken >> i) & 1u) && (key > best)) { best = key; best_e = e; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oe = __shfl_xor_sync(0xffffffffu, best_e, o);
        if (ob > best || (ob == best && oe < best_e)) { best = ob; best_e = oe; }
      }
      if ((best_e & 31) == lane && best_e < E) {
        taken |= 1u << (best_e >> 5);
        atomicAdd(&sm_hist[j * E + best_e], 1);
      }
      if (lane == j) { mine = best; mine_e = best_e; }
    }
    if constexpr (SIGMOID) mine = (lane < k && mine_e >= 0 && mine_e < E) ? scores[s * E + mine_e] : 0.0f;   // unbiased
    float denom = (lane < k) ? mine : 0.0f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) denom += __shfl_xor_sync(0xffffffffu, denom, o);
    if (lane < k) {
      float g = (normalize != 0 && k > 1) ? mine / fmaxf(denom, eps) : mine;
      if constexpr (SIGMOID) g *= sg.scale;
      idx[static_cast<long long>(lane) * S + s] = mine_e;
      top[static_cast<long long>(lane) * S + s] = mine;
      gates[static_cast<long long>(lane) * S + s] = g;
    }
    if constexpr (SIGMOID) __syncwarp();          // the next token overwrites this warp's score row
  }
#pragma unroll
  for (int i = 0; i < VPT; ++i)
    if (lane + 32 * i < E && me[i] != 0.0f) atomicAdd(&sm_me[lane + 32 * i], me[i]);
  __syncthreads();
  for (int i = threadIdx.x; i < k * E; i += kGateThreads) hist[static_cast<long long>(blockIdx.x) * k * E + i] = sm_hist[i];
  for (int i = threadIdx.x; i < E; i += kGateThreads) me_partial[static_cast<long long>(blockIdx.x) * E + i] = sm_me[i];
}

// ------------------------------------------------------------------------------------------------
// launch 2: queue offsets from the tile histograms, in-tile ranking, locations, slot map, counts, loss
// ------------------------------------------------------------------------------------------------
// Sigmoid mode: the loss, ce_out and `load` use the all-choice counts n_e, me_partial holds sums of s_se / T_s.
template <typename T, bool SIGMOID>
__global__ void __launch_bounds__(kTileTokens)
route_finish_kernel(const int* __restrict__ idx, const int* __restrict__ hist, const float* __restrict__ me_partial,
                    int* __restrict__ loc, int* __restrict__ counts, int* __restrict__ slot_src,
                    float* __restrict__ ce_out, T* __restrict__ l_aux, int S, int E, int k, int C, int ntiles,
                    float* __restrict__ load) {
  extern __shared__ int sm_dyn[];        // total[k*E] | base[k*E] | cnt[E]
  int* sm_total = sm_dyn;
  int* sm_base = sm_dyn + k * E;
  int* sm_cnt = sm_dyn + 2 * k * E;
  __shared__ float sm_red[kTileTokens / 32];
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // (1) per (choice, expert): tokens in all tiles / in the tiles before this one
  for (int p = threadIdx.x; p < k * E; p += kTileTokens) {
    int total = 0, before = 0;
    for (int t = 0; t < ntiles; ++t) {
      const int h = hist[static_cast<long long>(t) * k * E + p];
      total += h;
      before += (t < b) ? h : 0;
    }
    sm_total[p] = total;
    sm_base[p] = before;
  }
  __syncthreads();
  // (2) choice j queues behind ALL (j-1)-th choices (tutel/impls/fast_dispatch.py:160-166)
  for (int p = threadIdx.x; p < k * E; p += kTileTokens) {
    const int j = p / E, e = p - j * E;
    int prior = 0;
    for (int jj = 0; jj < j; ++jj) prior += sm_total[jj * E + e];
    sm_base[p] += prior;       // own slot only: no other thread reads sm_base[p] before the barrier below
  }
  __syncthreads();
  if (b == 0) {
    // per-expert token counts, first-choice counts (fp32, for the backward pass) and the GShard loss
    float part = 0.0f;
    for (int e = threadIdx.x; e < E; e += kTileTokens) {
      int c = 0;
      for (int j = 0; j < k; ++j) c += sm_total[j * E + e];
      counts[e] = c;
      const float ce = static_cast<float>(SIGMOID ? c : sm_total[e]);
      if (ce_out != nullptr) ce_out[e] = ce;
      if constexpr (SIGMOID)
        if (load != nullptr) load[e] += ce;
      float me = 0.0f;
      for (int t = 0; t < ntiles; ++t) me += me_partial[static_cast<long long>(t) * E + e];
      part += me * ce;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == 0) sm_red[warp] = part;
    __syncthreads();
    if (threadIdx.x == 0 && l_aux != nullptr) {
      float tot = 0.0f;
      for (int w = 0; w < kTileTokens / 32; ++w) tot += sm_red[w];
      const float ss = static_cast<float>(S) * static_cast<float>(S);
      stf<T>(l_aux, tot * static_cast<float>(E) / (SIGMOID ? static_cast<float>(k) * ss : ss));
    }
  }
  // (3) stable rank of every token inside its tile, choice by choice
  const int s = b * kTileTokens + threadIdx.x;
  for (int j = 0; j < k; ++j) {
    for (int e = threadIdx.x; e < E; e += kTileTokens) sm_cnt[e] = 0;
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
    for (int w = 0; w < kTileTokens / 32; ++w) {
      if (warp == w && e >= 0 && lane == leader) {
        base = sm_cnt[e];
        sm_cnt[e] = base + __popc(peers);
      }
      __syncthreads();
    }
    base = __shfl_sync(0xffffffffu, base, leader);
    if (s < S) {
      int l = kInvalidLoc;
      if (e >= 0) {
        l = sm_base[j * E + e] + base + rank_in_warp;
        if (slot_src != nullptr && l < C) slot_src[static_cast<long long>(e) * C + l] = s * k + j;
      }
      loc[static_cast<long long>(j) * S + s] = l;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// gate backward (one warp per token), dgates fp32 [k,S], dl / dlogits in the logits' dtype:
//   r_j  = p[idx_j], D = sum_j r_j, Dc = max(D, eps);  g_j = r_j / Dc (normalize && k>1)
//   dr_j = dg_j / Dc - [D > eps] * (sum_i dg_i r_i) / Dc^2
//   dp_e = dl * ce_e * E / S^2 + sum_j [idx_j == e] dr_j        (l_aux = E/S^2 * sum_e me_e ce_e; ce is constant)
//   dlogit_e = p_e * (dp_e - sum_e' dp_e' p_e')
// Sigmoid (p = sigmoid scores, ce = all-choice counts n, T = sum_e p_e, l_aux = E/(k S^2) sum_e n_e sum_s p_se / T_s):
//   dr_j scaled by routed_scaling_factor
//   dp_e = dl E / (k S^2 T) * (n_e - sum_e' n_e' p_e' / T) + sum_j [idx_j == e] dr_j
//   dlogit_e = p_e (1 - p_e) dp_e
// ------------------------------------------------------------------------------------------------
template <typename T, int VPT, bool SIGMOID>
__global__ void __launch_bounds__(256)
gate_route_bwd_kernel(const float* __restrict__ scores, const int* __restrict__ idx, const float* __restrict__ top,
                      const float* __restrict__ dgates, const float* __restrict__ ce, const T* __restrict__ dl,
                      T* __restrict__ dlogits, int S, int E, int k, int normalize, float eps, float scale) {
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const float ss = static_cast<float>(S) * static_cast<float>(S);
  const float aux_scale = (dl != nullptr ? ldf<T>(dl) : 0.0f) * static_cast<float>(E) /
                          (SIGMOID ? static_cast<float>(k) * ss : ss);
  for (long long s = static_cast<long long>(blockIdx.x) * 8 + warp; s < S; s += static_cast<long long>(gridDim.x) * 8) {
    float p[VPT], dp[VPT];
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int e = lane + 32 * i;
      p[i] = e < E ? scores[s * E + e] : 0.0f;
      if constexpr (SIGMOID) dp[i] = (e < E && ce != nullptr) ? ce[e] : 0.0f;
      else dp[i] = (e < E && ce != nullptr) ? aux_scale * ce[e] : 0.0f;
    }
    if constexpr (SIGMOID) {
      if (ce != nullptr) {
        float t = 0.0f, nd = 0.0f;
#pragma unroll
        for (int i = 0; i < VPT; ++i) {
          t += p[i];
          nd += dp[i] * p[i];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          t += __shfl_xor_sync(0xffffffffu, t, o);
          nd += __shfl_xor_sync(0xffffffffu, nd, o);
        }
        const float c = aux_scale / t, m = nd / t;
#pragma unroll
        for (int i = 0; i < VPT; ++i) dp[i] = c * (dp[i] - m);
      }
    }
    // lane j owns choice j
    const float r = lane < k ? top[static_cast<long long>(lane) * S + s] : 0.0f;
    const float dg = (lane < k && dgates != nullptr) ? dgates[static_cast<long long>(lane) * S + s] : 0.0f;
    const int my_e = lane < k ? idx[static_cast<long long>(lane) * S + s] : -1;
    float D = r, dot = dg * r;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      D += __shfl_xor_sync(0xffffffffu, D, o);
      dot += __shfl_xor_sync(0xffffffffu, dot, o);
    }
    float dr = dg;
    if (normalize != 0 && k > 1) {
      const float Dc = fmaxf(D, eps);
      dr = dg / Dc - (D > eps ? dot / (Dc * Dc) : 0.0f);
    }
    if constexpr (SIGMOID) dr *= scale;
    for (int j = 0; j < k; ++j) {
      const int e = __shfl_sync(0xffffffffu, my_e, j);
      const float d = __shfl_sync(0xffffffffu, dr, j);
      if (e >= 0 && (e & 31) == lane) {
#pragma unroll
        for (int i = 0; i < VPT; ++i)
          if (i == (e >> 5)) dp[i] += d;
      }
    }
    if constexpr (SIGMOID) {
#pragma unroll
      for (int i = 0; i < VPT; ++i) {
        const int e = lane + 32 * i;
        if (e < E) stf<T>(dlogits + s * E + e, p[i] * (1.0f - p[i]) * dp[i]);
      }
      continue;
    }
    float acc = 0.0f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) acc += dp[i] * p[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int e = lane + 32 * i;
      if (e < E) stf<T>(dlogits + s * E + e, p[i] * (dp[i] - acc));
    }
  }
}

// ------------------------------------------------------------------------------------------------
// auxiliary-loss-free balancing: bias_e += gamma * sign(mean(load) - load_e), then load = 0.  One block; the loads are
// integer-valued, so their fp32 sum is exact (below 2^24) and the result does not depend on the summation order.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
expert_bias_update_kernel(float* __restrict__ bias, float* __restrict__ load, int E, float gamma) {
  __shared__ float sm_red[32];
  float part = 0.0f;
  for (int e = threadIdx.x; e < E; e += 1024) part += load[e];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if ((threadIdx.x & 31) == 0) sm_red[threadIdx.x >> 5] = part;
  __syncthreads();
  float tot = 0.0f;
  for (int w = 0; w < 32; ++w) tot += sm_red[w];
  const float mean = tot / static_cast<float>(E);
  for (int e = threadIdx.x; e < E; e += 1024) {
    const float d = mean - load[e];
    bias[e] = bias[e] + gamma * static_cast<float>((d > 0.0f) - (d < 0.0f));
    load[e] = 0.0f;
  }
}

// ------------------------------------------------------------------------------------------------
// grouped column sums: out[g, n] = sum_t x[g, t, n]   (bias gradients), 16-byte loads, fp32 accumulate
// ------------------------------------------------------------------------------------------------
template <typename T> struct V16;
template <> struct V16<float> {
  static constexpr int N = 4;
  static __device__ __forceinline__ void add(const uint4& u, float* a) {
    a[0] += __uint_as_float(u.x); a[1] += __uint_as_float(u.y); a[2] += __uint_as_float(u.z); a[3] += __uint_as_float(u.w);
  }
};
template <> struct V16<__half> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void add(const uint4& u, float* a) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
      a[2 * i] += t.x; a[2 * i + 1] += t.y;
    }
  }
};
template <> struct V16<__nv_bfloat16> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void add(const uint4& u, float* a) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      a[2 * i] += __uint_as_float(w[i] << 16);
      a[2 * i + 1] += __uint_as_float(w[i] & 0xFFFF0000u);
    }
  }
};

// block = 256 threads = 16 row-lanes x 16 column-lanes; a block owns a strip of 16 * V columns of one group and the rows
// [split * rows_per_split, ...).  Each thread keeps 4 independent 16-byte loads in flight.
template <typename T, bool OFFS>
__global__ void __launch_bounds__(256)
colsum_kernel(const T* __restrict__ x, long long ld, long long group_stride, T* __restrict__ out, float* __restrict__ acc_out,
              int rows, int N, int rows_per_split, const int* __restrict__ offsets) {
  constexpr int V = V16<T>::N;
  __shared__ float sm[16][16 * V + 1];
  const int cl = threadIdx.x & 15;
  const int rl = threadIdx.x >> 4;
  const int col = (blockIdx.x * 16 + cl) * V;
  const int g = blockIdx.z;
  int r_lo = 0, r_hi = rows;
  if (OFFS) {   // segment g of one [rows, N] tensor, split evenly over the blocks of its strip
    r_lo = offsets[g];
    r_hi = min(rows, offsets[g + 1]);
    rows_per_split = (max(r_hi - r_lo, 0) + static_cast<int>(gridDim.y) - 1) / static_cast<int>(gridDim.y);
  }
  const int r_begin = r_lo + blockIdx.y * rows_per_split;
  const int r_end = min(r_hi, r_begin + rows_per_split);
  float a[V];
#pragma unroll
  for (int i = 0; i < V; ++i) a[i] = 0.0f;
  if (col < N) {
    const T* base = x + (OFFS ? 0LL : static_cast<long long>(g) * group_stride) + col;
    int r = r_begin + rl;
    for (; r + 48 < r_end; r += 64) {
      uint4 u[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) u[q] = ptx::ld_nc_v4(base + static_cast<long long>(r + 16 * q) * ld);
#pragma unroll
      for (int q = 0; q < 4; ++q) V16<T>::add(u[q], a);
    }
    for (; r < r_end; r += 16) V16<T>::add(ptx::ld_nc_v4(base + static_cast<long long>(r) * ld), a);
  }
#pragma unroll
  for (int i = 0; i < V; ++i) sm[rl][cl * V + i] = a[i];
  __syncthreads();
  for (int c = threadIdx.x; c < 16 * V; c += 256) {
    float t = 0.0f;
#pragma unroll
    for (int q = 0; q < 16; ++q) t += sm[q][c];
    const int n = blockIdx.x * 16 * V + c;
    if (n < N) {
      if (acc_out != nullptr) atomicAdd(acc_out + static_cast<long long>(g) * N + n, t);
      else stf<T>(out + static_cast<long long>(g) * N + n, t);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// public column scan (`tutel.moe.fast_cumsum_sub_one`): out[s, e] = sum_{s' <= s} in[s', e] - 1
// three linear passes over row tiles: tile sums, exclusive scan of the tile sums, in-tile scan
// ------------------------------------------------------------------------------------------------
constexpr int kScanRows = 32;

__global__ void __launch_bounds__(128)
cumsum_tile_kernel(const int* __restrict__ in, int* __restrict__ out, int* __restrict__ tile_sums, int S, int E,
                   int tiles_per_block, int apply) {
  const int ecols = E < 128 ? E : 128;
  const int tl = threadIdx.x / ecols;
  const int e = blockIdx.x * ecols + (threadIdx.x - tl * ecols);
  const long long tile = static_cast<long long>(blockIdx.y) * tiles_per_block + tl;
  if (tl >= tiles_per_block || e >= E || tile * kScanRows >= S) return;
  const int r0 = static_cast<int>(tile) * kScanRows;
  const int r1 = min(S, r0 + kScanRows);
  int run = apply ? tile_sums[tile * E + e] - 1 : 0;
  for (int r = r0; r < r1; ++r) {
    run += in[static_cast<long long>(r) * E + e];
    if (apply) out[static_cast<long long>(r) * E + e] = run;
  }
  if (!apply) tile_sums[tile * E + e] = run;
}

__global__ void __launch_bounds__(128)
cumsum_scan_kernel(int* __restrict__ tile_sums, int ntiles, int E) {
  const int e = blockIdx.x * 128 + threadIdx.x;
  if (e >= E) return;
  int run = 0;
  for (int t = 0; t < ntiles; ++t) {
    const int v = tile_sums[static_cast<long long>(t) * E + e];
    tile_sums[static_cast<long long>(t) * E + e] = run;
    run += v;
  }
}

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

}  // namespace

int gate_route_tiles(int S) { return (S + kTileTokens - 1) / kTileTokens; }

// Dynamic shared memory above the default 48 KB needs an opt-in per kernel (both launches grow with k * E: at E = 512
// and k = 32 the histograms take 68 KB and 133 KB).
static cudaError_t allow_dynamic_smem(const void* fn, size_t bytes) {
  if (bytes <= 48 * 1024) return cudaSuccess;
  int dev = 0, optin = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (e != cudaSuccess) return e;
  if (bytes > static_cast<size_t>(optin)) return cudaErrorInvalidValue;
  return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
}

template <typename T, bool SIGMOID>
static cudaError_t gate_route_forward_t(const void* logits, float* scores, int* idx, float* top, float* gates,
                                        float* me_partial, int* hist, int* loc, int* counts, int* slot_src,
                                        float* ce_out, void* l_aux, int S, int E, int k, int C, bool normalize, float eps,
                                        const SigmoidArgs& sg, cudaStream_t stream) {
  const int ntiles = gate_route_tiles(S);
  const long long slot_n = slot_src != nullptr ? static_cast<long long>(E) * C : 0;
  const size_t smem1 = sizeof(int) * static_cast<size_t>(k) * E + sizeof(float) * E +
                       (SIGMOID ? sizeof(float) * E * (1 + kGateThreads / 32) : 0);
  const size_t smem2 = sizeof(int) * (2 * static_cast<size_t>(k) * E + E);
  cudaError_t err = allow_dynamic_smem(reinterpret_cast<const void*>(route_finish_kernel<T, SIGMOID>), smem2);
  if (err != cudaSuccess) return err;
#define TB_GR(VPTv)                                                                                                   \
  do {                                                                                                                \
    const void* fn = reinterpret_cast<const void*>(gate_route_kernel<T, VPTv, SIGMOID>);                              \
    if ((err = allow_dynamic_smem(fn, smem1)) != cudaSuccess) return err;                                             \
    gate_route_kernel<T, VPTv, SIGMOID><<<ntiles, kGateThreads, smem1, stream>>>(                                     \
        static_cast<const T*>(logits), scores, idx, top, gates, me_partial, hist, slot_src, slot_n, S, E, k,          \
        normalize ? 1 : 0, eps, sg);                                                                                  \
  } while (0)
  if (E <= 32) TB_GR(1);
  else if (E <= 64) TB_GR(2);
  else if (E <= 128) TB_GR(4);
  else if (E <= 256) TB_GR(8);
  else if (E <= 512) TB_GR(16);
  else return cudaErrorInvalidValue;
#undef TB_GR
  route_finish_kernel<T, SIGMOID><<<ntiles, kTileTokens, smem2, stream>>>(idx, hist, me_partial, loc, counts, slot_src,
                                                                          ce_out, static_cast<T*>(l_aux), S, E, k, C,
                                                                          ntiles, sg.load);
  return cudaGetLastError();
}

cudaError_t gate_route_forward(const void* logits, float* scores, int* idx, float* top, float* gates, float* me_partial,
                               int* hist, int* loc, int* counts, int* slot_src, float* ce_out, void* l_aux, int S, int E,
                               int k, int C, bool normalize, float eps, int elem_type, cudaStream_t stream) {
  if (S <= 0 || k > 32 || k <= 0) return cudaErrorInvalidValue;
  const SigmoidArgs sg{nullptr, nullptr, 1, 1, 1.0f};
  switch (elem_type) {
    case ET_F32: return gate_route_forward_t<float, false>(logits, scores, idx, top, gates, me_partial, hist, loc, counts, slot_src, ce_out, l_aux, S, E, k, C, normalize, eps, sg, stream);
    case ET_F16: return gate_route_forward_t<__half, false>(logits, scores, idx, top, gates, me_partial, hist, loc, counts, slot_src, ce_out, l_aux, S, E, k, C, normalize, eps, sg, stream);
    case ET_BF16: return gate_route_forward_t<__nv_bfloat16, false>(logits, scores, idx, top, gates, me_partial, hist, loc, counts, slot_src, ce_out, l_aux, S, E, k, C, normalize, eps, sg, stream);
  }
  return cudaErrorInvalidValue;
}

cudaError_t sigmoid_gate_route_forward(const void* logits, const float* bias, float* scores, int* idx, float* top,
                                       float* gates, float* me_partial, int* hist, int* loc, int* counts, int* slot_src,
                                       float* ce_out, void* l_aux, float* load, int S, int E, int k, int C,
                                       bool normalize, float eps, int n_group, int topk_group, float scale,
                                       int elem_type, cudaStream_t stream) {
  if (S <= 0 || k > 32 || k <= 0 || bias == nullptr) return cudaErrorInvalidValue;
  if (n_group < 1 || n_group > 32 || E % n_group != 0 || topk_group < 1 || topk_group > n_group ||
      k > topk_group * (E / n_group))
    return cudaErrorInvalidValue;
  const SigmoidArgs sg{bias, load, n_group, topk_group, scale};
  switch (elem_type) {
    case ET_F32: return gate_route_forward_t<float, true>(logits, scores, idx, top, gates, me_partial, hist, loc, counts, slot_src, ce_out, l_aux, S, E, k, C, normalize, eps, sg, stream);
    case ET_F16: return gate_route_forward_t<__half, true>(logits, scores, idx, top, gates, me_partial, hist, loc, counts, slot_src, ce_out, l_aux, S, E, k, C, normalize, eps, sg, stream);
    case ET_BF16: return gate_route_forward_t<__nv_bfloat16, true>(logits, scores, idx, top, gates, me_partial, hist, loc, counts, slot_src, ce_out, l_aux, S, E, k, C, normalize, eps, sg, stream);
  }
  return cudaErrorInvalidValue;
}

template <typename T, bool SIGMOID>
static cudaError_t gate_route_backward_t(const float* scores, const int* idx, const float* top, const float* dgates,
                                         const float* ce, const void* dl, void* dlogits, int S, int E, int k,
                                         bool normalize, float eps, float scale, cudaStream_t stream) {
  const long long want = (static_cast<long long>(S) + 7) / 8;
  const int grid = static_cast<int>(want < 4LL * sm_count() ? want : 4LL * sm_count());
#define TB_GRB(VPTv)                                                                                             \
  gate_route_bwd_kernel<T, VPTv, SIGMOID><<<grid, 256, 0, stream>>>(scores, idx, top, dgates, ce,                \
                                                                    static_cast<const T*>(dl),                 \
                                                                    static_cast<T*>(dlogits), S, E, k,          \
                                                                    normalize ? 1 : 0, eps, scale)
  if (E <= 32) TB_GRB(1);
  else if (E <= 64) TB_GRB(2);
  else if (E <= 128) TB_GRB(4);
  else if (E <= 256) TB_GRB(8);
  else if (E <= 512) TB_GRB(16);
  else return cudaErrorInvalidValue;
#undef TB_GRB
  return cudaGetLastError();
}

cudaError_t gate_route_backward(const float* scores, const int* idx, const float* top, const float* dgates,
                                const float* ce, const void* dl, void* dlogits, int S, int E, int k, bool normalize,
                                float eps, int elem_type, cudaStream_t stream) {
  if (S <= 0) return cudaSuccess;
  if (k > 32) return cudaErrorInvalidValue;
  switch (elem_type) {
    case ET_F32: return gate_route_backward_t<float, false>(scores, idx, top, dgates, ce, dl, dlogits, S, E, k, normalize, eps, 1.0f, stream);
    case ET_F16: return gate_route_backward_t<__half, false>(scores, idx, top, dgates, ce, dl, dlogits, S, E, k, normalize, eps, 1.0f, stream);
    case ET_BF16: return gate_route_backward_t<__nv_bfloat16, false>(scores, idx, top, dgates, ce, dl, dlogits, S, E, k, normalize, eps, 1.0f, stream);
  }
  return cudaErrorInvalidValue;
}

cudaError_t sigmoid_gate_route_backward(const float* scores, const int* idx, const float* top, const float* dgates,
                                        const float* ce, const void* dl, void* dlogits, int S, int E, int k,
                                        bool normalize, float eps, float scale, int elem_type, cudaStream_t stream) {
  if (S <= 0) return cudaSuccess;
  if (k > 32) return cudaErrorInvalidValue;
  switch (elem_type) {
    case ET_F32: return gate_route_backward_t<float, true>(scores, idx, top, dgates, ce, dl, dlogits, S, E, k, normalize, eps, scale, stream);
    case ET_F16: return gate_route_backward_t<__half, true>(scores, idx, top, dgates, ce, dl, dlogits, S, E, k, normalize, eps, scale, stream);
    case ET_BF16: return gate_route_backward_t<__nv_bfloat16, true>(scores, idx, top, dgates, ce, dl, dlogits, S, E, k, normalize, eps, scale, stream);
  }
  return cudaErrorInvalidValue;
}

cudaError_t expert_bias_update(float* bias, float* load, int E, float gamma, cudaStream_t stream) {
  if (E <= 0) return cudaSuccess;
  expert_bias_update_kernel<<<1, 1024, 0, stream>>>(bias, load, E, gamma);
  return cudaGetLastError();
}

int colsum_row_splits(int G, int rows, int N, int elem_bytes) {
  const int strips = (N + 16 * (16 / elem_bytes) - 1) / (16 * (16 / elem_bytes));
  const long long blocks = static_cast<long long>(strips) * G;
  int splits = 1;
  while (blocks * splits < 2LL * sm_count() && rows / (splits * 2) >= 64) splits *= 2;
  return splits;
}

template <typename T>
static cudaError_t colsum_t(const void* x, long long ld, long long group_stride, void* out, float* acc, int G, int rows,
                            int N, int splits, const int* offsets, cudaStream_t stream) {
  constexpr int V = V16<T>::N;
  const int strips = (N + 16 * V - 1) / (16 * V);
  const int rps = (rows + splits - 1) / splits;
  dim3 grid(strips, splits, G);
  if (offsets != nullptr)
    colsum_kernel<T, true><<<grid, 256, 0, stream>>>(static_cast<const T*>(x), ld, group_stride, static_cast<T*>(out), acc, rows,
                                                     N, rps, offsets);
  else
    colsum_kernel<T, false><<<grid, 256, 0, stream>>>(static_cast<const T*>(x), ld, group_stride, static_cast<T*>(out), acc, rows,
                                                      N, rps, offsets);
  return cudaGetLastError();
}

cudaError_t grouped_colsum(const void* x, long long ld, long long group_stride, void* out, float* acc, int G, int rows,
                           int N, int splits, int elem_type, cudaStream_t stream, const int* offsets) {
  if (G <= 0 || rows <= 0 || N <= 0) return cudaSuccess;
  const int eb = elem_type == ET_F32 ? 4 : 2;
  if ((reinterpret_cast<uintptr_t>(x) & 15) || ((ld * eb) & 15) || ((group_stride * eb) & 15) || (N * eb) % 16)
    return cudaErrorInvalidValue;
  if (splits > 1 && acc == nullptr) return cudaErrorInvalidValue;
  if (splits <= 1) acc = nullptr;
  switch (elem_type) {
    case ET_F32: return colsum_t<float>(x, ld, group_stride, out, acc, G, rows, N, splits, offsets, stream);
    case ET_F16: return colsum_t<__half>(x, ld, group_stride, out, acc, G, rows, N, splits, offsets, stream);
    case ET_BF16: return colsum_t<__nv_bfloat16>(x, ld, group_stride, out, acc, G, rows, N, splits, offsets, stream);
  }
  return cudaErrorInvalidValue;
}

size_t cumsum_workspace_ints(int S, int E) { return static_cast<size_t>((S + kScanRows - 1) / kScanRows) * E; }

cudaError_t cumsum_sub_one(const int* in, int* out, int* workspace, int S, int E, cudaStream_t stream) {
  if (S <= 0 || E <= 0) return cudaSuccess;
  const int ntiles = (S + kScanRows - 1) / kScanRows;
  const int ecols = E < 128 ? E : 128;
  const int tpb = 128 / ecols;
  dim3 grid((E + ecols - 1) / ecols, (ntiles + tpb - 1) / tpb);
  cumsum_tile_kernel<<<grid, 128, 0, stream>>>(in, out, workspace, S, E, tpb, 0);
  cumsum_scan_kernel<<<(E + 127) / 128, 128, 0, stream>>>(workspace, ntiles, E);
  cumsum_tile_kernel<<<grid, 128, 0, stream>>>(in, out, workspace, S, E, tpb, 1);
  return cudaGetLastError();
}

}  // namespace tb
