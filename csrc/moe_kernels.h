// Host API of the routing / sparse dispatch kernels (moe_kernels.cu).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace tb {

enum ElemType : int { ET_F32 = 0, ET_F16 = 1, ET_BF16 = 2, ET_I32 = 3, ET_I64 = 4 };

// Stable slot assignment.  idx: [k, S] int32 expert id of the j-th choice of token s (or <0 = none).
// Produces loc[k, S] (position of the token inside its expert's queue: all 1st choices in token order, then all
// 2nd choices, ... - tutel/impls/fast_dispatch.py:155-171) and counts[E] (tokens routed to e, all choices).
// workspace: int32[ (nblocks + 1) * k * E ], nblocks = ceil(S / 1024).
cudaError_t route_locations(const int* idx, int* loc, int* counts, int* workspace, int S, int E, int k,
                            cudaStream_t stream);
size_t route_workspace_ints(int S, int E, int k);

// slot_src[E*C]: token*k + j occupying that slot, or -1.  Must be called after route_locations.
cudaError_t build_slot_map(const int* idx, const int* loc, int* slot_src, int S, int E, int k, int C,
                           cudaStream_t stream);

// out[slot, :] = scale * x[token(slot), :]   (zeros for empty slots);  scale = gates[j*S + token] or 1.
// dst_ptr_table (optional, uint64[E]): base pointer of expert e's [C, M] block - may be PEER memory (dispatch
// fusion); when null the block of expert e is out + e*C*M.
// signal_ptr_table/signal_rows (optional): after rows [r0, r0+signal_rows) of expert e are stored, the uint32
// counter at signal_ptr_table[e] + (r0/signal_rows) is set to `signal_value` with st.release.sys (each chunk has a
// single publisher - the block that finishes the chunk's last 16-row unit, elected through `chunk_counters`
// (uint32[E * ceil(C/signal_rows)], zero-initialised, self-resetting) - so the epoch number itself is published;
// 0 = increment instead).  valid_rows (optional, int[E]): rows >= valid_rows[e] of expert e are left untouched.
cudaError_t encode_rows(const void* x, const void* gates, const int* slot_src, void* out,
                        const unsigned long long* dst_ptr_table, const unsigned long long* signal_ptr_table,
                        unsigned int* chunk_counters, int signal_rows, int S, int E, int k, int C, int M, int elem_type,
                        int rot_chunks, int signal_value, const int* valid_rows, cudaStream_t stream);

// The same gather with per-row e4m3 quantisation: destination rows are M bytes, the row scales (max|row| / 448, fp32) go
// to scale_out[E*C] or - for a remote push - to scale_ptr_table[e][C].  16-bit sources, M % 16 == 0.
cudaError_t encode_rows_fp8(const void* x, const void* gates, const int* slot_src, void* out, float* scale_out,
                            const unsigned long long* dst_ptr_table, const unsigned long long* scale_ptr_table,
                            const unsigned long long* signal_ptr_table, unsigned int* chunk_counters, int signal_rows, int S,
                            int E, int k, int C, int M, int elem_type, int rot_chunks, int signal_value, cudaStream_t stream);

// out[s, :] = sum_j w_j * buf[idx_j[s]*C + loc_j[s], :]  (choices with loc >= C or idx < 0 contribute 0).
// wait_flags (optional): uint32[E] counters that must reach wait_target (acquire.sys) before expert e's rows
// are read (combine fusion).
// seg_off (optional, int[E]): expert-packed buffer, the row of (e, l) is seg_off[e] + l instead of e*C + l.
// base (optional, [S, M] of the buffer's type, 16-byte aligned rows for the vector path): shared experts' output, added
// after the routed terms as out[s] = T(fmaf(w_s, base[s], routed fp32 sum)) - one rounding - with w_s = 1, or
// sigmoid(shared_logit[s]) in fp32 when shared_logit (optional, fp32 [S]) is given.
cudaError_t decode_rows(const void* buf, const void* gates, const int* idx, const int* loc, void* out,
                        const uint32_t* wait_flags, uint32_t wait_target, int S, int E, int k, int C, int M,
                        int elem_type, cudaStream_t stream, const int* seg_off = nullptr, const void* base = nullptr,
                        const float* shared_logit = nullptr);

// dgate[j*S + s] = dot(a[s, :], buf[slot_j(s), :])   (fp32 accumulate, 0 for dropped choices).  seg_off: as decode_rows.
// Gated shared experts (shared_logit fp32 [S] given; base, d_base [S, M] of a's type; d_shared_logit fp32 [S]), in the same
// launch: d_base[s] = T(w_s * a[s]), d_shared_logit[s] = w_s (1 - w_s) dot(a[s], base[s]), w_s = sigmoid(shared_logit[s]).
// k may then be 0 (buf and dgate unused).
cudaError_t gate_grad(const void* a, const void* buf, const int* idx, const int* loc, void* dgate, int S, int E,
                      int k, int C, int M, int elem_type, cudaStream_t stream, const int* seg_off = nullptr,
                      const void* base = nullptr, const float* shared_logit = nullptr, void* d_base = nullptr,
                      float* d_shared_logit = nullptr);

// Expert-packed layout of R rows (R % 128 == 0, R >= sum_e roundup128(counts[e])), from device counts[E] with no host
// read: seg_off[E + 1] = exclusive scan of roundup128(counts), block_expert / block_rows [R / 128] = the expert and the
// valid rows of each 128-row block (0 past seg_off[E]), slot_src[R] = token*k + j of row seg_off[e] + loc, -1 for
// padding.  Three launches (layout, -1 fill, scatter).
cudaError_t packed_layout(const int* idx, const int* loc, const int* counts, int* seg_off, int* block_expert,
                          int* block_rows, int* slot_src, int S, int E, int k, int R, cudaStream_t stream);

// ---- fused gating + routing (gate_route.cu) ---------------------------------------------------------------------
// Two launches: logits [S,E] (fp32/fp16/bf16) -> softmax scores (fp32), top-k ids idx[k,S], raw top-k scores top[k,S],
// normalised gates[k,S] (fp32), queue locations loc[k,S], per-expert counts[E], the inverse slot map slot_src[E*C]
// (optional: pass null / C = 0 when the capacity is not known yet), first-choice counts ce[E] (fp32) and the GShard
// auxiliary loss l_aux (scalar of the logits' dtype, optional).  Workspaces: me_partial float[tiles*E], hist
// int[tiles*k*E] with tiles = gate_route_tiles(S).  Limits: E <= 512, k <= 32.
int gate_route_tiles(int S);
cudaError_t gate_route_forward(const void* logits, float* scores, int* idx, float* top, float* gates, float* me_partial,
                               int* hist, int* loc, int* counts, int* slot_src, float* ce_out, void* l_aux, int S, int E,
                               int k, int C, bool normalize, float eps, int elem_type, cudaStream_t stream);
// One launch: d logits [S,E] (dtype of the logits) from dgates fp32 [k,S] (may be null) and the loss gradient `dl`
// (device scalar of the logits' dtype, may be null; needs ce).
cudaError_t gate_route_backward(const float* scores, const int* idx, const float* top, const float* dgates,
                                const float* ce, const void* dl, void* dlogits, int S, int E, int k, bool normalize,
                                float eps, int elem_type, cudaStream_t stream);
// Sigmoid scoring (DeepSeek-V3 routing), same outputs and workspaces as gate_route_forward: scores = sigmoid(logits),
// ids chosen on scores + bias[E] (fp32) among the best `topk_group` of `n_group` expert groups (n_group <= 32),
// top = the unbiased scores, gates = scale * normalised top, ce = fp32 all-choice counts, l_aux the balance loss
// E / (k S^2) sum_e n_e sum_s s_se / T_s.  `load` (fp32 [E], may be null) accumulates the all-choice counts.
cudaError_t sigmoid_gate_route_forward(const void* logits, const float* bias, float* scores, int* idx, float* top,
                                       float* gates, float* me_partial, int* hist, int* loc, int* counts, int* slot_src,
                                       float* ce_out, void* l_aux, float* load, int S, int E, int k, int C,
                                       bool normalize, float eps, int n_group, int topk_group, float scale,
                                       int elem_type, cudaStream_t stream);
cudaError_t sigmoid_gate_route_backward(const float* scores, const int* idx, const float* top, const float* dgates,
                                        const float* ce, const void* dl, void* dlogits, int S, int E, int k,
                                        bool normalize, float eps, float scale, int elem_type, cudaStream_t stream);
// bias[e] += gamma * sign(mean(load) - load[e]); load = 0.  One launch, fp32 [E] both.
cudaError_t expert_bias_update(float* bias, float* load, int E, float gamma, cudaStream_t stream);

// out[g, n] = sum_r x[g, r, n]  (bias gradients).  splits = colsum_row_splits(..): 1 -> results are written to `out`
// (dtype of x); > 1 -> partial sums are atomically added to the zero-initialised fp32 buffer `acc` [G, N].
int colsum_row_splits(int G, int rows, int N, int elem_bytes);
// offsets (optional, int[G + 1]): group g is rows [offsets[g], offsets[g + 1]) of x (group_stride unused), split over
// `splits` blocks per column strip; `rows` only bounds the offsets.
cudaError_t grouped_colsum(const void* x, long long ld, long long group_stride, void* out, float* acc, int G, int rows,
                           int N, int splits, int elem_type, cudaStream_t stream, const int* offsets = nullptr);

// out[s, e] = (sum_{s' <= s} in[s', e]) - 1   (`tutel_ops.cumsum`, tutel/custom/custom_kernel.cpp:822-872)
size_t cumsum_workspace_ints(int S, int E);
cudaError_t cumsum_sub_one(const int* in, int* out, int* workspace, int S, int E, cudaStream_t stream);

// runtime spin-wait limit of the cross-GPU protocols (per translation unit; bindings call all of them)
cudaError_t set_spin_timeout_moe(unsigned long long ns);
cudaError_t set_spin_timeout_p2p(unsigned long long ns);
cudaError_t set_spin_timeout_gemm(unsigned long long ns);
cudaError_t set_spin_timeout_mx(unsigned long long ns);
cudaError_t set_spin_timeout_block_fp8(unsigned long long ns);

// q[r, :] = e4m3(x[r, :] / scale[r]),  scale[r] = max|x[r, :]| / 448   (one scale per row; rows are K-major GEMM
// operands, so the scale factors out of the dot product and is applied in the GEMM epilogue).
cudaError_t quantize_rows_e4m3(const void* x, void* q, float* scale, long long R, int K, int elem_type,
                               cudaStream_t stream);

// qT[g, k, r] = e4m3(x[g, r, k] / scale[g, k]),  scale[g, k] = max_r |x[g, r, k]| / 448: the transposed, row-scaled copy of a
// 16-bit weight (R % 128 == 0, K % 64 == 0).  amax_ws: fp32 [G, K] workspace.
cudaError_t quantize_transpose_e4m3(const void* x, void* qT, float* scale, float* amax_ws, int G, int R, int K, int elem_type,
                                    cudaStream_t stream);

// y[r, :] = q[r, :] * scale[r]  (e4m3 -> fp16 / bf16), K % 16 == 0
cudaError_t dequant_rows_e4m3(const void* q, const float* scale, void* y, long long R, int K, int elem_type,
                              cudaStream_t stream);

// Dropless / decoder inference: y[g, r, :] = act(x[g, r, :] @ W[g] + bias[g]) for r < counts[g] (device counts, no
// host sync); x [G, rows_cap, K], y [G, rows_cap, N], W [G, N, K] or (w_is_kn) [G, K, N].  Rows past the count are
// left untouched.  (csrc/skinny_gemm.cu)
cudaError_t skinny_grouped_gemm(const void* x, const void* w, const void* bias, void* y, const int* counts, int G,
                                int rows_cap, int N, int K, bool w_is_kn, bool relu, int elem_type, cudaStream_t stream);

// Whole two-layer expert FFN for a few rows per expert in ONE launch (dropless / decoder inference):
//   y[g, r, :] += act(x[g, r, :] @ W1[g]^T + b1[g]) @ W2[g] + b2[g]   for r < counts[g]
// x [G, rows_cap, K], W1 [G, H, K], W2 [G, H, N] (the reference's batched_fc1_w / batched_fc2_w layouts), y fp32
// [G, rows_cap, N] ZERO-INITIALISED (blocks split H and accumulate with atomics).  act: 0 none, 1 relu, 2 gelu, 3 silu.
cudaError_t skinny_grouped_ffn(const void* x, const void* w1, const void* b1, const void* w2, const void* b2, float* y,
                               const int* counts, int G, int rows_cap, int K, int H, int N, int act, int elem_type,
                               cudaStream_t stream);

// Whole SwiGLU expert for a few rows per expert in ONE launch (dropless / decoder inference):
//   y[g, r, :] += (act(x[g, r, :] @ W1[g]) * (x[g, r, :] @ W2[g])) @ W3[g]   for r < counts[g]
// x [G, rows_cap, M], W1 / W2 [G, M, H], W3 [G, H, N] (LlamaFFNNetwork's layouts, last dims contiguous), y fp32
// [G, rows_cap, N] ZERO-INITIALISED.  M, H, N multiples of 16 bytes' worth of elements; cudaErrorInvalidValue when the
// staged rows of x do not fit in the same 200 KB of shared memory as skinny_grouped_ffn (M > 12224).  act: as above.
cudaError_t skinny_grouped_glu_ffn(const void* x, const void* w1, const void* w2, const void* w3, float* y, const int* counts,
                                   int G, int rows_cap, int M, int H, int N, int act, int elem_type, cudaStream_t stream);

// Weight-only fp8 (W8A16) versions of the two kernels above, on the e4m3 copies the fp8 wgmma forward caches
// (ops/gemm.py: fp8_weight); x is fp16 / bf16 and is not quantised, accumulation is fp32, scales multiply finished dot
// products.  Same launch contract: y fp32 [G, rows_cap, N] ZERO-INITIALISED, rows r < min(counts[g], rows_cap) only.
//   skinny_grouped_ffn_fp8:     y[g, r] += act(s1[g] * (x[g, r] @ Q1[g]^T) + b1[g]) @ (s2[g] * Q2t[g])^T + b2[g]
//       Q1 [G, H, K] e4m3, s1 fp32 [G, H];  Q2t [G, N, H] e4m3, s2 fp32 [G, N];  biases [G, H] / [G, N] in x's dtype or null.
//   skinny_grouped_glu_ffn_fp8: y[g, r] += (act(s1[g] * (x @ Q1t[g]^T)) * (s2[g] * (x @ Q2t[g]^T))) @ (s3[g] * Q3t[g])^T
//       Q1t / Q2t [G, H, M] e4m3, s1 / s2 fp32 [G, H];  Q3t [G, N, H] e4m3, s3 fp32 [G, N].
// cudaErrorInvalidValue for a 32-bit x, unaligned x / e4m3 pointers, K (M), H or N not a multiple of 16, or staged rows of
// x beyond the 200 KB of shared memory of the 16-bit kernels.  act: 1 relu, 2 gelu, 3 silu.
cudaError_t skinny_grouped_ffn_fp8(const void* x, const void* q1, const float* s1, const void* b1, const void* q2t,
                                   const float* s2, const void* b2, float* y, const int* counts, int G, int rows_cap, int K,
                                   int H, int N, int act, int elem_type, cudaStream_t stream);
cudaError_t skinny_grouped_glu_ffn_fp8(const void* x, const void* q1t, const float* s1, const void* q2t, const float* s2,
                                       const void* q3t, const float* s3, float* y, const int* counts, int G, int rows_cap,
                                       int M, int H, int N, int act, int elem_type, cudaStream_t stream);
//   skinny_grouped_glu_ffn_block_fp8: the same SwiGLU expert on block-scaled e4m3 weights (DeepSeek-V3 format), x bf16:
//       Qglu [G, 2H, M]: W1^T and W2^T interleaved every 64 rows, Sglu fp32 [G, 2H / 64, M / 128];
//       Q3t [G, N, H], S3t fp32 [G, N / 128, H / 128]  (one scale per 128 x 128 block, applied per 128-deep K block).
// cudaErrorInvalidValue for unaligned pointers, M, H or N not a multiple of 128, or act outside 1..3.
cudaError_t skinny_grouped_glu_ffn_block_fp8(const void* x, const void* qglu, const float* sglu, const void* q3t,
                                             const float* s3t, float* y, const int* counts, int G, int rows_cap, int M, int H,
                                             int N, int act, cudaStream_t stream);
//   skinny_grouped_glu_ffn_int4: the same SwiGLU expert on group-32 int4 weights (W4A16), x bf16:
//       Qglu [G, 2H, M / 2] packed nibbles (W1^T and W2^T rows interleaved every 64), Sglu bf16 [G, 2H, M / 32];
//       Q3t [G, N, H / 2], S3t bf16 [G, N, H / 32]; nibble = q + 8, element 2j in bits 0-3 of byte j, 2j + 1 in bits 4-7.
// cudaErrorInvalidValue for unaligned pointers, M, H or N not a multiple of 128, or act outside 1..3.
cudaError_t skinny_grouped_glu_ffn_int4(const void* x, const void* qglu, const void* sglu, const void* q3t, const void* s3t,
                                        float* y, const int* counts, int G, int rows_cap, int M, int H, int N, int act,
                                        cudaStream_t stream);

}  // namespace tb
