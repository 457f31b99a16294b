// Host API of the block-scaled fp8 GEMM (DeepSeek-V3 recipe: e4m3 activations with one fp32 scale per 1 x 128 tile,
// e4m3 weights with one fp32 scale per 128 x 128 block, the MMA partial sum promoted into fp32 once per 128 K) and of
// its two quantisers; see gemm_block_fp8.cu and tutel_b200/ops/block_fp8.py.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace tb {

// Scale rule of every quantiser here (that of quantize_rows_kernel, per block): amax = the largest non-NaN magnitude,
// s = amax > 0 ? max(amax / 448, FLT_MIN) : 1, q = e4m3_rn_satfinite(x * (1 / s)).
//
// Activations x [G, R, K] bf16 -> q e4m3 [G, R, K] and scales fp32 [G, K / 128, Rp], Rp = roundup(R, 128): MN-major, so
// that one K step of a 128-row tile is 512 contiguous bytes.  Pad rows get scale 0.  K % 128 == 0.
// live_rows (optional device int32, groups == 1; the packed layout's seg_off[E]): rows at or past *live_rows are neither
// read nor written, rows below it are quantised bit for bit as without the bound.
cudaError_t block_fp8_quantize_act(const void* x, void* q, float* s, int groups, int rows, int k, cudaStream_t stream,
                                   const int* live_rows = nullptr);

// Weights w [G, R, C] bf16, 128 x 128 blocks (R % 128 == 0, C % 128 == 0), one launch for both orientations:
//   q [G, R, C] + s [G, R / 128, C / 128]      and      qT [G, C, R] + sT [G, C / 128, R / 128]
// (the same e4m3 bytes and scales, transposed).
cudaError_t block_fp8_quantize_weight(const void* w, void* q, float* s, void* qT, float* sT, int groups, int rows, int cols,
                                      cudaStream_t stream);

// SwiGLU gate / up weights w1, w2 [G, M, H] bf16 (M % 128 == 0, H % 128 == 0) in 128 x 128 blocks, one launch:
//   qcat [G, M, 2H] = [q(w1) q(w2)] + scat [G, M / 128, 2H / 128]           (B operand of dx = [dg du] [W1 W2]^T)
//   qglu [G, 2H, M]: w1^T and w2^T interleaved every 64 rows (rows 128 t + j = gate column 64 t + j, rows 128 t + 64 + j =
//   up column 64 t + j, j < 64) + sglu [G, 2H / 64, M / 128], one scale per 64 rows  (B operand of the GLU forward).
cudaError_t block_fp8_quantize_glu_weight(const void* w1, const void* w2, void* qcat, float* scat, void* qglu, float* sglu,
                                          int groups, int m, int h, cudaStream_t stream);

enum BlockFp8Epilogue : int {
  BF8_EPI_NONE = 0,       // D = acc (+ bias)
  BF8_EPI_RELU = 1,       // D = max(acc + bias, 0)
  BF8_EPI_RELU_BWD = 2,   // D = aux > 0 ? acc : 0
  BF8_EPI_GLU = 3,        // B tile = 64 gate + 64 up columns: D = act(g) * u, D2 = g, D3 = u (D* are [G, M, N / 2])
  BF8_EPI_GLU_BWD = 4,    // acc = dh; aux = g, aux2 = u: D = dh * u * act'(g) (dg), D2 = dh * act(g) (du)
};

struct BlockFp8GemmProblem {
  int M = 0, N = 0, K = 0, G = 1;
  const void* a = nullptr;       // e4m3 [G, M, K]
  const float* sa = nullptr;     // [G, K / 128, roundup(M, 128)]
  const void* b = nullptr;       // e4m3 [G, N, K]
  const float* sb = nullptr;     // [G, N / 128, K / 128]; BF8_EPI_GLU: [G, N / 64, K / 128]
  void* d = nullptr;             // bf16, row stride ldd, group stride d_group_stride
  void* d2 = nullptr;            // GLU: g;  GLU_BWD: du   (same strides as d)
  void* d3 = nullptr;            // GLU: u
  long long ldd = 0, d_group_stride = 0;
  const void* bias = nullptr;    // bf16 [G, N] (NONE / RELU only)
  long long bias_group_stride = 0;
  const void* aux = nullptr;     // RELU_BWD: forward activation;  GLU_BWD: g      bf16 [G, M, N]
  const void* aux2 = nullptr;    // GLU_BWD: u
  long long ld_aux = 0, aux_group_stride = 0;
  int epilogue = 0;              // BlockFp8Epilogue
  int act = 3;                   // GLU / GLU_BWD: 1 ReLU, 2 GELU, 3 SiLU
  int max_ctas = 0;              // 0: one CTA per SM
  // Optional device int32 [G]: only rows r < row_counts[g] of group g are live (dropless prefill).  Tiles whose first row
  // is at or past the count are skipped (no operand is loaded for them); every output row past the count is stored as
  // zero.  Null: all M rows, the same kernel as without the field.
  const int* row_counts = nullptr;
  // Optional device int32 [M / 128], the block-mapped launch of the expert-packed layout (tutel_b200/ops/packed.py): a is one
  // e4m3 [M, K] buffer (M = R packed rows, a multiple of 128) with scales [1, K / 128, M], d, d2, d3, aux and aux2 are
  // [M, *] (group strides unused), and row tile m is multiplied by B, sb and bias of group b_group_map[m] (G = the number
  // of B groups).  row_counts is then required and holds the live rows of each row tile: rows past it are stored as
  // zero in every output (whatever the epilogue), and a tile with no live rows loads and stores nothing.
  const int* b_group_map = nullptr;
};

cudaError_t block_fp8_gemm_launch(const BlockFp8GemmProblem& p, cudaStream_t stream, const char** why = nullptr);

// Activations x [G, R, K] bf16 (K % 128 == 0) quantised in both orientations from one read, for the weight gradients:
//   row-wise    q [G, R, K] + s [G, K / 128, Rp]: bit for bit what block_fp8_quantize_act writes (skipped when q and s
//               are null);
//   column-wise qT [G, K, Rp] e4m3 (x^T; rows R..Rp-1 of x are zero bytes) + sT [G, Rp / 128, K] fp32, one scale per
//               column of x and 128-row block, by the same rule over the block's real rows.
// live_rows (optional device int32, groups == 1, a multiple of 128): the 128-row tiles at or past *live_rows are neither read
// nor written; the others are bit for bit those of the unbounded launch.
cudaError_t block_fp8_quantize_act_dual(const void* x, void* q, float* s, void* qT, float* sT, int groups, int rows, int k,
                                        cudaStream_t stream, const int* live_rows = nullptr);

// Weight-gradient GEMM  D[g] = A[g] B[g]^T  with K the (padded) token dimension: A e4m3 [G, M, K], B e4m3 [G, N, K]
// (the column-wise outputs of block_fp8_quantize_act_dual), one fp32 scale per row and 128-deep K step for both, sa
// [G, K / 128, M] and sb [G, K / 128, N].  Every K step is promoted as acc = fmaf(part, sa[m] * sb[n], acc).  D is bf16
// [G, M, N]; with split = H > 0 (N == 2H), columns < H go to d [G, M, H] and columns >= H to d2 [G, M, H].
// M, N, K multiples of 128.
// Ragged K (optional device int32 k_offsets [G + 1], multiples of 128; the packed layout's seg_off): a [M, K] and b
// [N, K] are single operands with scales [1, K / 128, M] and [1, K / 128, N], and group g reduces over the K range
// [k_offsets[g], k_offsets[g + 1]) only; a group with an empty range gets zeros.
struct BlockFp8WgradProblem {
  int M = 0, N = 0, K = 0, G = 1;
  const void* a = nullptr;
  const float* sa = nullptr;
  const void* b = nullptr;
  const float* sb = nullptr;
  void* d = nullptr;
  void* d2 = nullptr;
  int split = 0;
  int max_ctas = 0;              // 0: one CTA per SM
  const int* k_offsets = nullptr;
};

cudaError_t block_fp8_wgrad_gemm_launch(const BlockFp8WgradProblem& p, cudaStream_t stream, const char** why = nullptr);

}  // namespace tb
