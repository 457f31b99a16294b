// Mixed-input grouped GEMM for group-32 int4 weights (W4A16) on sm_90a: D[g] = epilogue(A[g] * B[g]^T) with bf16
// activations A [G, M, K] and int4 weights B [G, N, K] (packed nibbles [G, N, K / 2], bf16 scales [G, N, K / 32]), the
// prefill path of LlamaFFNNetwork(weight_format='int4').  See gemm_w4a16.cu.
#pragma once

#include <cuda_runtime.h>

namespace tb {

enum W4A16Epilogue : int { W4A16_EPI_NONE = 0, W4A16_EPI_GLU = 1 };

struct W4A16GemmProblem {
  const void* a = nullptr;          // bf16 [G, M, K], K-major
  const void* b = nullptr;          // uint8 [G, N, K / 2]: element 2j in bits 0-3 of byte j, 2j + 1 in bits 4-7, as q + 8
  const void* sb = nullptr;         // bf16 [G, N, K / 32]
  void* d = nullptr;                // bf16 [G, M, N] (NONE) or [G, M, N / 2] (GLU: h = act(gate) * up)
  int G = 0, M = 0, N = 0, K = 0;
  int epilogue = W4A16_EPI_NONE;
  int act = 3;                      // GLU: 1 relu, 2 gelu, 3 silu
  const int* row_counts = nullptr;  // device int32 [G] or null: rows at or past the count are stored as zero
  int max_ctas = 0;
};

// cudaErrorInvalidValue (and *why) for shapes, alignment or an unknown epilogue / activation.
cudaError_t w4a16_gemm_launch(const W4A16GemmProblem& p, cudaStream_t stream, const char** why);

}  // namespace tb
