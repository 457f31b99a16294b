// Host API of the MX block-scaled fp8 GEMM (one e4m3 wgmma per 32-element K block, scales applied to the fp32 partial sums) and its quantiser; see gemm_mx.cu.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace tb {

// Scale factors (UE8M0, one per 32 consecutive K elements of a row) are stored in the tile order the tensor core
// reads them from shared memory:   sf[g][kb][rt][ (r % 32) * 16 + ((r % 128) / 32) * 4 + (k % 128) / 32 ]
// with kb = k / 128, rt = r / 128 - one 512-byte atom per 128 rows x 128 K elements, so a CTA stages the scales of a
// whole operand tile with a single bulk copy.  Rows are padded to a multiple of 128 with byte 0.  A block with a non-zero
// element has a byte in [1, 253] (e in [-126, 126]); byte 0 (a block that is all zero or NaN, a pad row) decodes to a scale of 0.
inline long long mx_sf_bytes(int groups, long long rows, long long k) {
  return static_cast<long long>(groups) * (k / 128) * ((rows + 127) / 128) * 512;
}

// x [G*R, K] (bf16 / fp16, contiguous) -> q e4m3 [G*R, K] and sf (layout above).  K % 128 == 0.
// elem_type: 0 fp32 (unsupported), 1 fp16, 2 bf16 (ElemType of moe_kernels.h).
cudaError_t mx_quantize(const void* x, void* q, void* sf, int groups, int rows, int k, int elem_type,
                        cudaStream_t stream);

// x [G, R, K] -> qT e4m3 [G, K, R] quantised along R, sf of an operand with K rows and reduction length R.
// R % 128 == 0, K % 64 == 0.
cudaError_t mx_quantize_transpose(const void* x, void* qT, void* sf, int groups, int rows, int k, int elem_type,
                                  cudaStream_t stream);

enum MxEpilogue : int { MX_EPI_NONE = 0, MX_EPI_RELU = 1, MX_EPI_RELU_BWD = 2 };   // RELU_BWD: D = aux > 0 ? acc : 0

struct MxGemmProblem {
  int M = 0, N = 0, K = 0, G = 1;
  const void* a = nullptr;       // e4m3 [G, M, K]
  const void* sfa = nullptr;     // scales of a
  const void* b = nullptr;       // e4m3 [G, N, K]   (an [N, K] weight: D = A * B^T)
  const void* sfb = nullptr;
  void* d = nullptr;             // bf16 [G, M, N]
  long long ldd = 0, d_group_stride = 0;
  const void* bias = nullptr;    // bf16 [G, N]: D = epilogue(acc + bias[n])
  long long bias_group_stride = 0;
  const void* aux = nullptr;     // MX_EPI_RELU_BWD: bf16 [G, M, N] forward activation
  long long ld_aux = 0, aux_group_stride = 0;
  int epilogue = 0;              // MxEpilogue
  int block_n = 0;               // 0, 128 or 256: tile-shape hint of callers written for wider tiles; the kernel tiles 128 x 128
  int cta_group = 0;             // 0, 1 or 2: likewise a hint only (Hopper has no CTA-pair MMA)
  int max_ctas = 0;              // 0: one CTA per SM
};

// sa * sb is formed in fp32, so ea + eb (byte_a + byte_b - 254) must stay in fp32's normal exponent range [-126, 127].
cudaError_t mx_gemm_launch(const MxGemmProblem& p, cudaStream_t stream, const char** why = nullptr);

}  // namespace tb
