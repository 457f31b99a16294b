// pybind11 / torch bindings for the tutel_b200 native runtime (`tutel_b200._C`).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <string>
#include <vector>

#include "cpu_kernels.h"
#include "gemm_block_fp8.h"
#include "gemm_mx.h"
#include "gemm_sm90.h"
#include "gemm_w4a16.h"
#include "jit_nvrtc.h"
#include "moe_kernels.h"
#include "p2p_kernels.h"
#include "symm_heap.h"

namespace {

#define TB_CHECK_CUDA(expr)                                                                          \
  do {                                                                                               \
    cudaError_t _e = (expr);                                                                         \
    TORCH_CHECK(_e == cudaSuccess, "tutel_b200 CUDA error: ", cudaGetErrorString(_e), " at ", #expr); \
  } while (0)

int gemm_dtype_of(const at::Tensor& t) {
  switch (t.scalar_type()) {
    case at::kBFloat16: return tb::DT_BF16;
    case at::kHalf: return tb::DT_FP16;
    case at::kFloat: return tb::DT_FP32;
    case at::kFloat8_e4m3fn: return tb::DT_E4M3;
    case at::kFloat8_e5m2: return tb::DT_E5M2;
    default: TORCH_CHECK(false, "unsupported dtype for tutel_b200 GEMM: ", t.scalar_type());
  }
}

int elem_type_of(const at::Tensor& t) {
  switch (t.scalar_type()) {
    case at::kFloat: return tb::ET_F32;
    case at::kHalf: return tb::ET_F16;
    case at::kBFloat16: return tb::ET_BF16;
    default: TORCH_CHECK(false, "unsupported dtype for tutel_b200 dispatch kernels: ", t.scalar_type());
  }
}

cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

// Optional packed-layout launch modes of the grouped GEMM (see GemmProblem): b_group_map int [G] (B group of each
// A group), k_offsets int [G + 1] (ragged K: a [1, K, M] / b [1, K, N], d [G, M, N]).
void set_packed_modes(tb::GemmProblem& p, const at::Tensor& a, const at::Tensor& b, const at::Tensor& d,
                      const c10::optional<at::Tensor>& b_group_map, const c10::optional<at::Tensor>& k_offsets) {
  if (b_group_map.has_value() && b_group_map->defined()) {
    TORCH_CHECK(b_group_map->is_cuda() && b_group_map->scalar_type() == at::kInt && b_group_map->is_contiguous() &&
                    b_group_map->numel() >= p.G, "tutel_b200.gemm: b_group_map must be a contiguous int32 [G]");
    p.b_group_map = b_group_map->data_ptr<int>();
    p.b_groups = static_cast<int>(b.size(0));
  }
  if (k_offsets.has_value() && k_offsets->defined()) {
    TORCH_CHECK(k_offsets->is_cuda() && k_offsets->scalar_type() == at::kInt && k_offsets->is_contiguous() &&
                    k_offsets->numel() == d.size(0) + 1 && a.size(0) == 1 && b.size(0) == 1,
                "tutel_b200.gemm: k_offsets must be a contiguous int32 [G + 1] with a [1, K, M], b [1, K, N] and d [G, M, N]");
    p.k_offsets = k_offsets->data_ptr<int>();
    p.G = static_cast<int>(d.size(0));
  }
}

// a: [G, M, K] (a_mn=false) or [G, K, M] (a_mn=true); b: [Gb, N, K] (b_mn=false) or [Gb, K, N] (b_mn=true);
// d: [G, M, N].  Innermost dims contiguous.  Pointer-table / flag arguments are raw device addresses (0 = off).
// b_group_map / k_offsets: see set_packed_modes.
void gemm_ex_packed(const at::Tensor& a, const at::Tensor& b, at::Tensor& d, bool a_mn, bool b_mn, int64_t epilogue,
             const c10::optional<at::Tensor>& bias, const c10::optional<at::Tensor>& aux,
             const c10::optional<at::Tensor>& row_counts, double alpha, int64_t b_group_div, int64_t cta_group,
             int64_t block_n, int64_t d_ptr_table, int64_t signal_ptr_table, int64_t wait_flags,
             int64_t wait_rows_per_flag, int64_t wait_flags_per_group, int64_t wait_target, int64_t max_ctas,
             int64_t group_rot, int64_t group_mod, const c10::optional<at::Tensor>& scale_a,
             const c10::optional<at::Tensor>& scale_b, const c10::optional<at::Tensor>& colsum,
             const c10::optional<at::Tensor>& d2, int64_t act, const c10::optional<at::Tensor>& b_group_map,
             const c10::optional<at::Tensor>& k_offsets) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && d.is_cuda(), "tutel_b200.gemm: CUDA tensors required");
  TORCH_CHECK(a.dim() == 3 && b.dim() == 3 && d.dim() == 3, "tutel_b200.gemm: expected 3-D operands");
  TORCH_CHECK(a.stride(2) == 1 && b.stride(2) == 1 && d.stride(2) == 1, "tutel_b200.gemm: innermost dim must be contiguous");
  TORCH_CHECK(a.scalar_type() == b.scalar_type(), "tutel_b200.gemm: A/B dtype mismatch");
  const c10::cuda::CUDAGuard guard(a.device());
  tb::GemmProblem p;
  p.G = static_cast<int>(a.size(0));
  p.M = static_cast<int>(a_mn ? a.size(2) : a.size(1));
  p.K = static_cast<int>(a_mn ? a.size(1) : a.size(2));
  p.N = static_cast<int>(b_mn ? b.size(2) : b.size(1));
  TORCH_CHECK((b_mn ? b.size(1) : b.size(2)) == p.K, "tutel_b200.gemm: K mismatch");
  set_packed_modes(p, a, b, d, b_group_map, k_offsets);
  TORCH_CHECK(d.size(0) == p.G && d.size(1) == p.M && d.size(2) == p.N, "tutel_b200.gemm: output shape mismatch");
  p.b_group_div = static_cast<int>(b_group_div > 0 ? b_group_div : 1);
  TORCH_CHECK(p.b_group_map != nullptr || p.k_offsets != nullptr || b.size(0) * p.b_group_div >= p.G,
              "tutel_b200.gemm: not enough B groups");
  p.a = a.data_ptr(); p.lda = a.stride(1); p.a_group_stride = a.stride(0); p.a_mn_major = a_mn;
  p.b = b.data_ptr(); p.ldb = b.stride(1); p.b_group_stride = b.stride(0); p.b_mn_major = b_mn;
  p.in_dtype = gemm_dtype_of(a);
  p.d = d.data_ptr(); p.ldd = d.stride(1); p.d_group_stride = d.stride(0);
  p.out_dtype = gemm_dtype_of(d);
  TORCH_CHECK(p.out_dtype <= tb::DT_FP32, "tutel_b200.gemm: output must be bf16/fp16/fp32");
  p.epilogue = static_cast<int>(epilogue);
  p.alpha = static_cast<float>(alpha);
  // groups of B (and rows of bias / scale_b / colsum) the kernel indexes: g / b_group_div for g < G (block-mapped B:
  // the map's values, which are below b.size(0); ragged K: g)
  const int64_t gb = p.b_group_map != nullptr ? b.size(0) : p.k_offsets != nullptr ? p.G : (p.G + p.b_group_div - 1) / p.b_group_div;
  // The epilogues read bias 16 bytes at a time (128 x 128) and scale_b 8 bytes at a time (128 x 256), from the row of
  // each B group: the base and the row stride must keep that alignment.
  auto aligned_rows = [](const at::Tensor& t, int64_t bytes) {
    return reinterpret_cast<uintptr_t>(t.data_ptr()) % bytes == 0 && (t.size(0) == 1 || (t.stride(0) * t.element_size()) % bytes == 0);
  };
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(bias->is_cuda() && bias->dim() == 2 && bias->stride(1) == 1 && bias->size(0) >= gb && bias->size(1) == p.N &&
                    (bias->scalar_type() == a.scalar_type() || (a.element_size() == 1 && bias->scalar_type() == d.scalar_type() && d.element_size() == 2)),
                "tutel_b200.gemm: bias must be [Gb, N] of the input dtype (fp8 inputs: of the 16-bit output dtype)");
    TORCH_CHECK(aligned_rows(*bias, 16), "tutel_b200.gemm: bias rows must start 16-byte aligned");
    p.bias = bias->data_ptr();
    p.bias_group_stride = bias->stride(0);
  }
  if (aux.has_value() && aux->defined()) {
    TORCH_CHECK(aux->is_cuda() && aux->scalar_type() == d.scalar_type() && aux->dim() == 3 && aux->stride(2) == 1 &&
                    aux->element_size() == 2,
                "tutel_b200.gemm: aux must be a 16-bit [G, M, N] tensor of the output dtype");
    p.aux = aux->data_ptr();
    p.ld_aux = aux->stride(1);
    p.aux_group_stride = aux->stride(0);
  }
  if (row_counts.has_value() && row_counts->defined()) {
    TORCH_CHECK(row_counts->is_cuda() && row_counts->scalar_type() == at::kInt && row_counts->numel() >= p.G);
    p.row_counts = row_counts->data_ptr<int>();
  }
  if (scale_a.has_value() && scale_a->defined()) {
    TORCH_CHECK(scale_a->is_cuda() && scale_a->scalar_type() == at::kFloat && scale_a->dim() == 2 && scale_a->stride(1) == 1 &&
                scale_a->size(0) == p.G && scale_a->size(1) == p.M, "tutel_b200.gemm: scale_a must be float [G, M]");
    p.scale_a = scale_a->data_ptr<float>();
    p.scale_a_group_stride = scale_a->stride(0);
  }
  if (scale_b.has_value() && scale_b->defined()) {
    TORCH_CHECK(scale_b->is_cuda() && scale_b->scalar_type() == at::kFloat && scale_b->dim() == 2 && scale_b->stride(1) == 1 &&
                scale_b->size(0) >= gb && scale_b->size(1) == p.N, "tutel_b200.gemm: scale_b must be float [Gb, N]");
    TORCH_CHECK(aligned_rows(*scale_b, 8), "tutel_b200.gemm: scale_b rows must start 8-byte aligned");
    p.scale_b = scale_b->data_ptr<float>();
    p.scale_b_group_stride = scale_b->stride(0);
  }
  if (colsum.has_value() && colsum->defined()) {
    TORCH_CHECK(colsum->is_cuda() && colsum->scalar_type() == at::kFloat && colsum->dim() == 2 && colsum->stride(1) == 1 &&
                colsum->size(0) >= gb && colsum->size(1) == p.N, "tutel_b200.gemm: colsum must be float [Gb, N]");
    p.colsum = colsum->data_ptr<float>();
    p.colsum_group_stride = colsum->stride(0);
  }
  p.cta_group = static_cast<int>(cta_group);
  p.block_n = static_cast<int>(block_n);
  p.max_ctas = static_cast<int>(max_ctas);
  p.d_ptr_table = reinterpret_cast<const unsigned long long*>(d_ptr_table);
  p.signal_ptr_table = reinterpret_cast<const unsigned long long*>(signal_ptr_table);
  p.wait_flags = reinterpret_cast<const uint32_t*>(wait_flags);
  p.wait_rows_per_flag = static_cast<int>(wait_rows_per_flag);
  p.wait_flags_per_group = static_cast<int>(wait_flags_per_group);
  p.wait_target = static_cast<uint32_t>(wait_target);
  p.group_rot = static_cast<int>(group_rot);
  p.group_mod = static_cast<int>(group_mod != 0 ? group_mod : 1);
  if (d2.has_value() && d2->defined()) {
    TORCH_CHECK(d2->is_cuda() && d2->scalar_type() == d.scalar_type() && d2->sizes() == d.sizes() && d2->strides() == d.strides(),
                "tutel_b200.gemm: d2 must look like d");
    p.d2 = d2->data_ptr();
  }
  if (act != 0) p.act = static_cast<int>(act);
  const char* why = nullptr;
  cudaError_t e = tb::gemm_sm90_launch(p, cur_stream(), &why);
  TORCH_CHECK(e == cudaSuccess, "tutel_b200.gemm launch failed: ", why ? why : cudaGetErrorString(e));
}

void gemm_ex(const at::Tensor& a, const at::Tensor& b, at::Tensor& d, bool a_mn, bool b_mn, int64_t epilogue,
             const c10::optional<at::Tensor>& bias, const c10::optional<at::Tensor>& aux,
             const c10::optional<at::Tensor>& row_counts, double alpha, int64_t b_group_div, int64_t cta_group,
             int64_t block_n, int64_t d_ptr_table, int64_t signal_ptr_table, int64_t wait_flags,
             int64_t wait_rows_per_flag, int64_t wait_flags_per_group, int64_t wait_target, int64_t max_ctas,
             int64_t group_rot, int64_t group_mod, const c10::optional<at::Tensor>& scale_a,
             const c10::optional<at::Tensor>& scale_b, const c10::optional<at::Tensor>& colsum,
             const c10::optional<at::Tensor>& d2, int64_t act) {
  gemm_ex_packed(a, b, d, a_mn, b_mn, epilogue, bias, aux, row_counts, alpha, b_group_div, cta_group, block_n, d_ptr_table,
                 signal_ptr_table, wait_flags, wait_rows_per_flag, wait_flags_per_group, wait_target, max_ctas, group_rot,
                 group_mod, scale_a, scale_b, colsum, d2, act, c10::nullopt, c10::nullopt);
}

void gemm(const at::Tensor& a, const at::Tensor& b, at::Tensor& d, bool a_mn, bool b_mn, int64_t epilogue,
          const c10::optional<at::Tensor>& bias, const c10::optional<at::Tensor>& aux,
          const c10::optional<at::Tensor>& row_counts, double alpha, int64_t b_group_div, int64_t cta_group,
          int64_t block_n, int64_t d_ptr_table, int64_t signal_ptr_table, int64_t wait_flags,
          int64_t wait_rows_per_flag, int64_t wait_flags_per_group, int64_t wait_target, int64_t max_ctas,
          int64_t group_rot, int64_t group_mod, const c10::optional<at::Tensor>& scale_a,
          const c10::optional<at::Tensor>& scale_b, const c10::optional<at::Tensor>& colsum) {
  gemm_ex(a, b, d, a_mn, b_mn, epilogue, bias, aux, row_counts, alpha, b_group_div, cta_group, block_n, d_ptr_table,
          signal_ptr_table, wait_flags, wait_rows_per_flag, wait_flags_per_group, wait_target, max_ctas, group_rot, group_mod,
          scale_a, scale_b, colsum, c10::nullopt, 0);
}

std::vector<at::Tensor> route_locations(const at::Tensor& idx, int64_t E, int64_t C) {
  TORCH_CHECK(idx.is_cuda() && idx.scalar_type() == at::kInt && idx.dim() == 2 && idx.is_contiguous());
  const c10::cuda::CUDAGuard guard(idx.device());
  const int k = static_cast<int>(idx.size(0)), S = static_cast<int>(idx.size(1));
  auto opts = idx.options();
  at::Tensor loc = at::empty({k, S}, opts);
  at::Tensor counts = at::empty({E}, opts);
  at::Tensor ws = at::empty({static_cast<int64_t>(tb::route_workspace_ints(S, static_cast<int>(E), k))}, opts);
  TB_CHECK_CUDA(tb::route_locations(idx.data_ptr<int>(), loc.data_ptr<int>(), counts.data_ptr<int>(),
                                    ws.data_ptr<int>(), S, static_cast<int>(E), k, cur_stream()));
  std::vector<at::Tensor> out{loc, counts};
  if (C > 0) {
    at::Tensor slot = at::empty({E * C}, opts);
    TB_CHECK_CUDA(tb::build_slot_map(idx.data_ptr<int>(), loc.data_ptr<int>(), slot.data_ptr<int>(), S,
                                     static_cast<int>(E), k, static_cast<int>(C), cur_stream()));
    out.push_back(slot);
  }
  return out;
}

at::Tensor build_slot_map(const at::Tensor& idx, const at::Tensor& loc, int64_t E, int64_t C) {
  TORCH_CHECK(idx.is_cuda() && loc.is_cuda() && idx.scalar_type() == at::kInt && loc.scalar_type() == at::kInt);
  TORCH_CHECK(idx.is_contiguous() && loc.is_contiguous() && idx.dim() == 2);
  const c10::cuda::CUDAGuard guard(idx.device());
  at::Tensor slot = at::empty({E * C}, idx.options());
  TB_CHECK_CUDA(tb::build_slot_map(idx.data_ptr<int>(), loc.data_ptr<int>(), slot.data_ptr<int>(),
                                   static_cast<int>(idx.size(1)), static_cast<int>(E), static_cast<int>(idx.size(0)),
                                   static_cast<int>(C), cur_stream()));
  return slot;
}

// x [S, M]; gates float [k, S] or None; slot_src int [E*C]; out [E*C, M] (ignored rows live in dst_ptr_table).
void encode_rows(const at::Tensor& x, const c10::optional<at::Tensor>& gates, const at::Tensor& slot_src,
                 at::Tensor& out, int64_t k, int64_t E, int64_t C, int64_t dst_ptr_table, int64_t signal_ptr_table,
                 int64_t signal_rows, int64_t rot_chunks, int64_t signal_value, int64_t chunk_counters,
                 const c10::optional<at::Tensor>& valid_rows) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.is_contiguous() && slot_src.is_cuda() && slot_src.is_contiguous());
  TORCH_CHECK(slot_src.scalar_type() == at::kInt && slot_src.numel() == E * C);
  const c10::cuda::CUDAGuard guard(x.device());
  const void* g = nullptr;
  if (gates.has_value() && gates->defined()) {
    TORCH_CHECK(gates->is_cuda() && gates->scalar_type() == at::kFloat && gates->is_contiguous());
    g = gates->data_ptr();
  }
  const int* vr = nullptr;
  if (valid_rows.has_value() && valid_rows->defined()) {
    TORCH_CHECK(valid_rows->is_cuda() && valid_rows->scalar_type() == at::kInt && valid_rows->numel() >= E);
    vr = valid_rows->data_ptr<int>();
  }
  if (dst_ptr_table == 0)
    TORCH_CHECK(out.is_cuda() && out.is_contiguous() && out.scalar_type() == x.scalar_type() &&
                out.numel() == E * C * x.size(1));
  TB_CHECK_CUDA(tb::encode_rows(x.data_ptr(), g, slot_src.data_ptr<int>(), out.data_ptr(),
                                reinterpret_cast<const unsigned long long*>(dst_ptr_table),
                                reinterpret_cast<const unsigned long long*>(signal_ptr_table),
                                reinterpret_cast<unsigned int*>(chunk_counters), static_cast<int>(signal_rows), static_cast<int>(x.size(0)), static_cast<int>(E),
                                static_cast<int>(k), static_cast<int>(C), static_cast<int>(x.size(1)), elem_type_of(x),
                                static_cast<int>(rot_chunks), static_cast<int>(signal_value), vr, cur_stream()));
}

// fp8 dispatch: x [S, M] (16-bit) -> e4m3 rows + fp32 row scales.  Local: returns [q [E*C, M], scale [E*C]]; remote push
// (dst_ptr_table != 0): rows / scales / flags go through the pointer tables and nothing is returned.
std::vector<at::Tensor> encode_rows_fp8(const at::Tensor& x, const c10::optional<at::Tensor>& gates, const at::Tensor& slot_src,
                                        int64_t k, int64_t E, int64_t C, int64_t dst_ptr_table, int64_t scale_ptr_table,
                                        int64_t signal_ptr_table, int64_t signal_rows, int64_t rot_chunks, int64_t signal_value,
                                        int64_t chunk_counters) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.is_contiguous() && slot_src.is_cuda() && slot_src.is_contiguous());
  TORCH_CHECK(slot_src.scalar_type() == at::kInt && slot_src.numel() == E * C && x.size(1) % 16 == 0 && x.element_size() == 2);
  const c10::cuda::CUDAGuard guard(x.device());
  const void* g = nullptr;
  if (gates.has_value() && gates->defined()) {
    TORCH_CHECK(gates->is_cuda() && gates->scalar_type() == at::kFloat && gates->is_contiguous());
    g = gates->data_ptr();
  }
  std::vector<at::Tensor> out;
  void* q = nullptr;
  float* sc = nullptr;
  if (dst_ptr_table == 0) {
    out.push_back(at::empty({E * C, x.size(1)}, x.options().dtype(at::kFloat8_e4m3fn)));
    out.push_back(at::empty({E * C}, x.options().dtype(at::kFloat)));
    q = out[0].data_ptr();
    sc = out[1].data_ptr<float>();
  } else {
    TORCH_CHECK(scale_ptr_table != 0, "encode_rows_fp8: a remote push needs scale_ptr_table");
  }
  TB_CHECK_CUDA(tb::encode_rows_fp8(x.data_ptr(), g, slot_src.data_ptr<int>(), q, sc,
                                    reinterpret_cast<const unsigned long long*>(dst_ptr_table),
                                    reinterpret_cast<const unsigned long long*>(scale_ptr_table),
                                    reinterpret_cast<const unsigned long long*>(signal_ptr_table),
                                    reinterpret_cast<unsigned int*>(chunk_counters), static_cast<int>(signal_rows),
                                    static_cast<int>(x.size(0)), static_cast<int>(E), static_cast<int>(k), static_cast<int>(C),
                                    static_cast<int>(x.size(1)), elem_type_of(x), static_cast<int>(rot_chunks),
                                    static_cast<int>(signal_value), cur_stream()));
  return out;
}

// Expert-packed buffers: seg_off int [E + 1] (or at least [E]) of the packed layout; the buffer is [R, M] and C is
// ignored (every location of a routed choice lies inside its expert's segment).
const int* packed_seg_off(const c10::optional<at::Tensor>& seg_off, int64_t E) {
  if (!seg_off.has_value() || !seg_off->defined()) return nullptr;
  TORCH_CHECK(seg_off->is_cuda() && seg_off->scalar_type() == at::kInt && seg_off->is_contiguous() && seg_off->numel() >= E,
              "tutel_b200: seg_off must be a contiguous int32 [E + 1]");
  return seg_off->data_ptr<int>();
}

// Shared experts' terms of the combine: base [S, M] of `like`'s dtype; shared_logit float [S] or None.
const void* shared_base(const c10::optional<at::Tensor>& base, const at::Tensor& like, int S, int64_t M) {
  if (!base.has_value() || !base->defined()) return nullptr;
  TORCH_CHECK(base->is_cuda() && base->is_contiguous() && base->scalar_type() == like.scalar_type() && base->dim() == 2 &&
                  base->size(0) == S && base->size(1) == M,
              "tutel_b200: the shared experts' output must be a contiguous [S, M] tensor of the routed buffer's dtype");
  return base->data_ptr();
}

const float* shared_logits(const c10::optional<at::Tensor>& shared_logit, int S) {
  if (!shared_logit.has_value() || !shared_logit->defined()) return nullptr;
  TORCH_CHECK(shared_logit->is_cuda() && shared_logit->scalar_type() == at::kFloat && shared_logit->is_contiguous() &&
                  shared_logit->numel() == S, "tutel_b200: shared_logit must be a contiguous float [S]");
  return shared_logit->data_ptr<float>();
}

// buf [E*C, M] (seg_off: [R, M]); gates float [k, S] or None; idx/loc int [k, S]; returns [S, M].
// base / shared_logit: the shared experts' output and gate logits (see tb::decode_rows), or None.
at::Tensor decode_rows_shared(const at::Tensor& buf, const c10::optional<at::Tensor>& gates, const at::Tensor& idx,
                              const at::Tensor& loc, int64_t E, int64_t C, int64_t wait_flags, int64_t wait_target,
                              const c10::optional<at::Tensor>& seg_off, const c10::optional<at::Tensor>& base,
                              const c10::optional<at::Tensor>& shared_logit) {
  TORCH_CHECK(buf.is_cuda() && buf.is_contiguous() && idx.is_cuda() && loc.is_cuda());
  TORCH_CHECK(idx.scalar_type() == at::kInt && loc.scalar_type() == at::kInt && idx.is_contiguous() && loc.is_contiguous());
  const c10::cuda::CUDAGuard guard(buf.device());
  const int k = static_cast<int>(idx.size(0)), S = static_cast<int>(idx.size(1));
  const int* so = packed_seg_off(seg_off, E);
  if (so != nullptr) {
    TORCH_CHECK(buf.dim() == 2, "decode_rows: a packed buffer is [R, M]");
    C = buf.size(0);
  }
  const int64_t rows = so != nullptr ? C : E * C;
  const bool has_base = base.has_value() && base->defined();
  // (an empty buffer, C = 0, takes the width from the shared experts' output or its own last dim)
  const int M = static_cast<int>(rows > 0 ? buf.numel() / rows : (has_base ? base->size(-1) : buf.size(-1)));
  const void* g = nullptr;
  if (gates.has_value() && gates->defined()) {
    TORCH_CHECK(gates->is_cuda() && gates->scalar_type() == at::kFloat && gates->is_contiguous());
    g = gates->data_ptr();
  }
  const void* b = shared_base(base, buf, S, M);
  const float* sl = shared_logits(shared_logit, S);
  TORCH_CHECK(sl == nullptr || b != nullptr, "decode_rows: shared_logit needs the shared experts' output");
  at::Tensor out = at::empty({S, M}, buf.options());
  TB_CHECK_CUDA(tb::decode_rows(buf.data_ptr(), g, idx.data_ptr<int>(), loc.data_ptr<int>(), out.data_ptr(),
                                reinterpret_cast<const uint32_t*>(wait_flags), static_cast<uint32_t>(wait_target), S,
                                static_cast<int>(E), k, static_cast<int>(C), M, elem_type_of(buf), cur_stream(), so, b, sl));
  return out;
}

at::Tensor decode_rows_packed(const at::Tensor& buf, const c10::optional<at::Tensor>& gates, const at::Tensor& idx,
                              const at::Tensor& loc, int64_t E, int64_t C, int64_t wait_flags, int64_t wait_target,
                              const c10::optional<at::Tensor>& seg_off) {
  return decode_rows_shared(buf, gates, idx, loc, E, C, wait_flags, wait_target, seg_off, c10::nullopt, c10::nullopt);
}

at::Tensor decode_rows(const at::Tensor& buf, const c10::optional<at::Tensor>& gates, const at::Tensor& idx,
                       const at::Tensor& loc, int64_t E, int64_t C, int64_t wait_flags, int64_t wait_target) {
  return decode_rows_packed(buf, gates, idx, loc, E, C, wait_flags, wait_target, c10::nullopt);
}

// a [S, M], buf [E*C, M] (seg_off: [R, M]) -> float [k, S]
at::Tensor gate_grad_packed(const at::Tensor& a, const at::Tensor& buf, const at::Tensor& idx, const at::Tensor& loc,
                            int64_t E, int64_t C, const c10::optional<at::Tensor>& seg_off) {
  TORCH_CHECK(a.is_cuda() && a.is_contiguous() && buf.is_cuda() && buf.is_contiguous());
  TORCH_CHECK(a.scalar_type() == buf.scalar_type());
  const c10::cuda::CUDAGuard guard(a.device());
  const int k = static_cast<int>(idx.size(0)), S = static_cast<int>(idx.size(1));
  const int* so = packed_seg_off(seg_off, E);
  if (so != nullptr) {
    TORCH_CHECK(buf.dim() == 2 && buf.size(1) == a.size(1), "gate_grad: a packed buffer is [R, M]");
    C = buf.size(0);
  }
  at::Tensor out = at::empty({k, S}, a.options().dtype(at::kFloat));
  TB_CHECK_CUDA(tb::gate_grad(a.data_ptr(), buf.data_ptr(), idx.data_ptr<int>(), loc.data_ptr<int>(), out.data_ptr(),
                              S, static_cast<int>(E), k, static_cast<int>(C), static_cast<int>(a.size(1)),
                              elem_type_of(a), cur_stream(), so));
  return out;
}

at::Tensor gate_grad(const at::Tensor& a, const at::Tensor& buf, const at::Tensor& idx, const at::Tensor& loc,
                     int64_t E, int64_t C) {
  return gate_grad_packed(a, buf, idx, loc, E, C, c10::nullopt);
}

// Gated shared experts: a [S, M] (dy of the combine), buf as gate_grad (None when idx / loc are [0, S]), base [S, M],
// shared_logit float [S] -> [dgate float [k, S], d_base [S, M] = w * a, d_shared_logit float [S]], one launch.
std::vector<at::Tensor> gate_grad_shared(const at::Tensor& a, const c10::optional<at::Tensor>& buf, const at::Tensor& idx,
                                         const at::Tensor& loc, int64_t E, int64_t C,
                                         const c10::optional<at::Tensor>& seg_off, const at::Tensor& base,
                                         const at::Tensor& shared_logit) {
  TORCH_CHECK(a.is_cuda() && a.is_contiguous() && a.dim() == 2);
  TORCH_CHECK(idx.scalar_type() == at::kInt && loc.scalar_type() == at::kInt && idx.is_contiguous() && loc.is_contiguous());
  const c10::cuda::CUDAGuard guard(a.device());
  const int k = static_cast<int>(idx.size(0)), S = static_cast<int>(idx.size(1));
  TORCH_CHECK(a.size(0) == S, "gate_grad: a is [S, M]");
  const void* bp = nullptr;
  const int* so = nullptr;
  if (k > 0) {
    TORCH_CHECK(buf.has_value() && buf->defined() && buf->is_cuda() && buf->is_contiguous() &&
                    buf->scalar_type() == a.scalar_type(), "gate_grad: the routed buffer is required when k > 0");
    so = packed_seg_off(seg_off, E);
    if (so != nullptr) {
      TORCH_CHECK(buf->dim() == 2 && buf->size(1) == a.size(1), "gate_grad: a packed buffer is [R, M]");
      C = buf->size(0);
    }
    bp = buf->data_ptr();
  }
  const void* b = shared_base(base, a, S, a.size(1));
  const float* sl = shared_logits(shared_logit, S);
  TORCH_CHECK(b != nullptr && sl != nullptr, "gate_grad: base and shared_logit are required");
  at::Tensor dgate = at::empty({k, S}, a.options().dtype(at::kFloat));
  at::Tensor d_base = at::empty_like(a);
  at::Tensor d_logit = at::empty({S}, a.options().dtype(at::kFloat));
  TB_CHECK_CUDA(tb::gate_grad(a.data_ptr(), bp, idx.data_ptr<int>(), loc.data_ptr<int>(), k > 0 ? dgate.data_ptr() : nullptr,
                              S, static_cast<int>(E), k, static_cast<int>(C), static_cast<int>(a.size(1)), elem_type_of(a),
                              cur_stream(), so, b, sl, d_base.data_ptr(), d_logit.data_ptr<float>()));
  return {dgate, d_base, d_logit};
}

// Expert-packed layout (see tb::packed_layout): idx / loc int [k, S], counts int [E], R rows ->
// [seg_off [E + 1], block_expert [R / 128], block_rows [R / 128], slot_src [R]]
std::vector<at::Tensor> packed_layout(const at::Tensor& idx, const at::Tensor& loc, const at::Tensor& counts, int64_t R) {
  TORCH_CHECK(idx.is_cuda() && loc.is_cuda() && counts.is_cuda() && idx.scalar_type() == at::kInt &&
              loc.scalar_type() == at::kInt && counts.scalar_type() == at::kInt && idx.is_contiguous() &&
              loc.is_contiguous() && counts.is_contiguous() && idx.dim() == 2 && loc.sizes() == idx.sizes(),
              "packed_layout: contiguous int32 CUDA idx / loc [k, S] and counts [E] expected");
  TORCH_CHECK(R > 0 && R % 128 == 0, "packed_layout: R must be a positive multiple of 128");
  const c10::cuda::CUDAGuard guard(idx.device());
  const int64_t E = counts.numel();
  auto opts = idx.options();
  at::Tensor seg_off = at::empty({E + 1}, opts), block_expert = at::empty({R / 128}, opts),
             block_rows = at::empty({R / 128}, opts), slot = at::empty({R}, opts);
  TB_CHECK_CUDA(tb::packed_layout(idx.data_ptr<int>(), loc.data_ptr<int>(), counts.data_ptr<int>(), seg_off.data_ptr<int>(),
                                  block_expert.data_ptr<int>(), block_rows.data_ptr<int>(), slot.data_ptr<int>(),
                                  static_cast<int>(idx.size(1)), static_cast<int>(E), static_cast<int>(idx.size(0)),
                                  static_cast<int>(R), cur_stream()));
  return {seg_off, block_expert, block_rows, slot};
}

// logits [S, E] (fp32 / fp16 / bf16) -> [scores fp32 [S,E], idx int [k,S], top fp32 [k,S], gates fp32 [k,S], loc int [k,S],
// counts int [E], ce fp32 [E], l_aux (scalar, logits dtype), slot_src int [E*C] (only when C > 0)]   - two launches
std::vector<at::Tensor> gate_route_forward(const at::Tensor& logits, int64_t k, int64_t C, bool normalize, double eps) {
  TORCH_CHECK(logits.is_cuda() && logits.dim() == 2 && logits.is_contiguous(), "gate_route_forward: contiguous CUDA [S, E] logits expected");
  const c10::cuda::CUDAGuard guard(logits.device());
  const int S = static_cast<int>(logits.size(0)), E = static_cast<int>(logits.size(1));
  TORCH_CHECK(E <= 512 && k >= 1 && k <= 32 && k <= E, "gate_route_forward: needs E <= 512 and 1 <= k <= min(32, E)");
  const int tiles = tb::gate_route_tiles(S);
  auto f32 = logits.options().dtype(at::kFloat);
  auto i32 = logits.options().dtype(at::kInt);
  at::Tensor scores = at::empty({S, E}, f32);
  at::Tensor idx = at::empty({k, S}, i32), loc = at::empty({k, S}, i32), counts = at::empty({E}, i32);
  at::Tensor top = at::empty({k, S}, f32), gates = at::empty({k, S}, f32), ce = at::empty({E}, f32);
  at::Tensor l_aux = at::empty({}, logits.options());
  at::Tensor me = at::empty({tiles, E}, f32);
  at::Tensor hist = at::empty({tiles, k, E}, i32);
  at::Tensor slot;
  if (C > 0) slot = at::empty({E * C}, i32);
  TB_CHECK_CUDA(tb::gate_route_forward(logits.data_ptr(), scores.data_ptr<float>(), idx.data_ptr<int>(), top.data_ptr<float>(),
                                       gates.data_ptr<float>(), me.data_ptr<float>(), hist.data_ptr<int>(), loc.data_ptr<int>(),
                                       counts.data_ptr<int>(), C > 0 ? slot.data_ptr<int>() : nullptr, ce.data_ptr<float>(),
                                       l_aux.data_ptr(), S, E, static_cast<int>(k), static_cast<int>(C), normalize,
                                       static_cast<float>(eps), elem_type_of(logits), cur_stream()));
  std::vector<at::Tensor> out{scores, idx, top, gates, loc, counts, ce, l_aux};
  if (C > 0) out.push_back(slot);
  return out;
}

// -> d logits [S, E] in `like`'s dtype; dgates fp32 [k, S] or None; dl: scalar of `like`'s dtype or None      - one launch
at::Tensor gate_route_backward(const at::Tensor& scores, const at::Tensor& idx, const at::Tensor& top,
                               const c10::optional<at::Tensor>& dgates, const c10::optional<at::Tensor>& ce,
                               const c10::optional<at::Tensor>& dl, const at::Tensor& like, bool normalize, double eps) {
  TORCH_CHECK(scores.is_cuda() && scores.scalar_type() == at::kFloat && scores.dim() == 2 && scores.is_contiguous());
  const int S = static_cast<int>(scores.size(0)), E = static_cast<int>(scores.size(1));
  const int k = static_cast<int>(idx.size(0));
  TORCH_CHECK(idx.scalar_type() == at::kInt && idx.is_contiguous() && idx.size(1) == S);
  TORCH_CHECK(top.scalar_type() == at::kFloat && top.is_contiguous() && top.sizes() == idx.sizes());
  const float* dg_p = nullptr;
  const float* ce_p = nullptr;
  const void* dl_p = nullptr;
  if (dgates.has_value() && dgates->defined()) {
    TORCH_CHECK(dgates->scalar_type() == at::kFloat && dgates->is_contiguous() && dgates->sizes() == idx.sizes());
    dg_p = dgates->data_ptr<float>();
  }
  if (ce.has_value() && ce->defined() && dl.has_value() && dl->defined()) {
    TORCH_CHECK(ce->is_cuda() && ce->scalar_type() == at::kFloat && ce->is_contiguous() && ce->numel() == E);
    TORCH_CHECK(dl->is_cuda() && dl->scalar_type() == like.scalar_type() && dl->numel() == 1);
    ce_p = ce->data_ptr<float>();
    dl_p = dl->data_ptr();
  }
  const c10::cuda::CUDAGuard guard(scores.device());
  at::Tensor out = at::empty({S, E}, like.options());
  TB_CHECK_CUDA(tb::gate_route_backward(scores.data_ptr<float>(), idx.data_ptr<int>(), top.data_ptr<float>(), dg_p, ce_p, dl_p,
                                        out.data_ptr(), S, E, k, normalize, static_cast<float>(eps), elem_type_of(like),
                                        cur_stream()));
  return out;
}

// Sigmoid scoring with a selection bias and group-limited choice: same outputs as gate_route_forward (top = unbiased
// scores, ce = fp32 all-choice counts); `expert_load` fp32 [E] (optional) accumulates the all-choice counts.
std::vector<at::Tensor> sigmoid_gate_route_forward(const at::Tensor& logits, const at::Tensor& bias, int64_t k, int64_t C,
                                                   bool normalize, double eps, int64_t n_group, int64_t topk_group,
                                                   double scale, const c10::optional<at::Tensor>& expert_load) {
  TORCH_CHECK(logits.is_cuda() && logits.dim() == 2 && logits.is_contiguous(), "sigmoid_gate_route_forward: contiguous CUDA [S, E] logits expected");
  const c10::cuda::CUDAGuard guard(logits.device());
  const int S = static_cast<int>(logits.size(0)), E = static_cast<int>(logits.size(1));
  TORCH_CHECK(E <= 512 && k >= 1 && k <= 32 && k <= E, "sigmoid_gate_route_forward: needs E <= 512 and 1 <= k <= min(32, E)");
  TORCH_CHECK(n_group >= 1 && n_group <= 32 && E % n_group == 0 && topk_group >= 1 && topk_group <= n_group &&
              k <= topk_group * (E / n_group),
              "sigmoid_gate_route_forward: needs n_group <= 32 dividing E, 1 <= topk_group <= n_group and k <= topk_group * E / n_group");
  TORCH_CHECK(bias.is_cuda() && bias.device() == logits.device() && bias.scalar_type() == at::kFloat && bias.is_contiguous() && bias.numel() == E,
              "sigmoid_gate_route_forward: fp32 [E] bias on the logits' device expected");
  float* load_p = nullptr;
  if (expert_load.has_value() && expert_load->defined()) {
    TORCH_CHECK(expert_load->is_cuda() && expert_load->device() == logits.device() && expert_load->scalar_type() == at::kFloat &&
                expert_load->is_contiguous() && expert_load->numel() == E,
                "sigmoid_gate_route_forward: fp32 [E] expert_load on the logits' device expected");
    load_p = expert_load->data_ptr<float>();
  }
  const int tiles = tb::gate_route_tiles(S);
  auto f32 = logits.options().dtype(at::kFloat);
  auto i32 = logits.options().dtype(at::kInt);
  at::Tensor scores = at::empty({S, E}, f32);
  at::Tensor idx = at::empty({k, S}, i32), loc = at::empty({k, S}, i32), counts = at::empty({E}, i32);
  at::Tensor top = at::empty({k, S}, f32), gates = at::empty({k, S}, f32), ce = at::empty({E}, f32);
  at::Tensor l_aux = at::empty({}, logits.options());
  at::Tensor me = at::empty({tiles, E}, f32);
  at::Tensor hist = at::empty({tiles, k, E}, i32);
  at::Tensor slot;
  if (C > 0) slot = at::empty({E * C}, i32);
  TB_CHECK_CUDA(tb::sigmoid_gate_route_forward(
      logits.data_ptr(), bias.data_ptr<float>(), scores.data_ptr<float>(), idx.data_ptr<int>(), top.data_ptr<float>(),
      gates.data_ptr<float>(), me.data_ptr<float>(), hist.data_ptr<int>(), loc.data_ptr<int>(), counts.data_ptr<int>(),
      C > 0 ? slot.data_ptr<int>() : nullptr, ce.data_ptr<float>(), l_aux.data_ptr(), load_p, S, E, static_cast<int>(k),
      static_cast<int>(C), normalize, static_cast<float>(eps), static_cast<int>(n_group), static_cast<int>(topk_group),
      static_cast<float>(scale), elem_type_of(logits), cur_stream()));
  std::vector<at::Tensor> out{scores, idx, top, gates, loc, counts, ce, l_aux};
  if (C > 0) out.push_back(slot);
  return out;
}

// -> d logits [S, E] in `like`'s dtype, as gate_route_backward with the sigmoid closed form; ce = all-choice counts
at::Tensor sigmoid_gate_route_backward(const at::Tensor& scores, const at::Tensor& idx, const at::Tensor& top,
                                       const c10::optional<at::Tensor>& dgates, const c10::optional<at::Tensor>& ce,
                                       const c10::optional<at::Tensor>& dl, const at::Tensor& like, bool normalize,
                                       double eps, double scale) {
  TORCH_CHECK(scores.is_cuda() && scores.scalar_type() == at::kFloat && scores.dim() == 2 && scores.is_contiguous());
  const int S = static_cast<int>(scores.size(0)), E = static_cast<int>(scores.size(1));
  const int k = static_cast<int>(idx.size(0));
  TORCH_CHECK(idx.scalar_type() == at::kInt && idx.is_contiguous() && idx.size(1) == S);
  TORCH_CHECK(top.scalar_type() == at::kFloat && top.is_contiguous() && top.sizes() == idx.sizes());
  const float* dg_p = nullptr;
  const float* ce_p = nullptr;
  const void* dl_p = nullptr;
  if (dgates.has_value() && dgates->defined()) {
    TORCH_CHECK(dgates->scalar_type() == at::kFloat && dgates->is_contiguous() && dgates->sizes() == idx.sizes());
    dg_p = dgates->data_ptr<float>();
  }
  if (ce.has_value() && ce->defined() && dl.has_value() && dl->defined()) {
    TORCH_CHECK(ce->is_cuda() && ce->scalar_type() == at::kFloat && ce->is_contiguous() && ce->numel() == E);
    TORCH_CHECK(dl->is_cuda() && dl->scalar_type() == like.scalar_type() && dl->numel() == 1);
    ce_p = ce->data_ptr<float>();
    dl_p = dl->data_ptr();
  }
  const c10::cuda::CUDAGuard guard(scores.device());
  at::Tensor out = at::empty({S, E}, like.options());
  TB_CHECK_CUDA(tb::sigmoid_gate_route_backward(scores.data_ptr<float>(), idx.data_ptr<int>(), top.data_ptr<float>(), dg_p,
                                                ce_p, dl_p, out.data_ptr(), S, E, k, normalize, static_cast<float>(eps),
                                                static_cast<float>(scale), elem_type_of(like), cur_stream()));
  return out;
}

// in place: bias[e] += gamma * sign(mean(load) - load[e]); load = 0      - one launch
void expert_bias_update(at::Tensor& bias, at::Tensor& load, double gamma) {
  TORCH_CHECK(bias.is_cuda() && bias.scalar_type() == at::kFloat && bias.is_contiguous(), "expert_bias_update: fp32 CUDA bias expected");
  TORCH_CHECK(load.device() == bias.device() && load.scalar_type() == at::kFloat && load.is_contiguous() &&
              load.numel() == bias.numel(), "expert_bias_update: fp32 load of the bias' shape and device expected");
  const c10::cuda::CUDAGuard guard(bias.device());
  TB_CHECK_CUDA(tb::expert_bias_update(bias.data_ptr<float>(), load.data_ptr<float>(), static_cast<int>(bias.numel()),
                                       static_cast<float>(gamma), cur_stream()));
}

// Segmented column sums: x [R, N] (rows contiguous), offsets int [G + 1] -> [G, N], row g = sum of rows
// [offsets[g], offsets[g + 1]) in x's dtype (fp32 accumulation; no host read of the offsets).
at::Tensor grouped_colsum_offsets(const at::Tensor& x, const at::Tensor& offsets) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.stride(1) == 1, "grouped_colsum: CUDA [R, N] tensor expected with offsets");
  TORCH_CHECK(offsets.is_cuda() && offsets.scalar_type() == at::kInt && offsets.is_contiguous() && offsets.numel() >= 2,
              "grouped_colsum: offsets must be a contiguous int32 [G + 1]");
  const c10::cuda::CUDAGuard guard(x.device());
  const int G = static_cast<int>(offsets.numel() - 1), R = static_cast<int>(x.size(0)), N = static_cast<int>(x.size(1));
  // the offsets are not known here: split as if one segment held every row (blocks of shorter segments finish early)
  const int splits = tb::colsum_row_splits(1, R, N, static_cast<int>(x.element_size()));
  at::Tensor acc = at::zeros({G, N}, x.options().dtype(at::kFloat));
  at::Tensor out = at::empty({G, N}, x.options());
  TB_CHECK_CUDA(tb::grouped_colsum(x.data_ptr(), x.stride(0), 0, out.data_ptr(), acc.data_ptr<float>(), G, R, N,
                                   splits > 1 ? splits : 2, elem_type_of(x), cur_stream(), offsets.data_ptr<int>()));
  out.copy_(acc);
  return out;
}

// x [G, T, N] (last dim contiguous) -> [G, N] column sums in x's dtype (fp32 accumulation)
at::Tensor grouped_colsum(const at::Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 3 && x.stride(2) == 1, "grouped_colsum: CUDA [G, T, N] tensor expected");
  const c10::cuda::CUDAGuard guard(x.device());
  const int G = static_cast<int>(x.size(0)), T = static_cast<int>(x.size(1)), N = static_cast<int>(x.size(2));
  const int splits = tb::colsum_row_splits(G, T, N, static_cast<int>(x.element_size()));
  at::Tensor out = at::empty({G, N}, x.options());
  at::Tensor acc;
  if (splits > 1) acc = at::zeros({G, N}, x.options().dtype(at::kFloat));
  TB_CHECK_CUDA(tb::grouped_colsum(x.data_ptr(), x.stride(1), x.stride(0), out.data_ptr(),
                                   splits > 1 ? acc.data_ptr<float>() : nullptr, G, T, N, splits, elem_type_of(x), cur_stream()));
  if (splits > 1) out.copy_(acc);
  return out;
}

// int [S, E] -> cumsum along dim 0 minus one (int32)
at::Tensor cumsum_sub_one(const at::Tensor& data) {
  TORCH_CHECK(data.is_cuda() && data.dim() == 2, "cumsum_sub_one: CUDA [S, E] tensor expected");
  const c10::cuda::CUDAGuard guard(data.device());
  at::Tensor x = data.to(at::kInt).contiguous();
  const int S = static_cast<int>(x.size(0)), E = static_cast<int>(x.size(1));
  at::Tensor out = at::empty_like(x);
  at::Tensor ws = at::empty({static_cast<int64_t>(tb::cumsum_workspace_ints(S, E))}, x.options());
  TB_CHECK_CUDA(tb::cumsum_sub_one(x.data_ptr<int>(), out.data_ptr<int>(), ws.data_ptr<int>(), S, E, cur_stream()));
  return out;
}

std::vector<at::Tensor> quantize_rows(const at::Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous() && x.dim() >= 2, "quantize_rows: contiguous CUDA tensor [.., K] expected");
  const c10::cuda::CUDAGuard guard(x.device());
  const int K = static_cast<int>(x.size(-1));
  const int64_t R = x.numel() / K;
  at::Tensor q = at::empty(x.sizes(), x.options().dtype(at::kFloat8_e4m3fn));
  auto lead = x.sizes().vec();
  lead.pop_back();
  at::Tensor scale = at::empty(lead, x.options().dtype(at::kFloat));
  TB_CHECK_CUDA(tb::quantize_rows_e4m3(x.data_ptr(), q.data_ptr(), scale.data_ptr<float>(), R, K, elem_type_of(x), cur_stream()));
  return {q, scale};
}

// x [G, R, K] (16 bit) -> [qT e4m3 [G, K, R], scale fp32 [G, K]]   (transposed copy with one scale per output row)
std::vector<at::Tensor> quantize_transpose(const at::Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous() && x.dim() == 3 && x.element_size() == 2 && x.size(1) % 128 == 0 && x.size(2) % 64 == 0,
              "quantize_transpose: contiguous 16-bit CUDA tensor [G, R, K] with R % 128 == 0 and K % 64 == 0 expected");
  const c10::cuda::CUDAGuard guard(x.device());
  const int G = static_cast<int>(x.size(0)), R = static_cast<int>(x.size(1)), K = static_cast<int>(x.size(2));
  at::Tensor q = at::empty({G, K, R}, x.options().dtype(at::kFloat8_e4m3fn));
  at::Tensor scale = at::empty({G, K}, x.options().dtype(at::kFloat));
  at::Tensor ws = at::empty({G, K}, x.options().dtype(at::kFloat));
  TB_CHECK_CUDA(tb::quantize_transpose_e4m3(x.data_ptr(), q.data_ptr(), scale.data_ptr<float>(), ws.data_ptr<float>(), G, R, K,
                                            elem_type_of(x), cur_stream()));
  return {q, scale};
}

// q e4m3 [.., K], scale fp32 [..] -> 16-bit [.., K]
at::Tensor dequant_rows(const at::Tensor& q, const at::Tensor& scale, at::ScalarType dtype) {
  TORCH_CHECK(q.is_cuda() && q.is_contiguous() && q.scalar_type() == at::kFloat8_e4m3fn && scale.is_cuda() && scale.is_contiguous() &&
              scale.scalar_type() == at::kFloat && q.dim() >= 2 && scale.numel() * q.size(-1) == q.numel());
  const c10::cuda::CUDAGuard guard(q.device());
  at::Tensor y = at::empty(q.sizes(), q.options().dtype(dtype));
  TB_CHECK_CUDA(tb::dequant_rows_e4m3(q.data_ptr(), scale.data_ptr<float>(), y.data_ptr(), scale.numel(), static_cast<int>(q.size(-1)),
                                      elem_type_of(y), cur_stream()));
  return y;
}

// MX block-scaled fp8 (OCP MX: e4m3 elements, one UE8M0 scale per 32 K elements); see csrc/gemm_mx.cu.
// x [G, R, K] (16 bit, K % 128 == 0) -> [q e4m3 [G, R, K], sf uint8 (tile-ordered scale atoms, csrc/gemm_mx.h)]
std::vector<at::Tensor> mx_quantize(const at::Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous() && x.dim() == 3 && x.element_size() == 2 && x.size(2) % 128 == 0,
              "mx_quantize: contiguous 16-bit CUDA tensor [G, R, K] with K % 128 == 0 expected");
  const c10::cuda::CUDAGuard guard(x.device());
  const int G = static_cast<int>(x.size(0)), R = static_cast<int>(x.size(1)), K = static_cast<int>(x.size(2));
  at::Tensor q = at::empty({G, R, K}, x.options().dtype(at::kFloat8_e4m3fn));
  const long long sf_bytes = tb::mx_sf_bytes(G, R, K);
  at::Tensor sf = (R % 128 == 0) ? at::empty({sf_bytes}, x.options().dtype(at::kByte))
                                 : at::zeros({sf_bytes}, x.options().dtype(at::kByte));
  TB_CHECK_CUDA(tb::mx_quantize(x.data_ptr(), q.data_ptr(), sf.data_ptr(), G, R, K, elem_type_of(x), cur_stream()));
  return {q, sf};
}

// x [G, R, K] (16 bit, R % 128 == 0, K % 64 == 0) -> [qT e4m3 [G, K, R] quantised along R, sf]
std::vector<at::Tensor> mx_quantize_transpose(const at::Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous() && x.dim() == 3 && x.element_size() == 2 && x.size(1) % 128 == 0 && x.size(2) % 64 == 0,
              "mx_quantize_transpose: contiguous 16-bit CUDA tensor [G, R, K] with R % 128 == 0 and K % 64 == 0 expected");
  const c10::cuda::CUDAGuard guard(x.device());
  const int G = static_cast<int>(x.size(0)), R = static_cast<int>(x.size(1)), K = static_cast<int>(x.size(2));
  at::Tensor q = at::empty({G, K, R}, x.options().dtype(at::kFloat8_e4m3fn));
  const long long sf_bytes = tb::mx_sf_bytes(G, K, R);
  at::Tensor sf = (K % 128 == 0) ? at::empty({sf_bytes}, x.options().dtype(at::kByte))
                                 : at::zeros({sf_bytes}, x.options().dtype(at::kByte));
  TB_CHECK_CUDA(tb::mx_quantize_transpose(x.data_ptr(), q.data_ptr(), sf.data_ptr(), G, R, K, elem_type_of(x), cur_stream()));
  return {q, sf};
}

// d[g] = epilogue(a[g] * b[g]^T + bias[g]) :  a e4m3 [G, M, K], b e4m3 [G, N, K], scales from mx_quantize -> bf16 [G, M, N]
// epilogue: 0 none, 1 ReLU, 2 ReLU backward (d = aux > 0 ? acc : 0 with aux bf16 [G, M, N])
at::Tensor mx_gemm(const at::Tensor& a, const at::Tensor& sfa, const at::Tensor& b, const at::Tensor& sfb,
                   const c10::optional<at::Tensor>& bias, const c10::optional<at::Tensor>& aux, int64_t epilogue,
                   int64_t block_n, int64_t cta_group, int64_t max_ctas) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && sfa.is_cuda() && sfb.is_cuda() && a.dim() == 3 && b.dim() == 3);
  TORCH_CHECK(a.is_contiguous() && b.is_contiguous() && sfa.is_contiguous() && sfb.is_contiguous());
  TORCH_CHECK(a.scalar_type() == at::kFloat8_e4m3fn && b.scalar_type() == at::kFloat8_e4m3fn &&
              sfa.scalar_type() == at::kByte && sfb.scalar_type() == at::kByte, "mx_gemm: e4m3 operands and uint8 scales expected");
  TORCH_CHECK(a.size(0) == b.size(0) && a.size(2) == b.size(2), "mx_gemm: a [G, M, K] and b [G, N, K] expected");
  const c10::cuda::CUDAGuard guard(a.device());
  tb::MxGemmProblem p;
  p.G = static_cast<int>(a.size(0)); p.M = static_cast<int>(a.size(1)); p.K = static_cast<int>(a.size(2));
  p.N = static_cast<int>(b.size(1));
  TORCH_CHECK(sfa.numel() == tb::mx_sf_bytes(p.G, p.M, p.K) && sfb.numel() == tb::mx_sf_bytes(p.G, p.N, p.K),
              "mx_gemm: scale arrays do not match the operand shapes");
  at::Tensor d = at::empty({p.G, p.M, p.N}, a.options().dtype(at::kBFloat16));
  p.a = a.data_ptr(); p.sfa = sfa.data_ptr(); p.b = b.data_ptr(); p.sfb = sfb.data_ptr(); p.d = d.data_ptr();
  p.ldd = p.N; p.d_group_stride = static_cast<long long>(p.M) * p.N;
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(bias->is_cuda() && bias->scalar_type() == at::kBFloat16 && bias->is_contiguous() && bias->numel() == static_cast<long long>(p.G) * p.N,
                "mx_gemm: bias must be a contiguous bf16 [G, N]");
    p.bias = bias->data_ptr(); p.bias_group_stride = p.N;
  }
  if (aux.has_value() && aux->defined()) {
    TORCH_CHECK(aux->is_cuda() && aux->scalar_type() == at::kBFloat16 && aux->is_contiguous() && aux->numel() == d.numel(),
                "mx_gemm: aux must be a contiguous bf16 [G, M, N]");
    p.aux = aux->data_ptr(); p.ld_aux = p.N; p.aux_group_stride = p.d_group_stride;
  }
  p.epilogue = static_cast<int>(epilogue);
  p.block_n = static_cast<int>(block_n);
  p.cta_group = static_cast<int>(cta_group);
  p.max_ctas = static_cast<int>(max_ctas);
  const char* why = nullptr;
  cudaError_t e = tb::mx_gemm_launch(p, cur_stream(), &why);
  TORCH_CHECK(e == cudaSuccess, "mx_gemm: ", why ? why : cudaGetErrorString(e));
  return d;
}

// Block-scaled fp8 (DeepSeek-V3: 1 x 128 activation tiles, 128 x 128 weight blocks, fp32 scales); see csrc/gemm_block_fp8.cu.
// x [G, R, K] bf16 (K % 128 == 0) -> [q e4m3 [G, R, K], s fp32 [G, K / 128, roundup(R, 128)]]
std::vector<at::Tensor> block_fp8_quantize_act(const at::Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous() && x.dim() == 3 && x.scalar_type() == at::kBFloat16 && x.size(2) % 128 == 0,
              "block_fp8_quantize_act: contiguous bf16 CUDA tensor [G, R, K] with K % 128 == 0 expected");
  const c10::cuda::CUDAGuard guard(x.device());
  const int G = static_cast<int>(x.size(0)), R = static_cast<int>(x.size(1)), K = static_cast<int>(x.size(2));
  at::Tensor q = at::empty({G, R, K}, x.options().dtype(at::kFloat8_e4m3fn));
  at::Tensor s = at::empty({G, K / 128, (R + 127) / 128 * 128}, x.options().dtype(at::kFloat));
  TB_CHECK_CUDA(tb::block_fp8_quantize_act(x.data_ptr(), q.data_ptr(), s.data_ptr<float>(), G, R, K, cur_stream()));
  return {q, s};
}

// The same for one group x [1, R, K] bounded by live_rows (device int32 [1], the packed layout's seg_off[E]): rows at or
// past it are neither read nor written (q and s are left uninitialised there).
std::vector<at::Tensor> block_fp8_quantize_act_bounded(const at::Tensor& x, const at::Tensor& live_rows) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous() && x.dim() == 3 && x.size(0) == 1 && x.scalar_type() == at::kBFloat16 &&
                  x.size(2) % 128 == 0,
              "block_fp8_quantize_act: a bounded launch takes a contiguous bf16 CUDA tensor [1, R, K] with K % 128 == 0");
  TORCH_CHECK(live_rows.is_cuda() && live_rows.scalar_type() == at::kInt && live_rows.numel() == 1 && live_rows.device() == x.device(),
              "block_fp8_quantize_act: live_rows must be a one-element int32 tensor on x's device");
  const c10::cuda::CUDAGuard guard(x.device());
  const int R = static_cast<int>(x.size(1)), K = static_cast<int>(x.size(2));
  at::Tensor q = at::empty({1, R, K}, x.options().dtype(at::kFloat8_e4m3fn));
  at::Tensor s = at::empty({1, K / 128, (R + 127) / 128 * 128}, x.options().dtype(at::kFloat));
  TB_CHECK_CUDA(tb::block_fp8_quantize_act(x.data_ptr(), q.data_ptr(), s.data_ptr<float>(), 1, R, K, cur_stream(),
                                           live_rows.data_ptr<int>()));
  return {q, s};
}

// w [G, R, C] bf16 (R, C % 128 == 0) -> [q [G, R, C], s [G, R / 128, C / 128], qT [G, C, R], sT [G, C / 128, R / 128]]
std::vector<at::Tensor> block_fp8_quantize_weight(const at::Tensor& w) {
  TORCH_CHECK(w.is_cuda() && w.is_contiguous() && w.dim() == 3 && w.scalar_type() == at::kBFloat16 && w.size(1) % 128 == 0 &&
                  w.size(2) % 128 == 0,
              "block_fp8_quantize_weight: contiguous bf16 CUDA tensor [G, R, C] with R % 128 == 0 and C % 128 == 0 expected");
  const c10::cuda::CUDAGuard guard(w.device());
  const int G = static_cast<int>(w.size(0)), R = static_cast<int>(w.size(1)), C = static_cast<int>(w.size(2));
  at::Tensor q = at::empty({G, R, C}, w.options().dtype(at::kFloat8_e4m3fn));
  at::Tensor qT = at::empty({G, C, R}, w.options().dtype(at::kFloat8_e4m3fn));
  at::Tensor s = at::empty({G, R / 128, C / 128}, w.options().dtype(at::kFloat));
  at::Tensor sT = at::empty({G, C / 128, R / 128}, w.options().dtype(at::kFloat));
  TB_CHECK_CUDA(tb::block_fp8_quantize_weight(w.data_ptr(), q.data_ptr(), s.data_ptr<float>(), qT.data_ptr(), sT.data_ptr<float>(),
                                              G, R, C, cur_stream()));
  return {q, s, qT, sT};
}

// SwiGLU gate / up weights w1, w2 [G, M, H] bf16 -> [qcat [G, M, 2H], scat [G, M / 128, 2H / 128],
// qglu [G, 2H, M] (interleaved every 64 rows), sglu [G, 2H / 64, M / 128]]  (csrc/gemm_block_fp8.h)
std::vector<at::Tensor> block_fp8_quantize_glu_weight(const at::Tensor& w1, const at::Tensor& w2) {
  TORCH_CHECK(w1.is_cuda() && w1.is_contiguous() && w2.is_contiguous() && w1.dim() == 3 && w1.sizes() == w2.sizes() &&
                  w1.scalar_type() == at::kBFloat16 && w2.scalar_type() == at::kBFloat16 && w2.device() == w1.device() &&
                  w1.size(1) % 128 == 0 && w1.size(2) % 128 == 0,
              "block_fp8_quantize_glu_weight: two contiguous bf16 CUDA tensors [G, M, H] with M % 128 == 0 and H % 128 == 0 expected");
  const c10::cuda::CUDAGuard guard(w1.device());
  const int G = static_cast<int>(w1.size(0)), M = static_cast<int>(w1.size(1)), H = static_cast<int>(w1.size(2));
  at::Tensor qcat = at::empty({G, M, 2 * H}, w1.options().dtype(at::kFloat8_e4m3fn));
  at::Tensor qglu = at::empty({G, 2 * H, M}, w1.options().dtype(at::kFloat8_e4m3fn));
  at::Tensor scat = at::empty({G, M / 128, 2 * H / 128}, w1.options().dtype(at::kFloat));
  at::Tensor sglu = at::empty({G, 2 * H / 64, M / 128}, w1.options().dtype(at::kFloat));
  TB_CHECK_CUDA(tb::block_fp8_quantize_glu_weight(w1.data_ptr(), w2.data_ptr(), qcat.data_ptr(), scat.data_ptr<float>(),
                                                  qglu.data_ptr(), sglu.data_ptr<float>(), G, M, H, cur_stream()));
  return {qcat, scat, qglu, sglu};
}

// d[g] = epilogue(a[g] * b[g]^T):  a e4m3 [G, M, K] + sa, b e4m3 [G, N, K] + sb (shapes above) -> bf16.
// epilogue 0 none / 1 ReLU (+ bias [G, N]) -> [d [G, M, N]];  2 ReLU backward (aux = forward activation) -> [d];
// 3 GLU (b = the interleaved gate / up copy, sb [G, N / 64, K / 128]) -> [h, g, u], each [G, M, N / 2];
// 4 GLU backward (acc = dh, aux = g, aux2 = u) -> [dgu [G, M, 2N]] with dg in columns [0, N) and du in [N, 2N).
// Block-mapped (b_group_map, csrc/gemm_block_fp8.h): a is [R, K] with sa [1, K / 128, R], aux / aux2 and the results are
// [R, *], and G is b's group count.
std::vector<at::Tensor> block_fp8_gemm_impl(const at::Tensor& a, const at::Tensor& sa, const at::Tensor& b, const at::Tensor& sb,
                                            const c10::optional<at::Tensor>& bias, const c10::optional<at::Tensor>& aux,
                                            const c10::optional<at::Tensor>& aux2, int64_t epilogue, int64_t act, int64_t max_ctas,
                                            const int* row_counts, const int* b_group_map = nullptr) {
  const bool mapped = b_group_map != nullptr;
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && sa.is_cuda() && sb.is_cuda() && a.dim() == (mapped ? 2 : 3) && b.dim() == 3 &&
              sa.dim() == 3 && sb.dim() == 3, mapped ? "block_fp8_gemm: a [R, K] and 3-D b, sa, sb CUDA tensors expected"
                                                     : "block_fp8_gemm: 3-D CUDA tensors expected");
  TORCH_CHECK(a.is_contiguous() && b.is_contiguous() && sa.is_contiguous() && sb.is_contiguous(),
              "block_fp8_gemm: contiguous operands expected");
  TORCH_CHECK(a.scalar_type() == at::kFloat8_e4m3fn && b.scalar_type() == at::kFloat8_e4m3fn &&
              sa.scalar_type() == at::kFloat && sb.scalar_type() == at::kFloat, "block_fp8_gemm: e4m3 operands and fp32 scales expected");
  TORCH_CHECK(mapped ? a.size(1) == b.size(2) : (a.size(0) == b.size(0) && a.size(2) == b.size(2)),
              mapped ? "block_fp8_gemm: a [R, K] and b [G, N, K] expected" : "block_fp8_gemm: a [G, M, K] and b [G, N, K] expected");
  TORCH_CHECK(epilogue >= tb::BF8_EPI_NONE && epilogue <= tb::BF8_EPI_GLU_BWD, "block_fp8_gemm: unknown epilogue");
  const c10::cuda::CUDAGuard guard(a.device());
  tb::BlockFp8GemmProblem p;
  p.G = static_cast<int>(b.size(0)); p.M = static_cast<int>(a.size(-2)); p.K = static_cast<int>(a.size(-1));
  p.N = static_cast<int>(b.size(1));
  const int64_t ga = mapped ? 1 : p.G;                 // groups of a, sa, aux and the results
  const bool glu = epilogue == tb::BF8_EPI_GLU, glu_bwd = epilogue == tb::BF8_EPI_GLU_BWD;
  const int64_t kb = (p.K + 127) / 128, mp = (p.M + 127) / 128 * 128, nb = glu ? (p.N + 63) / 64 : (p.N + 127) / 128;
  TORCH_CHECK(sa.size(0) == ga && sa.size(1) == kb && sa.size(2) == mp && sb.size(0) == p.G && sb.size(1) == nb && sb.size(2) == kb,
              glu ? "block_fp8_gemm: scale arrays do not match the operand shapes (sa [G, K / 128, roundup(M, 128)], sb [G, N / 64, K / 128] expected)"
                  : "block_fp8_gemm: scale arrays do not match the operand shapes (sa [G, K / 128, roundup(M, 128)], sb [G, N / 128, K / 128] expected)");
  const auto bf = a.options().dtype(at::kBFloat16);
  auto shape = [&](int64_t cols) { return mapped ? std::vector<int64_t>{p.M, cols} : std::vector<int64_t>{p.G, p.M, cols}; };
  auto check_mn = [&](const c10::optional<at::Tensor>& t, const char* name) -> const void* {
    if (!t.has_value() || !t->defined()) return nullptr;
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kBFloat16 && t->is_contiguous() && t->sizes() == at::IntArrayRef(shape(p.N)),
                "block_fp8_gemm: ", name, mapped ? " must be a contiguous bf16 [R, N]" : " must be a contiguous bf16 [G, M, N]");
    return t->data_ptr();
  };
  p.aux = check_mn(aux, "aux");
  p.aux2 = check_mn(aux2, "aux2");
  p.ld_aux = p.N; p.aux_group_stride = static_cast<long long>(p.M) * p.N;
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(bias->is_cuda() && bias->scalar_type() == at::kBFloat16 && bias->is_contiguous() && bias->numel() == static_cast<long long>(p.G) * p.N,
                "block_fp8_gemm: bias must be a contiguous bf16 [G, N]");
    p.bias = bias->data_ptr(); p.bias_group_stride = p.N;
  }
  std::vector<at::Tensor> out;
  if (glu) {
    for (int i = 0; i < 3; ++i) out.push_back(at::empty(shape(p.N / 2), bf));
    p.d = out[0].data_ptr(); p.d2 = out[1].data_ptr(); p.d3 = out[2].data_ptr();
    p.ldd = p.N / 2;
  } else if (glu_bwd) {
    out.push_back(at::empty(shape(2LL * p.N), bf));
    p.d = out[0].data_ptr(); p.d2 = static_cast<__nv_bfloat16*>(p.d) + p.N;
    p.ldd = 2LL * p.N;
  } else {
    out.push_back(at::empty(shape(p.N), bf));
    p.d = out[0].data_ptr();
    p.ldd = p.N;
  }
  p.d_group_stride = p.ldd * p.M;
  p.a = a.data_ptr(); p.sa = sa.data_ptr<float>(); p.b = b.data_ptr(); p.sb = sb.data_ptr<float>();
  p.epilogue = static_cast<int>(epilogue);
  p.act = static_cast<int>(act);
  p.max_ctas = static_cast<int>(max_ctas);
  p.row_counts = row_counts;
  p.b_group_map = b_group_map;
  const char* why = nullptr;
  cudaError_t e = tb::block_fp8_gemm_launch(p, cur_stream(), &why);
  TORCH_CHECK(e == cudaSuccess, "block_fp8_gemm: ", why ? why : cudaGetErrorString(e));
  return out;
}

std::vector<at::Tensor> block_fp8_gemm(const at::Tensor& a, const at::Tensor& sa, const at::Tensor& b, const at::Tensor& sb,
                                       const c10::optional<at::Tensor>& bias, const c10::optional<at::Tensor>& aux,
                                       const c10::optional<at::Tensor>& aux2, int64_t epilogue, int64_t act, int64_t max_ctas) {
  return block_fp8_gemm_impl(a, sa, b, sb, bias, aux, aux2, epilogue, act, max_ctas, nullptr);
}

// block_fp8_gemm with device row counts (int32 [G]): rows r >= row_counts[g] of every output are zero, and tiles that
// start at or past the count are skipped.
std::vector<at::Tensor> block_fp8_gemm_counts(const at::Tensor& a, const at::Tensor& sa, const at::Tensor& b, const at::Tensor& sb,
                                              const c10::optional<at::Tensor>& bias, const c10::optional<at::Tensor>& aux,
                                              const c10::optional<at::Tensor>& aux2, int64_t epilogue, int64_t act, int64_t max_ctas,
                                              const at::Tensor& row_counts) {
  TORCH_CHECK(row_counts.is_cuda() && row_counts.scalar_type() == at::kInt && row_counts.is_contiguous() &&
                  row_counts.numel() == a.size(0) && row_counts.device() == a.device(),
              "block_fp8_gemm: row_counts must be a contiguous int32 CUDA tensor [G] on a's device");
  return block_fp8_gemm_impl(a, sa, b, sb, bias, aux, aux2, epilogue, act, max_ctas, row_counts.data_ptr<int>());
}

// block_fp8_gemm, block-mapped over an expert-packed buffer: a e4m3 [R, K] (R % 128 == 0) + sa [1, K / 128, R], b the
// [E, N, K] expert operand; row tile m (128 rows) is multiplied by b[b_group_map[m]] (and that expert's sb and bias), and
// only its first row_counts[m] rows are live (both int32 [R / 128]).  Results and aux are [R, *]; rows past a tile's count
// are zero, tiles with no live rows are neither loaded nor stored.
std::vector<at::Tensor> block_fp8_gemm_packed(const at::Tensor& a, const at::Tensor& sa, const at::Tensor& b, const at::Tensor& sb,
                                              const c10::optional<at::Tensor>& bias, const c10::optional<at::Tensor>& aux,
                                              const c10::optional<at::Tensor>& aux2, int64_t epilogue, int64_t act, int64_t max_ctas,
                                              const at::Tensor& row_counts, const at::Tensor& b_group_map) {
  TORCH_CHECK(a.dim() == 2 && a.size(0) % 128 == 0, "block_fp8_gemm: a block-mapped a must be [R, K] with R % 128 == 0");
  for (const at::Tensor* t : {&row_counts, &b_group_map})
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kInt && t->is_contiguous() && t->numel() == a.size(0) / 128 &&
                    t->device() == a.device(),
                "block_fp8_gemm: row_counts and b_group_map must be contiguous int32 CUDA tensors [R / 128] on a's device");
  return block_fp8_gemm_impl(a, sa, b, sb, bias, aux, aux2, epilogue, act, max_ctas, row_counts.data_ptr<int>(),
                             b_group_map.data_ptr<int>());
}

// x [G, R, K] bf16 (K % 128 == 0), both orientations from one read (csrc/gemm_block_fp8.h) ->
// rowwise: [q [G, R, K], s [G, K / 128, Rp], qT [G, K, Rp], sT [G, Rp / 128, K]];  otherwise [qT, sT].  Rp = roundup(R, 128).
// live_rows (optional device int32 [1], G == 1, a multiple of 128): the 128-row tiles at or past it are neither read nor
// written.
std::vector<at::Tensor> block_fp8_quantize_act_dual_impl(const at::Tensor& x, bool rowwise, const int* live_rows) {
  TORCH_CHECK(x.is_cuda() && x.is_contiguous() && x.dim() == 3 && x.scalar_type() == at::kBFloat16 && x.size(2) % 128 == 0 &&
                  x.size(0) <= 65535,
              "block_fp8_quantize_act_dual: contiguous bf16 CUDA tensor [G, R, K] with K % 128 == 0 and G <= 65535 expected");
  const c10::cuda::CUDAGuard guard(x.device());
  const int G = static_cast<int>(x.size(0)), R = static_cast<int>(x.size(1)), K = static_cast<int>(x.size(2));
  const int Rp = (R + 127) / 128 * 128;
  const auto f8 = x.options().dtype(at::kFloat8_e4m3fn), f32 = x.options().dtype(at::kFloat);
  at::Tensor qT = at::empty({G, K, Rp}, f8);
  at::Tensor sT = at::empty({G, Rp / 128, K}, f32);
  at::Tensor q, s;
  if (rowwise) {
    q = at::empty({G, R, K}, f8);
    s = at::empty({G, K / 128, Rp}, f32);
  }
  TB_CHECK_CUDA(tb::block_fp8_quantize_act_dual(x.data_ptr(), rowwise ? q.data_ptr() : nullptr, rowwise ? s.data_ptr<float>() : nullptr,
                                                qT.data_ptr(), sT.data_ptr<float>(), G, R, K, cur_stream(), live_rows));
  if (rowwise) return {q, s, qT, sT};
  return {qT, sT};
}

std::vector<at::Tensor> block_fp8_quantize_act_dual(const at::Tensor& x, bool rowwise) {
  return block_fp8_quantize_act_dual_impl(x, rowwise, nullptr);
}

std::vector<at::Tensor> block_fp8_quantize_act_dual_bounded(const at::Tensor& x, bool rowwise, const at::Tensor& live_rows) {
  TORCH_CHECK(x.dim() == 3 && x.size(0) == 1, "block_fp8_quantize_act_dual: a bounded launch takes one group [1, R, K]");
  TORCH_CHECK(live_rows.is_cuda() && live_rows.scalar_type() == at::kInt && live_rows.numel() == 1 && live_rows.device() == x.device(),
              "block_fp8_quantize_act_dual: live_rows must be a one-element int32 tensor on x's device");
  return block_fp8_quantize_act_dual_impl(x, rowwise, live_rows.data_ptr<int>());
}

// Weight-gradient GEMM d[g] = a[g] * b[g]^T over the padded token dimension K: a e4m3 [G, M, K] + sa fp32 [G, K / 128, M],
// b e4m3 [G, N, K] + sb fp32 [G, K / 128, N] (one scale per row and K step) -> [d bf16 [G, M, N]]; split = H > 0
// (N == 2H) -> [d1 [G, M, H] (columns < H), d2 [G, M, H] (columns >= H)].
// Ragged K (k_offsets int32 [E + 1], multiples of 128): a [1, M, R] and b [1, N, R] are single operands with scales
// [1, R / 128, M] and [1, R / 128, N], and d[e] reduces over K in [k_offsets[e], k_offsets[e + 1]) -> d [E, M, N] (or split).
std::vector<at::Tensor> block_fp8_wgrad_gemm_impl(const at::Tensor& a, const at::Tensor& sa, const at::Tensor& b, const at::Tensor& sb,
                                                  int64_t split, int64_t max_ctas, const at::Tensor* k_offsets) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && sa.is_cuda() && sb.is_cuda() && a.dim() == 3 && b.dim() == 3 && sa.dim() == 3 &&
              sb.dim() == 3, "block_fp8_wgrad_gemm: 3-D CUDA tensors expected");
  TORCH_CHECK(b.device() == a.device() && sa.device() == a.device() && sb.device() == a.device(),
              "block_fp8_wgrad_gemm: operands on one device expected");
  TORCH_CHECK(a.is_contiguous() && b.is_contiguous() && sa.is_contiguous() && sb.is_contiguous(),
              "block_fp8_wgrad_gemm: contiguous operands expected");
  TORCH_CHECK(a.scalar_type() == at::kFloat8_e4m3fn && b.scalar_type() == at::kFloat8_e4m3fn &&
              sa.scalar_type() == at::kFloat && sb.scalar_type() == at::kFloat,
              "block_fp8_wgrad_gemm: e4m3 operands and fp32 scales expected");
  TORCH_CHECK(a.size(0) == b.size(0) && a.size(2) == b.size(2), "block_fp8_wgrad_gemm: a [G, M, K] and b [G, N, K] expected");
  if (k_offsets != nullptr)
    TORCH_CHECK(a.size(0) == 1 && k_offsets->is_cuda() && k_offsets->scalar_type() == at::kInt && k_offsets->is_contiguous() &&
                    k_offsets->numel() >= 2 && k_offsets->device() == a.device(),
                "block_fp8_wgrad_gemm: ragged K takes single operands [1, M, R], [1, N, R] and contiguous int32 CUDA k_offsets [E + 1]");
  const c10::cuda::CUDAGuard guard(a.device());
  tb::BlockFp8WgradProblem p;
  p.G = k_offsets != nullptr ? static_cast<int>(k_offsets->numel() - 1) : static_cast<int>(a.size(0));
  p.M = static_cast<int>(a.size(1)); p.K = static_cast<int>(a.size(2));
  p.N = static_cast<int>(b.size(1));
  TORCH_CHECK(p.M % 128 == 0 && p.N % 128 == 0 && p.K % 128 == 0, "block_fp8_wgrad_gemm: M, N and K must be multiples of 128");
  const int64_t kb = p.K / 128;
  TORCH_CHECK(sa.size(0) == a.size(0) && sa.size(1) == kb && sa.size(2) == p.M && sb.size(0) == a.size(0) && sb.size(1) == kb && sb.size(2) == p.N,
              "block_fp8_wgrad_gemm: scale arrays do not match the operand shapes (sa [G, K / 128, M], sb [G, K / 128, N] expected)");
  TORCH_CHECK(split == 0 || (split % 128 == 0 && 2 * split == p.N),
              "block_fp8_wgrad_gemm: split must be 0 or N / 2, a multiple of 128");
  const auto bf = a.options().dtype(at::kBFloat16);
  std::vector<at::Tensor> out;
  if (split == 0) {
    out.push_back(at::empty({p.G, p.M, p.N}, bf));
  } else {
    out.push_back(at::empty({p.G, p.M, split}, bf));
    out.push_back(at::empty({p.G, p.M, split}, bf));
    p.d2 = out[1].data_ptr();
  }
  p.d = out[0].data_ptr();
  p.split = static_cast<int>(split);
  p.a = a.data_ptr(); p.sa = sa.data_ptr<float>(); p.b = b.data_ptr(); p.sb = sb.data_ptr<float>();
  p.max_ctas = static_cast<int>(max_ctas);
  p.k_offsets = k_offsets != nullptr ? k_offsets->data_ptr<int>() : nullptr;
  const char* why = nullptr;
  cudaError_t e = tb::block_fp8_wgrad_gemm_launch(p, cur_stream(), &why);
  TORCH_CHECK(e == cudaSuccess, "block_fp8_wgrad_gemm: ", why ? why : cudaGetErrorString(e));
  return out;
}

std::vector<at::Tensor> block_fp8_wgrad_gemm(const at::Tensor& a, const at::Tensor& sa, const at::Tensor& b, const at::Tensor& sb,
                                             int64_t split, int64_t max_ctas) {
  return block_fp8_wgrad_gemm_impl(a, sa, b, sb, split, max_ctas, nullptr);
}

std::vector<at::Tensor> block_fp8_wgrad_gemm_ragged(const at::Tensor& a, const at::Tensor& sa, const at::Tensor& b,
                                                    const at::Tensor& sb, int64_t split, int64_t max_ctas,
                                                    const at::Tensor& k_offsets) {
  return block_fp8_wgrad_gemm_impl(a, sa, b, sb, split, max_ctas, &k_offsets);
}

// Gated-linear-unit GEMMs (SwiGLU / GeGLU / ReGLU experts; reference: tutel/experts/llama_ffn.py:38-41 runs three
// cuBLAS GEMMs plus separate activation and multiply kernels).
//   forward  (b2 given):  h = act(a*b) .* (a*b2)   [+ g = a*b -> d2, u = a*b2 -> d3 when given]   ONE launch
//   backward (aux given): acc = a*b (= dh);  d = dh .* u .* act'(g),  d2 = dh .* act(g)   with g = aux, u = aux2
void gemm_glu_packed(const at::Tensor& a, const at::Tensor& b, const c10::optional<at::Tensor>& b2, at::Tensor& d,
              const c10::optional<at::Tensor>& d2, const c10::optional<at::Tensor>& d3,
              const c10::optional<at::Tensor>& aux, const c10::optional<at::Tensor>& aux2, bool b_mn, int64_t act,
              const c10::optional<at::Tensor>& scale_a, const c10::optional<at::Tensor>& scale_b,
              const c10::optional<at::Tensor>& scale_b2, const c10::optional<at::Tensor>& row_counts,
              int64_t b_group_div, int64_t cta_group, int64_t wait_flags, int64_t wait_rows_per_flag,
              int64_t wait_flags_per_group, int64_t wait_target, int64_t group_rot, int64_t group_mod,
              const c10::optional<at::Tensor>& b_group_map) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && d.is_cuda() && a.dim() == 3 && b.dim() == 3 && d.dim() == 3);
  TORCH_CHECK(a.stride(2) == 1 && b.stride(2) == 1 && d.stride(2) == 1 && a.scalar_type() == b.scalar_type());
  const c10::cuda::CUDAGuard guard(a.device());
  const bool fwd = b2.has_value() && b2->defined();
  tb::GemmProblem p;
  p.G = static_cast<int>(a.size(0));
  p.M = static_cast<int>(a.size(1));
  p.K = static_cast<int>(a.size(2));
  p.N = static_cast<int>(b_mn ? b.size(2) : b.size(1));
  TORCH_CHECK((b_mn ? b.size(1) : b.size(2)) == p.K, "tutel_b200.gemm_glu: K mismatch");
  p.b_group_div = static_cast<int>(b_group_div > 0 ? b_group_div : 1);
  set_packed_modes(p, a, b, d, b_group_map, c10::nullopt);
  TORCH_CHECK((p.b_group_map != nullptr || b.size(0) * p.b_group_div >= p.G) && d.size(0) == p.G && d.size(1) == p.M &&
              d.size(2) == p.N && d.element_size() == 2);
  p.cta_group = static_cast<int>(cta_group);
  p.wait_flags = reinterpret_cast<const uint32_t*>(wait_flags);
  p.wait_rows_per_flag = static_cast<int>(wait_rows_per_flag);
  p.wait_flags_per_group = static_cast<int>(wait_flags_per_group);
  p.wait_target = static_cast<uint32_t>(wait_target);
  p.group_rot = static_cast<int>(group_rot);
  p.group_mod = static_cast<int>(group_mod != 0 ? group_mod : 1);
  p.a = a.data_ptr(); p.lda = a.stride(1); p.a_group_stride = a.stride(0);
  p.b = b.data_ptr(); p.ldb = b.stride(1); p.b_group_stride = b.stride(0); p.b_mn_major = b_mn;
  p.in_dtype = gemm_dtype_of(a);
  p.d = d.data_ptr(); p.ldd = d.stride(1); p.d_group_stride = d.stride(0);
  p.out_dtype = gemm_dtype_of(d);
  p.act = static_cast<int>(act);
  auto same_as_d = [&](const at::Tensor& t) {
    return t.is_cuda() && t.scalar_type() == d.scalar_type() && t.sizes() == d.sizes() && t.strides() == d.strides();
  };
  if (fwd) {
    TORCH_CHECK(b2->scalar_type() == b.scalar_type() && b2->sizes() == b.sizes() && b2->strides() == b.strides(),
                "tutel_b200.gemm_glu: b2 must have the layout of b");
    p.epilogue = tb::EPI_GLU;
    p.b2 = b2->data_ptr();
    if (d2.has_value() && d2->defined()) {
      TORCH_CHECK(d3.has_value() && d3->defined() && same_as_d(*d2) && same_as_d(*d3), "tutel_b200.gemm_glu: d2/d3 must look like d");
      p.d2 = d2->data_ptr();
      p.d3 = d3->data_ptr();
    }
  } else {
    TORCH_CHECK(aux.has_value() && aux2.has_value() && d2.has_value() && same_as_d(*d2) && same_as_d(*aux) &&
                    aux2->scalar_type() == d.scalar_type() && aux2->sizes() == aux->sizes() && aux2->strides() == aux->strides(),
                "tutel_b200.gemm_glu: backward needs aux, aux2 and d2 shaped like d");
    p.epilogue = tb::EPI_GLU_BWD;
    p.aux = aux->data_ptr(); p.ld_aux = aux->stride(1); p.aux_group_stride = aux->stride(0);
    p.aux2 = aux2->data_ptr();
    p.d2 = d2->data_ptr();
  }
  auto scale = [&](const c10::optional<at::Tensor>& t, int64_t cols, const float** ptr, long long* stride) {
    if (!t.has_value() || !t->defined()) return;
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kFloat && t->dim() == 2 && t->stride(1) == 1 && t->size(1) == cols);
    *ptr = t->data_ptr<float>();
    if (stride) *stride = t->stride(0);
  };
  scale(scale_a, p.M, &p.scale_a, &p.scale_a_group_stride);
  scale(scale_b, p.N, &p.scale_b, &p.scale_b_group_stride);
  long long s2 = p.scale_b_group_stride;
  scale(scale_b2, p.N, &p.scale_b2, &s2);
  TORCH_CHECK(s2 == p.scale_b_group_stride, "tutel_b200.gemm_glu: scale_b / scale_b2 stride mismatch");
  if (row_counts.has_value() && row_counts->defined()) {
    TORCH_CHECK(row_counts->is_cuda() && row_counts->scalar_type() == at::kInt && row_counts->numel() >= p.G);
    p.row_counts = row_counts->data_ptr<int>();
  }
  const char* why = nullptr;
  cudaError_t e = tb::gemm_sm90_launch(p, cur_stream(), &why);
  TORCH_CHECK(e == cudaSuccess, "tutel_b200.gemm_glu launch failed: ", why ? why : cudaGetErrorString(e));
}

void gemm_glu(const at::Tensor& a, const at::Tensor& b, const c10::optional<at::Tensor>& b2, at::Tensor& d,
              const c10::optional<at::Tensor>& d2, const c10::optional<at::Tensor>& d3,
              const c10::optional<at::Tensor>& aux, const c10::optional<at::Tensor>& aux2, bool b_mn, int64_t act,
              const c10::optional<at::Tensor>& scale_a, const c10::optional<at::Tensor>& scale_b,
              const c10::optional<at::Tensor>& scale_b2, const c10::optional<at::Tensor>& row_counts,
              int64_t b_group_div, int64_t cta_group, int64_t wait_flags, int64_t wait_rows_per_flag,
              int64_t wait_flags_per_group, int64_t wait_target, int64_t group_rot, int64_t group_mod) {
  gemm_glu_packed(a, b, b2, d, d2, d3, aux, aux2, b_mn, act, scale_a, scale_b, scale_b2, row_counts, b_group_div, cta_group,
                  wait_flags, wait_rows_per_flag, wait_flags_per_group, wait_target, group_rot, group_mod, c10::nullopt);
}

at::Tensor skinny_gemm(const at::Tensor& x, const at::Tensor& w, const c10::optional<at::Tensor>& bias,
                       const c10::optional<at::Tensor>& counts, bool w_is_kn, bool relu) {
  TORCH_CHECK(x.is_cuda() && w.is_cuda() && x.dim() == 3 && w.dim() == 3 && x.is_contiguous() && w.is_contiguous());
  TORCH_CHECK(x.scalar_type() == w.scalar_type() && x.size(0) == w.size(0));
  const c10::cuda::CUDAGuard guard(x.device());
  const int G = static_cast<int>(x.size(0)), R = static_cast<int>(x.size(1)), K = static_cast<int>(x.size(2));
  const int N = static_cast<int>(w_is_kn ? w.size(2) : w.size(1));
  TORCH_CHECK((w_is_kn ? w.size(1) : w.size(2)) == K, "skinny_gemm: K mismatch");
  at::Tensor y = at::zeros({G, R, N}, x.options());
  const void* b = nullptr;
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(bias->is_cuda() && bias->is_contiguous() && bias->scalar_type() == x.scalar_type() && bias->numel() == static_cast<int64_t>(G) * N);
    b = bias->data_ptr();
  }
  const int* c = nullptr;
  if (counts.has_value() && counts->defined()) {
    TORCH_CHECK(counts->is_cuda() && counts->scalar_type() == at::kInt && counts->numel() >= G);
    c = counts->data_ptr<int>();
  }
  TB_CHECK_CUDA(tb::skinny_grouped_gemm(x.data_ptr(), w.data_ptr(), b, y.data_ptr(), c, G, R, N, K, w_is_kn, relu,
                                        elem_type_of(x), cur_stream()));
  return y;
}

// x [G, R, K], w1 [G, H, K], w2 [G, H, N], biases [G, H] / [G, N] or None, counts int [G] or None -> fp32 [G, R, N]
at::Tensor skinny_ffn(const at::Tensor& x, const at::Tensor& w1, const c10::optional<at::Tensor>& b1, const at::Tensor& w2,
                      const c10::optional<at::Tensor>& b2, const c10::optional<at::Tensor>& counts, int64_t act) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 3 && w1.dim() == 3 && w2.dim() == 3 && x.is_contiguous() && w1.is_contiguous() && w2.is_contiguous());
  TORCH_CHECK(x.scalar_type() == w1.scalar_type() && x.scalar_type() == w2.scalar_type() && x.size(0) == w1.size(0) && x.size(0) == w2.size(0));
  const c10::cuda::CUDAGuard guard(x.device());
  const int G = static_cast<int>(x.size(0)), R = static_cast<int>(x.size(1)), K = static_cast<int>(x.size(2));
  const int H = static_cast<int>(w1.size(1)), N = static_cast<int>(w2.size(2));
  TORCH_CHECK(w1.size(2) == K && w2.size(1) == H, "skinny_ffn: weight shapes do not match");
  at::Tensor y = at::zeros({G, R, N}, x.options().dtype(at::kFloat));
  auto opt_ptr = [&](const c10::optional<at::Tensor>& t, int64_t n) -> const void* {
    if (!t.has_value() || !t->defined()) return nullptr;
    TORCH_CHECK(t->is_cuda() && t->is_contiguous() && t->scalar_type() == x.scalar_type() && t->numel() == n);
    return t->data_ptr();
  };
  const int* c = nullptr;
  if (counts.has_value() && counts->defined()) {
    TORCH_CHECK(counts->is_cuda() && counts->scalar_type() == at::kInt && counts->numel() >= G);
    c = counts->data_ptr<int>();
  }
  TB_CHECK_CUDA(tb::skinny_grouped_ffn(x.data_ptr(), w1.data_ptr(), opt_ptr(b1, static_cast<int64_t>(G) * H), w2.data_ptr(),
                                       opt_ptr(b2, static_cast<int64_t>(G) * N), y.data_ptr<float>(), c, G, R, K, H, N,
                                       static_cast<int>(act), elem_type_of(x), cur_stream()));
  return y;
}

// x [G, R, M], w1 / w2 [G, M, H], w3 [G, H, N], counts int [G] or None -> fp32 [G, R, N]
at::Tensor skinny_glu_ffn(const at::Tensor& x, const at::Tensor& w1, const at::Tensor& w2, const at::Tensor& w3,
                          const c10::optional<at::Tensor>& counts, int64_t act) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 3 && w1.dim() == 3 && w2.dim() == 3 && w3.dim() == 3 && x.is_contiguous() &&
              w1.is_contiguous() && w2.is_contiguous() && w3.is_contiguous(), "skinny_glu_ffn: needs contiguous 3-d CUDA tensors");
  TORCH_CHECK(x.scalar_type() == w1.scalar_type() && x.scalar_type() == w2.scalar_type() && x.scalar_type() == w3.scalar_type(),
              "skinny_glu_ffn: x and the weights must have one dtype");
  TORCH_CHECK(x.size(0) == w1.size(0) && x.size(0) == w2.size(0) && x.size(0) == w3.size(0), "skinny_glu_ffn: group count mismatch");
  const c10::cuda::CUDAGuard guard(x.device());
  const int G = static_cast<int>(x.size(0)), R = static_cast<int>(x.size(1)), M = static_cast<int>(x.size(2));
  const int H = static_cast<int>(w1.size(2)), N = static_cast<int>(w3.size(2));
  TORCH_CHECK(w1.size(1) == M && w2.sizes() == w1.sizes() && w3.size(1) == H, "skinny_glu_ffn: weight shapes do not match");
  TORCH_CHECK(act >= 1 && act <= 3, "skinny_glu_ffn: act must be 1 (relu), 2 (gelu) or 3 (silu)");
  at::Tensor y = at::zeros({G, R, N}, x.options().dtype(at::kFloat));
  const int* c = nullptr;
  if (counts.has_value() && counts->defined()) {
    TORCH_CHECK(counts->is_cuda() && counts->scalar_type() == at::kInt && counts->numel() >= G);
    c = counts->data_ptr<int>();
  }
  TB_CHECK_CUDA(tb::skinny_grouped_glu_ffn(x.data_ptr(), w1.data_ptr(), w2.data_ptr(), w3.data_ptr(), y.data_ptr<float>(), c, G,
                                           R, M, H, N, static_cast<int>(act), elem_type_of(x), cur_stream()));
  return y;
}

// Checks shared by the weight-only fp8 skinny kernels.
void check_fp8_x(const at::Tensor& x, const char* fn) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 3 && x.is_contiguous(), fn, ": x must be a contiguous 3-d CUDA tensor");
  TORCH_CHECK(x.scalar_type() == at::kHalf || x.scalar_type() == at::kBFloat16, fn, ": x must be float16 or bfloat16");
}

void check_fp8_weight(const at::Tensor& q, const at::Tensor& s, int64_t G, int64_t rows, int64_t cols, const char* fn,
                      const char* name) {
  TORCH_CHECK(q.is_cuda() && q.scalar_type() == at::kFloat8_e4m3fn && q.is_contiguous(), fn, ": ", name,
              " must be a contiguous float8_e4m3fn CUDA tensor");
  TORCH_CHECK(q.dim() == 3 && q.size(0) == G && q.size(1) == rows && q.size(2) == cols, fn, ": ", name, " must be [", G, ", ",
              rows, ", ", cols, "], got ", q.sizes());
  TORCH_CHECK(s.is_cuda() && s.scalar_type() == at::kFloat && s.is_contiguous() && s.numel() == G * rows, fn, ": the scales of ",
              name, " must be contiguous float32 with ", G * rows, " elements");
}

const int* opt_counts(const c10::optional<at::Tensor>& counts, int64_t G) {
  if (!counts.has_value() || !counts->defined()) return nullptr;
  TORCH_CHECK(counts->is_cuda() && counts->scalar_type() == at::kInt && counts->numel() >= G);
  return counts->data_ptr<int>();
}

// x [G, R, K] (fp16 / bf16), q1 [G, H, K] + s1 [G, H], q2t [G, N, H] + s2 [G, N] (e4m3 + fp32), biases [G, H] / [G, N] in
// x's dtype or None, counts int [G] or None -> fp32 [G, R, N]
at::Tensor skinny_ffn_fp8(const at::Tensor& x, const at::Tensor& q1, const at::Tensor& s1, const c10::optional<at::Tensor>& b1,
                          const at::Tensor& q2t, const at::Tensor& s2, const c10::optional<at::Tensor>& b2,
                          const c10::optional<at::Tensor>& counts, int64_t act) {
  check_fp8_x(x, "skinny_ffn_fp8");
  const int64_t G = x.size(0), R = x.size(1), K = x.size(2), H = q1.dim() == 3 ? q1.size(1) : -1;
  const int64_t N = q2t.dim() == 3 ? q2t.size(1) : -1;
  check_fp8_weight(q1, s1, G, H, K, "skinny_ffn_fp8", "q1");
  check_fp8_weight(q2t, s2, G, N, H, "skinny_ffn_fp8", "q2t");
  TORCH_CHECK(act >= 1 && act <= 3, "skinny_ffn_fp8: act must be 1 (relu), 2 (gelu) or 3 (silu)");
  const c10::cuda::CUDAGuard guard(x.device());
  auto opt_ptr = [&](const c10::optional<at::Tensor>& t, int64_t n) -> const void* {
    if (!t.has_value() || !t->defined()) return nullptr;
    TORCH_CHECK(t->is_cuda() && t->is_contiguous() && t->scalar_type() == x.scalar_type() && t->numel() == n,
                "skinny_ffn_fp8: biases must be contiguous, in x's dtype, with G * H / G * N elements");
    return t->data_ptr();
  };
  const void* pb1 = opt_ptr(b1, G * H);
  const void* pb2 = opt_ptr(b2, G * N);
  at::Tensor y = at::zeros({G, R, N}, x.options().dtype(at::kFloat));
  TB_CHECK_CUDA(tb::skinny_grouped_ffn_fp8(x.data_ptr(), q1.data_ptr(), s1.data_ptr<float>(), pb1, q2t.data_ptr(),
                                           s2.data_ptr<float>(), pb2, y.data_ptr<float>(), opt_counts(counts, G),
                                           static_cast<int>(G), static_cast<int>(R), static_cast<int>(K), static_cast<int>(H),
                                           static_cast<int>(N), static_cast<int>(act), elem_type_of(x), cur_stream()));
  return y;
}

// x [G, R, M] (fp16 / bf16), q1t / q2t [G, H, M] + s1 / s2 [G, H], q3t [G, N, H] + s3 [G, N], counts int [G] or None
// -> fp32 [G, R, N]
at::Tensor skinny_glu_ffn_fp8(const at::Tensor& x, const at::Tensor& q1t, const at::Tensor& s1, const at::Tensor& q2t,
                              const at::Tensor& s2, const at::Tensor& q3t, const at::Tensor& s3,
                              const c10::optional<at::Tensor>& counts, int64_t act) {
  check_fp8_x(x, "skinny_glu_ffn_fp8");
  const int64_t G = x.size(0), R = x.size(1), M = x.size(2), H = q1t.dim() == 3 ? q1t.size(1) : -1;
  const int64_t N = q3t.dim() == 3 ? q3t.size(1) : -1;
  check_fp8_weight(q1t, s1, G, H, M, "skinny_glu_ffn_fp8", "q1t");
  check_fp8_weight(q2t, s2, G, H, M, "skinny_glu_ffn_fp8", "q2t");
  check_fp8_weight(q3t, s3, G, N, H, "skinny_glu_ffn_fp8", "q3t");
  TORCH_CHECK(act >= 1 && act <= 3, "skinny_glu_ffn_fp8: act must be 1 (relu), 2 (gelu) or 3 (silu)");
  const c10::cuda::CUDAGuard guard(x.device());
  at::Tensor y = at::zeros({G, R, N}, x.options().dtype(at::kFloat));
  TB_CHECK_CUDA(tb::skinny_grouped_glu_ffn_fp8(x.data_ptr(), q1t.data_ptr(), s1.data_ptr<float>(), q2t.data_ptr(),
                                               s2.data_ptr<float>(), q3t.data_ptr(), s3.data_ptr<float>(), y.data_ptr<float>(),
                                               opt_counts(counts, G), static_cast<int>(G), static_cast<int>(R),
                                               static_cast<int>(M), static_cast<int>(H), static_cast<int>(N),
                                               static_cast<int>(act), elem_type_of(x), cur_stream()));
  return y;
}

// x [G, R, M] bf16, qglu [G, 2H, M] e4m3 (gate / up interleaved every 64 rows) + sglu [G, 2H / 64, M / 128],
// q3t [G, N, H] e4m3 + s3t [G, N / 128, H / 128], counts int [G] or None -> fp32 [G, R, N], rows past the counts zero
at::Tensor skinny_glu_ffn_block_fp8(const at::Tensor& x, const at::Tensor& qglu, const at::Tensor& sglu, const at::Tensor& q3t,
                                    const at::Tensor& s3t, const c10::optional<at::Tensor>& counts, int64_t act) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 3 && x.is_contiguous() && x.scalar_type() == at::kBFloat16,
              "skinny_glu_ffn_block_fp8: x must be a contiguous bf16 CUDA tensor [G, R, M]");
  const int64_t G = x.size(0), R = x.size(1), M = x.size(2);
  TORCH_CHECK(qglu.dim() == 3 && q3t.dim() == 3, "skinny_glu_ffn_block_fp8: 3-D weights expected");
  const int64_t H = qglu.size(1) / 2, N = q3t.size(1);
  TORCH_CHECK(M % 128 == 0 && H % 128 == 0 && N % 128 == 0, "skinny_glu_ffn_block_fp8: M, H and N must be multiples of 128");
  auto ok = [&](const at::Tensor& t, at::ScalarType dt, int64_t d0, int64_t d1, int64_t d2) {
    return t.is_cuda() && t.device() == x.device() && t.is_contiguous() && t.scalar_type() == dt && t.dim() == 3 &&
           t.size(0) == d0 && t.size(1) == d1 && t.size(2) == d2;
  };
  TORCH_CHECK(ok(qglu, at::kFloat8_e4m3fn, G, 2 * H, M), "skinny_glu_ffn_block_fp8: qglu must be a contiguous e4m3 CUDA tensor [G, 2H, M]");
  TORCH_CHECK(ok(sglu, at::kFloat, G, 2 * H / 64, M / 128),
              "skinny_glu_ffn_block_fp8: sglu must be a contiguous fp32 CUDA tensor [G, 2H / 64, M / 128]");
  TORCH_CHECK(ok(q3t, at::kFloat8_e4m3fn, G, N, H), "skinny_glu_ffn_block_fp8: q3t must be a contiguous e4m3 CUDA tensor [G, N, H]");
  TORCH_CHECK(ok(s3t, at::kFloat, G, N / 128, H / 128),
              "skinny_glu_ffn_block_fp8: s3t must be a contiguous fp32 CUDA tensor [G, N / 128, H / 128]");
  TORCH_CHECK(act >= 1 && act <= 3, "skinny_glu_ffn_block_fp8: act must be 1 (relu), 2 (gelu) or 3 (silu)");
  const c10::cuda::CUDAGuard guard(x.device());
  at::Tensor y = at::zeros({G, R, N}, x.options().dtype(at::kFloat));
  TB_CHECK_CUDA(tb::skinny_grouped_glu_ffn_block_fp8(x.data_ptr(), qglu.data_ptr(), sglu.data_ptr<float>(), q3t.data_ptr(),
                                                     s3t.data_ptr<float>(), y.data_ptr<float>(), opt_counts(counts, G),
                                                     static_cast<int>(G), static_cast<int>(R), static_cast<int>(M),
                                                     static_cast<int>(H), static_cast<int>(N), static_cast<int>(act), cur_stream()));
  return y;
}

bool int4_operand_ok(const at::Tensor& t, const at::Tensor& like, at::ScalarType dt, int64_t d0, int64_t d1, int64_t d2) {
  return t.is_cuda() && t.device() == like.device() && t.is_contiguous() && t.scalar_type() == dt && t.dim() == 3 &&
         t.size(0) == d0 && t.size(1) == d1 && t.size(2) == d2;
}

// x [G, R, M] bf16, qglu [G, 2H, M / 2] uint8 (packed int4, gate / up rows interleaved every 64) + sglu bf16 [G, 2H, M / 32],
// q3t [G, N, H / 2] uint8 + s3t bf16 [G, N, H / 32], counts int [G] or None -> fp32 [G, R, N], rows past the counts zero
at::Tensor skinny_glu_ffn_int4(const at::Tensor& x, const at::Tensor& qglu, const at::Tensor& sglu, const at::Tensor& q3t,
                               const at::Tensor& s3t, const c10::optional<at::Tensor>& counts, int64_t act) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 3 && x.is_contiguous() && x.scalar_type() == at::kBFloat16,
              "skinny_glu_ffn_int4: x must be a contiguous bf16 CUDA tensor [G, R, M]");
  const int64_t G = x.size(0), R = x.size(1), M = x.size(2);
  TORCH_CHECK(qglu.dim() == 3 && q3t.dim() == 3, "skinny_glu_ffn_int4: 3-D weights expected");
  const int64_t H = qglu.size(1) / 2, N = q3t.size(1);
  TORCH_CHECK(M % 128 == 0 && H % 128 == 0 && N % 128 == 0, "skinny_glu_ffn_int4: M, H and N must be multiples of 128");
  TORCH_CHECK(int4_operand_ok(qglu, x, at::kByte, G, 2 * H, M / 2),
              "skinny_glu_ffn_int4: qglu must be a contiguous uint8 CUDA tensor [G, 2H, M / 2]");
  TORCH_CHECK(int4_operand_ok(sglu, x, at::kBFloat16, G, 2 * H, M / 32),
              "skinny_glu_ffn_int4: sglu must be a contiguous bf16 CUDA tensor [G, 2H, M / 32]");
  TORCH_CHECK(int4_operand_ok(q3t, x, at::kByte, G, N, H / 2),
              "skinny_glu_ffn_int4: q3t must be a contiguous uint8 CUDA tensor [G, N, H / 2]");
  TORCH_CHECK(int4_operand_ok(s3t, x, at::kBFloat16, G, N, H / 32),
              "skinny_glu_ffn_int4: s3t must be a contiguous bf16 CUDA tensor [G, N, H / 32]");
  TORCH_CHECK(act >= 1 && act <= 3, "skinny_glu_ffn_int4: act must be 1 (relu), 2 (gelu) or 3 (silu)");
  const c10::cuda::CUDAGuard guard(x.device());
  at::Tensor y = at::zeros({G, R, N}, x.options().dtype(at::kFloat));
  TB_CHECK_CUDA(tb::skinny_grouped_glu_ffn_int4(x.data_ptr(), qglu.data_ptr(), sglu.data_ptr(), q3t.data_ptr(), s3t.data_ptr(),
                                                y.data_ptr<float>(), opt_counts(counts, G), static_cast<int>(G),
                                                static_cast<int>(R), static_cast<int>(M), static_cast<int>(H),
                                                static_cast<int>(N), static_cast<int>(act), cur_stream()));
  return y;
}

// a bf16 [G, M, K], b uint8 [G, N, K / 2] packed int4 + sb bf16 [G, N, K / 32], row_counts int32 [G] or None ->
// epilogue 0 (none): bf16 [G, M, N];  1 (GLU, b's rows interleaved every 64 gate / up): h = act(gate) * up, bf16 [G, M, N / 2].
// Rows at or past a group's count are zero.
at::Tensor w4a16_gemm(const at::Tensor& a, const at::Tensor& b, const at::Tensor& sb, const c10::optional<at::Tensor>& row_counts,
                      int64_t epilogue, int64_t act) {
  TORCH_CHECK(a.is_cuda() && a.dim() == 3 && a.is_contiguous() && a.scalar_type() == at::kBFloat16,
              "w4a16_gemm: a must be a contiguous bf16 CUDA tensor [G, M, K]");
  const int64_t G = a.size(0), M = a.size(1), K = a.size(2);
  TORCH_CHECK(b.dim() == 3 && b.size(0) == G && b.size(2) * 2 == K, "w4a16_gemm: b must be uint8 [G, N, K / 2]");
  const int64_t N = b.size(1);
  TORCH_CHECK(K % 64 == 0 && N % 128 == 0, "w4a16_gemm: K must be a multiple of 64 and N of 128");
  TORCH_CHECK(int4_operand_ok(b, a, at::kByte, G, N, K / 2), "w4a16_gemm: b must be a contiguous uint8 CUDA tensor [G, N, K / 2]");
  TORCH_CHECK(int4_operand_ok(sb, a, at::kBFloat16, G, N, K / 32),
              "w4a16_gemm: sb must be a contiguous bf16 CUDA tensor [G, N, K / 32]");
  TORCH_CHECK(epilogue == tb::W4A16_EPI_NONE || epilogue == tb::W4A16_EPI_GLU, "w4a16_gemm: epilogue must be 0 (none) or 1 (glu)");
  TORCH_CHECK(epilogue != tb::W4A16_EPI_GLU || (act >= 1 && act <= 3), "w4a16_gemm: act must be 1 (relu), 2 (gelu) or 3 (silu)");
  if (row_counts.has_value() && row_counts->defined())
    TORCH_CHECK(row_counts->is_cuda() && row_counts->scalar_type() == at::kInt && row_counts->is_contiguous() &&
                    row_counts->numel() == G && row_counts->device() == a.device(),
                "w4a16_gemm: row_counts must be a contiguous int32 CUDA tensor [G] on a's device");
  const c10::cuda::CUDAGuard guard(a.device());
  const bool glu = epilogue == tb::W4A16_EPI_GLU;
  at::Tensor d = at::empty({G, M, glu ? N / 2 : N}, a.options());
  if (G == 0 || M == 0) return d;
  tb::W4A16GemmProblem p;
  p.a = a.data_ptr();
  p.b = b.data_ptr();
  p.sb = sb.data_ptr();
  p.d = d.data_ptr();
  p.G = static_cast<int>(G); p.M = static_cast<int>(M); p.N = static_cast<int>(N); p.K = static_cast<int>(K);
  p.epilogue = static_cast<int>(epilogue);
  p.act = static_cast<int>(act);
  p.row_counts = opt_counts(row_counts, G);
  const char* why = nullptr;
  const cudaError_t e = tb::w4a16_gemm_launch(p, cur_stream(), &why);
  TORCH_CHECK(e == cudaSuccess, "w4a16_gemm: ", why != nullptr ? why : cudaGetErrorString(e));
  return d;
}

}  // namespace

void register_symm_bindings(pybind11::module& m);  // symm_heap.cpp / p2p bindings
void register_cpu_bindings(pybind11::module& m);   // cpu_kernels.cpp
void register_jit_bindings(pybind11::module& m);   // jit_nvrtc.cpp

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "tutel_b200 native runtime: sm_90a wgmma grouped GEMM, routing/dispatch kernels, symmetric heap, "
            "P2P collectives, NVRTC JIT";
  m.def("gemm", &gemm);
  m.def("gemm_ex", &gemm_ex);
  m.def("gemm_ex", &gemm_ex_packed);   // + b_group_map, k_offsets
  m.def("gemm_glu", &gemm_glu);
  m.def("gemm_glu", &gemm_glu_packed); // + b_group_map
  m.def("route_locations", &route_locations);
  m.def("build_slot_map", &build_slot_map);
  m.def("encode_rows", &encode_rows);
  m.def("encode_rows_fp8", &encode_rows_fp8);
  m.def("decode_rows", &decode_rows);
  m.def("decode_rows", &decode_rows_packed);
  m.def("decode_rows", &decode_rows_shared);
  m.def("gate_grad", &gate_grad);
  m.def("gate_grad", &gate_grad_packed);
  m.def("gate_grad", &gate_grad_shared);
  m.def("packed_layout", &packed_layout);
  m.def("gate_route_forward", &gate_route_forward);
  m.def("gate_route_backward", &gate_route_backward);
  m.def("sigmoid_gate_route_forward", &sigmoid_gate_route_forward);
  m.def("sigmoid_gate_route_backward", &sigmoid_gate_route_backward);
  m.def("expert_bias_update", &expert_bias_update);
  m.def("grouped_colsum", &grouped_colsum);
  m.def("grouped_colsum", &grouped_colsum_offsets);
  m.def("cumsum_sub_one", &cumsum_sub_one);
  m.def("skinny_gemm", &skinny_gemm);
  m.def("skinny_ffn", &skinny_ffn);
  m.def("skinny_glu_ffn", &skinny_glu_ffn);
  m.def("skinny_ffn_fp8", &skinny_ffn_fp8);
  m.def("skinny_glu_ffn_fp8", &skinny_glu_ffn_fp8);
  m.def("quantize_rows", &quantize_rows);
  m.def("dequant_rows", &dequant_rows);
  m.def("quantize_transpose", &quantize_transpose);
  m.def("mx_quantize", &mx_quantize);
  m.def("mx_quantize_transpose", &mx_quantize_transpose);
  m.def("mx_gemm", &mx_gemm);
  m.def("block_fp8_quantize_act", &block_fp8_quantize_act);
  m.def("block_fp8_quantize_act", &block_fp8_quantize_act_bounded);   // + live_rows
  m.def("block_fp8_quantize_weight", &block_fp8_quantize_weight);
  m.def("block_fp8_quantize_glu_weight", &block_fp8_quantize_glu_weight);
  m.def("block_fp8_gemm", &block_fp8_gemm);
  m.def("block_fp8_gemm", &block_fp8_gemm_counts);   // + row_counts
  m.def("block_fp8_gemm", &block_fp8_gemm_packed);   // + row_counts, b_group_map
  m.def("block_fp8_quantize_act_dual", &block_fp8_quantize_act_dual);
  m.def("block_fp8_quantize_act_dual", &block_fp8_quantize_act_dual_bounded);   // + live_rows
  m.def("block_fp8_wgrad_gemm", &block_fp8_wgrad_gemm);
  m.def("block_fp8_wgrad_gemm", &block_fp8_wgrad_gemm_ragged);   // + k_offsets
  m.def("skinny_glu_ffn_block_fp8", &skinny_glu_ffn_block_fp8);
  m.def("skinny_glu_ffn_int4", &skinny_glu_ffn_int4);
  m.def("w4a16_gemm", &w4a16_gemm);
  register_symm_bindings(m);
  register_cpu_bindings(m);
  register_jit_bindings(m);
}
