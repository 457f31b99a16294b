#include "symm_heap.h"

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda_runtime.h>
#include <torch/extension.h>

#include <cstring>
#include <memory>
#include <stdexcept>

#include "moe_kernels.h"
#include "p2p_kernels.h"

namespace tb {

#define TB_CUDA_OK(expr)                                                                              \
  do {                                                                                                \
    cudaError_t _e = (expr);                                                                          \
    if (_e != cudaSuccess)                                                                            \
      throw std::runtime_error(std::string("tutel_b200 symm_heap: ") + cudaGetErrorString(_e) + " at " #expr); \
  } while (0)

SymmHeap::SymmHeap(size_t bytes, int device) : bytes_(bytes), device_(device) {
  c10::cuda::CUDAGuard guard(device);
  TB_CUDA_OK(cudaMalloc(&local_, bytes));
  TB_CUDA_OK(cudaMemset(local_, 0, bytes));
  TB_CUDA_OK(cudaMalloc(reinterpret_cast<void**>(&d_peer_table_), sizeof(unsigned long long) * kMaxPeers));
  peer_base_.assign(1, local_);
  unsigned long long self = reinterpret_cast<unsigned long long>(local_);
  TB_CUDA_OK(cudaMemcpy(d_peer_table_, &self, sizeof(self), cudaMemcpyHostToDevice));
  TB_CUDA_OK(cudaDeviceSynchronize());
}

SymmHeap::~SymmHeap() {
  try { close(); } catch (...) {}
}

std::string SymmHeap::ipc_handle() const {
  cudaIpcMemHandle_t h;
  TB_CUDA_OK(cudaIpcGetMemHandle(&h, local_));
  return std::string(reinterpret_cast<const char*>(&h), sizeof(h));
}

void SymmHeap::open_peers(int rank, const std::vector<std::string>& handles) {
  c10::cuda::CUDAGuard guard(device_);
  const int world = static_cast<int>(handles.size());
  if (world > kMaxPeers) throw std::runtime_error("tutel_b200 symm_heap: more peers than kMaxPeers");
  rank_ = rank;
  peer_base_.assign(world, nullptr);
  std::vector<unsigned long long> table(world, 0);
  for (int r = 0; r < world; ++r) {
    if (r == rank) {
      peer_base_[r] = local_;
    } else {
      if (handles[r].size() != sizeof(cudaIpcMemHandle_t)) throw std::runtime_error("bad IPC handle size");
      cudaIpcMemHandle_t h;
      std::memcpy(&h, handles[r].data(), sizeof(h));
      void* p = nullptr;
      TB_CUDA_OK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
      peer_base_[r] = p;
    }
    table[r] = reinterpret_cast<unsigned long long>(peer_base_[r]);
  }
  TB_CUDA_OK(cudaMemcpy(d_peer_table_, table.data(), sizeof(unsigned long long) * world, cudaMemcpyHostToDevice));
  TB_CUDA_OK(cudaDeviceSynchronize());
}

void BlockPool::reset(long long off, long long bytes) {
  std::lock_guard<std::mutex> g(mu_);
  free_.clear();
  used_.clear();
  if (bytes > 0) free_[off] = bytes;
}

long long BlockPool::alloc(long long bytes) {
  bytes = (bytes + 255) / 256 * 256;
  if (bytes <= 0) bytes = 256;
  std::lock_guard<std::mutex> g(mu_);
  for (auto it = free_.begin(); it != free_.end(); ++it) {
    if (it->second >= bytes) {
      const long long off = it->first, len = it->second;
      free_.erase(it);
      if (len > bytes) free_[off + bytes] = len - bytes;
      used_[off] = bytes;
      return off;
    }
  }
  return -1;
}

void BlockPool::free(long long off) {
  std::lock_guard<std::mutex> g(mu_);
  auto u = used_.find(off);
  if (u == used_.end()) return;
  long long len = u->second;
  used_.erase(u);
  auto next = free_.lower_bound(off);
  if (next != free_.end() && off + len == next->first) {   // merge with the following free block
    len += next->second;
    next = free_.erase(next);
  }
  if (next != free_.begin()) {                              // merge with the preceding free block
    auto prev = std::prev(next);
    if (prev->first + prev->second == off) {
      prev->second += len;
      return;
    }
  }
  free_[off] = len;
}

long long BlockPool::free_bytes() {
  std::lock_guard<std::mutex> g(mu_);
  long long n = 0;
  for (auto& kv : free_) n += kv.second;
  return n;
}

long long BlockPool::largest_free_block() {
  std::lock_guard<std::mutex> g(mu_);
  long long n = 0;
  for (auto& kv : free_) n = kv.second > n ? kv.second : n;
  return n;
}

size_t BlockPool::live_blocks() {
  std::lock_guard<std::mutex> g(mu_);
  return used_.size();
}

void SymmHeap::close() {
  if (closed_) return;
  closed_ = true;
  for (size_t r = 0; r < peer_base_.size(); ++r)
    if (static_cast<int>(r) != rank_ && peer_base_[r] != nullptr) cudaIpcCloseMemHandle(peer_base_[r]);
  if (d_peer_table_) cudaFree(d_peer_table_);
  if (local_) cudaFree(local_);
  d_peer_table_ = nullptr;
  local_ = nullptr;
}

}  // namespace tb

namespace {

cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

#define TB_CHECK_CUDA(expr)                                                                          \
  do {                                                                                               \
    cudaError_t _e = (expr);                                                                         \
    TORCH_CHECK(_e == cudaSuccess, "tutel_b200 CUDA error: ", cudaGetErrorString(_e), " at ", #expr); \
  } while (0)

int et_of(at::ScalarType t) {
  switch (t) {
    case at::kFloat: return tb::ET_F32;
    case at::kHalf: return tb::ET_F16;
    case at::kBFloat16: return tb::ET_BF16;
    case at::kInt: return tb::ET_I32;
    case at::kLong: return tb::ET_I64;
    default: TORCH_CHECK(false, "unsupported dtype for P2P reduce: ", t);
  }
}

}  // namespace

void register_symm_bindings(pybind11::module& m) {
  namespace py = pybind11;
  py::class_<tb::BlockPool>(m, "BlockPool")
      .def(py::init<>())
      .def("reset", &tb::BlockPool::reset)
      .def("alloc", &tb::BlockPool::alloc)
      .def("free", &tb::BlockPool::free)
      .def("free_bytes", &tb::BlockPool::free_bytes)
      .def("largest_free_block", &tb::BlockPool::largest_free_block)
      .def("live_blocks", &tb::BlockPool::live_blocks);
  py::class_<tb::SymmHeap, std::shared_ptr<tb::SymmHeap>>(m, "SymmHeap")
      .def(py::init([](int64_t bytes, int64_t device) {
        return std::make_shared<tb::SymmHeap>(static_cast<size_t>(bytes), static_cast<int>(device));
      }))
      .def("ipc_handle", [](const tb::SymmHeap& h) { return py::bytes(h.ipc_handle()); })
      .def("open_peers",
           [](tb::SymmHeap& h, int64_t rank, const std::vector<py::bytes>& handles) {
             std::vector<std::string> hs;
             for (const auto& b : handles) hs.emplace_back(static_cast<std::string>(b));
             h.open_peers(static_cast<int>(rank), hs);
           })
      .def("close", &tb::SymmHeap::close)
      .def("set_pool", [](tb::SymmHeap& h, int64_t off, int64_t bytes) { h.set_pool(off, bytes); })
      .def("bytes", [](const tb::SymmHeap& h) { return static_cast<int64_t>(h.bytes()); })
      .def("world", &tb::SymmHeap::world)
      .def("rank", &tb::SymmHeap::rank)
      .def("base_ptr", [](const tb::SymmHeap& h, int64_t r) { return reinterpret_cast<int64_t>(h.base(static_cast<int>(r))); })
      .def("peer_table_ptr", [](const tb::SymmHeap& h) { return reinterpret_cast<int64_t>(h.device_peer_table()); })
      // Non-owning tensor view of `rank`'s heap at byte offset `off` (keep the heap alive while it is used).
      .def("tensor",
           [](std::shared_ptr<tb::SymmHeap> h, int64_t rank, int64_t off, std::vector<int64_t> sizes,
              at::ScalarType dtype, int64_t device) {
             uint8_t* p = static_cast<uint8_t*>(h->base(static_cast<int>(rank))) + off;
             auto opts = at::TensorOptions().dtype(dtype).device(at::kCUDA, static_cast<int>(device));
             return at::from_blob(p, sizes, [h](void*) {}, opts);
           });

  // One-call collective: allocate the receive buffer from the arena pool (or use the bounce region), announce it to
  // the peers through the mailboxes, push this rank's payload, and return the received data as a tensor that lives
  // in the arena (its deleter frees the pool block).  `src_off/dst_off/nbytes` are per-peer byte offsets/sizes.
  m.def("p2p_collective", [](std::shared_ptr<tb::SymmHeap> h, const at::Tensor& src, std::vector<int64_t> src_off,
                             std::vector<int64_t> dst_off, std::vector<int64_t> nbytes, std::vector<int64_t> out_sizes,
                             int64_t slot_off, int64_t epoch, int64_t blocks_per_peer, int64_t bounce_off,
                             int64_t bounce_bytes, bool small_blocks) {
    TORCH_CHECK(src.is_cuda() && src.is_contiguous());
    const int world = h->world(), rank = h->rank();
    TORCH_CHECK(world <= tb::kMaxPeers && (int)src_off.size() == world && (int)dst_off.size() == world && (int)nbytes.size() == world);
    const c10::cuda::CUDAGuard guard(src.device());
    int64_t out_elems = 1;
    for (auto v : out_sizes) out_elems *= v;
    const int64_t out_bytes = out_elems * static_cast<int64_t>(src.element_size());
    long long off = h->pool_alloc(out_bytes);
    const bool pooled = off >= 0;
    if (!pooled) {
      TORCH_CHECK(out_bytes <= bounce_bytes, "tutel_b200: P2P receive buffer does not fit the arena");
      off = bounce_off;
    }
    tb::PushPlan plan{};
    for (int p = 0; p < world; ++p) { plan.src_off[p] = src_off[p]; plan.dst_off[p] = dst_off[p]; plan.bytes[p] = nbytes[p]; }
    TB_CHECK_CUDA(tb::p2p_push(src.data_ptr(), plan, h->device_peer_table(), off, slot_off, slot_off + 128, slot_off + 256,
                               rank, world, static_cast<uint32_t>(epoch), static_cast<int>(blocks_per_peer), small_blocks, cur_stream()));
    uint8_t* ptr = static_cast<uint8_t*>(h->base(rank)) + off;
    auto opts = src.options();
    if (pooled) {
      return at::from_blob(ptr, out_sizes, [h, off](void*) { h->pool_free(off); }, opts);
    }
    return at::from_blob(ptr, out_sizes, [h](void*) {}, opts).clone();
  });
  m.def("p2p_push", [](const at::Tensor& src, std::vector<int64_t> src_off, std::vector<int64_t> dst_off,
                       std::vector<int64_t> nbytes, int64_t peer_table, int64_t dst_heap_off, int64_t ready_off,
                       int64_t done_off, int64_t scratch_off, int64_t rank, int64_t world, int64_t epoch,
                       int64_t blocks_per_peer) {
    TORCH_CHECK(src.is_cuda() && src.is_contiguous());
    TORCH_CHECK(world <= tb::kMaxPeers && (int64_t)src_off.size() == world && (int64_t)dst_off.size() == world &&
                (int64_t)nbytes.size() == world);
    const c10::cuda::CUDAGuard guard(src.device());
    tb::PushPlan plan{};
    for (int p = 0; p < world; ++p) { plan.src_off[p] = src_off[p]; plan.dst_off[p] = dst_off[p]; plan.bytes[p] = nbytes[p]; }
    TB_CHECK_CUDA(tb::p2p_push(src.data_ptr(), plan, reinterpret_cast<const unsigned long long*>(peer_table),
                               dst_heap_off, ready_off, done_off, scratch_off, static_cast<int>(rank), static_cast<int>(world),
                               static_cast<uint32_t>(epoch), static_cast<int>(blocks_per_peer), false, cur_stream()));
  });
  m.def("p2p_reduce_slice", [](at::Tensor& out, int64_t peer_table, int64_t stage_off, int64_t slice_off_bytes,
                               int64_t rank, int64_t world, bool is_max) {
    TORCH_CHECK(out.is_cuda() && out.is_contiguous());
    const c10::cuda::CUDAGuard guard(out.device());
    TB_CHECK_CUDA(tb::p2p_reduce_slice(out.data_ptr(), reinterpret_cast<const unsigned long long*>(peer_table),
                                       stage_off, slice_off_bytes, out.numel(), et_of(out.scalar_type()),
                                       static_cast<int>(rank), static_cast<int>(world), is_max, cur_stream()));
  });
  m.def("p2p_allreduce_oneshot", [](const at::Tensor& in, at::Tensor& out, int64_t peer_table, int64_t inbox_off,
                                    int64_t slot_bytes, int64_t flag_off, int64_t rank, int64_t world, int64_t epoch,
                                    bool is_max) {
    TORCH_CHECK(in.is_cuda() && in.is_contiguous() && out.is_cuda() && out.is_contiguous() &&
                in.scalar_type() == out.scalar_type() && in.numel() == out.numel());
    const c10::cuda::CUDAGuard guard(in.device());
    TB_CHECK_CUDA(tb::p2p_allreduce_oneshot(in.data_ptr(), out.data_ptr(), reinterpret_cast<const unsigned long long*>(peer_table),
                                            inbox_off, slot_bytes, flag_off, in.numel(), et_of(in.scalar_type()),
                                            static_cast<int>(rank), static_cast<int>(world), static_cast<uint32_t>(epoch),
                                            is_max, cur_stream()));
  });
  m.def("p2p_oneshot_max_blocks", []() { return static_cast<int64_t>(tb::kOneShotMaxBlocks); });
  // [rows, cols, width] -> [cols, rows, width] record transpose (2-D hierarchical all-to-all phases)
  m.def("p2p_stride_copy", [](const at::Tensor& src, at::Tensor& dst, int64_t rows, int64_t cols) {
    TORCH_CHECK(src.is_cuda() && src.is_contiguous() && dst.is_cuda() && dst.is_contiguous() &&
                src.numel() == dst.numel() && src.scalar_type() == dst.scalar_type() && rows * cols > 0 &&
                src.numel() % (rows * cols) == 0);
    const c10::cuda::CUDAGuard guard(src.device());
    const int64_t width = src.numel() / (rows * cols) * static_cast<int64_t>(src.element_size());
    TB_CHECK_CUDA(tb::p2p_stride_copy(src.data_ptr(), dst.data_ptr(), static_cast<int>(rows), static_cast<int>(cols), width,
                                      cur_stream()));
  });
  m.def("set_spin_timeout", [](double seconds) {
    const unsigned long long ns = static_cast<unsigned long long>(seconds * 1e9);
    TB_CHECK_CUDA(tb::set_spin_timeout_moe(ns));
    TB_CHECK_CUDA(tb::set_spin_timeout_p2p(ns));
    TB_CHECK_CUDA(tb::set_spin_timeout_gemm(ns));
    TB_CHECK_CUDA(tb::set_spin_timeout_mx(ns));
    TB_CHECK_CUDA(tb::set_spin_timeout_block_fp8(ns));
  });
  m.def("p2p_barrier", [](int64_t peer_table, int64_t bar_off, int64_t rank, int64_t world, int64_t epoch) {
    TB_CHECK_CUDA(tb::p2p_barrier(reinterpret_cast<const unsigned long long*>(peer_table), bar_off,
                                  static_cast<int>(rank), static_cast<int>(world), static_cast<uint32_t>(epoch),
                                  cur_stream()));
  });
}
