// Symmetric heap: one cudaMalloc'd arena per rank, exported with CUDA IPC and mapped into every peer process on the
// node, so that kernels can address any rank's buffers directly over NVLink.  H100-native replacement for the
// reference's private NCCL communicators (tutel/custom/custom_kernel.cpp:327-431).
#pragma once
#include <cstddef>
#include <cstdint>
#include <map>
#include <mutex>
#include <string>
#include <vector>

namespace tb {

// First-fit block allocator over an offset range (256-byte granularity, adjacent free blocks coalesce).  Owns no
// memory: the symmetric heap uses it for the receive-buffer pool inside the arena; thread safe.
class BlockPool {
 public:
  void reset(long long off, long long bytes);
  long long alloc(long long bytes);   // offset of a block of at least `bytes`, -1 when no free block fits
  void free(long long off);           // unknown offsets are ignored
  long long free_bytes();
  long long largest_free_block();
  size_t live_blocks();

 private:
  std::mutex mu_;
  std::map<long long, long long> free_;   // offset -> length of free blocks
  std::map<long long, long long> used_;   // offset -> length of live blocks
};

class SymmHeap {
 public:
  SymmHeap(size_t bytes, int device);
  ~SymmHeap();
  SymmHeap(const SymmHeap&) = delete;
  SymmHeap& operator=(const SymmHeap&) = delete;

  std::string ipc_handle() const;                                   // 64 opaque bytes
  void open_peers(int rank, const std::vector<std::string>& handles);  // handles[r] from rank r (own entry ignored)
  void close();

  size_t bytes() const { return bytes_; }
  int rank() const { return rank_; }
  int world() const { return static_cast<int>(peer_base_.size()); }
  void* base(int r) const { return peer_base_.at(r); }
  const unsigned long long* device_peer_table() const { return d_peer_table_; }

  // Receive-buffer pool inside the arena (first-fit free list, 256-byte granularity).  Collectives allocate their
  // output here and hand it out as a tensor whose deleter returns the block - no copy out of a staging area.
  void set_pool(long long off, long long bytes) { pool_.reset(off, bytes); }
  long long pool_alloc(long long bytes) { return pool_.alloc(bytes); }   // -1 when no block fits
  void pool_free(long long off) { pool_.free(off); }

 private:
  size_t bytes_ = 0;
  int device_ = 0;
  int rank_ = 0;
  void* local_ = nullptr;
  std::vector<void*> peer_base_;
  unsigned long long* d_peer_table_ = nullptr;
  bool closed_ = false;
  BlockPool pool_;
};

}  // namespace tb
