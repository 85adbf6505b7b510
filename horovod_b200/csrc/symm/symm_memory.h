// Symmetric (peer-mapped) GPU memory for one team of ranks on an NVSwitch box,
// plus GPU / NVLink topology discovery done once in hvd.init().
//
// The reference never sees the fabric: NCCL does discovery and buffer
// registration internally (ops/nccl_operations.cc:87-131 only bootstraps a
// communicator).  Here every rank allocates its fusion buffers and a flag page
// with the CUDA VMM API (cuMemCreate, POSIX-fd shareable), passes the fds to its
// peers over abstract Unix sockets (SCM_RIGHTS), maps all peers' allocations
// (cuMemMap + cuMemSetAccess) and — when the driver exposes NVLS — binds the
// buffers to a multicast object so multimem.ld_reduce / multimem.st work on
// them.  Fallback when fd export is not permitted: cudaMalloc + cudaIpc handles
// (no multicast).
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <vector>
#include "../kernels/p2p_kernels.h"
#include "../transport/transport.h"

namespace hvd {

struct GpuTopology {
  int device = -1;
  int device_count = 0;
  std::string name;
  int sm_count = 0;
  int cc_major = 0, cc_minor = 0;
  size_t total_mem = 0;
  bool vmm_supported = false;          // CU_DEVICE_ATTRIBUTE_VIRTUAL_MEMORY_MANAGEMENT_SUPPORTED
  bool fd_handles_supported = false;   // POSIX fd export of VMM allocations
  bool multicast_supported = false;    // CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED (NVLS)
  std::vector<int> peer_access;        // [device_count]: 1 if this device can map that device's memory
  std::vector<int> p2p_native_atomics; // [device_count]
  int numa_node = -1;
  std::string DebugString() const;
};

// Queries the local device (no communication). Safe without a GPU (device = -1).
GpuTopology DiscoverGpuTopology(int device);

class SymmTeam {
 public:
  // Collective over `transport` (the team's ranks; all on one host, one GPU
  // each). `device` = this rank's CUDA device. Returns nullptr (on every rank)
  // when peer mapping is not possible; `why` gets the reason.
  static std::shared_ptr<SymmTeam> Create(Transport* transport, int device, size_t buffer_bytes, bool want_multicast,
                                          const std::string& unique_tag, std::string* why);
  // Single-process variant for kernel unit tests on ONE GPU: all "ranks" are
  // plain allocations on `device`; returns one team object per simulated rank.
  static std::vector<std::shared_ptr<SymmTeam>> CreateSimulated(int nranks, int device, size_t buffer_bytes);
  ~SymmTeam();

  int nranks() const { return nranks_; }
  int device() const { return device_; }            // the CUDA device this rank's buffers live on
  int rank() const { return rank_; }
  // bytes of one buffer slot available to ordinary ops; the reserved tail [buffer_bytes(), buffer_bytes() + reserved_tail())
  // belongs to the latency lane
  size_t buffer_bytes() const { return buffer_bytes_ - reserved_tail_; }
  size_t reserved_tail() const { return reserved_tail_; }
  void set_reserved_tail(size_t b) { reserved_tail_ = b < buffer_bytes_ ? b : 0; }
  bool has_multicast() const { return mc_va_[0] != nullptr; }
  // CommParams for buffer slot `which` (0/1 ping-pong).  `channel` selects an independent set of barrier flags + epochs:
  // kernels of different channels may run concurrently (channel 0 = the cycle thread's stream, kGraphChannel = collectives
  // captured into CUDA graphs on framework streams, the rest = extra engine streams).  The data slots are shared: only
  // zero-copy (registered-region) kernels may use a channel other than the one that owns the slots.
  // `byte_offset` shifts the data pointers (buffers and multicast alias) into a sub-area of the slot.
  kern::CommParams Params(int which, int channel = 0, int64_t byte_offset = 0) const;
  // Next ping-pong slot (ops alternate so a fast rank never overwrites data a
  // slow peer is still reading).
  int NextSlot() { int s = slot_; slot_ ^= 1; return s; }
  int NextLatencySlot() { int s = lat_slot_; lat_slot_ ^= 1; return s; }  // the latency lane alternates on its own
  int* host_abort_flag() { return abort_host_; }
  void Abort() { if (abort_host_) *abort_host_ = 1; }
  // 0 = healthy, 1 = aborted by the host, 2 = a kernel timed out waiting for a peer
  int abort_state() const { return abort_host_ ? *(volatile int*)abort_host_ : 0; }
  void set_timeout_seconds(double s) { timeout_ns_ = s > 0 ? (unsigned long long)(s * 1e9) : 0; }
  const std::string& backend() const { return backend_; }  // "vmm", "vmm+mc", "ipc", "sim"

  // ---- registered regions: user tensors allocated in peer-mapped memory get a zero-copy collective path ----
  struct RegionView { void* ptr[kern::kMaxPeers] = {}; void* mc = nullptr; size_t bytes = 0; };
  // Collective over the team's transport (background thread). Returns the region index or -1.
  int AllocRegion(Transport* t, size_t bytes, const std::string& unique_tag, std::string* why);
  // Is [p, p+len) inside a registered region of THIS rank?
  bool FindRegion(const void* p, size_t len, RegionView* view, int64_t* offset, int* index = nullptr) const;
  void* RegionPtr(int index) const;

 private:
  SymmTeam() = default;
  struct Impl;
  int nranks_ = 0, rank_ = 0, device_ = 0;
  size_t buffer_bytes_ = 0, reserved_tail_ = 0;
  void* buf_[2][kern::kMaxPeers] = {};
  uint32_t* flags_[kern::kMaxPeers] = {};
  void* mc_va_[2] = {nullptr, nullptr};
  uint32_t* epochs_ = nullptr;
  int* abort_host_ = nullptr;   // pinned, mapped
  int* abort_dev_ = nullptr;    // device alias of abort_host_
  int slot_ = 0, lat_slot_ = 0;
  unsigned long long timeout_ns_ = 0;
  std::string backend_;
  std::vector<RegionView> regions_;
  std::shared_ptr<Impl> impl_;  // owns driver handles / mappings

 public:
  // Token that keeps every mapping of this team alive (framework tensors placed in registered regions hold one, so a
  // tensor that outlives hvd.shutdown() / an elastic reset never points at unmapped memory).
  std::shared_ptr<void> KeepAlive() const;
};

}  // namespace hvd
