// GPU collective ops: the NVLink peer-to-peer product path, the NCCL baseline
// path (reference-equivalent: pack kernel -> ncclAllReduce -> unpack kernel)
// and the host-staged fallback, plus the per-device CUDA plumbing (private
// high-priority stream, pooled events, descriptor staging ring).
//
// Parity: horovod/common/ops/gpu_operations.{h,cc} (GPUContext / GPUOpContext /
// GPUAllreduce...), ops/cuda_operations.cc (streams, event pool),
// ops/nccl_operations.{h,cc} (NCCL ops).
#pragma once
#include <atomic>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>
#include <cuda_runtime.h>
#include "../common/common.h"
#include "../common/controller.h"
#include "../common/process_set.h"
#include "../common/timeline.h"
#include "../kernels/p2p_kernels.h"
#include "../symm/symm_memory.h"
#include "collective_plan.h"

namespace hvd {

// Completion event shared by every entry of a fused response.
struct SharedEvent {
  cudaEvent_t ev = nullptr;
  std::atomic<int> refs{0};
  int device = 0;
};

class GpuContext {
 public:
  static GpuContext& Get();
  bool Available();
  int DeviceCount();
  cudaStream_t Stream(int device);
  cudaStream_t LatencyStream(int device);  // small responses (GpuOpEnv::latency_lane_bytes)
  void* GridSyncBlock(int device);         // 256 zeroed bytes: grid-barrier state of the persistent Adasum kernel
  SharedEvent* NewEvent(int device, int refs);
  void Release(SharedEvent* e);
  // Copies a small host table to device memory on `s` (pinned ring -> device ring).
  const void* Stage(int device, const void* host, size_t bytes, cudaStream_t s);
  // zero-filled / scratch device memory that lives until the stream reaches this point
  void* TempAlloc(int device, size_t bytes, bool zero, cudaStream_t s);
  // Grow-only pinned host staging buffer (one per device; used by the background thread only).
  void* PinnedHost(int device, size_t bytes);
  void TempFreeAll(int device, cudaStream_t s);
  void Reset();

 private:
  struct PerDevice {
    cudaStream_t stream = nullptr;
    cudaStream_t lat_stream = nullptr;
    void* grid_sync = nullptr;
    std::vector<cudaEvent_t> pool;
    char* host_ring = nullptr; char* dev_ring = nullptr; size_t ring_off = 0;
    std::vector<void*> temps;
    void* pinned = nullptr; size_t pinned_bytes = 0;
  };
  PerDevice& Dev(int device);
  std::mutex mu_;
  std::map<int, PerDevice> devs_;
  int count_ = -2;
};

using Entries = std::vector<std::shared_ptr<TensorTableEntry>>;

struct GpuOpEnv {
  const TunableParams* params = nullptr;
  Timeline* timeline = nullptr;
  std::string backend = "p2p";        // p2p | nccl | cpu
  std::string variant = "auto";       // auto | oneshot | twoshot | nvls
  DataType wire_dtype = DataType::FLOAT32;  // FLOAT32 = no compression
  size_t symm_buffer_bytes = 128ull << 20;
  bool want_multicast = true;
  int64_t large_msg_ctas = 256;   // CTAs for >= 64 MiB fused messages (two per SM)
  bool broadcast_multicast = true;
  // allreduce responses of at most this many fused bytes run on the latency lane (own stream / barrier channel / reserved
  // buffer tail) instead of queueing behind large ones on the main stream; 0 = off
  int64_t latency_lane_bytes = 256 << 10;
  bool adasum_persistent = true;   // single-launch Adasum (grid barriers inside the kernel) instead of 2 + 2 log2(N) launches
  // teams of up to this many ranks reduce IPC-registered plain tensors in place with the P2P two-shot kernel; larger
  // teams keep the fused pack + NVLS + unpack kernel for sums and use IPC only for MIN / MAX / PRODUCT
  int ipc_max_ranks = 4;  // at 4 GPUs zero-copy P2P beat the three-phase NVLS kernel where it was measured; at 8 GPUs the two tied
  // Kernel-variant crossovers measured on this box when the global set's team is created (cached per topology under
  // HVD_CACHE_DIR): the engine applies them to the tunable parameters unless the environment pinned those.
  int64_t zero_copy_nvls_min_bytes = 1 << 20;  // registered tensors: multimem from this size (two-shot P2P below)
  bool calibrate = true;
  std::function<void(int64_t oneshot_max_bytes, int64_t nvls_min_bytes)> on_calibrated;
};

class GpuOps {
 public:
  explicit GpuOps(GpuOpEnv env) : env_(std::move(env)) {}
  GpuOpEnv& env() { return env_; }
  // Each op enqueues its kernels on the hvd stream and returns a shared
  // completion event in *done (refs preset to entries.size()).
  Status Allreduce(ProcessSet& ps, Entries& es, const Response& r, int device, SharedEvent** done);
  Status Adasum(ProcessSet& ps, Entries& es, const Response& r, int device, SharedEvent** done);
  Status Allgather(ProcessSet& ps, Entries& es, const Response& r, int device, SharedEvent** done);
  Status Broadcast(ProcessSet& ps, Entries& es, const Response& r, int device, SharedEvent** done);
  Status Alltoall(ProcessSet& ps, Entries& es, const Response& r, int device, SharedEvent** done);
  Status Reducescatter(ProcessSet& ps, Entries& es, const Response& r, int device, SharedEvent** done);
  // Description of the data path chosen for a set (for hvd.gpu_backend_info()).
  std::string Describe(ProcessSet& ps);

  // Zero-copy allreduce of a registered tensor as ONE kernel on `stream` (which may be capturing into a CUDA graph), on
  // barrier channel `channel` (kern::kGraphChannel; kern::kSyncBnChannel for hvd.SyncBatchNorm), with no negotiation:
  // callable from framework threads.
  Status CapturedAllreduce(ProcessSet& ps, void* ptr, int64_t bytes, DataType dtype, ReduceOp op, double prescale,
                           double postscale, int max_ctas, cudaStream_t stream, int channel);
  // Sharded optimizer step (ZeRO-1), same launch contract as CapturedAllreduce: rank r owns [r*S, (r+1)*S), S = bytes / n,
  // and bytes must be a multiple of 16 * n.  Reduce-scatter: rank r's shard of its own tensor receives the reduction.
  // Allgather: every owner's shard is copied into every peer's tensor.
  Status CapturedReducescatter(ProcessSet& ps, void* ptr, int64_t bytes, DataType dtype, ReduceOp op, double prescale,
                               double postscale, int max_ctas, cudaStream_t stream);
  Status CapturedAllgather(ProcessSet& ps, void* ptr, int64_t bytes, int max_ctas, cudaStream_t stream, int channel);
  // Alltoall of `rows` rows of `row_bytes` at `in` (inside a registered region) whose splits (n int32 / int64 values) exist
  // only on the device: ONE kernel on `stream` on barrier channel kern::kAlltoallChannel, same launch contract as the other
  // captured collectives; every rank passes the same grid (`max_ctas`).  Writes up to `capacity` rows to `out`, the
  // received splits to `recv_splits` and the verdict (kern::AlltoallStatus) to `status`.
  Status CapturedAlltoall(ProcessSet& ps, const void* in, int64_t rows, int64_t row_bytes, const void* splits, int64_t nsplits,
                          bool splits_int64, void* out, int64_t capacity, int64_t* recv_splits, int* status, int max_ctas,
                          cudaStream_t stream);
  bool BuildInplaceArgs(SymmTeam& team, const void* ptr, int64_t bytes, DataType dtype, ReduceOp op, double prescale,
                        double postscale, int64_t expect_off, int max_ctas, kern::InplaceArgs* out);

  // allreduces that ran zero-copy on IPC-registered plain tensors
  uint64_t ipc_launches() const { return ipc_launches_.load(std::memory_order_relaxed); }

  // Lazily creates (collectively) the peer-mapped team of a process set.
  std::shared_ptr<SymmTeam> EnsureTeam(ProcessSet& ps, int device);

 private:
  Status NcclAllreduce(ProcessSet& ps, Entries& es, const Response& r, int device, cudaStream_t s);
  Status StagedOnHost(ProcessSet& ps, Entries& es, const Response& r, int device, cudaStream_t s);
  // Multi-host sets with the same number of GPUs per host: intra-host reduce-scatter kernel, cross-host CPU-transport
  // allreduce of the 1/L shard, intra-host allgather kernel (the role of NCCLHierarchicalAllreduce).
  bool EnsureHierarchy(ProcessSet& ps, int device);
  Status HierarchicalAllreduce(ProcessSet& ps, Entries& es, const Response& r, int device, cudaStream_t s);
  // returns InProgress() when the kernel path does not apply (caller falls back to host staging)
  Status AdasumP2P(ProcessSet& ps, SymmTeam& team, Entries& es, const Response& r, const std::vector<int64_t>& counts,
                   int device, cudaStream_t s);
  void Calibrate(ProcessSet& ps, SymmTeam& team, int device);
  // Stages and launches every entry of a plan (collective_plan.h) in order, each on the team's next buffer slot, or on
  // its next latency-lane slot.  `es`: the entries of an allreduce, whose timelines record each launch's kernel.
  Status LaunchPlan(SymmTeam& team, int device, cudaStream_t s, const Plan& plan, const char* what, Entries* es = nullptr,
                    bool latency_lane = false);
  // What the captured collectives share: the set's team, the zero-copy arguments of the registered range and the launch
  // on the caller's stream.  `launch` is kern::LaunchInplaceAllreduce, LaunchInplaceReducescatter or LaunchInplaceAllgather.
  using InplaceLaunch = cudaError_t (*)(const kern::CommParams&, const kern::InplaceArgs&, cudaStream_t);
  Status LaunchCaptured(ProcessSet& ps, const char* what, InplaceLaunch launch, void* ptr, int64_t bytes, DataType dtype, ReduceOp op,
                        double prescale, double postscale, int max_ctas, cudaStream_t stream, int channel);
  GpuOpEnv env_;
  uint64_t team_counter_ = 0;
  std::atomic<uint64_t> ipc_launches_{0};
};

// Row split of dim 0 for reducescatter: the first dim0 % size ranks get one extra row
// (reference ops/collective_operations.cc:314-330).
inline void ReducescatterRows(int64_t dim0, int size, std::vector<int64_t>* rows) {
  rows->assign(size, dim0 / size);
  for (int i = 0; i < dim0 % size; ++i) (*rows)[i]++;
}

}  // namespace hvd
