// The runtime: global state, the background cycle thread, the Enqueue* API the
// framework bindings call, and response execution.
//
// Capability parity with horovod/common/operations.{h,cc} + global_state.h:
// InitializeHorovodOnce / BackgroundThreadLoop / RunLoopOnce / PerformOperation
// (operations.cc:277-334, 409-851, 856-908) and EnqueueTensor* (:1408-2057).
// Differences by design: the loop is event driven (an enqueue wakes it, the
// cycle time is only an upper bound on latency for idle ranks), GPU responses
// complete asynchronously through a shared CUDA event handed to the framework
// (the reference's HOROVOD_ENABLE_ASYNC_COMPLETION is the only mode), the
// collective itself is one fused NVLink kernel (ops/gpu_ops.cc).
#pragma once
#include <atomic>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include "../ops/gpu_ops.h"
#include "common.h"
#include "parameter_manager.h"
#include "process_set.h"
#include "thread_pool.h"
#include "timeline.h"

namespace hvd {

struct InitConfig {
  int rank = 0, size = 1;
  int local_rank = 0, local_size = 1, cross_rank = 0, cross_size = 1;
  std::string rendezvous_addr;
  int rendezvous_port = 0;
  std::string scope = "hvd";
  std::string hostname;
  std::vector<std::vector<int>> process_sets;  // static sets registered at init (ids 1..k)
  std::shared_ptr<Transport> transport;        // pre-built transport (unit tests with the loopback hub)
};

class Engine {
 public:
  Engine();
  ~Engine();
  static Engine& Get();  // process-wide instance used by the C API / framework bindings

  Status Init(const InitConfig& cfg);
  void Shutdown();
  bool initialized() const { return initialized_.load(); }
  bool running() const { return initialized_.load() && !loop_exited_.load(); }  // the background loop is alive

  int rank() const { return cfg_.rank; }
  int size() const { return cfg_.size; }
  int local_rank() const { return cfg_.local_rank; }
  int local_size() const { return cfg_.local_size; }
  int cross_rank() const { return cfg_.cross_rank; }
  int cross_size() const { return cfg_.cross_size; }
  bool is_homogeneous() const { return homogeneous_; }

  // ---- enqueue API (framework threads) ----
  // Entries must have name/input/output/dtype/shape/device/callback (+ready_event) filled in.
  Status EnqueueAllreduces(std::vector<std::shared_ptr<TensorTableEntry>>& es, int32_t process_set_id);
  Status EnqueueAllgathers(std::vector<std::shared_ptr<TensorTableEntry>>& es, int32_t process_set_id);
  Status EnqueueBroadcast(std::shared_ptr<TensorTableEntry> e, int32_t process_set_id);  // e->root_rank is a GLOBAL rank
  Status EnqueueAlltoall(std::shared_ptr<TensorTableEntry> e, int32_t process_set_id);
  Status EnqueueReducescatters(std::vector<std::shared_ptr<TensorTableEntry>>& es, int32_t process_set_id);
  Status EnqueueJoin(std::shared_ptr<TensorTableEntry> e, int32_t process_set_id);
  Status EnqueueBarrier(std::shared_ptr<TensorTableEntry> e, int32_t process_set_id);

  // ---- batching hints from the framework binding ----
  void RequestFlush();  // start a cycle now (someone polls a handle)
  void BeginWait();     // a framework thread blocks on a handle: cycle continuously until EndWait()
  void EndWait();

  // ---- process sets ----
  // Collective over the global set; blocks until every rank asked for the same set. Returns id or <0.
  int32_t AddProcessSet(const std::vector<int>& ranks, std::string* err);
  int32_t RemoveProcessSet(int32_t id, std::string* err);
  ProcessSetTable& process_sets() { return sets_; }
  // Collective allocation of registered (peer-mapped) memory; returns the local address or nullptr (+err).
  // `keep_alive` (optional) receives a token that keeps the region mapped for as long as the caller holds it
  void* AllocSymmetric(size_t bytes, int device, int32_t process_set_id, std::string* err, std::shared_ptr<void>* keep_alive = nullptr);

  // Zero-copy allreduce of a registered tensor launched on the caller's stream (CUDA-graph capturable, no negotiation);
  // `stream` is a cudaStream_t.  See GpuOps::CapturedAllreduce.  `channel`: the barrier channel (kern::kGraphChannel,
  // or kern::kSyncBnChannel for hvd.SyncBatchNorm).
  Status CapturedAllreduce(void* ptr, int64_t bytes, DataType dtype, ReduceOp op, double prescale, double postscale,
                           int32_t process_set_id, int max_ctas, void* stream, int channel = 1);
  // The two halves of a sharded optimizer step, same contract (see GpuOps::CapturedReducescatter / CapturedAllgather).
  Status CapturedReducescatter(void* ptr, int64_t bytes, DataType dtype, ReduceOp op, double prescale, double postscale,
                               int32_t process_set_id, int max_ctas, void* stream);
  Status CapturedAllgather(void* ptr, int64_t bytes, int32_t process_set_id, int max_ctas, void* stream, int channel = 1);
  // Alltoall with device-resident splits, same launch contract (see GpuOps::CapturedAlltoall); needs a set of >= 2 ranks.
  Status CapturedAlltoall(const void* in, int64_t rows, int64_t row_bytes, const void* splits, int64_t nsplits, bool splits_int64,
                          void* out, int64_t capacity, int64_t* recv_splits, int* status, int32_t process_set_id, int max_ctas,
                          void* stream);
  // Ulysses sequence-parallel exchange, same launch contract (see GpuOps::CapturedUlyssesExchange); `nranks` is the set
  // size the caller sized the output for, and the split dim (dims[1] or dims[3]) must be a multiple of it.
  Status CapturedUlyssesExchange(const void* in, void* out, const int64_t* dims, int64_t elem_bytes, int direction, bool head_first,
                                 void* staging, int64_t staging_bytes, int* status, int nranks, int32_t process_set_id, int max_ctas,
                                 void* stream);

  // ---- timeline ----
  Status StartTimeline(const std::string& file, bool mark_cycles);
  Status StopTimeline();

  GpuOps& gpu_ops() { return *gpu_ops_; }
  ParameterManager& parameter_manager() { return params_; }
  Timeline& timeline() { return timeline_; }
  std::string TopologyString() const { return topology_str_; }
  std::string ControlPlaneString(int process_set_id = 0);
  std::string last_error() const { std::lock_guard<std::mutex> l(err_mu_); return last_error_; }
  // statistics for tests / bench
  uint64_t cycles() const { return cycles_.load(); }
  uint64_t fast_path_cycles() const { return fast_cycles_.load(); }
  uint64_t responses_executed() const { return responses_.load(); }
  uint64_t captured_launches() const { return captured_launches_.load(); }
  // Host-path latency probes (sums of nanoseconds + sample counts since init): where a collective's time goes before the
  // GPU sees it.  0 queue = enqueue -> its cycle starts, 1 negotiate = ComputeResponseList, 2 execute = PerformOperation
  // (pack descriptors, launch, record events, callbacks), 3 total = enqueue -> completion callback.
  static constexpr int kLatKinds = 4;
  uint64_t latency_sum_ns(int k) const { return lat_sum_[k].load(std::memory_order_relaxed); }
  uint64_t latency_count(int k) const { return lat_cnt_[k].load(std::memory_order_relaxed); }
  // Named monotonic counters (hvd.metrics()): per collective type the number of executed (fused) responses, tensors and
  // payload bytes, split by where they ran (gpu / host), plus errors.  Index = type * kPerType + field.
  static constexpr int kMetricTypes = 12, kPerType = 5;
  enum MetricField { kResponses = 0, kTensors = 1, kBytes = 2, kOnGpu = 3, kErrors = 4 };
  uint64_t metric(int type, int field) const { return op_metrics_[type * kPerType + field].load(std::memory_order_relaxed); }

 private:
  void BackgroundThread();
  bool RunLoopOnce();
  void PerformOperation(ProcessSet& ps, Response& r);
  Status ExecuteCpu(ProcessSet& ps, Entries& es, const Response& r);
  std::shared_ptr<ProcessSet> MakeProcessSet(const std::vector<int>& ranks);
  Status CheckSet(int32_t id, std::shared_ptr<ProcessSet>* out);
  void Wake();
  void NotePending(int64_t bytes);
  void FailAll(const Status& s);
  void SetError(const std::string& m) { std::lock_guard<std::mutex> l(err_mu_); last_error_ = m; }

  InitConfig cfg_;
  std::atomic<bool> initialized_{false}, init_done_{false}, init_failed_{false}, shutdown_requested_{false},
      loop_exited_{false};
  std::thread thread_;
  std::shared_ptr<Transport> transport_;
  ProcessSetTable sets_;
  ParameterManager params_;
  Timeline timeline_;
  ThreadPool finalizers_;
  std::unique_ptr<GpuOps> gpu_ops_;
  bool homogeneous_ = true;
  bool elastic_ = false;
  std::string topology_str_;
  std::vector<char> fusion_host_;  // CPU fusion buffer (reference FusionBufferManager for the host path)

  std::mutex wake_mu_;
  std::condition_variable wake_cv_;
  bool wake_flag_ = false;
  std::atomic<int64_t> pending_bytes_{0};
  std::atomic<uint64_t> first_pending_ns_{0};
  std::atomic<bool> flush_{false};
  std::atomic<int> waiters_{0};

  // pending timeline commands (applied by the cycle thread)
  std::mutex tl_mu_;
  std::string tl_pending_file_;
  bool tl_pending_start_ = false, tl_pending_stop_ = false, tl_pending_mark_ = false;

  mutable std::mutex err_mu_;
  std::string last_error_;
  std::atomic<uint64_t> cycles_{0}, fast_cycles_{0}, responses_{0};
  std::atomic<uint64_t> op_metrics_[kMetricTypes * kPerType] = {};
  std::atomic<uint64_t> captured_launches_{0};
  int64_t ipc_min_bytes_ = 0;  // plain in-place GPU tensors of at least this size are offered for IPC registration (0 = off)
  std::atomic<uint64_t> lat_sum_[kLatKinds] = {}, lat_cnt_[kLatKinds] = {};
  uint64_t cycle_start_ns_ = 0;
  void NoteLatency(int k, uint64_t ns) { lat_sum_[k].fetch_add(ns, std::memory_order_relaxed); lat_cnt_[k].fetch_add(1, std::memory_order_relaxed); }
  std::atomic<int> noname_counter_{0};
  std::atomic<int> symm_alloc_counter_{0};
  std::atomic<int> join_device_{-1};  // CUDA device a joined rank contributes zeros from
};

}  // namespace hvd
