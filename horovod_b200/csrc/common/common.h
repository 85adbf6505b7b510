// Core value types of the hvd runtime: Status, dtypes, reduce ops, shapes,
// tensor-table entries and the knob names read from the environment.
//
// Capability parity: horovod/common/common.h:79-404 (Status, TensorShape,
// TensorTableEntry, activity names, env knob macros) and message.h:30-54
// (DataType / ReduceOp).  The layout here is new: entries carry raw device
// pointers + CUDA events + std::function allocation hooks instead of the
// reference's virtual Tensor/OpContext/ReadyEvent adapter hierarchy, and
// BFLOAT16 is a first-class dtype (the reference has none).
#pragma once
#include <cstdint>
#include <cstring>
#include <functional>
#include <memory>
#include <string>
#include <vector>

namespace hvd {

enum class DataType : uint8_t {
  UINT8 = 0, INT8 = 1, UINT16 = 2, INT16 = 3, INT32 = 4, INT64 = 5,
  FLOAT16 = 6, FLOAT32 = 7, FLOAT64 = 8, BOOL = 9, BFLOAT16 = 10,
};
constexpr int kNumDataTypes = 11;

inline size_t DataTypeSize(DataType t) {
  switch (t) {
    case DataType::UINT8: case DataType::INT8: case DataType::BOOL: return 1;
    case DataType::UINT16: case DataType::INT16: case DataType::FLOAT16:
    case DataType::BFLOAT16: return 2;
    case DataType::INT32: case DataType::FLOAT32: return 4;
    case DataType::INT64: case DataType::FLOAT64: return 8;
  }
  return 0;
}
const char* DataTypeName(DataType t);
inline bool IsFloatType(DataType t) {
  return t == DataType::FLOAT16 || t == DataType::FLOAT32 ||
         t == DataType::FLOAT64 || t == DataType::BFLOAT16;
}

enum class ReduceOp : uint8_t { AVERAGE = 0, SUM = 1, ADASUM = 2, MIN = 3, MAX = 4, PRODUCT = 5 };
const char* ReduceOpName(ReduceOp op);

constexpr int CPU_DEVICE_ID = -1;
constexpr int32_t kUniformSplits = -2;  // Request/Response::root_rank of an alltoall without explicit splits

// Names with special meaning in the negotiation stream.
constexpr const char* JOIN_TENSOR_NAME = "join.noname";
constexpr const char* BARRIER_TENSOR_NAME = "barrier.noname";
constexpr const char* PS_ADD_PREFIX = "__process_set_add__:";
constexpr const char* PS_REMOVE_PREFIX = "__process_set_remove__:";
constexpr const char* SYMM_ALLOC_PREFIX = "__symm_alloc__:";

// Every fused tensor starts on a 128 B boundary so that 16 B vector accesses
// and multimem.* never straddle two tensors (the reference pads
// to 16 B: controller.cc:922-930).
constexpr int64_t FUSION_ALIGN_BYTES = 128;

enum class StatusType : uint8_t { OK, UNKNOWN_ERROR, PRECONDITION_ERROR, ABORTED, INVALID_ARGUMENT, IN_PROGRESS };

class Status {
 public:
  Status() = default;
  static Status OK() { return Status(); }
  static Status UnknownError(const std::string& m) { return Status(StatusType::UNKNOWN_ERROR, m); }
  static Status PreconditionError(const std::string& m) { return Status(StatusType::PRECONDITION_ERROR, m); }
  static Status Aborted(const std::string& m) { return Status(StatusType::ABORTED, m); }
  static Status InvalidArgument(const std::string& m) { return Status(StatusType::INVALID_ARGUMENT, m); }
  static Status InProgress() { return Status(StatusType::IN_PROGRESS, ""); }
  bool ok() const { return type_ == StatusType::OK; }
  bool in_progress() const { return type_ == StatusType::IN_PROGRESS; }
  StatusType type() const { return type_; }
  const std::string& reason() const { return reason_; }

 private:
  Status(StatusType t, std::string r) : type_(t), reason_(std::move(r)) {}
  StatusType type_ = StatusType::OK;
  std::string reason_;
};

// Error texts asserted on by API-level tests (reference common.h:233-262).
extern const char* const SHUT_DOWN_ERROR_MSG;
extern const char* const NOT_INITIALIZED_ERROR_MSG;
std::string DuplicateNameError(const std::string& name);

class TensorShape {
 public:
  TensorShape() = default;
  explicit TensorShape(std::vector<int64_t> d) : dims_(std::move(d)) {}
  void AddDim(int64_t d) { dims_.push_back(d); }
  int ndim() const { return (int)dims_.size(); }
  int64_t dim(int i) const { return dims_[i]; }
  int64_t num_elements() const { int64_t n = 1; for (auto d : dims_) n *= d; return n; }
  const std::vector<int64_t>& dims() const { return dims_; }
  bool operator==(const TensorShape& o) const { return dims_ == o.dims_; }
  bool operator!=(const TensorShape& o) const { return dims_ != o.dims_; }
  std::string DebugString() const;

 private:
  std::vector<int64_t> dims_;
};

enum class RequestType : uint8_t {
  ALLREDUCE = 0, ALLGATHER = 1, BROADCAST = 2, JOIN = 3, ADASUM = 4,
  ALLTOALL = 5, BARRIER = 6, REDUCESCATTER = 7, PROCESS_SET_ADD = 8, PROCESS_SET_REMOVE = 9,
  SYMM_ALLOC = 11,  // collective allocation of a registered (peer-mapped) region; 10 is ResponseType::ERROR
};
const char* RequestTypeName(RequestType t);

// Completion record handed to the framework binding.
struct Completion {
  Status status;
  void* done_event = nullptr;            // cudaEvent_t recorded on the hvd stream (GPU ops), else null
  std::vector<int32_t> received_splits;  // alltoall
  int32_t last_joined_rank = -1;         // join
  void* aux_ptr = nullptr;               // SYMM_ALLOC: local address of the new region
};
using CompletionCallback = std::function<void(const Completion&)>;
// Allocates (or resizes) the framework-owned output for ops whose size is only
// known after negotiation (allgather / alltoall / reducescatter). Returns the
// data pointer.  Runs on the background thread.
using OutputAllocator = std::function<void*(const std::vector<int64_t>& shape)>;

struct TensorTableEntry {
  std::string name;
  RequestType type = RequestType::ALLREDUCE;
  const void* input = nullptr;
  void* output = nullptr;
  DataType dtype = DataType::FLOAT32;
  TensorShape shape;
  int device = CPU_DEVICE_ID;
  int root_rank = 0;  // set-relative rank for broadcast
  int32_t process_set_id = 0;
  double prescale = 1.0, postscale = 1.0;
  ReduceOp reduce_op = ReduceOp::SUM;
  std::vector<int32_t> splits;  // alltoall send splits (rows per destination)
  void* ready_event = nullptr;  // cudaEvent_t recorded on the framework stream
  int32_t group_id = -1;
  OutputAllocator alloc_output;
  CompletionCallback callback;
  // filled in during execution
  std::vector<int32_t> received_splits;
  std::shared_ptr<void> nvtx_range;  // NvtxOpRange: ends when the entry is destroyed (after its callback ran)
  uint64_t enqueue_ns = 0;
  size_t bytes() const { return (size_t)shape.num_elements() * DataTypeSize(dtype); }
};

// ---- environment knobs (names kept where the reference meaning carries over,
// operations.cc:460-650; HVD_* are new knobs of this library) -----------------
#define HOROVOD_FUSION_THRESHOLD "HOROVOD_FUSION_THRESHOLD"
#define HOROVOD_CYCLE_TIME "HOROVOD_CYCLE_TIME"
#define HOROVOD_CACHE_CAPACITY "HOROVOD_CACHE_CAPACITY"
#define HOROVOD_TIMELINE "HOROVOD_TIMELINE"
#define HOROVOD_TIMELINE_MARK_CYCLES "HOROVOD_TIMELINE_MARK_CYCLES"
#define HOROVOD_AUTOTUNE "HOROVOD_AUTOTUNE"
#define HOROVOD_AUTOTUNE_LOG "HOROVOD_AUTOTUNE_LOG"
#define HOROVOD_AUTOTUNE_WARMUP_SAMPLES "HOROVOD_AUTOTUNE_WARMUP_SAMPLES"
#define HOROVOD_AUTOTUNE_STEPS_PER_SAMPLE "HOROVOD_AUTOTUNE_STEPS_PER_SAMPLE"
#define HOROVOD_AUTOTUNE_BAYES_OPT_MAX_SAMPLES "HOROVOD_AUTOTUNE_BAYES_OPT_MAX_SAMPLES"
#define HOROVOD_AUTOTUNE_GAUSSIAN_PROCESS_NOISE "HOROVOD_AUTOTUNE_GAUSSIAN_PROCESS_NOISE"
#define HOROVOD_STALL_CHECK_DISABLE "HOROVOD_STALL_CHECK_DISABLE"
#define HOROVOD_STALL_CHECK_TIME_SECONDS "HOROVOD_STALL_CHECK_TIME_SECONDS"
#define HOROVOD_STALL_SHUTDOWN_TIME_SECONDS "HOROVOD_STALL_SHUTDOWN_TIME_SECONDS"
#define HOROVOD_DISABLE_GROUP_FUSION "HOROVOD_DISABLE_GROUP_FUSION"
#define HOROVOD_THREAD_AFFINITY "HOROVOD_THREAD_AFFINITY"
#define HOROVOD_NUM_STREAMS "HOROVOD_NUM_NCCL_STREAMS"
#define HOROVOD_ELASTIC "HOROVOD_ELASTIC"
#define HOROVOD_DYNAMIC_PROCESS_SETS "HOROVOD_DYNAMIC_PROCESS_SETS"
#define HOROVOD_LOG_LEVEL "HOROVOD_LOG_LEVEL"
#define HOROVOD_LOG_HIDE_TIME "HOROVOD_LOG_HIDE_TIME"
#define HOROVOD_ADASUM_CHUNK_SIZE "HOROVOD_ADASUM_MPI_CHUNK_SIZE"
#define HOROVOD_RENDEZVOUS_ADDR "HOROVOD_GLOO_RENDEZVOUS_ADDR"
#define HOROVOD_RENDEZVOUS_PORT "HOROVOD_GLOO_RENDEZVOUS_PORT"
#define HOROVOD_TIMEOUT_SECONDS "HOROVOD_GLOO_TIMEOUT_SECONDS"
#define HOROVOD_RANK "HOROVOD_RANK"
#define HOROVOD_SIZE "HOROVOD_SIZE"
#define HOROVOD_LOCAL_RANK "HOROVOD_LOCAL_RANK"
#define HOROVOD_LOCAL_SIZE "HOROVOD_LOCAL_SIZE"
#define HOROVOD_CROSS_RANK "HOROVOD_CROSS_RANK"
#define HOROVOD_CROSS_SIZE "HOROVOD_CROSS_SIZE"
#define HOROVOD_HOSTNAME "HOROVOD_HOSTNAME"
// new knobs
#define HVD_GPU_BACKEND "HVD_GPU_BACKEND"            // p2p (default) | nccl | cpu
#define HVD_ALLREDUCE_VARIANT "HVD_ALLREDUCE_VARIANT"  // auto | oneshot | twoshot | nvls
#define HVD_ONESHOT_MAX_BYTES "HVD_ONESHOT_MAX_BYTES"
#define HVD_NVLS_MIN_BYTES "HVD_NVLS_MIN_BYTES"
#define HVD_COMM_CTAS "HVD_COMM_CTAS"
#define HVD_SYMM_BUFFER_BYTES "HVD_SYMM_BUFFER_BYTES"
#define HVD_CONTROL_PLANE "HVD_CONTROL_PLANE"        // auto | shm | tcp
#define HVD_WIRE_DTYPE "HVD_WIRE_DTYPE"              // none | bf16 | fp16 (in-kernel compression)

uint64_t NowNs();

}  // namespace hvd
