// PyTorch binding: wraps at::Tensor arguments into TensorTableEntry objects,
// records a ready event on the caller's current CUDA stream, enqueues into the
// engine and hands back an integer handle.  Completion is event-chained: for
// GPU collectives `wait_and_clear` makes the caller's stream wait on the
// engine's completion event instead of blocking the host.
//
// Capability parity: horovod/torch/mpi_ops_v2.cc (Do{Allreduce,...}, PollHandle,
// WaitAndClear), adapter_v2.cc (TorchTensor / TorchOpContext allocation),
// ready_event.cc (pooled events on the current stream), handle_manager.cc,
// cuda_util.cc (device guard).
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <cuda_runtime.h>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <map>
#include <mutex>
#include <set>
#include <unordered_map>
#include "../common/engine.h"
#include "../kernels/p2p_kernels.h"

namespace py = pybind11;
using namespace hvd;

namespace {

// ---- handle manager --------------------------------------------------------
struct HandleState {
  std::atomic<bool> done{false};
  Status status;
  std::vector<SharedEvent*> events;  // one per fused response that carried members of this handle
  int device = CPU_DEVICE_ID;
  std::vector<int32_t> received_splits;
  int32_t last_joined_rank = -1;
  std::vector<at::Tensor> keep_alive;
  at::Tensor received_splits_out;
  int pending = 1;  // grouped ops complete when every member did
};

class HandleManager {
 public:
  int Allocate(int pending = 1) {
    std::lock_guard<std::mutex> l(mu_);
    int h = next_++;
    auto st = std::make_shared<HandleState>();
    st->pending = pending;
    map_[h] = st;
    return h;
  }
  std::shared_ptr<HandleState> Get(int h) {
    std::lock_guard<std::mutex> l(mu_);
    auto it = map_.find(h);
    return it == map_.end() ? nullptr : it->second;
  }
  void MarkDone(int h, const Completion& c) {
    std::lock_guard<std::mutex> l(mu_);
    auto it = map_.find(h);
    if (it == map_.end()) { if (c.done_event) GpuContext::Get().Release((SharedEvent*)c.done_event); return; }
    auto& st = *it->second;
    if (!c.status.ok() && st.status.ok()) st.status = c.status;
    if (c.done_event) {
      auto* ev = (SharedEvent*)c.done_event;
      bool dup = false;
      for (auto* x : st.events) if (x == ev) dup = true;
      if (dup) GpuContext::Get().Release(ev);  // grouped members fused into one response share the event
      else st.events.push_back(ev);
    }
    if (!c.received_splits.empty()) st.received_splits = c.received_splits;
    if (c.last_joined_rank >= 0) st.last_joined_rank = c.last_joined_rank;
    if (--st.pending <= 0) { st.done = true; cv_.notify_all(); }
  }
  void Wait(const std::shared_ptr<HandleState>& st) {
    // a fused NVLink allreduce completes in tens of microseconds: spin briefly before paying a futex sleep + wake-up
    const auto spin_end = std::chrono::steady_clock::now() + std::chrono::microseconds(200);
    while (!st->done.load(std::memory_order_acquire) && std::chrono::steady_clock::now() < spin_end) {
#if defined(__x86_64__)
      __builtin_ia32_pause();
#endif
    }
    if (st->done.load(std::memory_order_acquire)) { std::lock_guard<std::mutex> l(mu_); return; }
    std::unique_lock<std::mutex> l(mu_);
    cv_.wait(l, [&] { return st->done.load(); });
  }
  bool Done(const std::shared_ptr<HandleState>& st) { return st->done.load(std::memory_order_acquire); }
  void Release(int h) { std::lock_guard<std::mutex> l(mu_); map_.erase(h); }
  void Reset() {
    std::lock_guard<std::mutex> l(mu_);
    for (auto& kv : map_) for (auto* ev : kv.second->events) GpuContext::Get().Release(ev);
    map_.clear();
  }

 private:
  std::mutex mu_;
  std::condition_variable cv_;
  std::unordered_map<int, std::shared_ptr<HandleState>> map_;
  int next_ = 0;
};
HandleManager g_handles;

// ---- ready events ----------------------------------------------------------
class EventPool {
 public:
  cudaEvent_t Get(int device) {
    {
      std::lock_guard<std::mutex> l(mu_);
      auto& v = pool_[device];
      if (!v.empty()) { auto e = v.back(); v.pop_back(); return e; }
    }
    cudaEvent_t e;
    C10_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    return e;
  }
  void Put(int device, cudaEvent_t e) { std::lock_guard<std::mutex> l(mu_); pool_[device].push_back(e); }

 private:
  std::mutex mu_;
  std::unordered_map<int, std::vector<cudaEvent_t>> pool_;
};
EventPool g_events;

DataType MapDtype(at::ScalarType t) {
  switch (t) {
    case at::kByte: return DataType::UINT8;
    case at::kChar: return DataType::INT8;
    case at::kShort: return DataType::INT16;
    case at::kInt: return DataType::INT32;
    case at::kLong: return DataType::INT64;
    case at::kHalf: return DataType::FLOAT16;
    case at::kBFloat16: return DataType::BFLOAT16;
    case at::kFloat: return DataType::FLOAT32;
    case at::kDouble: return DataType::FLOAT64;
    case at::kBool: return DataType::BOOL;
    default: throw std::invalid_argument(std::string("Horovod: unsupported tensor dtype ") + c10::toString(t));
  }
}

int DeviceOf(const at::Tensor& t) { return t.is_cuda() ? (int)t.get_device() : CPU_DEVICE_ID; }

// Unnamed ops are numbered per (op type, process set) — not by handle: handle counters diverge between ranks as soon as
// one rank issues an extra op (around hvd.join(), or inside a process set the other rank is not a member of, e.g. the
// unnamed allreduce in an autograd backward), and the names must match across the ranks of the set.
std::mutex g_noname_mu;
std::unordered_map<std::string, int> g_noname_counters;
std::string OpName(const char* op, const std::string& name, int process_set_id) {
  if (!name.empty()) return std::string(op) + "." + name;
  std::lock_guard<std::mutex> l(g_noname_mu);
  const std::string key = std::string(op) + (process_set_id ? ".ps" + std::to_string(process_set_id) : "");
  return key + ".noname." + std::to_string(g_noname_counters[key]++);
}

// Process-set ids are recycled: a new set must start numbering from zero on every member.
void ResetNonameCounters(int process_set_id) {
  std::lock_guard<std::mutex> l(g_noname_mu);
  const std::string tag = ".ps" + std::to_string(process_set_id);
  for (auto it = g_noname_counters.begin(); it != g_noname_counters.end();) {
    const std::string& k = it->first;
    if (k.size() >= tag.size() && k.compare(k.size() - tag.size(), tag.size(), tag) == 0) it = g_noname_counters.erase(it);
    else ++it;
  }
}

void ThrowIfError(const Status& st) {
  if (st.ok()) return;
  switch (st.type()) {
    case StatusType::INVALID_ARGUMENT: throw std::invalid_argument(st.reason());
    case StatusType::PRECONDITION_ERROR: throw std::logic_error(st.reason());
    default: throw std::runtime_error(st.reason());
  }
}

std::shared_ptr<TensorTableEntry> MakeEntry(const at::Tensor& in, const std::string& name) {
  TORCH_CHECK(in.is_non_overlapping_and_dense(), "Horovod: tensor must be dense (contiguous in some memory format)");
  auto e = std::make_shared<TensorTableEntry>();
  e->name = name;
  e->input = in.data_ptr();
  e->dtype = MapDtype(in.scalar_type());
  e->device = DeviceOf(in);
  std::vector<int64_t> dims(in.sizes().begin(), in.sizes().end());
  e->shape = TensorShape(dims);
  if (in.is_cuda()) {
    c10::cuda::CUDAGuard guard(in.device());
    cudaEvent_t ev = g_events.Get(e->device);
    C10_CUDA_CHECK(cudaEventRecord(ev, c10::cuda::getCurrentCUDAStream(e->device)));
    e->ready_event = ev;
  }
  return e;
}

CompletionCallback MakeCallback(int handle, int device, void* ready_event) {
  return [handle, device, ready_event](const Completion& c) {
    if (ready_event) g_events.Put(device, (cudaEvent_t)ready_event);
    g_handles.MarkDone(handle, c);
  };
}

// Output allocation for collectives whose size is negotiated: runs on the
// background thread; for CUDA the freshly allocated block is ordered before
// the hvd stream touches it.
OutputAllocator MakeAllocator(at::Tensor output) {
  return [output](const std::vector<int64_t>& shape) mutable -> void* {
    if (output.is_cuda()) {
      c10::cuda::CUDAGuard guard(output.device());
      output.resize_(shape);
      int dev = (int)output.get_device();
      cudaEvent_t ev = g_events.Get(dev);
      cudaEventRecord(ev, c10::cuda::getCurrentCUDAStream(dev));
      cudaStreamWaitEvent(GpuContext::Get().Stream(dev), ev, 0);
      g_events.Put(dev, ev);
    } else {
      output.resize_(shape);
    }
    return output.data_ptr();
  };
}

// ---- ops --------------------------------------------------------------------

int DoAllreduce(at::Tensor tensor, at::Tensor output, const std::string& name, int op, double prescale, double postscale,
                int process_set_id) {
  int h = g_handles.Allocate();
  auto e = MakeEntry(tensor, OpName("allreduce", name, process_set_id));
  e->output = output.data_ptr();
  e->reduce_op = (ReduceOp)op; e->prescale = prescale; e->postscale = postscale;
  e->callback = MakeCallback(h, e->device, e->ready_event);
  auto st = g_handles.Get(h);
  st->device = e->device; st->keep_alive = {tensor, output};
  std::vector<std::shared_ptr<TensorTableEntry>> es{e};
  Status s = Engine::Get().EnqueueAllreduces(es, process_set_id);
  if (!s.ok()) { if (e->ready_event) g_events.Put(e->device, (cudaEvent_t)e->ready_event); g_handles.Release(h); ThrowIfError(s); }
  return h;
}

int DoGroupedAllreduce(std::vector<at::Tensor> tensors, std::vector<at::Tensor> outputs, const std::string& name, int op,
                       double prescale, double postscale, int process_set_id) {
  TORCH_CHECK(tensors.size() == outputs.size() && !tensors.empty(), "grouped_allreduce: bad tensor lists");
  int h = g_handles.Allocate((int)tensors.size());
  auto st = g_handles.Get(h);
  std::vector<std::shared_ptr<TensorTableEntry>> es;
  std::string base = OpName("grouped_allreduce", name, process_set_id);
  for (size_t i = 0; i < tensors.size(); ++i) {
    auto e = MakeEntry(tensors[i], base + "_" + std::to_string(i + 1) + "of" + std::to_string(tensors.size()));
    e->output = outputs[i].data_ptr();
    e->reduce_op = (ReduceOp)op; e->prescale = prescale; e->postscale = postscale;
    e->callback = MakeCallback(h, e->device, e->ready_event);
    st->device = e->device;
    st->keep_alive.push_back(tensors[i]); st->keep_alive.push_back(outputs[i]);
    es.push_back(e);
  }
  Status s = Engine::Get().EnqueueAllreduces(es, process_set_id);
  if (!s.ok()) { for (auto& e : es) if (e->ready_event) g_events.Put(e->device, (cudaEvent_t)e->ready_event); g_handles.Release(h); ThrowIfError(s); }
  return h;
}

int DoAllgather(at::Tensor tensor, at::Tensor output, const std::string& name, int process_set_id) {
  int h = g_handles.Allocate();
  auto e = MakeEntry(tensor, OpName("allgather", name, process_set_id));
  e->alloc_output = MakeAllocator(output);
  e->callback = MakeCallback(h, e->device, e->ready_event);
  auto st = g_handles.Get(h);
  st->device = e->device; st->keep_alive = {tensor, output};
  std::vector<std::shared_ptr<TensorTableEntry>> es{e};
  Status s = Engine::Get().EnqueueAllgathers(es, process_set_id);
  if (!s.ok()) { if (e->ready_event) g_events.Put(e->device, (cudaEvent_t)e->ready_event); g_handles.Release(h); ThrowIfError(s); }
  return h;
}

int DoGroupedAllgather(std::vector<at::Tensor> tensors, std::vector<at::Tensor> outputs, const std::string& name,
                       int process_set_id) {
  TORCH_CHECK(tensors.size() == outputs.size() && !tensors.empty(), "grouped_allgather: bad tensor lists");
  int h = g_handles.Allocate((int)tensors.size());
  auto st = g_handles.Get(h);
  std::vector<std::shared_ptr<TensorTableEntry>> es;
  std::string base = OpName("grouped_allgather", name, process_set_id);
  for (size_t i = 0; i < tensors.size(); ++i) {
    auto e = MakeEntry(tensors[i], base + "_" + std::to_string(i + 1) + "of" + std::to_string(tensors.size()));
    e->alloc_output = MakeAllocator(outputs[i]);
    e->callback = MakeCallback(h, e->device, e->ready_event);
    st->device = e->device;
    st->keep_alive.push_back(tensors[i]); st->keep_alive.push_back(outputs[i]);
    es.push_back(e);
  }
  Status s = Engine::Get().EnqueueAllgathers(es, process_set_id);
  if (!s.ok()) { for (auto& e : es) if (e->ready_event) g_events.Put(e->device, (cudaEvent_t)e->ready_event); g_handles.Release(h); ThrowIfError(s); }
  return h;
}

int DoBroadcast(at::Tensor tensor, at::Tensor output, int root_rank, const std::string& name, int process_set_id) {
  int h = g_handles.Allocate();
  auto e = MakeEntry(tensor, OpName("broadcast", name, process_set_id));
  e->output = output.data_ptr();
  e->root_rank = root_rank;
  e->callback = MakeCallback(h, e->device, e->ready_event);
  auto st = g_handles.Get(h);
  st->device = e->device; st->keep_alive = {tensor, output};
  Status s = Engine::Get().EnqueueBroadcast(e, process_set_id);
  if (!s.ok()) { if (e->ready_event) g_events.Put(e->device, (cudaEvent_t)e->ready_event); g_handles.Release(h); ThrowIfError(s); }
  return h;
}

int DoAlltoall(at::Tensor tensor, at::Tensor splits, at::Tensor output, at::Tensor received_splits, const std::string& name,
               int process_set_id) {
  int h = g_handles.Allocate();
  auto e = MakeEntry(tensor, OpName("alltoall", name, process_set_id));
  if (splits.defined() && splits.numel() > 0) {
    at::Tensor cpu_splits = splits.to(at::kCPU, at::kInt).contiguous();  // synchronous D2H when splits live on the GPU (mpi_ops_v2.cc:603-650)
    e->splits.assign(cpu_splits.data_ptr<int32_t>(), cpu_splits.data_ptr<int32_t>() + cpu_splits.numel());
  }
  e->alloc_output = MakeAllocator(output);
  e->callback = MakeCallback(h, e->device, e->ready_event);
  auto st = g_handles.Get(h);
  st->device = e->device; st->keep_alive = {tensor, output};
  st->received_splits_out = received_splits;
  Status s = Engine::Get().EnqueueAlltoall(e, process_set_id);
  if (!s.ok()) { if (e->ready_event) g_events.Put(e->device, (cudaEvent_t)e->ready_event); g_handles.Release(h); ThrowIfError(s); }
  return h;
}

int DoReducescatter(at::Tensor tensor, at::Tensor output, const std::string& name, int op, double prescale, double postscale,
                    int process_set_id) {
  int h = g_handles.Allocate();
  auto e = MakeEntry(tensor, OpName("reducescatter", name, process_set_id));
  e->alloc_output = MakeAllocator(output);
  e->reduce_op = (ReduceOp)op; e->prescale = prescale; e->postscale = postscale;
  e->callback = MakeCallback(h, e->device, e->ready_event);
  auto st = g_handles.Get(h);
  st->device = e->device; st->keep_alive = {tensor, output};
  std::vector<std::shared_ptr<TensorTableEntry>> es{e};
  Status s = Engine::Get().EnqueueReducescatters(es, process_set_id);
  if (!s.ok()) { if (e->ready_event) g_events.Put(e->device, (cudaEvent_t)e->ready_event); g_handles.Release(h); ThrowIfError(s); }
  return h;
}

int DoGroupedReducescatter(std::vector<at::Tensor> tensors, std::vector<at::Tensor> outputs, const std::string& name, int op,
                           double prescale, double postscale, int process_set_id) {
  TORCH_CHECK(tensors.size() == outputs.size() && !tensors.empty(), "grouped_reducescatter: bad tensor lists");
  int h = g_handles.Allocate((int)tensors.size());
  auto st = g_handles.Get(h);
  std::vector<std::shared_ptr<TensorTableEntry>> es;
  std::string base = OpName("grouped_reducescatter", name, process_set_id);
  for (size_t i = 0; i < tensors.size(); ++i) {
    auto e = MakeEntry(tensors[i], base + "_" + std::to_string(i + 1) + "of" + std::to_string(tensors.size()));
    e->alloc_output = MakeAllocator(outputs[i]);
    e->reduce_op = (ReduceOp)op; e->prescale = prescale; e->postscale = postscale;
    e->callback = MakeCallback(h, e->device, e->ready_event);
    st->device = e->device;
    st->keep_alive.push_back(tensors[i]); st->keep_alive.push_back(outputs[i]);
    es.push_back(e);
  }
  Status s = Engine::Get().EnqueueReducescatters(es, process_set_id);
  if (!s.ok()) { for (auto& e : es) if (e->ready_event) g_events.Put(e->device, (cudaEvent_t)e->ready_event); g_handles.Release(h); ThrowIfError(s); }
  return h;
}

int DoJoin(int device, int process_set_id) {
  int h = g_handles.Allocate();
  auto e = std::make_shared<TensorTableEntry>();
  e->device = device;
  e->callback = MakeCallback(h, device, nullptr);
  Status s = Engine::Get().EnqueueJoin(e, process_set_id);
  if (!s.ok()) { g_handles.Release(h); ThrowIfError(s); }
  return h;
}

int DoBarrier(int process_set_id) {
  int h = g_handles.Allocate();
  auto e = std::make_shared<TensorTableEntry>();
  e->callback = MakeCallback(h, CPU_DEVICE_ID, nullptr);
  Status s = Engine::Get().EnqueueBarrier(e, process_set_id);
  if (!s.ok()) { g_handles.Release(h); ThrowIfError(s); }
  return h;
}

bool PollHandle(int h) {
  auto st = g_handles.Get(h);
  if (!st) throw std::invalid_argument("Handle " + std::to_string(h) + " was not created or has been cleared.");
  if (!g_handles.Done(st)) { Engine::Get().RequestFlush(); return false; }
  if (st->status.ok()) {
    for (auto* ev : st->events) {
      cudaError_t q = cudaEventQuery(ev->ev);
      if (q == cudaErrorNotReady) { cudaGetLastError(); return false; }
    }
  }
  return true;
}

// Returns last_joined_rank (join) or -1.
int WaitAndClear(int h) {
  auto st = g_handles.Get(h);
  if (!st) throw std::invalid_argument("Handle " + std::to_string(h) + " was not created or has been cleared.");
  if (!g_handles.Done(st)) {
    py::gil_scoped_release release;
    Engine::Get().BeginWait();
    g_handles.Wait(st);
    Engine::Get().EndWait();
  }
  Status status = st->status;
  for (auto* ev : st->events) {
    if (status.ok()) {
      // chain instead of block: the caller's current stream waits for the collective
      cudaStream_t cur = c10::cuda::getCurrentCUDAStream(ev->device);
      cudaStreamWaitEvent(cur, ev->ev, 0);
    }
    GpuContext::Get().Release(ev);
  }
  st->events.clear();
  if (st->received_splits_out.defined() && !st->received_splits.empty()) {
    at::Tensor cpu = at::from_blob(st->received_splits.data(), {(int64_t)st->received_splits.size()}, at::kInt).clone();
    st->received_splits_out.resize_({(int64_t)st->received_splits.size()});
    st->received_splits_out.copy_(cpu);
  }
  int joined = st->last_joined_rank;
  g_handles.Release(h);
  ThrowIfError(status);
  return joined;
}

void Reset() {
  g_handles.Reset();
  std::lock_guard<std::mutex> l(g_noname_mu);
  g_noname_counters.clear();
}

// ---- registered symmetric memory -------------------------------------------------------------
// Collective: returns a uint8 CUDA tensor of `nbytes` that lives in peer-mapped memory. In-place allreduces on (views
// of) it skip the fusion-buffer pack/unpack and run the zero-copy NVLink kernel. The memory stays valid until
// hvd.shutdown().
at::Tensor SymmEmpty(int64_t nbytes, int device, int process_set_id) {
  TORCH_CHECK(nbytes > 0, "symm_empty: size must be positive");
  std::string err;
  void* p = nullptr;
  std::shared_ptr<void> keep;
  {
    py::gil_scoped_release release;
    p = Engine::Get().AllocSymmetric((size_t)nbytes, device, process_set_id, &err, &keep);
  }
  if (!p) throw std::runtime_error("symm_empty failed: " + err);
  auto opts = at::TensorOptions().dtype(at::kByte).device(at::kCUDA, device);
  // the tensor co-owns the team's mappings: it stays valid memory after hvd.shutdown() / an elastic reset (it then simply
  // is no longer registered with the new team and takes the packed path)
  return at::from_blob(p, {nbytes}, [keep](void*) mutable { keep.reset(); }, opts);
}

// In-place allreduce of a tensor that lives in registered symmetric memory, launched as ONE kernel on the current CUDA
// stream of the calling thread — which may be capturing into a CUDA graph.  No handle, no negotiation, no host
// synchronisation: ordering is the stream's.  reduce_op follows hvd.ReduceOp (0 Average, 1 Sum, 3 Min, 4 Max, 5 Product).
// `channel`: the barrier channel, kGraphChannel for the public hvd.captured_* functions, kSyncBnChannel for
// hvd.SyncBatchNorm, whose collectives can be resident together with graph-channel ones.
void CheckCapturedChannel(const char* op, int channel) {
  TORCH_CHECK(channel == kern::kGraphChannel || channel == kern::kSyncBnChannel, op, ": channel must be ",
              kern::kGraphChannel, " or ", kern::kSyncBnChannel, ", got ", channel);
}

void CapturedAllreduce(at::Tensor tensor, int reduce_op, double prescale, double postscale, int process_set_id, int max_ctas,
                       int channel) {
  CheckCapturedChannel("captured_allreduce_", channel);
  TORCH_CHECK(tensor.is_cuda(), "captured_allreduce_: CUDA tensor expected");
  TORCH_CHECK(tensor.is_non_overlapping_and_dense(), "captured_allreduce_: tensor must be dense");
  c10::cuda::CUDAGuard guard(tensor.device());
  cudaStream_t stream = c10::cuda::getCurrentCUDAStream(tensor.get_device());
  const int64_t bytes = (int64_t)tensor.numel() * (int64_t)tensor.element_size();
  ThrowIfError(Engine::Get().CapturedAllreduce(tensor.data_ptr(), bytes, MapDtype(tensor.scalar_type()), (ReduceOp)reduce_op, prescale,
                                               postscale, process_set_id, max_ctas, (void*)stream, channel));
}

// The two halves of a sharded optimizer step on a registered tensor, launched like CapturedAllreduce.  Rank r owns the
// contiguous slice [r*S, (r+1)*S) of the tensor's bytes, S = bytes / set size.
void CapturedReducescatter(at::Tensor tensor, int reduce_op, double prescale, double postscale, int process_set_id, int max_ctas) {
  TORCH_CHECK(tensor.is_cuda(), "captured_reducescatter_: CUDA tensor expected");
  TORCH_CHECK(tensor.is_non_overlapping_and_dense(), "captured_reducescatter_: tensor must be dense");
  c10::cuda::CUDAGuard guard(tensor.device());
  cudaStream_t stream = c10::cuda::getCurrentCUDAStream(tensor.get_device());
  const int64_t bytes = (int64_t)tensor.numel() * (int64_t)tensor.element_size();
  ThrowIfError(Engine::Get().CapturedReducescatter(tensor.data_ptr(), bytes, MapDtype(tensor.scalar_type()), (ReduceOp)reduce_op,
                                                   prescale, postscale, process_set_id, max_ctas, (void*)stream));
}

void CapturedAllgather(at::Tensor tensor, int process_set_id, int max_ctas, int channel) {
  CheckCapturedChannel("captured_allgather_", channel);
  TORCH_CHECK(tensor.is_cuda(), "captured_allgather_: CUDA tensor expected");
  TORCH_CHECK(tensor.is_non_overlapping_and_dense(), "captured_allgather_: tensor must be dense");
  c10::cuda::CUDAGuard guard(tensor.device());
  cudaStream_t stream = c10::cuda::getCurrentCUDAStream(tensor.get_device());
  const int64_t bytes = (int64_t)tensor.numel() * (int64_t)tensor.element_size();
  ThrowIfError(Engine::Get().CapturedAllgather(tensor.data_ptr(), bytes, process_set_id, max_ctas, (void*)stream, channel));
}

// Alltoall of the rows (dim 0) of a registered tensor with splits that only the device reads, launched like
// CapturedAllreduce.  The outputs are allocated on the current stream (from the graph's pool under capture):
// output [capacity, *row] in the tensor's dtype, recv_splits int64 [n] and status int32 [1] (kern::AlltoallStatus).
std::tuple<at::Tensor, at::Tensor, at::Tensor> CapturedAlltoall(at::Tensor tensor, at::Tensor splits, int64_t capacity,
                                                                int process_set_id, int max_ctas) {
  const char* op = "captured_alltoall";
  TORCH_CHECK(tensor.is_cuda(), op, ": CUDA tensor expected");
  TORCH_CHECK(tensor.dim() >= 1, op, ": tensor must have at least one dimension (its rows)");
  TORCH_CHECK(tensor.is_contiguous(), op, ": tensor must be contiguous");
  TORCH_CHECK(splits.is_cuda() && splits.device() == tensor.device(), op, ": splits must be on the tensor's device ", tensor.device(),
              ", got ", splits.device());
  TORCH_CHECK(splits.scalar_type() == at::kInt || splits.scalar_type() == at::kLong, op, ": splits must be int32 or int64, got ",
              splits.scalar_type());
  TORCH_CHECK(splits.dim() == 1 && splits.is_contiguous(), op, ": splits must be a contiguous 1-D tensor, got sizes ", splits.sizes());
  TORCH_CHECK(capacity >= 0, op, ": capacity must be >= 0, got ", capacity);
  c10::cuda::CUDAGuard guard(tensor.device());
  cudaStream_t stream = c10::cuda::getCurrentCUDAStream(tensor.get_device());
  const int64_t rows = tensor.size(0);
  const int64_t row_bytes = c10::multiply_integers(tensor.sizes().slice(1)) * (int64_t)tensor.element_size();
  std::vector<int64_t> out_sizes = tensor.sizes().vec();
  out_sizes[0] = capacity;
  at::Tensor out = at::empty(out_sizes, tensor.options());
  at::Tensor recv = at::empty({splits.numel()}, tensor.options().dtype(at::kLong));
  at::Tensor status = at::empty({1}, tensor.options().dtype(at::kInt));
  ThrowIfError(Engine::Get().CapturedAlltoall(tensor.data_ptr(), rows, row_bytes, splits.data_ptr(), splits.numel(),
                                              splits.scalar_type() == at::kLong, out.data_ptr(), capacity,
                                              recv.data_ptr<int64_t>(), status.data_ptr<int>(), process_set_id, max_ctas,
                                              (void*)stream));
  return {out, recv, status};
}

// ---- fused optimizer kernels (an extra of this library; see kernels/optim_kernels.cu) --------------
// The kernels address every tensor of entry i with the element index of params[i] and take one element type per list, so
// each companion tensor must have the param's sizes and strides, one dtype per list, and live on the param's device.
// Checked here, before anything is staged: a mismatch would otherwise become an out-of-bounds access or silent garbage.
void CheckOptimizerPeer(const char* op, const char* what, size_t i, const at::Tensor& param, const at::Tensor& t,
                        at::ScalarType dtype) {
  TORCH_CHECK(t.device() == param.device(), op, ": ", what, "[", i, "] is on ", t.device(), ", params[", i, "] on ",
              param.device());
  TORCH_CHECK(t.scalar_type() == dtype, op, ": ", what, "[", i, "] is ", t.scalar_type(), ", expected ", dtype);
  TORCH_CHECK(t.sizes() == param.sizes(), op, ": ", what, "[", i, "] has size ", t.sizes(), ", params[", i, "] has ",
              param.sizes());
  TORCH_CHECK(t.strides() == param.strides(), op, ": ", what, "[", i, "] has strides ", t.strides(), ", params[", i,
              "] has ", param.strides());
}

void CheckOptimizerParam(const char* op, size_t i, const at::Tensor& param, const at::Tensor& first) {
  TORCH_CHECK(param.is_cuda() && param.is_non_overlapping_and_dense(), op, ": params[", i, "] must be a dense CUDA tensor");
  TORCH_CHECK(param.device() == first.device(), op, ": params[", i, "] is on ", param.device(), ", params[0] on ",
              first.device());
  TORCH_CHECK(param.scalar_type() == first.scalar_type(), op, ": params[", i, "] is ", param.scalar_type(),
              ", params[0] is ", first.scalar_type(), " (one dtype per call)");
}

// A device-side scalar the kernels read: one fp32 element on the params' device (nullptr when absent).
const float* DeviceScalar(const char* op, const char* what, const c10::optional<at::Tensor>& t, const at::Tensor& param) {
  if (!t.has_value() || !t->defined()) return nullptr;
  TORCH_CHECK(t->is_cuda() && t->device() == param.device(), op, ": ", what, " must be on ", param.device(), ", got ", t->device());
  TORCH_CHECK(t->scalar_type() == at::kFloat, op, ": ", what, " must be float32, got ", t->scalar_type());
  TORCH_CHECK(t->numel() == 1, op, ": ", what, " must have one element, got ", t->numel());
  return t->data_ptr<float>();
}

// fp32 master weights (optional, empty: none): one fp32 tensor per param with its sizes, strides and device.  Only for
// bf16 / fp16 params with gradients of the same dtype, the pairs the master kernels are instantiated for.  Call after
// the params themselves are checked.  Returns whether masters are in use.
bool CheckMasters(const char* op, const std::vector<at::Tensor>& params, const std::vector<at::Tensor>& grads,
                  const std::vector<at::Tensor>& masters) {
  if (masters.empty()) return false;
  const auto pt = params[0].scalar_type();
  TORCH_CHECK(pt == at::kBFloat16 || pt == at::kHalf, op, ": master_params are for bfloat16 / float16 params, params are ", pt);
  TORCH_CHECK(grads[0].scalar_type() == pt, op, ": with master_params the grads must be ", pt, ", got ", grads[0].scalar_type());
  for (size_t i = 0; i < params.size(); ++i) CheckOptimizerPeer(op, "master_params", i, params[i], masters[i], at::kFloat);
  return true;
}

// One state list of an optimizer call and the table field it fills.  States are fp32, except a list marked
// `param_dtype` (SGD momentum), which has the param's dtype without masters.
struct OptState {
  const char* name;
  const std::vector<at::Tensor>& list;
  void* kern::OptTensor::*field;
  bool param_dtype = false;
};

// A checked call of the kern::Launch* optimizer launchers: the table, its dtypes and what the launchers take besides.
struct OptPlan {
  std::vector<kern::OptTensor> table;
  int64_t max_count = 0, partials = 0;
  int param_dtype = 0, grad_dtype = 0;
  bool master = false;
  const float* grad_scale_dev = nullptr;
  kern::OptEma ema;
};

// The EMA of one optimizer call (optional, empty list: none): one fp32 tensor per param with its sizes, strides and
// device, updated after the parameter with weight = 1 - decay; `start` begins every one of them at the updated value.
struct EmaArgs {
  const std::vector<at::Tensor>& list;
  double weight;
  bool start;
};
const std::vector<at::Tensor> kNoTensors;
const EmaArgs kNoEma{kNoTensors, 0.0, false};

// Checks every argument of one optimizer call and builds its table; nothing is staged or launched here.  Entry i is
// params[i] with grads[i], masters[i] and each state list's element in its field.  `norms` (LAMB and LARS; nullptr:
// none) is a contiguous fp32 tensor on the params' device with 2 floats per slot: entry i gets norm slot slots[i]
// (empty: i) and the offset of its stage-1 partials.  Zero-size params get no entry.
OptPlan PlanOpt(const char* op, const std::vector<at::Tensor>& params, const std::vector<at::Tensor>& grads,
                const std::vector<OptState>& states, const std::vector<at::Tensor>& masters,
                const c10::optional<at::Tensor>& grad_scale_dev, const at::Tensor* norms = nullptr,
                const std::vector<int64_t>& slots = {}, const EmaArgs& ema = kNoEma) {
  bool sizes = params.size() == grads.size();
  for (const auto& st : states) sizes = sizes && st.list.size() == params.size();
  TORCH_CHECK(sizes, op, ": list sizes differ");
  TORCH_CHECK(masters.empty() || masters.size() == params.size(), op, ": ", masters.size(), " master params for ",
              params.size(), " params");
  TORCH_CHECK(slots.empty() || slots.size() == params.size(), op, ": ", slots.size(), " slots for ", params.size(), " params");
  TORCH_CHECK(ema.list.empty() || ema.list.size() == params.size(), op, ": ", ema.list.size(), " ema params for ",
              params.size(), " params");
  OptPlan plan;
  if (params.empty()) return plan;
  for (size_t i = 0; i < params.size(); ++i) {
    CheckOptimizerParam(op, i, params[i], params[0]);
    CheckOptimizerPeer(op, "grads", i, params[i], grads[i], grads[0].scalar_type());
  }
  plan.master = CheckMasters(op, params, grads, masters);
  for (size_t i = 0; i < ema.list.size(); ++i) CheckOptimizerPeer(op, "ema_params", i, params[i], ema.list[i], at::kFloat);
  plan.ema = kern::OptEma{!ema.list.empty(), (float)ema.weight, ema.start ? 1 : 0};
  for (const auto& st : states)
    for (size_t i = 0; i < params.size(); ++i)
      CheckOptimizerPeer(op, st.name, i, params[i], st.list[i],
                         st.param_dtype && !plan.master ? params[i].scalar_type() : at::kFloat);
  if (norms != nullptr) {
    TORCH_CHECK(norms->is_cuda() && norms->device() == params[0].device() && norms->scalar_type() == at::kFloat &&
                norms->is_contiguous(), op, ": norms must be a contiguous float32 tensor on ", params[0].device());
    const int64_t nslots = norms->numel() / 2;
    std::set<int64_t> seen;
    for (size_t i = 0; i < params.size(); ++i) {
      const int64_t s = slots.empty() ? (int64_t)i : slots[i];
      TORCH_CHECK(s >= 0 && s < nslots, op, ": slot ", s, " of params[", i, "] is out of range for norms with room for ",
                  nslots, " slots");
      TORCH_CHECK(seen.insert(s).second, op, ": slot ", s, " appears twice in one call");
    }
  }
  plan.grad_scale_dev = DeviceScalar(op, "grad_scale_dev", grad_scale_dev, params[0]);
  plan.param_dtype = (int)MapDtype(params[0].scalar_type());
  plan.grad_dtype = (int)MapDtype(grads[0].scalar_type());
  for (size_t i = 0; i < params.size(); ++i) {
    if (params[i].numel() == 0) continue;
    kern::OptTensor t{};
    t.param = params[i].data_ptr(); t.grad = grads[i].data_ptr();
    t.master = plan.master ? masters[i].data_ptr() : nullptr;
    t.ema = plan.ema.on ? ema.list[i].data_ptr() : nullptr;
    for (const auto& st : states) t.*st.field = st.list[i].data_ptr();
    t.count = params[i].numel();
    if (norms != nullptr) {
      t.partial = plan.partials;
      t.slot = slots.empty() ? (int64_t)i : slots[i];
      plan.partials += kern::NormPartials(t.count);
    }
    plan.max_count = std::max(plan.max_count, t.count);
    plan.table.push_back(t);
  }
  return plan;
}

// The optimizer kernels select the table entry with blockIdx.y, which CUDA caps at 65535.  A piece of that many entries
// (72 B each) also fits the 8 MiB staging ring of GpuContext::Stage.
constexpr size_t kOptMaxEntries = 65535;

// One launch's share of a plan's table: `n` entries staged on the device and the longest of their counts.
struct OptPiece {
  const kern::OptTensor* table;
  int n;
  int64_t max_count;
};

// Stages the plan's table on the params' device in pieces of at most kOptMaxEntries entries (one piece, so one launch
// per phase, when the table fits) and runs launch(piece, current stream) for each, which makes one or more kern::Launch*
// calls and returns the first error.  Every entry keeps its norm slot and partial offset, so the LAMB / LARS phases run
// piece by piece unchanged.
template <typename F>
void RunPlan(const char* op, const OptPlan& plan, const std::vector<at::Tensor>& params, F&& launch) {
  if (plan.table.empty()) return;
  const int device = (int)params[0].get_device();
  c10::cuda::CUDAGuard guard(params[0].device());
  cudaStream_t s = c10::cuda::getCurrentCUDAStream(device);
  for (size_t lo = 0; lo < plan.table.size(); lo += kOptMaxEntries) {
    const size_t n = std::min(kOptMaxEntries, plan.table.size() - lo);
    int64_t max_count = 0;
    for (size_t i = lo; i < lo + n; ++i) max_count = std::max(max_count, plan.table[i].count);
    const auto* dt = (const kern::OptTensor*)GpuContext::Get().Stage(device, plan.table.data() + lo,
                                                                      n * sizeof(kern::OptTensor), s);
    TORCH_CHECK(dt != nullptr, op, ": table too large");
    const cudaError_t e = launch(OptPiece{dt, (int)n, max_count}, s);
    TORCH_CHECK(e == cudaSuccess, op, " launch failed: ", cudaGetErrorString(e));
  }
}

std::vector<OptState> MomentStates(const std::vector<at::Tensor>& exp_avg, const std::vector<at::Tensor>& exp_avg_sq) {
  return {{"exp_avgs", exp_avg, &kern::OptTensor::state0}, {"exp_avg_sqs", exp_avg_sq, &kern::OptTensor::state1}};
}

// Adam's and LAMB's bias correction 1 - beta^step; step is 1-based: step 0 would make it 0 and every parameter inf / NaN
float BiasCorrection(const char* op, double beta, int64_t step) {
  TORCH_CHECK(step >= 1, op, ": step must be >= 1, got ", step);
  return 1.0f - (float)std::pow(beta, (double)step);
}

void FusedSgdStep(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> momenta, double lr,
                  double momentum, double dampening, double weight_decay, bool nesterov, double grad_scale, bool first_step,
                  c10::optional<at::Tensor> grad_scale_dev, std::vector<at::Tensor> masters, std::vector<at::Tensor> emas,
                  double ema_weight, bool ema_start) {
  const bool has_mom = momentum != 0.0;
  // without momentum the buffers are not read: none, or a list of the params' length
  TORCH_CHECK(has_mom || momenta.empty() || momenta.size() == params.size(),
              "fused_sgd: ", momenta.size(), " momentum buffers for ", params.size(), " params");
  std::vector<OptState> states;
  if (has_mom) states.push_back({"momentum_buffers", momenta, &kern::OptTensor::state0, true});
  const OptPlan plan = PlanOpt("fused_sgd", params, grads, states, masters, grad_scale_dev, nullptr, {},
                               EmaArgs{emas, ema_weight, ema_start});
  RunPlan("fused_sgd", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    return kern::LaunchFusedSgd(pc.table, pc.n, pc.max_count, (float)lr, (float)momentum, (float)dampening,
                                (float)weight_decay, nesterov ? 1 : 0, (float)grad_scale, first_step ? 1 : 0,
                                plan.param_dtype, plan.grad_dtype, s, plan.grad_scale_dev, plan.master, plan.ema);
  });
}

void FusedAdamStep(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> exp_avg,
                   std::vector<at::Tensor> exp_avg_sq, double lr, double beta1, double beta2, double eps, double weight_decay,
                   int64_t step, double grad_scale, bool adamw, c10::optional<at::Tensor> grad_scale_dev,
                   std::vector<at::Tensor> masters, std::vector<at::Tensor> emas, double ema_weight, bool ema_start) {
  const float c1 = BiasCorrection("fused_adam", beta1, step), c2 = BiasCorrection("fused_adam", beta2, step);
  const OptPlan plan = PlanOpt("fused_adam", params, grads, MomentStates(exp_avg, exp_avg_sq), masters, grad_scale_dev,
                               nullptr, {}, EmaArgs{emas, ema_weight, ema_start});
  RunPlan("fused_adam", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    return kern::LaunchFusedAdamW(pc.table, pc.n, pc.max_count, (float)lr, (float)beta1, (float)beta2,
                                  (float)eps, (float)weight_decay, c1, c2, (float)grad_scale, adamw ? 1 : 0,
                                  plan.param_dtype, plan.grad_dtype, s, plan.grad_scale_dev, plan.master, plan.ema);
  });
}

// ---- fused LAMB and LARS: a norms phase (two launches) and an apply phase (one launch) on one table with a norm slot
// per entry, so that the norms can be allreduced in between.

// stream-ordered scratch from torch's caching allocator: one pair of sums of squares per stage-1 CTA
at::Tensor NormsScratch(const OptPlan& plan, const at::Tensor& norms) { return at::empty({2 * plan.partials}, norms.options()); }

struct LambArgs { double beta1, beta2, eps, weight_decay; float c1, c2; };

LambArgs LambHyper(const char* op, double beta1, double beta2, double eps, double weight_decay, int64_t step,
                   bool bias_correction) {
  const float c1 = BiasCorrection(op, beta1, step), c2 = BiasCorrection(op, beta2, step);  // checks step in any case
  return bias_correction ? LambArgs{beta1, beta2, eps, weight_decay, c1, c2} : LambArgs{beta1, beta2, eps, weight_decay, 1.f, 1.f};
}

cudaError_t LambNormsPhase(const OptPlan& plan, const OptPiece& pc, const LambArgs& a, double grad_scale,
                           at::Tensor& norms, cudaStream_t s) {
  at::Tensor work = NormsScratch(plan, norms);
  return kern::LaunchLambNorms(pc.table, pc.n, pc.max_count, (float)a.beta1, (float)a.beta2, (float)a.eps,
                               (float)a.weight_decay, a.c1, a.c2, (float)grad_scale, plan.grad_scale_dev,
                               work.data_ptr<float>(), norms.data_ptr<float>(), plan.param_dtype, plan.grad_dtype,
                               plan.master, s);
}

cudaError_t LambApplyPhase(const OptPlan& plan, const OptPiece& pc, const LambArgs& a, double lr, bool adapt,
                           const at::Tensor& norms, cudaStream_t s) {
  return kern::LaunchLambApply(pc.table, pc.n, pc.max_count, (float)lr, (float)a.eps, (float)a.weight_decay,
                               a.c1, a.c2, adapt ? 1 : 0, norms.data_ptr<float>(), plan.param_dtype, plan.master, s,
                               plan.ema);
}

// Phase 1: moments, then the squared norms of every entry ADDED into norms[2 * slot], norms[2 * slot + 1].
void LambNorms(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> exp_avg,
               std::vector<at::Tensor> exp_avg_sq, double beta1, double beta2, double eps, double weight_decay, int64_t step,
               bool bias_correction, double grad_scale, c10::optional<at::Tensor> grad_scale_dev,
               std::vector<at::Tensor> masters, at::Tensor out, std::vector<int64_t> slots) {
  const LambArgs a = LambHyper("lamb_norms", beta1, beta2, eps, weight_decay, step, bias_correction);
  const OptPlan plan = PlanOpt("lamb_norms", params, grads, MomentStates(exp_avg, exp_avg_sq), masters, grad_scale_dev,
                               &out, slots);
  RunPlan("lamb_norms", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    return LambNormsPhase(plan, pc, a, grad_scale, out, s);
  });
}

// Phase 2: w -= lr * r * u with r from the (allreduced) norms.  `grads` are checked like phase 1's, not read.
void LambApply(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> exp_avg,
               std::vector<at::Tensor> exp_avg_sq, double lr, double beta1, double beta2, double eps, double weight_decay,
               int64_t step, bool bias_correction, bool adapt, std::vector<at::Tensor> masters, at::Tensor norms,
               std::vector<int64_t> slots, std::vector<at::Tensor> emas, double ema_weight, bool ema_start) {
  const LambArgs a = LambHyper("lamb_apply", beta1, beta2, eps, weight_decay, step, bias_correction);
  const OptPlan plan = PlanOpt("lamb_apply", params, grads, MomentStates(exp_avg, exp_avg_sq), masters, c10::nullopt,
                               &norms, slots, EmaArgs{emas, ema_weight, ema_start});
  RunPlan("lamb_apply", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    return LambApplyPhase(plan, pc, a, lr, adapt, norms, s);
  });
}

// A fresh norms buffer for both phases on one device (slot i = params[i]).
at::Tensor FreshNorms(const char* op, const std::vector<at::Tensor>& params) {
  TORCH_CHECK(params.empty() || params[0].is_cuda(), op, ": params[0] must be a dense CUDA tensor");
  return params.empty() ? at::Tensor() : at::zeros({2 * (int64_t)params.size()}, params[0].options().dtype(at::kFloat));
}

// Both phases: three launches per staged piece of the table (one piece up to 65535 entries).
void FusedLambStep(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> exp_avg,
                   std::vector<at::Tensor> exp_avg_sq, double lr, double beta1, double beta2, double eps, double weight_decay,
                   int64_t step, bool bias_correction, bool adapt, double grad_scale,
                   c10::optional<at::Tensor> grad_scale_dev, std::vector<at::Tensor> masters, std::vector<at::Tensor> emas,
                   double ema_weight, bool ema_start) {
  at::Tensor norms = FreshNorms("fused_lamb", params);
  const LambArgs a = LambHyper("fused_lamb", beta1, beta2, eps, weight_decay, step, bias_correction);
  const OptPlan plan = PlanOpt("fused_lamb", params, grads, MomentStates(exp_avg, exp_avg_sq), masters, grad_scale_dev,
                               &norms, {}, EmaArgs{emas, ema_weight, ema_start});
  RunPlan("fused_lamb", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    const cudaError_t e = LambNormsPhase(plan, pc, a, grad_scale, norms, s);
    return e != cudaSuccess ? e : LambApplyPhase(plan, pc, a, lr, adapt, norms, s);
  });
}

// LARS keeps one fp32 state, the momentum buffer.
std::vector<OptState> LarsStates(const std::vector<at::Tensor>& momentum_buffers) {
  return {{"momentum_buffers", momentum_buffers, &kern::OptTensor::state0}};
}

cudaError_t LarsNormsPhase(const OptPlan& plan, const OptPiece& pc, double grad_scale, at::Tensor& norms,
                           cudaStream_t s) {
  at::Tensor work = NormsScratch(plan, norms);
  return kern::LaunchLarsNorms(pc.table, pc.n, pc.max_count, (float)grad_scale, plan.grad_scale_dev,
                               work.data_ptr<float>(), norms.data_ptr<float>(), plan.param_dtype, plan.grad_dtype,
                               plan.master, s);
}

cudaError_t LarsApplyPhase(const OptPlan& plan, const OptPiece& pc, double lr, double momentum, double weight_decay,
                           double trust_coefficient, double eps, bool adapt, double grad_scale, const at::Tensor& norms,
                           cudaStream_t s) {
  return kern::LaunchLarsApply(pc.table, pc.n, pc.max_count, (float)lr, (float)momentum, (float)weight_decay,
                               (float)trust_coefficient, (float)eps, adapt ? 1 : 0, (float)grad_scale, plan.grad_scale_dev,
                               norms.data_ptr<float>(), plan.param_dtype, plan.grad_dtype, plan.master, s, plan.ema);
}

// LARS phase 1: the squared norms of every entry's parameter and scaled gradient ADDED into norms[2 * slot],
// norms[2 * slot + 1].  The momentum buffers are checked like phase 2's, not read.
void LarsNorms(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> momentum_buffers,
               double grad_scale, c10::optional<at::Tensor> grad_scale_dev, std::vector<at::Tensor> masters, at::Tensor out,
               std::vector<int64_t> slots) {
  const OptPlan plan = PlanOpt("lars_norms", params, grads, LarsStates(momentum_buffers), masters, grad_scale_dev, &out,
                               slots);
  RunPlan("lars_norms", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    return LarsNormsPhase(plan, pc, grad_scale, out, s);
  });
}

// LARS phase 2: momentum and parameter update with r from the (allreduced) norms; reads the gradient again, scaled the
// same way as in phase 1.
void LarsApply(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> momentum_buffers,
               double lr, double momentum, double weight_decay, double trust_coefficient, double eps, bool adapt,
               double grad_scale, c10::optional<at::Tensor> grad_scale_dev, std::vector<at::Tensor> masters,
               at::Tensor norms, std::vector<int64_t> slots, std::vector<at::Tensor> emas, double ema_weight,
               bool ema_start) {
  const OptPlan plan = PlanOpt("lars_apply", params, grads, LarsStates(momentum_buffers), masters, grad_scale_dev, &norms,
                               slots, EmaArgs{emas, ema_weight, ema_start});
  RunPlan("lars_apply", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    return LarsApplyPhase(plan, pc, lr, momentum, weight_decay, trust_coefficient, eps, adapt, grad_scale, norms, s);
  });
}

// Both LARS phases: three launches per staged piece of the table (one piece up to 65535 entries).
void FusedLarsStep(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> momentum_buffers,
                   double lr, double momentum, double weight_decay, double trust_coefficient, double eps, bool adapt,
                   double grad_scale, c10::optional<at::Tensor> grad_scale_dev, std::vector<at::Tensor> masters,
                   std::vector<at::Tensor> emas, double ema_weight, bool ema_start) {
  at::Tensor norms = FreshNorms("fused_lars", params);
  const OptPlan plan = PlanOpt("fused_lars", params, grads, LarsStates(momentum_buffers), masters, grad_scale_dev, &norms,
                               {}, EmaArgs{emas, ema_weight, ema_start});
  RunPlan("fused_lars", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    const cudaError_t e = LarsNormsPhase(plan, pc, grad_scale, norms, s);
    return e != cudaSuccess ? e : LarsApplyPhase(plan, pc, lr, momentum, weight_decay, trust_coefficient, eps, adapt,
                                                 grad_scale, norms, s);
  });
}

// ---- fused Adafactor: the OptTensor table of PlanOpt (variance of dim <= 1 params in state0, one norm slot per param)
// plus a geometry table parallel to it for the factored params.  Both tables and all scratch live in tensors of torch's
// caching allocator on the current stream, and the tables reach the device through kernel parameters, so the call can
// be captured into a CUDA graph.

// Checks that `f` is params[i]'s row (`dim` = -1) or column (`dim` = -2) factor: fp32, contiguous, on its device, with
// its sizes except 1 at `dim`.
void CheckAdafactorFactor(const char* op, const char* what, size_t i, const at::Tensor& param,
                          const c10::optional<at::Tensor>& f, int64_t dim) {
  TORCH_CHECK(f.has_value() && f->defined(), op, ": ", what, "[", i, "] is missing for params[", i, "] of dim ", param.dim());
  TORCH_CHECK(f->device() == param.device(), op, ": ", what, "[", i, "] is on ", f->device(), ", params[", i, "] on ",
              param.device());
  TORCH_CHECK(f->scalar_type() == at::kFloat, op, ": ", what, "[", i, "] is ", f->scalar_type(), ", expected Float");
  std::vector<int64_t> want = param.sizes().vec();
  want[want.size() + dim] = 1;
  TORCH_CHECK(f->sizes() == at::IntArrayRef(want), op, ": ", what, "[", i, "] has size ", f->sizes(), ", expected ",
              at::IntArrayRef(want));
  TORCH_CHECK(f->is_contiguous(), op, ": ", what, "[", i, "] must be contiguous");
}

void FusedAdafactorStep(std::vector<at::Tensor> params, std::vector<at::Tensor> grads,
                        std::vector<c10::optional<at::Tensor>> row_vars, std::vector<c10::optional<at::Tensor>> col_vars,
                        std::vector<c10::optional<at::Tensor>> variances, double lr, double beta2_decay, double eps1,
                        double eps2, double d, double weight_decay, int64_t step, double grad_scale,
                        c10::optional<at::Tensor> grad_scale_dev, std::vector<at::Tensor> masters,
                        std::vector<at::Tensor> emas, double ema_weight, bool ema_start) {
  const char* op = "fused_adafactor";
  TORCH_CHECK(row_vars.size() == params.size() && col_vars.size() == params.size() && variances.size() == params.size(),
              op, ": list sizes differ");
  TORCH_CHECK(step >= 1, op, ": step must be >= 1, got ", step);
  TORCH_CHECK(eps1 >= 0.0 && d > 0.0, op, ": eps1 must be >= 0 and d > 0, got eps1 = ", eps1, ", d = ", d);
  if (params.empty()) return;
  // the kernels address a parameter's elements with 32-bit unsigned offsets, and the geometry of a factored parameter
  // holds its sizes and strides as int32
  for (size_t i = 0; i < params.size(); ++i) {
    const at::Tensor& p = params[i];
    TORCH_CHECK(p.numel() < ((int64_t)1 << 32), op, ": params[", i, "] has ", p.numel(),
                " elements, at most 2^32 - 1 are supported");
    if (p.dim() < 2) continue;
    for (int64_t k = 0; k < p.dim(); ++k)
      TORCH_CHECK(p.size(k) < ((int64_t)1 << 31) && (p.size(k) == 1 || p.stride(k) < ((int64_t)1 << 31)), op,
                  ": params[", i, "] has size ", p.size(k), " and stride ", p.stride(k), " in dim ", k,
                  ", at most 2^31 - 1 are supported in each dim of a factored parameter");
  }
  // not zeroed yet: nothing is launched before every argument is checked
  at::Tensor norms = at::empty({2 * (int64_t)params.size()}, params[0].options().dtype(at::kFloat));
  OptPlan plan = PlanOpt(op, params, grads, {}, masters, grad_scale_dev, &norms, {}, EmaArgs{emas, ema_weight, ema_start});
  for (size_t i = 0; i < params.size(); ++i) {
    const at::Tensor& p = params[i];
    TORCH_CHECK(p.dim() <= kern::kAdafactorMaxDims, op, ": params[", i, "] has ", p.dim(), " dims, at most ",
                kern::kAdafactorMaxDims, " are supported");
    if (p.dim() >= 2) {
      CheckAdafactorFactor(op, "row_vars", i, p, row_vars[i], -1);
      CheckAdafactorFactor(op, "col_vars", i, p, col_vars[i], -2);
      TORCH_CHECK(!(variances[i].has_value() && variances[i]->defined()), op, ": variances[", i,
                  "] is given for params[", i, "] of dim ", p.dim(), ", which keeps row / column factors");
    } else {
      TORCH_CHECK(!(row_vars[i].has_value() && row_vars[i]->defined()) && !(col_vars[i].has_value() && col_vars[i]->defined()),
                  op, ": row_vars[", i, "] / col_vars[", i, "] are given for params[", i, "] of dim ", p.dim(),
                  ", which keeps a variance");
      TORCH_CHECK(variances[i].has_value() && variances[i]->defined(), op, ": variances[", i, "] is missing for params[",
                  i, "] of dim ", p.dim());
      CheckOptimizerPeer(op, "variances", i, p, *variances[i], at::kFloat);
    }
  }
  // the geometry of every table entry (PlanOpt gives zero-size params no entry) and the scratch offsets
  std::vector<kern::AdafactorGeom> geom;
  int64_t colparts = 0, batches = 0, stats_ctas = 1, factor_ctas = 1;
  for (size_t i = 0, e = 0; i < params.size(); ++i) {
    const at::Tensor& p = params[i];
    if (p.numel() == 0) continue;
    kern::AdafactorGeom g{};
    for (int k = 0; k < kern::kAdafactorMaxDims; ++k) { g.size[k] = 1; g.stride[k] = 1; }
    if (p.dim() >= 2) {
      for (int64_t k = 0; k < p.dim(); ++k) {
        const int slot = kern::kAdafactorMaxDims - (int)p.dim() + (int)k;
        g.size[slot] = (int32_t)p.size(k);
        g.stride[slot] = p.size(k) == 1 ? 1 : (int32_t)p.stride(k);
      }
      g.row_var = row_vars[i]->data_ptr<float>();
      g.col_var = col_vars[i]->data_ptr<float>();
      const int64_t B = (int64_t)g.size[0] * g.size[1] * g.size[2], R = g.size[3], C = g.size[4];
      g.col_off = colparts;
      g.batch_off = batches;
      colparts += B * C * kern::AdafactorRowChunks(R);
      batches += B;
      stats_ctas = std::max(stats_ctas, kern::AdafactorStatsCtas(B, R, C));
      factor_ctas = std::max(factor_ctas, kern::AdafactorFactorCtas(B, C));
    } else {
      plan.table[e].state0 = variances[i]->data_ptr();
    }
    geom.push_back(g);
    ++e;
  }
  if (plan.table.empty()) return;
  TORCH_CHECK(plan.table.size() <= 65535, op, ": at most 65535 non-empty params per call, got ", plan.table.size());
  kern::AdafactorHyper h;
  const double t = (double)step;
  h.beta_w = (float)std::pow(t, beta2_decay);
  h.rho = (float)std::min(lr, 1.0 / std::sqrt(t));
  h.eps1 = (float)eps1;
  h.eps1_sq = (float)(eps1 * eps1);
  h.eps2 = (float)eps2;
  h.d = (float)d;
  h.decay = (float)(1.0 - lr * weight_decay);
  const size_t tab_bytes = plan.table.size() * sizeof(kern::OptTensor);
  const size_t geom_at = (tab_bytes + 255) / 256 * 256, bytes = geom_at + geom.size() * sizeof(kern::AdafactorGeom);
  std::vector<unsigned char> host(bytes);
  memcpy(host.data(), plan.table.data(), tab_bytes);
  memcpy(host.data() + geom_at, geom.data(), geom.size() * sizeof(kern::AdafactorGeom));
  c10::cuda::CUDAGuard guard(params[0].device());
  cudaStream_t s = c10::cuda::getCurrentCUDAStream(params[0].get_device());
  at::Tensor tables = at::empty({(int64_t)bytes}, params[0].options().dtype(at::kByte));
  at::Tensor work = at::empty({colparts + batches + 2 * plan.partials}, norms.options());
  norms.zero_();
  float* w = work.data_ptr<float>();
  cudaError_t e = kern::LaunchUploadBytes(tables.data_ptr(), host.data(), bytes, s);
  if (e == cudaSuccess) {
    const auto* dt = reinterpret_cast<const kern::OptTensor*>(tables.data_ptr<uint8_t>());
    const auto* dg = reinterpret_cast<const kern::AdafactorGeom*>(tables.data_ptr<uint8_t>() + geom_at);
    // the float2 CTA partials first, where the allocator's alignment holds; then the column partials and batch means
    float* part = w;
    float* cols = part + 2 * plan.partials;
    e = kern::LaunchAdafactor(dt, dg, (int)plan.table.size(), plan.max_count, stats_ctas, factor_ctas, h,
                              (float)grad_scale, plan.grad_scale_dev, cols, cols + colparts, part,
                              norms.data_ptr<float>(), plan.param_dtype, plan.grad_dtype, plan.master, s, plan.ema);
  }
  TORCH_CHECK(e == cudaSuccess, op, " launch failed: ", cudaGetErrorString(e));
}

// The stats kernel's last-CTA ticket: one zeroed counter per (device, stream), which every launch leaves zeroed again.
// Launches on one stream run one after the other, so they can share it; launches on different streams may overlap and
// must not.  Kept for the life of the process (4 bytes per stream that ever ran the kernel).
unsigned* StatsTicket(int device, cudaStream_t s) {
  static std::mutex mu;
  static std::map<std::pair<int, cudaStream_t>, unsigned*> tickets;
  std::lock_guard<std::mutex> l(mu);
  unsigned*& t = tickets[{device, s}];
  if (!t) {
    void* p = nullptr;
    TORCH_CHECK(cudaMalloc(&p, sizeof(unsigned)) == cudaSuccess, "grad_shard_stats: cannot allocate the ticket counter");
    TORCH_CHECK(cudaMemset(p, 0, sizeof(unsigned)) == cudaSuccess, "grad_shard_stats: cannot zero the ticket counter");
    t = static_cast<unsigned*>(p);
  }
  return t;
}

// One launch of the gradient statistics kernel over `grads` (one dtype: fp32 / bf16 / fp16), folded into out[0:2].
void GradShardStats(std::vector<at::Tensor> grads, at::Tensor out, c10::optional<at::Tensor> inv_scale, bool norm_inf) {
  TORCH_CHECK(out.is_cuda() && out.scalar_type() == at::kFloat && out.is_contiguous() && out.numel() >= 2,
              "grad_shard_stats: out must be a contiguous float32 CUDA tensor with at least 2 elements");
  for (size_t i = 0; i < grads.size(); ++i) {
    TORCH_CHECK(grads[i].is_cuda() && grads[i].is_non_overlapping_and_dense(), "grad_shard_stats: tensors[", i,
                "] must be a dense CUDA tensor");
    TORCH_CHECK(grads[i].device() == out.device(), "grad_shard_stats: tensors[", i, "] is on ", grads[i].device(),
                ", out on ", out.device());
    TORCH_CHECK(grads[i].scalar_type() == grads[0].scalar_type(), "grad_shard_stats: tensors[", i, "] is ",
                grads[i].scalar_type(), ", tensors[0] is ", grads[0].scalar_type(), " (one dtype per call)");
  }
  if (!grads.empty()) {
    const auto st = grads[0].scalar_type();
    TORCH_CHECK(st == at::kFloat || st == at::kBFloat16 || st == at::kHalf,
                "grad_shard_stats: gradients must be float32, bfloat16 or float16, got ", st);
  }
  const float* isc = DeviceScalar("grad_shard_stats", "inv_scale", inv_scale, out);
  std::vector<kern::StatTensor> table;
  int64_t tiles = 0, row_tiles = 0;  // one CTA per tile of every tensor
  for (auto& g : grads) {
    if (g.numel() == 0) continue;
    table.push_back({g.data_ptr(), g.numel(), tiles});
    const int64_t t = kern::GradShardStatsTiles(g.numel());
    tiles += t;
    row_tiles = std::max(row_tiles, t);
  }
  if (table.empty()) return;
  TORCH_CHECK(tiles <= 0x7fffffff, "grad_shard_stats: ", tiles, " tiles exceed one launch's grid");
  int device = (int)out.get_device();
  c10::cuda::CUDAGuard guard(out.device());
  cudaStream_t s = c10::cuda::getCurrentCUDAStream(device);
  // stream-ordered scratch from torch's caching allocator: fp32 partials followed by int flags
  at::Tensor work = at::empty({2 * tiles}, out.options());
  const auto* dt = (const kern::StatTensor*)GpuContext::Get().Stage(device, table.data(), table.size() * sizeof(kern::StatTensor), s);
  TORCH_CHECK(dt != nullptr, "grad_shard_stats: table too large");
  cudaError_t e = kern::LaunchGradShardStats(dt, (int)table.size(), tiles, row_tiles, isc, norm_inf ? 1 : 0,
                                             work.data_ptr<float>(), reinterpret_cast<int*>(work.data_ptr<float>() + tiles),
                                             StatsTicket(device, s), out.data_ptr<float>(),
                                             (int)MapDtype(grads[0].scalar_type()), s);
  TORCH_CHECK(e == cudaSuccess, "grad_shard_stats launch failed: ", cudaGetErrorString(e));
}

// Fold bf16 / fp16 gradients into fp32 accumulators (kern::LaunchGradAccumulate): mode 0 first, 1 add, 2 last.  Every
// argument is checked before anything is launched; one launch per kAccMaxTensors non-empty entries, on the current stream,
// with the table as a kernel parameter, so the call can be captured into a CUDA graph.
void GradAccumulate(std::vector<at::Tensor> grads, std::vector<at::Tensor> accs, int64_t mode) {
  TORCH_CHECK(mode >= kern::kAccFirst && mode <= kern::kAccLast, "grad_accumulate: mode must be 0 (first), 1 (add) or 2 "
              "(last), got ", mode);
  TORCH_CHECK(grads.size() == accs.size(), "grad_accumulate: ", grads.size(), " gradients but ", accs.size(), " accumulators");
  if (grads.empty()) return;
  const auto st = grads[0].scalar_type();
  TORCH_CHECK(st == at::kBFloat16 || st == at::kHalf, "grad_accumulate: gradients must be bfloat16 or float16, got ", st);
  for (size_t i = 0; i < grads.size(); ++i) {
    const at::Tensor& g = grads[i];
    const at::Tensor& a = accs[i];
    TORCH_CHECK(g.is_cuda() && g.is_non_overlapping_and_dense(), "grad_accumulate: grads[", i, "] must be a dense CUDA tensor");
    TORCH_CHECK(g.scalar_type() == st, "grad_accumulate: grads[", i, "] is ", g.scalar_type(), ", grads[0] is ", st,
                " (one dtype per call)");
    TORCH_CHECK(a.is_cuda() && a.scalar_type() == at::kFloat, "grad_accumulate: accs[", i, "] must be a float32 CUDA tensor");
    TORCH_CHECK(a.device() == grads[0].device() && g.device() == grads[0].device(), "grad_accumulate: entry ", i,
                " is not on ", grads[0].device());
    TORCH_CHECK(a.sizes() == g.sizes() && a.strides() == g.strides(), "grad_accumulate: accs[", i,
                "] must have the shape and strides of grads[", i, "]");
  }
  std::vector<kern::AccTensor> entries;
  int64_t maxc = 0;
  for (size_t i = 0; i < grads.size(); ++i) {
    if (grads[i].numel() == 0) continue;
    entries.push_back({grads[i].data_ptr(), accs[i].data_ptr<float>(), grads[i].numel()});
  }
  if (entries.empty()) return;
  c10::cuda::CUDAGuard guard(grads[0].device());
  cudaStream_t s = c10::cuda::getCurrentCUDAStream(grads[0].get_device());
  for (size_t lo = 0; lo < entries.size(); lo += kern::kAccMaxTensors) {
    kern::AccTable table;
    table.n = (int)std::min<size_t>(kern::kAccMaxTensors, entries.size() - lo);
    maxc = 0;
    for (int k = 0; k < table.n; ++k) {
      table.t[k] = entries[lo + k];
      maxc = std::max(maxc, table.t[k].count);
    }
    cudaError_t e = kern::LaunchGradAccumulate(table, maxc, (int)mode, (int)MapDtype(st), s);
    TORCH_CHECK(e == cudaSuccess, "grad_accumulate launch failed: ", cudaGetErrorString(e));
  }
}

// ---- hvd.SyncBatchNorm kernels (see kernels/sync_bn_kernels.cu) ------------------------------------------------------
// Every argument is checked here, before anything is launched.

// The view of an input with channels at dim 1: rows [M, C] when, walking dims 1, d-1, ..., 2, 0, the strides are those of
// a packed array (channels_last, [N, C], spatial size 1; dims of size 1 do not matter), else planes [N, C, L] when it is
// contiguous.  Other layouts are the caller's to make contiguous.
kern::BnGeom BnView(const char* op, const at::Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.dim() >= 2 && x.size(1) > 0, op, ": x must be a CUDA tensor with at least 2 dimensions "
              "and at least one channel");
  const auto st = x.scalar_type();
  TORCH_CHECK(st == at::kFloat || st == at::kBFloat16 || st == at::kHalf, op, ": x must be float32, bfloat16 or float16, got ", st);
  const int64_t d = x.dim(), C = x.size(1);
  std::vector<int64_t> order {1};
  for (int64_t k = d - 1; k >= 2; --k) order.push_back(k);
  order.push_back(0);
  bool rows = true;
  int64_t expect = 1;
  for (int64_t k : order) {
    if (x.size(k) != 1 && x.stride(k) != expect) { rows = false; break; }
    expect *= x.size(k);
  }
  if (rows) return kern::BnGeom {kern::kBnRows, x.numel() / C, C, 1};
  TORCH_CHECK(x.is_contiguous(), op, ": x must be contiguous or channels-last (channels innermost), got strides ", x.strides());
  const int64_t N = x.size(0);
  return kern::BnGeom {kern::kBnPlanes, N, C, N > 0 ? x.numel() / (N * C) : 0};
}

// a per-channel vector: C contiguous elements on x's device, of one of `dtypes`
void CheckBnVec(const char* op, const char* what, const at::Tensor& t, int64_t C, const at::Tensor& x,
                std::initializer_list<at::ScalarType> dtypes) {
  TORCH_CHECK(t.is_cuda() && t.device() == x.device(), op, ": ", what, " must be on ", x.device(), ", got ", t.device());
  TORCH_CHECK(t.is_contiguous() && t.numel() == C, op, ": ", what, " must be contiguous with ", C, " elements, got sizes ",
              t.sizes());
  bool ok = false;
  for (auto d : dtypes) ok |= t.scalar_type() == d;
  TORCH_CHECK(ok, op, ": ", what, " has dtype ", t.scalar_type(), ", which is not allowed here");
}

// weight / bias: fp32 or x's dtype, both the same
int BnAffineDtype(const char* op, const c10::optional<at::Tensor>& w, const c10::optional<at::Tensor>& b, int64_t C,
                  const at::Tensor& x) {
  const at::Tensor* first = w ? &*w : (b ? &*b : nullptr);
  if (!first) return (int)MapDtype(at::kFloat);
  if (w) CheckBnVec(op, "weight", *w, C, x, {at::kFloat, x.scalar_type()});
  if (b) CheckBnVec(op, "bias", *b, C, x, {at::kFloat, x.scalar_type()});
  TORCH_CHECK(!(w && b) || w->scalar_type() == b->scalar_type(), op, ": weight and bias must have the same dtype");
  return (int)MapDtype(first->scalar_type());
}

// The stats kernels' last-CTA tickets: a zeroed int32 array per (device, stream), grown to the most channel tiles seen,
// which every launch leaves zeroed.  Launches on one stream run one after another and share it.  It comes from torch's
// allocator and is zeroed on the stream, so a stream first seen while it is being captured (hvd.GraphedStep captures on
// a stream of its own) gets its array from the graph's pool, zeroed by the graph.  Arrays are kept for the life of the
// process: a captured graph may still refer to them.
unsigned* BnTickets(int device, cudaStream_t s, int64_t n) {
  static std::mutex mu;
  static std::map<std::pair<int, cudaStream_t>, at::Tensor> tickets;
  static std::vector<at::Tensor> outgrown;
  std::lock_guard<std::mutex> l(mu);
  at::Tensor& t = tickets[{device, s}];
  if (!t.defined() || t.numel() < n) {
    if (t.defined()) outgrown.push_back(t);
    t = at::zeros({std::max<int64_t>(n, 1024)}, at::TensorOptions().dtype(at::kInt).device(at::kCUDA, device));
  }
  return reinterpret_cast<unsigned*>(t.data_ptr<int>());
}

void CheckBnSums(const char* op, const char* what, const at::Tensor& t, int64_t need, const at::Tensor& x) {
  TORCH_CHECK(t.is_cuda() && t.device() == x.device() && t.scalar_type() == at::kDouble && t.is_contiguous() &&
              t.numel() >= need, op, ": ", what, " must be a contiguous float64 tensor on ", x.device(), " with at least ",
              need, " elements");
}

// This rank's {count, mean, M2} of every channel of x, as fp64 triples, into slot[0 : 3C].
void SyncBnStats(at::Tensor x, at::Tensor slot) {
  const kern::BnGeom g = BnView("sync_bn_stats", x);
  CheckBnSums("sync_bn_stats", "slot", slot, 3 * g.C, x);
  c10::cuda::CUDAGuard guard(x.device());
  cudaStream_t s = c10::cuda::getCurrentCUDAStream(x.get_device());
  const int dt = (int)MapDtype(x.scalar_type());
  const kern::BnPlan plan = kern::BnReducePlan(g, dt);
  at::Tensor part = at::empty({plan.splits * g.C * 2}, x.options().dtype(at::kDouble));  // 16 B per partial
  cudaError_t e = kern::LaunchBnStats(x.data_ptr(), g, dt, part.data_ptr(), BnTickets(x.get_device(), s, plan.tiles),
                                      slot.data_ptr<double>(), s);
  TORCH_CHECK(e == cudaSuccess, "sync_bn_stats launch failed: ", cudaGetErrorString(e));
}

// Merges the slots (rows of `slots`, in rank order) of C channels: returns (mean, invstd, count) as float32 and updates
// the running statistics where given.
std::tuple<at::Tensor, at::Tensor, at::Tensor> SyncBnCombine(at::Tensor slots, int64_t C, double eps, double momentum,
                                                             c10::optional<at::Tensor> running_mean,
                                                             c10::optional<at::Tensor> running_var,
                                                             c10::optional<at::Tensor> num_batches_tracked) {
  const char* op = "sync_bn_combine";
  TORCH_CHECK(C > 0, op, ": C must be positive");
  TORCH_CHECK(slots.is_cuda() && slots.scalar_type() == at::kDouble && slots.is_contiguous() && slots.dim() == 2 &&
              slots.size(0) >= 1 && slots.size(0) <= kern::kMaxPeers && slots.size(1) >= 3 * C, op,
              ": slots must be a contiguous float64 CUDA tensor [nranks <= ", kern::kMaxPeers, ", >= 3 * C], got ",
              slots.scalar_type(), " ", slots.sizes());
  TORCH_CHECK(running_mean.has_value() == running_var.has_value(), op, ": running_mean and running_var go together");
  int sdt = (int)MapDtype(at::kFloat);
  if (running_mean) {
    for (const at::Tensor* t : {&*running_mean, &*running_var})
      CheckBnVec(op, t == &*running_mean ? "running_mean" : "running_var", *t, C, slots, {at::kFloat, at::kBFloat16, at::kHalf});
    TORCH_CHECK(running_mean->scalar_type() == running_var->scalar_type(), op, ": running stats must have one dtype");
    sdt = (int)MapDtype(running_mean->scalar_type());
  }
  if (num_batches_tracked)
    TORCH_CHECK(running_mean && num_batches_tracked->is_cuda() && num_batches_tracked->device() == slots.device() &&
                num_batches_tracked->scalar_type() == at::kLong && num_batches_tracked->numel() == 1, op,
                ": num_batches_tracked must be a one-element int64 tensor on ", slots.device(), ", with running stats");
  c10::cuda::CUDAGuard guard(slots.device());
  cudaStream_t s = c10::cuda::getCurrentCUDAStream(slots.get_device());
  at::Tensor mean = at::empty({C}, slots.options().dtype(at::kFloat)), invstd = at::empty_like(mean);
  at::Tensor count = at::empty({1}, mean.options());
  cudaError_t e = kern::LaunchBnCombine(slots.data_ptr<double>(), (int)slots.size(0), slots.size(1), C, eps, momentum,
                                        num_batches_tracked ? num_batches_tracked->data_ptr<int64_t>() : nullptr,
                                        mean.data_ptr<float>(), invstd.data_ptr<float>(), count.data_ptr<float>(),
                                        running_mean ? running_mean->data_ptr() : nullptr,
                                        running_var ? running_var->data_ptr() : nullptr, sdt, s);
  TORCH_CHECK(e == cudaSuccess, "sync_bn_combine launch failed: ", cudaGetErrorString(e));
  return {mean, invstd, count};
}

at::Tensor SyncBnElemt(at::Tensor x, at::Tensor mean, at::Tensor invstd, c10::optional<at::Tensor> weight,
                       c10::optional<at::Tensor> bias) {
  const char* op = "sync_bn_elemt";
  const kern::BnGeom g = BnView(op, x);
  CheckBnVec(op, "mean", mean, g.C, x, {at::kFloat});
  CheckBnVec(op, "invstd", invstd, g.C, x, {at::kFloat});
  const int wdt = BnAffineDtype(op, weight, bias, g.C, x);
  c10::cuda::CUDAGuard guard(x.device());
  cudaStream_t s = c10::cuda::getCurrentCUDAStream(x.get_device());
  at::Tensor y = at::empty_like(x);  // x is dense, so y gets its strides
  cudaError_t e = kern::LaunchBnElemt(x.data_ptr(), y.data_ptr(), g, (int)MapDtype(x.scalar_type()), mean.data_ptr<float>(),
                                      invstd.data_ptr<float>(), weight ? weight->data_ptr() : nullptr,
                                      bias ? bias->data_ptr() : nullptr, wdt, s);
  TORCH_CHECK(e == cudaSuccess, "sync_bn_elemt launch failed: ", cudaGetErrorString(e));
  return y;
}

void CheckBnGrad(const char* op, const at::Tensor& dy, const at::Tensor& x) {
  TORCH_CHECK(dy.device() == x.device() && dy.scalar_type() == x.scalar_type() && dy.sizes() == x.sizes() &&
              dy.strides() == x.strides(), op, ": grad_output must have x's device, dtype, sizes and strides");
}

// sums[2c] = sum dy, sums[2c+1] = sum dy * (x - mean) over this rank's batch; returns the local (grad_weight, grad_bias)
// in the weight's dtype where asked for (None otherwise).
std::tuple<at::Tensor, at::Tensor> SyncBnBackwardReduce(at::Tensor dy, at::Tensor x, at::Tensor mean, at::Tensor invstd,
                                                        c10::optional<at::Tensor> weight, at::Tensor sums,
                                                        bool need_weight_grad, bool need_bias_grad) {
  const char* op = "sync_bn_backward_reduce";
  const kern::BnGeom g = BnView(op, x);
  CheckBnGrad(op, dy, x);
  CheckBnVec(op, "mean", mean, g.C, x, {at::kFloat});
  CheckBnVec(op, "invstd", invstd, g.C, x, {at::kFloat});
  CheckBnSums(op, "sums", sums, 2 * g.C, x);
  const int wdt = BnAffineDtype(op, weight, c10::nullopt, g.C, x);
  const auto wopt = x.options().dtype(weight ? weight->scalar_type() : at::kFloat);
  at::Tensor gw = need_weight_grad ? at::empty({g.C}, wopt) : at::Tensor();
  at::Tensor gb = need_bias_grad ? at::empty({g.C}, wopt) : at::Tensor();
  c10::cuda::CUDAGuard guard(x.device());
  cudaStream_t s = c10::cuda::getCurrentCUDAStream(x.get_device());
  const int dt = (int)MapDtype(x.scalar_type());
  const kern::BnPlan plan = kern::BnReducePlan(g, dt);
  at::Tensor part = at::empty({plan.splits * g.C * 2}, x.options().dtype(at::kFloat));  // 8 B per partial
  cudaError_t e = kern::LaunchBnBackwardReduce(dy.data_ptr(), x.data_ptr(), g, dt, mean.data_ptr<float>(),
                                               invstd.data_ptr<float>(), part.data_ptr(),
                                               BnTickets(x.get_device(), s, plan.tiles), sums.data_ptr<double>(),
                                               gw.defined() ? gw.data_ptr() : nullptr, gb.defined() ? gb.data_ptr() : nullptr,
                                               wdt, s);
  TORCH_CHECK(e == cudaSuccess, "sync_bn_backward_reduce launch failed: ", cudaGetErrorString(e));
  return {gw, gb};
}

at::Tensor SyncBnBackwardElemt(at::Tensor dy, at::Tensor x, at::Tensor mean, at::Tensor invstd,
                               c10::optional<at::Tensor> weight, at::Tensor sums, at::Tensor count) {
  const char* op = "sync_bn_backward_elemt";
  const kern::BnGeom g = BnView(op, x);
  CheckBnGrad(op, dy, x);
  CheckBnVec(op, "mean", mean, g.C, x, {at::kFloat});
  CheckBnVec(op, "invstd", invstd, g.C, x, {at::kFloat});
  CheckBnSums(op, "sums", sums, 2 * g.C, x);
  CheckBnVec(op, "count", count, 1, x, {at::kFloat});
  const int wdt = BnAffineDtype(op, weight, c10::nullopt, g.C, x);
  c10::cuda::CUDAGuard guard(x.device());
  cudaStream_t s = c10::cuda::getCurrentCUDAStream(x.get_device());
  at::Tensor dx = at::empty_like(x);
  cudaError_t e = kern::LaunchBnBackwardElemt(dy.data_ptr(), x.data_ptr(), dx.data_ptr(), g, (int)MapDtype(x.scalar_type()),
                                              mean.data_ptr<float>(), invstd.data_ptr<float>(),
                                              weight ? weight->data_ptr() : nullptr, wdt, sums.data_ptr<double>(),
                                              count.data_ptr<float>(), s);
  TORCH_CHECK(e == cudaSuccess, "sync_bn_backward_elemt launch failed: ", cudaGetErrorString(e));
  return dx;
}

// ---- hvd.ExpertDispatcher kernels (see kernels/moe_kernels.cu) -------------------------------------------------------
// Every argument is checked here, before anything is launched.  Rows are the dim-1 slices of contiguous 2-D tensors of
// fp32 / bf16 / fp16; positions and row indices are int32, byte offsets int64.

// a contiguous [rows, h] tensor of `dtype` on `dev`
void CheckMoeRows(const char* op, const char* what, const at::Tensor& t, int64_t h, at::ScalarType dtype, const at::Device& dev) {
  TORCH_CHECK(t.is_cuda() && t.device() == dev, op, ": ", what, " must be on ", dev, ", got ", t.device());
  TORCH_CHECK(t.dim() == 2 && t.size(1) == h && t.is_contiguous(), op, ": ", what, " must be a contiguous [rows, ", h,
              "] tensor, got sizes ", t.sizes(), " and strides ", t.strides());
  TORCH_CHECK(t.scalar_type() == dtype, op, ": ", what, " must be ", dtype, ", got ", t.scalar_type());
  TORCH_CHECK(t.size(0) <= 0x7fffffff, op, ": ", what, " has ", t.size(0), " rows, more than int32 row indices reach");
}

at::ScalarType MoeDtype(const char* op, const at::Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.size(1) >= 1, op, ": rows must be a 2-D CUDA tensor [rows, hidden] with "
              "hidden >= 1, got sizes ", x.sizes());
  const auto st = x.scalar_type();
  TORCH_CHECK(st == at::kFloat || st == at::kBFloat16 || st == at::kHalf, op, ": rows must be float32, bfloat16 or float16, "
              "got ", st);
  return st;
}

void CheckMoePos(const char* op, const at::Tensor& pos, int64_t ntok, const at::Device& dev) {
  TORCH_CHECK(pos.is_cuda() && pos.device() == dev && pos.scalar_type() == at::kInt && pos.dim() == 2 && pos.is_contiguous(),
              op, ": pos must be a contiguous int32 [tokens, k] tensor on ", dev);
  TORCH_CHECK(pos.size(0) == ntok && pos.size(1) >= 1 && pos.size(1) <= kern::kMoeMaxTopK, op, ": pos must be [", ntok,
              ", k] with 1 <= k <= ", kern::kMoeMaxTopK, ", got sizes ", pos.sizes());
}

// gates: [tokens, k] contiguous, fp32 or the rows' dtype
const void* MoeGates(const char* op, const c10::optional<at::Tensor>& gates, const at::Tensor& pos, at::ScalarType dtype,
                     int* gate_dtype) {
  *gate_dtype = (int)MapDtype(at::kFloat);
  if (!gates) return nullptr;
  const at::Tensor& g = *gates;
  TORCH_CHECK(g.is_cuda() && g.device() == pos.device() && g.sizes() == pos.sizes() && g.is_contiguous(), op,
              ": gates must be a contiguous ", pos.sizes(), " tensor on ", pos.device());
  TORCH_CHECK(g.scalar_type() == at::kFloat || g.scalar_type() == dtype, op, ": gates must be float32 or ", dtype, ", got ",
              g.scalar_type());
  *gate_dtype = (int)MapDtype(g.scalar_type());
  return g.data_ptr();
}

const int* MoeStatus(const char* op, const c10::optional<at::Tensor>& status, const at::Device& dev) {
  if (!status) return nullptr;
  TORCH_CHECK(status->is_cuda() && status->device() == dev && status->scalar_type() == at::kInt && status->numel() == 1,
              op, ": status must be a one-element int32 tensor on ", dev);
  return status->data_ptr<int>();
}

// The stable order by expert of expert_idx [T, k] (int32 / int64), and the copy of every token's row x[t] to its k
// send-buffer rows.  counts: this rank's num_experts per-expert counts (int64, contiguous), written by the kernel.
// Returns (pos int32 [T, k], splits int32 [nranks]).
std::tuple<at::Tensor, at::Tensor> MoePermute(at::Tensor x, at::Tensor expert_idx, at::Tensor send, at::Tensor counts,
                                              int64_t num_experts, int64_t nranks, int64_t ctas) {
  const char* op = "moe_permute";
  const auto dt = MoeDtype(op, x);
  const at::Device dev = x.device();
  const int64_t T = x.size(0), h = x.size(1);
  CheckMoeRows(op, "x", x, h, dt, dev);
  CheckMoeRows(op, "send", send, h, dt, dev);
  TORCH_CHECK(num_experts >= 1 && num_experts <= kern::kMoeMaxExperts, op, ": num_experts must be in [1, ",
              kern::kMoeMaxExperts, "], got ", num_experts);
  TORCH_CHECK(nranks >= 1 && num_experts % nranks == 0, op, ": num_experts (", num_experts, ") must be a multiple of nranks (",
              nranks, ")");
  TORCH_CHECK(expert_idx.is_cuda() && expert_idx.device() == dev && expert_idx.dim() == 2 && expert_idx.is_contiguous() &&
              (expert_idx.scalar_type() == at::kInt || expert_idx.scalar_type() == at::kLong), op,
              ": expert_idx must be a contiguous int32 or int64 [tokens, k] tensor on ", dev);
  const int64_t k = expert_idx.size(1);
  TORCH_CHECK(expert_idx.size(0) == T && k >= 1 && k <= kern::kMoeMaxTopK, op, ": expert_idx must be [", T, ", k] with 1 <= k <= ",
              kern::kMoeMaxTopK, ", got sizes ", expert_idx.sizes());
  TORCH_CHECK(send.size(0) >= T * k, op, ": send holds ", send.size(0), " rows, fewer than the ", T * k, " assignments");
  TORCH_CHECK(counts.is_cuda() && counts.device() == dev && counts.scalar_type() == at::kLong && counts.is_contiguous() &&
              counts.numel() == num_experts, op, ": counts must be a contiguous int64 tensor of ", num_experts, " elements on ", dev);
  TORCH_CHECK(ctas >= 0, op, ": ctas must be >= 0");
  c10::cuda::CUDAGuard guard(dev);
  cudaStream_t s = c10::cuda::getCurrentCUDAStream(x.get_device());
  auto iopt = x.options().dtype(at::kInt);
  at::Tensor pos = at::empty({T, k}, iopt);
  at::Tensor splits = at::empty({nranks}, iopt);
  const int64_t tiles = kern::MoeRouteTiles(T * k);
  at::Tensor hist = at::empty({tiles * (num_experts + 1)}, iopt);
  cudaError_t e = kern::LaunchMoeRoute(expert_idx.data_ptr(), expert_idx.scalar_type() == at::kLong, T * k, (int)num_experts,
                                       (int)nranks, hist.data_ptr<int>(), BnTickets(x.get_device(), s, 1),
                                       counts.data_ptr<int64_t>(), splits.data_ptr<int>(), pos.data_ptr<int>(), s);
  if (e == cudaSuccess) {
    kern::MoeRows a {};
    a.src = x.data_ptr(); a.dst = send.data_ptr(); a.src_rows = T; a.dst_rows = send.size(0);
    a.pos = pos.data_ptr<int>(); a.ntok = T; a.k = (int)k; a.h = h; a.dtype = (int)MapDtype(dt);
    a.gate_dtype = (int)MapDtype(at::kFloat); a.ctas = (int)ctas;
    e = kern::LaunchMoeScatter(a, s);
  }
  TORCH_CHECK(e == cudaSuccess, op, " launch failed: ", cudaGetErrorString(e));
  return {pos, splits};
}

// dst[pos[t, j]] = src[t] (no gates) or round(gates[t, j] * src[t]); with dot_rows also returns grad_gates [T, k] in the
// gates' dtype, grad_gates[t, j] = <src[t], dot_rows[pos[t, j]]>.
c10::optional<at::Tensor> MoeScatter(at::Tensor src, at::Tensor pos, at::Tensor dst, c10::optional<at::Tensor> gates,
                                     c10::optional<at::Tensor> dot_rows, c10::optional<at::Tensor> status, int64_t ctas) {
  const char* op = "moe_scatter";
  const auto dt = MoeDtype(op, src);
  const at::Device dev = src.device();
  const int64_t T = src.size(0), h = src.size(1);
  CheckMoeRows(op, "src", src, h, dt, dev);
  CheckMoeRows(op, "dst", dst, h, dt, dev);
  CheckMoePos(op, pos, T, dev);
  int gdt = 0;
  const void* g = MoeGates(op, gates, pos, dt, &gdt);
  TORCH_CHECK(!dot_rows || gates, op, ": dot_rows needs gates (the gate gradient has the gates' dtype)");
  if (dot_rows) CheckMoeRows(op, "dot_rows", *dot_rows, h, dt, dev);
  TORCH_CHECK(!dot_rows || dot_rows->size(0) >= dst.size(0), op, ": dot_rows must have at least dst's ", dst.size(0), " rows");
  const int* st = MoeStatus(op, status, dev);
  TORCH_CHECK(ctas >= 0, op, ": ctas must be >= 0");
  c10::cuda::CUDAGuard guard(dev);
  cudaStream_t s = c10::cuda::getCurrentCUDAStream(src.get_device());
  c10::optional<at::Tensor> grad_gates;
  if (dot_rows) grad_gates = at::empty(pos.sizes(), gates->options());
  kern::MoeRows a {};
  a.src = src.data_ptr(); a.dst = dst.data_ptr(); a.src_rows = T; a.dst_rows = dst.size(0);
  a.pos = pos.data_ptr<int>(); a.ntok = T; a.k = (int)pos.size(1); a.h = h; a.dtype = (int)MapDtype(dt);
  a.gates = g; a.gate_dtype = gdt; a.dot_rows = dot_rows ? dot_rows->data_ptr() : nullptr;
  a.grad_gates = grad_gates ? grad_gates->data_ptr() : nullptr; a.status = st; a.ctas = (int)ctas;
  cudaError_t e = kern::LaunchMoeScatter(a, s);
  TORCH_CHECK(e == cudaSuccess, op, " launch failed: ", cudaGetErrorString(e));
  return grad_gates;
}

// y[t] = round(sum_j gates[t, j] * src[pos[t, j]]) in fp32, j ascending (no gates: unit gates); zeros under a non-zero
// status.  Returns y [T, hidden] in src's dtype.
at::Tensor MoeGather(at::Tensor src, at::Tensor pos, c10::optional<at::Tensor> gates, c10::optional<at::Tensor> status,
                     int64_t ctas) {
  const char* op = "moe_gather";
  const auto dt = MoeDtype(op, src);
  const at::Device dev = src.device();
  const int64_t h = src.size(1);
  CheckMoeRows(op, "src", src, h, dt, dev);
  TORCH_CHECK(pos.dim() == 2, op, ": pos must be [tokens, k], got sizes ", pos.sizes());
  const int64_t T = pos.size(0);
  CheckMoePos(op, pos, T, dev);
  int gdt = 0;
  const void* g = MoeGates(op, gates, pos, dt, &gdt);
  const int* st = MoeStatus(op, status, dev);
  TORCH_CHECK(ctas >= 0, op, ": ctas must be >= 0");
  c10::cuda::CUDAGuard guard(dev);
  cudaStream_t s = c10::cuda::getCurrentCUDAStream(src.get_device());
  at::Tensor y = at::empty({T, h}, src.options());
  kern::MoeRows a {};
  a.src = src.data_ptr(); a.dst = y.data_ptr(); a.src_rows = src.size(0); a.dst_rows = T;
  a.pos = pos.data_ptr<int>(); a.ntok = T; a.k = (int)pos.size(1); a.h = h; a.dtype = (int)MapDtype(dt);
  a.gates = g; a.gate_dtype = gdt; a.status = st; a.ctas = (int)ctas;
  cudaError_t e = kern::LaunchMoeGather(a, s);
  TORCH_CHECK(e == cudaSuccess, op, " launch failed: ", cudaGetErrorString(e));
  return y;
}

// Source-major <-> expert-major rows (kern::LaunchMoeRegroup) with counts [nranks, experts_per_rank] int64.  Returns the
// group ends (int32 [experts_per_rank]) forward, the return splits (int32 [nranks]) in reverse.
at::Tensor MoeRegroup(at::Tensor src, at::Tensor counts, c10::optional<at::Tensor> status, at::Tensor dst, bool reverse,
                      int64_t ctas) {
  const char* op = reverse ? "moe_regroup_reverse" : "moe_regroup";
  const auto dt = MoeDtype(op, src);
  const at::Device dev = src.device();
  const int64_t rows = src.size(0), h = src.size(1);
  CheckMoeRows(op, "src", src, h, dt, dev);
  CheckMoeRows(op, "dst", dst, h, dt, dev);
  TORCH_CHECK(dst.size(0) == rows, op, ": dst must have src's ", rows, " rows, got ", dst.size(0));
  TORCH_CHECK(counts.is_cuda() && counts.device() == dev && counts.scalar_type() == at::kLong && counts.dim() == 2 &&
              counts.is_contiguous() && counts.size(0) >= 1 && counts.size(1) >= 1 &&
              counts.numel() <= kern::kMoeMaxExperts, op, ": counts must be a contiguous int64 [nranks, experts_per_rank] "
              "tensor of at most ", kern::kMoeMaxExperts, " elements on ", dev, ", got sizes ", counts.sizes());
  const int n = (int)counts.size(0), el = (int)counts.size(1);
  TORCH_CHECK(src.data_ptr() != dst.data_ptr() || el == 1, op, ": src and dst may only be the same tensor with one expert per rank");
  const int* st = MoeStatus(op, status, dev);
  TORCH_CHECK(ctas >= 0, op, ": ctas must be >= 0");
  c10::cuda::CUDAGuard guard(dev);
  cudaStream_t s = c10::cuda::getCurrentCUDAStream(src.get_device());
  at::Tensor out = at::empty({reverse ? n : el}, src.options().dtype(at::kInt));
  cudaError_t e = kern::LaunchMoeRegroup(src.data_ptr(), dst.data_ptr(), h * (int64_t)src.element_size(), rows,
                                         counts.data_ptr<int64_t>(), n, el, st, reverse, reverse ? nullptr : out.data_ptr<int>(),
                                         reverse ? out.data_ptr<int>() : nullptr, (int)ctas, s);
  TORCH_CHECK(e == cudaSuccess, op, " launch failed: ", cudaGetErrorString(e));
  return out;
}

}  // namespace

PYBIND11_MODULE(_hvd_torch, m) {
  m.doc() = "horovod_b200 PyTorch binding";
  m.def("allreduce_async", &DoAllreduce);
  m.def("grouped_allreduce_async", &DoGroupedAllreduce);
  m.def("allgather_async", &DoAllgather);
  m.def("grouped_allgather_async", &DoGroupedAllgather);
  m.def("broadcast_async", &DoBroadcast);
  m.def("alltoall_async", &DoAlltoall);
  m.def("reducescatter_async", &DoReducescatter);
  m.def("grouped_reducescatter_async", &DoGroupedReducescatter);
  m.def("join", &DoJoin);
  m.def("barrier", &DoBarrier);
  m.def("poll", &PollHandle);
  m.def("wait_and_clear", &WaitAndClear);
  m.def("reset", &Reset);
  m.def("reset_noname_counters", &ResetNonameCounters);
  m.def("symm_empty", &SymmEmpty);
  m.def("captured_allreduce_", &CapturedAllreduce, py::arg("tensor"), py::arg("reduce_op"), py::arg("prescale"),
        py::arg("postscale"), py::arg("process_set_id"), py::arg("max_ctas"), py::arg("channel") = kern::kGraphChannel);
  m.def("captured_reducescatter_", &CapturedReducescatter);
  m.def("captured_allgather_", &CapturedAllgather, py::arg("tensor"), py::arg("process_set_id"), py::arg("max_ctas"),
        py::arg("channel") = kern::kGraphChannel);
  m.def("captured_alltoall", &CapturedAlltoall, py::arg("tensor"), py::arg("splits"), py::arg("capacity"),
        py::arg("process_set_id"), py::arg("max_ctas"));
  m.def("fused_sgd_step", &FusedSgdStep, py::arg("params"), py::arg("grads"), py::arg("momenta"), py::arg("lr"),
        py::arg("momentum"), py::arg("dampening"), py::arg("weight_decay"), py::arg("nesterov"), py::arg("grad_scale"),
        py::arg("first_step"), py::arg("grad_scale_dev") = py::none(), py::arg("master_params") = std::vector<at::Tensor>(),
        py::arg("ema_params") = std::vector<at::Tensor>(), py::arg("ema_weight") = 0.0, py::arg("ema_start") = false);
  m.def("fused_adam_step", &FusedAdamStep, py::arg("params"), py::arg("grads"), py::arg("exp_avg"), py::arg("exp_avg_sq"),
        py::arg("lr"), py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("weight_decay"), py::arg("step"),
        py::arg("grad_scale"), py::arg("adamw"), py::arg("grad_scale_dev") = py::none(),
        py::arg("master_params") = std::vector<at::Tensor>(),
        py::arg("ema_params") = std::vector<at::Tensor>(), py::arg("ema_weight") = 0.0, py::arg("ema_start") = false);
  m.def("fused_lamb_step", &FusedLambStep, py::arg("params"), py::arg("grads"), py::arg("exp_avg"), py::arg("exp_avg_sq"),
        py::arg("lr"), py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("weight_decay"), py::arg("step"),
        py::arg("bias_correction"), py::arg("adapt"), py::arg("grad_scale"), py::arg("grad_scale_dev") = py::none(),
        py::arg("master_params") = std::vector<at::Tensor>(),
        py::arg("ema_params") = std::vector<at::Tensor>(), py::arg("ema_weight") = 0.0, py::arg("ema_start") = false);
  m.def("lamb_norms", &LambNorms, py::arg("params"), py::arg("grads"), py::arg("exp_avg"), py::arg("exp_avg_sq"),
        py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("weight_decay"), py::arg("step"),
        py::arg("bias_correction"), py::arg("grad_scale"), py::arg("grad_scale_dev"), py::arg("master_params"),
        py::arg("out"), py::arg("slots"));
  m.def("lamb_apply", &LambApply, py::arg("params"), py::arg("grads"), py::arg("exp_avg"), py::arg("exp_avg_sq"),
        py::arg("lr"), py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("weight_decay"), py::arg("step"),
        py::arg("bias_correction"), py::arg("adapt"), py::arg("master_params"), py::arg("norms"), py::arg("slots"),
        py::arg("ema_params") = std::vector<at::Tensor>(), py::arg("ema_weight") = 0.0, py::arg("ema_start") = false);
  m.def("fused_lars_step", &FusedLarsStep, py::arg("params"), py::arg("grads"), py::arg("momentum_buffers"), py::arg("lr"),
        py::arg("momentum"), py::arg("weight_decay"), py::arg("trust_coefficient"), py::arg("eps"), py::arg("adapt"),
        py::arg("grad_scale"), py::arg("grad_scale_dev") = py::none(), py::arg("master_params") = std::vector<at::Tensor>(),
        py::arg("ema_params") = std::vector<at::Tensor>(), py::arg("ema_weight") = 0.0, py::arg("ema_start") = false);
  m.def("lars_norms", &LarsNorms, py::arg("params"), py::arg("grads"), py::arg("momentum_buffers"), py::arg("grad_scale"),
        py::arg("grad_scale_dev"), py::arg("master_params"), py::arg("out"), py::arg("slots"));
  m.def("lars_apply", &LarsApply, py::arg("params"), py::arg("grads"), py::arg("momentum_buffers"), py::arg("lr"),
        py::arg("momentum"), py::arg("weight_decay"), py::arg("trust_coefficient"), py::arg("eps"), py::arg("adapt"),
        py::arg("grad_scale"), py::arg("grad_scale_dev"), py::arg("master_params"), py::arg("norms"), py::arg("slots"),
        py::arg("ema_params") = std::vector<at::Tensor>(), py::arg("ema_weight") = 0.0, py::arg("ema_start") = false);
  m.def("fused_adafactor_step", &FusedAdafactorStep, py::arg("params"), py::arg("grads"), py::arg("row_vars"),
        py::arg("col_vars"), py::arg("variances"), py::arg("lr"), py::arg("beta2_decay"), py::arg("eps1"), py::arg("eps2"),
        py::arg("d"), py::arg("weight_decay"), py::arg("step"), py::arg("grad_scale"), py::arg("grad_scale_dev"),
        py::arg("master_params"), py::arg("ema_params"), py::arg("ema_weight"), py::arg("ema_start"));
  m.def("grad_shard_stats", &GradShardStats, py::arg("grads"), py::arg("out"), py::arg("inv_scale") = py::none(),
        py::arg("norm_inf") = false);
  m.def("grad_accumulate", &GradAccumulate, py::arg("grads"), py::arg("accs"), py::arg("mode"));
  m.def("sync_bn_stats", &SyncBnStats, py::arg("x"), py::arg("slot"));
  m.def("sync_bn_combine", &SyncBnCombine, py::arg("slots"), py::arg("num_features"), py::arg("eps"), py::arg("momentum"),
        py::arg("running_mean") = py::none(), py::arg("running_var") = py::none(),
        py::arg("num_batches_tracked") = py::none());
  m.def("sync_bn_elemt", &SyncBnElemt, py::arg("x"), py::arg("mean"), py::arg("invstd"), py::arg("weight") = py::none(),
        py::arg("bias") = py::none());
  m.def("sync_bn_backward_reduce", &SyncBnBackwardReduce, py::arg("grad_output"), py::arg("x"), py::arg("mean"),
        py::arg("invstd"), py::arg("weight"), py::arg("sums"), py::arg("need_weight_grad"), py::arg("need_bias_grad"));
  m.def("sync_bn_backward_elemt", &SyncBnBackwardElemt, py::arg("grad_output"), py::arg("x"), py::arg("mean"),
        py::arg("invstd"), py::arg("weight"), py::arg("sums"), py::arg("count"));
  m.def("moe_permute", &MoePermute, py::arg("x"), py::arg("expert_idx"), py::arg("send"), py::arg("counts"),
        py::arg("num_experts"), py::arg("nranks"), py::arg("ctas") = 0);
  m.def("moe_scatter", &MoeScatter, py::arg("src"), py::arg("pos"), py::arg("dst"), py::arg("gates") = py::none(),
        py::arg("dot_rows") = py::none(), py::arg("status") = py::none(), py::arg("ctas") = 0);
  m.def("moe_gather", &MoeGather, py::arg("src"), py::arg("pos"), py::arg("gates") = py::none(),
        py::arg("status") = py::none(), py::arg("ctas") = 0);
  m.def("moe_regroup", &MoeRegroup, py::arg("src"), py::arg("counts"), py::arg("status"), py::arg("dst"),
        py::arg("reverse"), py::arg("ctas") = 0);
}
