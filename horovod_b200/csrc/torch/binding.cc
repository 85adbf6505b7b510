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
// The fused optimizer, SyncBatchNorm and MoE entry points are in optim_binding.cc, sync_bn_binding.cc and
// moe_binding.cc; PYBIND11_MODULE below registers them.
#include <cuda_runtime.h>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <unordered_map>
#include "../common/engine.h"
#include "../kernels/p2p_kernels.h"
#include "binding_util.h"
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
    const OnDevice on(in);
    cudaEvent_t ev = g_events.Get(e->device);
    C10_CUDA_CHECK(cudaEventRecord(ev, on.stream));
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
      const OnDevice on(output);
      output.resize_(shape);
      int dev = (int)output.get_device();
      cudaEvent_t ev = g_events.Get(dev);
      cudaEventRecord(ev, on.stream);
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
  const OnDevice on(tensor);
  const int64_t bytes = (int64_t)tensor.numel() * (int64_t)tensor.element_size();
  ThrowIfError(Engine::Get().CapturedAllreduce(tensor.data_ptr(), bytes, MapDtype(tensor.scalar_type()), (ReduceOp)reduce_op, prescale,
                                               postscale, process_set_id, max_ctas, (void*)on.stream, channel));
}

// The two halves of a sharded optimizer step on a registered tensor, launched like CapturedAllreduce.  Rank r owns the
// contiguous slice [r*S, (r+1)*S) of the tensor's bytes, S = bytes / set size.
void CapturedReducescatter(at::Tensor tensor, int reduce_op, double prescale, double postscale, int process_set_id, int max_ctas) {
  TORCH_CHECK(tensor.is_cuda(), "captured_reducescatter_: CUDA tensor expected");
  TORCH_CHECK(tensor.is_non_overlapping_and_dense(), "captured_reducescatter_: tensor must be dense");
  const OnDevice on(tensor);
  const int64_t bytes = (int64_t)tensor.numel() * (int64_t)tensor.element_size();
  ThrowIfError(Engine::Get().CapturedReducescatter(tensor.data_ptr(), bytes, MapDtype(tensor.scalar_type()), (ReduceOp)reduce_op,
                                                   prescale, postscale, process_set_id, max_ctas, (void*)on.stream));
}

void CapturedAllgather(at::Tensor tensor, int process_set_id, int max_ctas, int channel) {
  CheckCapturedChannel("captured_allgather_", channel);
  TORCH_CHECK(tensor.is_cuda(), "captured_allgather_: CUDA tensor expected");
  TORCH_CHECK(tensor.is_non_overlapping_and_dense(), "captured_allgather_: tensor must be dense");
  const OnDevice on(tensor);
  const int64_t bytes = (int64_t)tensor.numel() * (int64_t)tensor.element_size();
  ThrowIfError(Engine::Get().CapturedAllgather(tensor.data_ptr(), bytes, process_set_id, max_ctas, (void*)on.stream, channel));
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
  const OnDevice on(tensor);
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
                                              (void*)on.stream));
  return {out, recv, status};
}

// Ulysses exchange of a contiguous tensor between sequence shards and head shards (hvd.UlyssesExchange), launched like
// CapturedAllreduce through this rank's registered staging buffer.  direction 0 (seq -> heads) splits head_dim into
// nranks blocks and concatenates the ranks' blocks along seq_dim; direction 1 (heads -> seq) splits seq_dim and
// concatenates along head_dim.  The output is allocated on the current stream; `status` (int32 [1]) keeps the first
// non-zero kern::AlltoallStatus.
at::Tensor CapturedUlyssesExchange(at::Tensor tensor, at::Tensor staging, at::Tensor status, int64_t seq_dim, int64_t head_dim,
                                   int direction, int nranks, int process_set_id, int max_ctas) {
  const char* op = "ulysses_exchange";
  TORCH_CHECK(tensor.is_cuda(), op, ": CUDA tensor expected");
  TORCH_CHECK(tensor.is_contiguous(), op, ": tensor must be contiguous");
  TORCH_CHECK(direction == kern::kUlySeqToHeads || direction == kern::kUlyHeadsToSeq, op, ": direction must be 0 or 1, got ", direction);
  TORCH_CHECK(nranks >= 1 && nranks <= kern::kMaxPeers, op, ": nranks must be in [1, ", kern::kMaxPeers, "], got ", nranks);
  const int64_t nd = tensor.dim();
  TORCH_CHECK(seq_dim >= 0 && seq_dim < nd && head_dim >= 0 && head_dim < nd && seq_dim != head_dim, op,
              ": seq_dim and head_dim must be two distinct dims of a ", nd, "-D tensor, got ", seq_dim, " and ", head_dim);
  const int64_t split = direction == kern::kUlySeqToHeads ? head_dim : seq_dim;
  TORCH_CHECK(tensor.size(split) % nranks == 0, op, ": dim ", split, " (size ", tensor.size(split), ") must be a multiple of ",
              nranks);
  TORCH_CHECK(staging.is_cuda() && staging.device() == tensor.device() && staging.is_contiguous(), op,
              ": staging must be a contiguous tensor on ", tensor.device());
  const int64_t bytes = tensor.numel() * (int64_t)tensor.element_size();
  const int64_t staging_bytes = staging.numel() * (int64_t)staging.element_size();
  TORCH_CHECK(staging_bytes >= bytes, op, ": the tensor has ", bytes, " bytes, the staging buffer ", staging_bytes);
  CheckVector(op, "status", status, tensor.device(), {at::kInt}, 1);
  const OnDevice on(tensor);
  const int64_t lo = std::min(seq_dim, head_dim), hi = std::max(seq_dim, head_dim);
  const auto sz = tensor.sizes();
  const int64_t dims[5] = {c10::multiply_integers(sz.slice(0, lo)), sz[lo], c10::multiply_integers(sz.slice(lo + 1, hi - lo - 1)),
                           sz[hi], c10::multiply_integers(sz.slice(hi + 1))};
  std::vector<int64_t> out_sizes = sz.vec();
  const int64_t concat = split == head_dim ? seq_dim : head_dim;
  out_sizes[split] /= nranks;
  out_sizes[concat] *= nranks;
  at::Tensor out = at::empty(out_sizes, tensor.options());
  ThrowIfError(Engine::Get().CapturedUlyssesExchange(tensor.data_ptr(), out.data_ptr(), dims, tensor.element_size(), direction,
                                                     head_dim < seq_dim, staging.data_ptr(), staging_bytes, status.data_ptr<int>(),
                                                     nranks, process_set_id, max_ctas, (void*)on.stream));
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
  m.def("captured_ulysses_exchange", &CapturedUlyssesExchange, py::arg("tensor"), py::arg("staging"), py::arg("status"),
        py::arg("seq_dim"), py::arg("head_dim"), py::arg("direction"), py::arg("nranks"), py::arg("process_set_id"),
        py::arg("max_ctas"));
  DefOptim(m);
  DefSyncBn(m);
  DefMoe(m);
}
