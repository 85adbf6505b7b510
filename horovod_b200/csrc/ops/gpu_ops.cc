#include "gpu_ops.h"
#include <sys/stat.h>
#include <unistd.h>
#include <sstream>
#include <algorithm>
#include <atomic>
#include <cstring>
#include "../common/env.h"
#include "../common/logging.h"
#include "../kernels/p2p_kernels.h"
#include "../symm/symm_memory.h"
#include "collective_plan.h"
#include "cpu_ops.h"
#include "ipc_registry.h"
#include "nccl_baseline.h"

namespace hvd {

#define HVD_CUDA(call)                                                                      \
  do {                                                                                      \
    cudaError_t _e = (call);                                                                \
    if (_e != cudaSuccess) return Status::UnknownError(std::string(#call) + " failed: " + cudaGetErrorString(_e)); \
  } while (0)

namespace {
constexpr size_t kRingBytes = 8 << 20;
constexpr int64_t kLatencyAreaBytes = 1 << 20;  // tail of each symmetric buffer slot reserved for the latency lane
int64_t Align128(int64_t b) { return (b + 127) / 128 * 128; }
}  // namespace

// ---------------------------------------------------------------------------
// GpuContext

GpuContext& GpuContext::Get() { static GpuContext c; return c; }

int GpuContext::DeviceCount() {
  std::lock_guard<std::mutex> l(mu_);  // several engines may live in one process (native self-test)
  if (count_ == -2) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); n = 0; }
    count_ = n;
  }
  return count_;
}
bool GpuContext::Available() { return DeviceCount() > 0; }

GpuContext::PerDevice& GpuContext::Dev(int device) {
  auto it = devs_.find(device);
  if (it != devs_.end()) return it->second;
  PerDevice& d = devs_[device];
  cudaSetDevice(device);
  int lo = 0, hi = 0;
  cudaDeviceGetStreamPriorityRange(&lo, &hi);
  cudaStreamCreateWithPriority(&d.stream, cudaStreamNonBlocking, hi);  // highest priority, like the reference (cuda_operations.cc:202-209)
  cudaHostAlloc((void**)&d.host_ring, kRingBytes, cudaHostAllocDefault);
  cudaMalloc((void**)&d.dev_ring, kRingBytes);
  return d;
}

cudaStream_t GpuContext::Stream(int device) { std::lock_guard<std::mutex> l(mu_); return Dev(device).stream; }
cudaStream_t GpuContext::LatencyStream(int device) {
  std::lock_guard<std::mutex> l(mu_);
  PerDevice& d = Dev(device);
  if (!d.lat_stream) {
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    cudaStreamCreateWithPriority(&d.lat_stream, cudaStreamNonBlocking, hi);
  }
  return d.lat_stream;
}
void* GpuContext::GridSyncBlock(int device) {
  std::lock_guard<std::mutex> l(mu_);
  PerDevice& d = Dev(device);
  if (!d.grid_sync) {
    if (cudaMalloc(&d.grid_sync, 256) != cudaSuccess) { cudaGetLastError(); d.grid_sync = nullptr; return nullptr; }
    cudaMemset(d.grid_sync, 0, 256);
  }
  return d.grid_sync;
}

SharedEvent* GpuContext::NewEvent(int device, int refs) {
  std::lock_guard<std::mutex> l(mu_);
  PerDevice& d = Dev(device);
  auto* e = new SharedEvent();
  e->device = device;
  e->refs = refs;
  if (!d.pool.empty()) { e->ev = d.pool.back(); d.pool.pop_back(); }
  else { cudaSetDevice(device); cudaEventCreateWithFlags(&e->ev, cudaEventDisableTiming); }
  return e;
}

void GpuContext::Release(SharedEvent* e) {
  if (!e) return;
  if (e->refs.fetch_sub(1) > 1) return;
  {
    std::lock_guard<std::mutex> l(mu_);
    auto it = devs_.find(e->device);
    if (it != devs_.end() && e->ev) it->second.pool.push_back(e->ev);
  }
  delete e;
}

const void* GpuContext::Stage(int device, const void* host, size_t bytes, cudaStream_t s) {
  std::lock_guard<std::mutex> l(mu_);
  PerDevice& d = Dev(device);
  const size_t raw = bytes;
  bytes = (bytes + 255) / 256 * 256;
  if (bytes > kRingBytes) return nullptr;
  if (d.ring_off + bytes > kRingBytes) {  // wrap: everything older must have been consumed, on every stream that stages here
    cudaStreamSynchronize(s);
    if (d.stream && d.stream != s) cudaStreamSynchronize(d.stream);
    if (d.lat_stream && d.lat_stream != s) cudaStreamSynchronize(d.lat_stream);
    d.ring_off = 0;
  }
  char* h = d.host_ring + d.ring_off;
  char* dv = d.dev_ring + d.ring_off;
  d.ring_off += bytes;
  memcpy(h, host, raw);
  cudaMemcpyAsync(dv, h, raw, cudaMemcpyHostToDevice, s);
  return dv;
}

void* GpuContext::TempAlloc(int device, size_t bytes, bool zero, cudaStream_t s) {
  void* p = nullptr;
  cudaSetDevice(device);
  if (cudaMallocAsync(&p, bytes ? bytes : 16, s) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  if (zero) cudaMemsetAsync(p, 0, bytes ? bytes : 16, s);
  std::lock_guard<std::mutex> l(mu_);
  Dev(device).temps.push_back(p);
  return p;
}
void GpuContext::TempFreeAll(int device, cudaStream_t s) {
  std::vector<void*> t;
  { std::lock_guard<std::mutex> l(mu_); t.swap(Dev(device).temps); }
  for (void* p : t) cudaFreeAsync(p, s);
}

void* GpuContext::PinnedHost(int device, size_t bytes) {
  std::lock_guard<std::mutex> l(mu_);
  PerDevice& d = Dev(device);
  if (d.pinned_bytes < bytes) {
    if (d.pinned) cudaFreeHost(d.pinned);
    d.pinned = nullptr; d.pinned_bytes = 0;
    size_t want = std::max<size_t>(bytes, 1 << 20);
    if (cudaHostAlloc(&d.pinned, want, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); d.pinned = nullptr; return nullptr; }
    d.pinned_bytes = want;
  }
  return d.pinned;
}

void GpuContext::Reset() {
  std::lock_guard<std::mutex> l(mu_);
  for (auto& kv : devs_) {
    cudaSetDevice(kv.first);
    if (kv.second.pinned) cudaFreeHost(kv.second.pinned);
    if (kv.second.stream) { cudaStreamSynchronize(kv.second.stream); cudaStreamDestroy(kv.second.stream); }
    if (kv.second.lat_stream) { cudaStreamSynchronize(kv.second.lat_stream); cudaStreamDestroy(kv.second.lat_stream); }
    if (kv.second.grid_sync) cudaFree(kv.second.grid_sync);
    for (auto e : kv.second.pool) cudaEventDestroy(e);
    if (kv.second.host_ring) cudaFreeHost(kv.second.host_ring);
    if (kv.second.dev_ring) cudaFree(kv.second.dev_ring);
  }
  devs_.clear();
  cudaGetLastError();
}

// ---------------------------------------------------------------------------
// helpers

namespace {

struct Piece { const char* in; char* out; int64_t count; };

void WaitReady(Entries& es, cudaStream_t s) {
  void* last = nullptr;
  for (auto& e : es) {
    if (e && e->ready_event && e->ready_event != last) { cudaStreamWaitEvent(s, (cudaEvent_t)e->ready_event, 0); last = e->ready_event; }
  }
}

Status FinishEvent(int device, cudaStream_t s, size_t nrefs, SharedEvent** done) {
  SharedEvent* ev = GpuContext::Get().NewEvent(device, (int)std::max<size_t>(nrefs, 1));
  cudaError_t e = cudaEventRecord(ev->ev, s);
  if (e != cudaSuccess) { GpuContext::Get().Release(ev); return Status::UnknownError(std::string("cudaEventRecord: ") + cudaGetErrorString(e)); }
  *done = ev;
  return Status::OK();
}

// Allreduce pieces: real entries, or zero placeholders for tensors this (joined) rank never submitted.
Status BuildPieces(Entries& es, const Response& r, int device, cudaStream_t s, std::vector<Piece>* pieces) {
  const size_t esz = DataTypeSize(r.dtype);
  for (size_t i = 0; i < es.size(); ++i) {
    if (es[i]) {
      pieces->push_back({(const char*)es[i]->input, (char*)es[i]->output, es[i]->shape.num_elements()});
    } else {
      int64_t cnt = i < r.tensor_sizes.size() ? r.tensor_sizes[i] : 0;
      char* z = (char*)GpuContext::Get().TempAlloc(device, (size_t)cnt * esz, true, s);
      if (!z) return Status::UnknownError("out of device memory for join placeholder");
      pieces->push_back({z, z, cnt});
    }
  }
  return Status::OK();
}

// The pieces' packed layout in a fusion buffer, each at the next 128-byte boundary; returns the buffer's bytes.
int64_t PackDescs(const std::vector<Piece>& pieces, int64_t esz, std::vector<kern::TensorDesc>* descs) {
  int64_t total = 0;
  for (auto& p : pieces) {
    descs->push_back({p.in, p.out, total, p.count});
    total += Align128(p.count * esz);
  }
  return total;
}

// Arguments of the zero-copy kernel over every rank's copy of a tensor, ptr[p] + off as mapped into this process, without
// multicast; false when the kernel cannot apply the scale factors to `op` (it scales sums only).
bool FillInplaceArgs(int n, void* const* ptr, int64_t off, int64_t bytes, DataType dtype, ReduceOp op, double prescale,
                     double postscale, int max_ctas, kern::InplaceArgs* ia) {
  if (op != ReduceOp::SUM && op != ReduceOp::AVERAGE && !(prescale == 1.0 && postscale == 1.0)) return false;
  *ia = kern::InplaceArgs {};
  for (int p = 0; p < n; ++p) ia->ptr[p] = (char*)ptr[p] + off;
  ia->bytes = bytes;
  ia->scale = prescale * postscale;
  ia->op = (int)op;
  ia->dtype = (int)dtype;
  ia->ctas = (int)std::max<int64_t>(1, std::min<int64_t>(max_ctas, (bytes + 4096ll * n - 1) / (4096ll * n)));
  return true;
}

}  // namespace

std::shared_ptr<SymmTeam> GpuOps::EnsureTeam(ProcessSet& ps, int device) {
  if (ps.team_tried) {
    if (ps.team && ps.team->abort_state() == 2)
      throw TransportError("a peer GPU did not reach the collective's flag barrier within HVD_KERNEL_TIMEOUT_SECONDS");
    // one symmetric team per process set, on the device of the set's first GPU collective.  A tensor that lives on ANOTHER
    // device of this process (a model split over two GPUs, reference test_model_parallelism) cannot use it: that response is
    // staged through the host instead (every rank of a symmetric program takes the same branch).
    if (ps.team && ps.team->device() != device) {
      static std::atomic<bool> warned{false};
      if (!warned.exchange(true))
        LOG(WARNING) << "a GPU tensor on device " << device << " meets the process set's peer-mapped team on device " << ps.team->device()
                     << ": its collectives are staged through host memory (one process per GPU is the fast path)";
      return nullptr;
    }
    return ps.team;
  }
  ps.team_tried = true;
  Transport* t = ps.transport.get();
  // unique tag for the fd-passing sockets: coordinator pid + counter, agreed through the transport
  int64_t tag[2] = {(int64_t)getpid(), (int64_t)(++team_counter_)};
  t->Bcast(tag, sizeof tag, 0);
  std::string why;
  bool single = t->single_host();
  uint64_t ok = single ? 1 : 0;
  t->AllreduceBits(&ok, 1, nullptr, 0);
  if (!ok) { LOG(INFO) << "process set " << ps.id << " spans hosts: no set-wide peer mapping (allreduce goes hierarchical when hosts are uniform)"; return nullptr; }
  size_t bytes = ps.id == 0 ? env_.symm_buffer_bytes : std::min<size_t>(env_.symm_buffer_bytes, 32ull << 20);
  std::shared_ptr<SymmTeam> created = SymmTeam::Create(t, device, bytes, env_.want_multicast,
                             std::to_string(tag[0]) + "-" + std::to_string(tag[1]) + "-" + std::to_string(ps.id), &why);
  { std::lock_guard<std::mutex> l(ps.team_mu); ps.team = created; }
  if (!ps.team) LOG(WARNING) << "peer-mapped symmetric memory unavailable for process set " << ps.id << " (" << why
                             << "); GPU collectives fall back to host staging";
  if (ps.team) ps.team->set_timeout_seconds(EnvDouble("HVD_KERNEL_TIMEOUT_SECONDS", 60.0));
  if (ps.team && env_.latency_lane_bytes > 0 && ps.team->buffer_bytes() >= (size_t)(8 * kLatencyAreaBytes)) ps.team->set_reserved_tail((size_t)kLatencyAreaBytes);
  if (ps.team) LOG(INFO) << "process set " << ps.id << ": symmetric team of " << ps.team->nranks() << " GPUs, backend "
                 << ps.team->backend() << ", 2 x " << (ps.team->buffer_bytes() >> 20) << " MiB";
  // (same decision on every rank: a team exists everywhere or nowhere, the flags come from the shared environment)
  if (ps.team && ps.id == 0 && env_.calibrate && env_.variant == "auto") Calibrate(ps, *ps.team, device);
  return ps.team;
}

bool GpuOps::EnsureHierarchy(ProcessSet& ps, int device) {
  if (ps.hier_tried) {
    if (ps.local_team && ps.local_team->abort_state() == 2)
      throw TransportError("a peer GPU did not reach the collective's flag barrier within HVD_KERNEL_TIMEOUT_SECONDS");
    return ps.local_team != nullptr;
  }
  ps.hier_tried = true;
  Transport* t = ps.transport.get();
  const int n = t->size(), me = t->rank();
  // group the members by host (host ids come from the bootstrap hostname exchange, identical on every rank)
  std::map<int, std::vector<int>> by_host;
  for (int i = 0; i < n; ++i) by_host[t->host_id(i)].push_back(i);
  const std::vector<int>& mine = by_host[t->host_id(me)];
  const int L = (int)mine.size();
  // on by default for uniform multi-host sets; HOROVOD_HIERARCHICAL_ALLREDUCE=0 (hvdrun --no-hierarchical-allreduce) forces
  // the flat host-staged path
  // HOROVOD_TORUS_ALLREDUCE (the reference's 2-D variant whose cross step stays on the GPU fabric) selects the same two-level
  // schedule here: intra-host kernels + cross-host shard exchange
  bool uniform = L >= 2 && L <= kern::kMaxPeers &&
                 EnvBool("HVD_HIERARCHICAL_ALLREDUCE", EnvBool("HOROVOD_HIERARCHICAL_ALLREDUCE", true) || EnvBool("HOROVOD_TORUS_ALLREDUCE", false));
  for (auto& kv : by_host) if ((int)kv.second.size() != L) uniform = false;
  int64_t tag[2] = {(int64_t)getpid(), (int64_t)(++team_counter_)};
  t->Bcast(tag, sizeof tag, 0);
  if (!uniform) return false;  // same decision on every rank: it only depends on the shared host table
  const int li = (int)(std::find(mine.begin(), mine.end(), me) - mine.begin());
  std::vector<int> cross;
  for (auto& kv : by_host) cross.push_back(kv.second[li]);
  ps.local_transport = t->Split(mine);
  ps.cross_transport = t->Split(cross);
  std::string why;
  size_t bytes = ps.id == 0 ? env_.symm_buffer_bytes : std::min<size_t>(env_.symm_buffer_bytes, 32ull << 20);
  std::shared_ptr<SymmTeam> created = SymmTeam::Create(ps.local_transport.get(), device, bytes, env_.want_multicast,
      std::to_string(tag[0]) + "-" + std::to_string(tag[1]) + "-" + std::to_string(ps.id) + "-h" + std::to_string(t->host_id(me)), &why);
  uint64_t ok = created ? 1 : 0;
  t->AllreduceBits(&ok, 1, nullptr, 0);  // all hosts or none
  if (!ok) {
    LOG(WARNING) << "hierarchical allreduce unavailable for process set " << ps.id << (why.empty() ? "" : " (" + why + ")") << "; staging through the host";
    return false;
  }
  created->set_timeout_seconds(EnvDouble("HVD_KERNEL_TIMEOUT_SECONDS", 60.0));
  { std::lock_guard<std::mutex> l(ps.team_mu); ps.local_team = created; }
  LOG(INFO) << "process set " << ps.id << ": hierarchical allreduce over " << by_host.size() << " hosts x " << L << " GPUs (intra-host "
            << created->backend() << ")";
  return true;
}

// reduce-scatter (intra-host kernel) -> shard allreduce over the cross-host CPU transport -> allgather (intra-host kernel)
Status GpuOps::HierarchicalAllreduce(ProcessSet& ps, Entries& es, const Response& r, int device, cudaStream_t s) {
  GpuContext& ctx = GpuContext::Get();
  SymmTeam& team = *ps.local_team;
  const int L = team.nranks(), li = team.rank();
  const int64_t esz = (int64_t)DataTypeSize(r.dtype);
  std::vector<Piece> pieces;
  Status st = BuildPieces(es, r, device, s, &pieces);
  if (!st.ok()) return st;
  std::vector<kern::TensorDesc> descs;
  const int64_t total = PackDescs(pieces, esz, &descs);
  if (total == 0) return Status::OK();
  const int64_t B = Align128((total + L - 1) / L);  // shard bytes per local GPU
  char* F = (char*)ctx.TempAlloc(device, (size_t)(B * L), true, s);
  char* S = (char*)ctx.TempAlloc(device, (size_t)B, false, s);
  if (!F || !S) return Status::UnknownError("out of device memory for the hierarchical fusion buffer");
  const auto* dtab = (const kern::TensorDesc*)ctx.Stage(device, descs.data(), descs.size() * sizeof(kern::TensorDesc), s);
  if (!dtab) return Status::UnknownError("descriptor table too large");
  if (env_.timeline && env_.timeline->Initialized()) env_.timeline->ActivityStartAll(es, HVD_ACT_HIER_ALLREDUCE);
  HVD_CUDA(kern::LaunchPackUnpack(F, dtab, (int)descs.size(), total, (int)r.dtype, (int)r.dtype, r.prescale, 0, 132, s));
  // ---- 1. intra-host reduce-scatter: local GPU q ends up with block q of the host-local reduction ----
  PlanTensor fused;
  fused.in = F; fused.out = S; fused.dims = {L * B / esz};
  ReduceParams rp;
  rp.dtype = r.dtype; rp.op = r.reduce_op;
  Plan plan;
  st = PlanReducescatter(li, L, {fused}, rp, (int64_t)team.buffer_bytes(), env_.params->comm_ctas, &plan);
  if (st.ok()) st = LaunchPlan(team, device, s, plan, "hierarchical reduce-scatter");
  if (!st.ok()) return st;
  // ---- 2. cross-host allreduce of the shard (pinned staging; the CPU transport is the inter-node fabric here) ----
  char* host = (char*)ctx.PinnedHost(device, (size_t)B);
  if (!host) return Status::UnknownError("out of pinned host memory for the hierarchical shard");
  HVD_CUDA(cudaMemcpyAsync(host, S, (size_t)B, cudaMemcpyDeviceToHost, s));
  HVD_CUDA(cudaStreamSynchronize(s));
  if (team.abort_state() == 2) return Status::UnknownError("intra-host reduce-scatter timed out waiting for a peer GPU");
  cpu::Allreduce(ps.cross_transport.get(), host, B / esz, r.dtype, r.reduce_op);
  HVD_CUDA(cudaMemcpyAsync(S, host, (size_t)B, cudaMemcpyHostToDevice, s));
  // ---- 3. intra-host allgather of the shards back into the fusion buffer ----
  PlanTensor shard;
  shard.in = S; shard.out = F; shard.dims.assign(L, B);
  plan.clear();
  st = PlanAllgather(li, L, {shard}, 1, (int64_t)team.buffer_bytes(), env_.params->comm_ctas, &plan);
  if (st.ok()) st = LaunchPlan(team, device, s, plan, "hierarchical allgather");
  if (!st.ok()) return st;
  HVD_CUDA(kern::LaunchPackUnpack(F, dtab, (int)descs.size(), total, (int)r.dtype, (int)r.dtype, r.postscale, 1, 132, s));
  return Status::OK();
}

// Arguments of the zero-copy kernel for [ptr, ptr + bytes) if that range lies in a registered region of `team` (at byte
// offset `expect_off` when >= 0 — the offset every rank agreed on during negotiation).
bool GpuOps::BuildInplaceArgs(SymmTeam& team, const void* ptr, int64_t bytes, DataType dtype, ReduceOp op, double prescale,
                              double postscale, int64_t expect_off, int max_ctas, kern::InplaceArgs* out) {
  const int n = team.nranks();
  SymmTeam::RegionView view;
  int64_t off = 0;
  if (bytes <= 0 || (bytes & 15) || !team.FindRegion(ptr, (size_t)bytes, &view, &off) || (off & 15)) return false;
  if (expect_off >= 0 && expect_off != off) return false;
  if (!FillInplaceArgs(n, view.ptr, off, bytes, dtype, op, prescale, postscale, max_ctas, out)) return false;
  out->mc = view.mc ? (char*)view.mc + off : nullptr;
  // (the crossover of THIS kernel — no pack / unpack around the NVLink phase — is not the packed kernels' nvls_min_bytes)
  out->use_multicast = (out->mc && MultimemReduces(dtype, op) && env_.variant != "twoshot" && (n >= 4 || env_.variant == "nvls") &&
                        bytes >= env_.zero_copy_nvls_min_bytes) ? 1 : 0;
  return true;
}

// Collective as a CUDA-graph node: launches the zero-copy allreduce of a registered tensor on the CALLER's stream — which
// may be capturing — on the graph channel's flags, without a negotiation round.  Every rank must issue the same sequence
// of captured collectives (same tensors, same order), which is what capturing the same training step on every rank
// does; the kernel's own flag barrier is the only synchronisation, so a replayed step needs no host work at all.
// Nothing like it exists in the reference (its cycle loop negotiates every tensor every step, controller.cc:209-252).
Status GpuOps::CapturedAllreduce(ProcessSet& ps, void* ptr, int64_t bytes, DataType dtype, ReduceOp op, double prescale,
                                 double postscale, int max_ctas, cudaStream_t stream, int channel) {
  return LaunchCaptured(ps, "allreduce", kern::LaunchInplaceAllreduce, ptr, bytes, dtype, op, prescale, postscale, max_ctas, stream,
                        channel);
}

// The two halves of a sharded optimizer step, launched exactly like CapturedAllreduce (caller's stream, graph channel, no
// negotiation).  Rank r owns the contiguous slice [r*S, (r+1)*S), S = bytes / n, of the registered range.
Status GpuOps::CapturedReducescatter(ProcessSet& ps, void* ptr, int64_t bytes, DataType dtype, ReduceOp op, double prescale,
                                     double postscale, int max_ctas, cudaStream_t stream) {
  return LaunchCaptured(ps, "reducescatter", kern::LaunchInplaceReducescatter, ptr, bytes, dtype, op, prescale, postscale, max_ctas,
                        stream, kern::kGraphChannel);
}

Status GpuOps::CapturedAllgather(ProcessSet& ps, void* ptr, int64_t bytes, int max_ctas, cudaStream_t stream, int channel) {
  // a byte copy: described as an fp32 SUM so that the multicast store follows the same policy as the reductions
  return LaunchCaptured(ps, "allgather", kern::LaunchInplaceAllgather, ptr, bytes, DataType::FLOAT32, ReduceOp::SUM, 1.0, 1.0, max_ctas,
                        stream, channel);
}

// The inputs are read in place from every sender's registered region, and each rank publishes the byte offset of its own
// input with its splits, so only the region (not the offset) has to be the same on every rank.
Status GpuOps::CapturedAlltoall(ProcessSet& ps, const void* in, int64_t rows, int64_t row_bytes, const void* splits, int64_t nsplits,
                                bool splits_int64, void* out, int64_t capacity, int64_t* recv_splits, int* status, int max_ctas,
                                cudaStream_t stream) {
  const std::string name = "captured alltoall";
  std::shared_ptr<SymmTeam> team;
  { std::lock_guard<std::mutex> l(ps.team_mu); team = ps.team; }
  if (!team) return Status::PreconditionError(name + ": the process set has no peer-mapped team (allocate the tensor with hvd.symm_empty first)");
  if (team->abort_state() != 0) return Status::Aborted(name + ": the team was aborted");
  const int n = team->nranks();
  if (nsplits != n) return Status::InvalidArgument(name + ": splits must have one entry per rank of the team");
  SymmTeam::RegionView view;
  int64_t off = 0;
  if (!team->FindRegion(in, (size_t)(rows * row_bytes), &view, &off))
    return Status::InvalidArgument(name + ": tensor is not (entirely) inside registered symmetric memory");
  kern::CapturedAlltoallArgs a {};
  for (int p = 0; p < n; ++p) { a.in[p] = view.ptr[p]; a.counts[p] = team->CountRegion(p); }
  a.in_offset = off; a.rows = rows; a.capacity = capacity; a.row_bytes = row_bytes;
  a.splits = splits; a.splits_int64 = splits_int64 ? 1 : 0;
  a.out = out; a.recv_splits = recv_splits; a.status = status;
  a.ctas = std::min(max_ctas > 0 ? max_ctas : env_.params->comm_ctas, kern::kMaxCtas);
  cudaError_t ce = kern::LaunchCapturedAlltoall(team->Params(0, kern::kAlltoallChannel), a, stream);
  if (ce != cudaSuccess) return Status::UnknownError(name + " launch failed: " + cudaGetErrorString(ce));
  return Status::OK();
}

// Each rank publishes the offset of its own staging buffer, so only the region (not the offset) has to be the same on
// every rank.
Status GpuOps::CapturedUlyssesExchange(ProcessSet& ps, const void* in, void* out, const int64_t* dims, int64_t elem_bytes,
                                       int direction, bool head_first, void* staging, int64_t staging_bytes, int* status,
                                       int max_ctas, cudaStream_t stream) {
  const std::string name = "ulysses exchange";
  std::shared_ptr<SymmTeam> team;
  { std::lock_guard<std::mutex> l(ps.team_mu); team = ps.team; }
  if (!team) return Status::PreconditionError(name + ": the process set has no peer-mapped team (allocate the staging buffer with hvd.symm_empty first)");
  if (team->abort_state() != 0) return Status::Aborted(name + ": the team was aborted");
  const int n = team->nranks();
  SymmTeam::RegionView view;
  int64_t off = 0;
  if (staging_bytes <= 0 || !team->FindRegion(staging, (size_t)staging_bytes, &view, &off))
    return Status::InvalidArgument(name + ": the staging buffer is not (entirely) inside registered symmetric memory");
  kern::UlyssesArgs a {};
  for (int p = 0; p < n; ++p) { a.staging[p] = view.ptr[p]; a.counts[p] = team->CountRegion(p); }
  a.staging_offset = off; a.staging_bytes = staging_bytes;
  a.in = in; a.out = out;
  for (int k = 0; k < 5; ++k) a.dims[k] = dims[k];
  a.elem_bytes = elem_bytes; a.direction = direction; a.head_first = head_first ? 1 : 0; a.status = status;
  a.ctas = std::min(max_ctas > 0 ? max_ctas : env_.params->comm_ctas, kern::kMaxCtas);
  cudaError_t ce = kern::LaunchUlyssesExchange(team->Params(0, kern::kAlltoallChannel), a, stream);
  if (ce != cudaSuccess) return Status::UnknownError(name + " launch failed: " + cudaGetErrorString(ce));
  return Status::OK();
}

Status GpuOps::LaunchCaptured(ProcessSet& ps, const char* what, InplaceLaunch launch, void* ptr, int64_t bytes, DataType dtype,
                              ReduceOp op, double prescale, double postscale, int max_ctas, cudaStream_t stream, int channel) {
  const std::string name = std::string("captured ") + what;
  std::shared_ptr<SymmTeam> team;
  { std::lock_guard<std::mutex> l(ps.team_mu); team = ps.team; }
  if (!team) return Status::PreconditionError(name + ": the process set has no peer-mapped team (allocate the tensor with hvd.symm_empty first)");
  if (team->abort_state() != 0) return Status::Aborted(name + ": the team was aborted");
  // reducescatter and allgather split the range into one contiguous shard per rank
  if (launch != kern::LaunchInplaceAllreduce && bytes % (16 * (int64_t)team->nranks()) != 0)
    return Status::InvalidArgument(name + ": the byte size must be a multiple of 16 * the process set size");
  kern::InplaceArgs ia {};
  if (max_ctas <= 0) max_ctas = env_.params->comm_ctas;
  if (!BuildInplaceArgs(*team, ptr, bytes, dtype, op, prescale, postscale, -1, std::min(max_ctas, kern::kMaxCtas), &ia))
    return Status::InvalidArgument(name + (launch == kern::LaunchInplaceAllgather
        ? ": tensor is not (entirely) inside registered symmetric memory or is not 16 B aligned"
        : ": tensor is not (entirely) inside registered symmetric memory, is not 16 B aligned, or combines MIN/MAX/PRODUCT with scale factors"));
  cudaError_t ce = launch(team->Params(0, channel), ia, stream);
  if (ce != cudaSuccess) return Status::UnknownError(name + " launch failed: " + cudaGetErrorString(ce));
  return Status::OK();
}

// Measures, on THIS box and team, where the allreduce variants cross over (SURVEY 5.8: "variant picked per message size
// from measured bus bandwidth"): every rank runs the same short sequence of real launches on scratch tensors, rank 0's
// device-timed results decide, the decision is broadcast and cached per (GPU, team size, NVLS) so later jobs skip the
// ~10 ms measurement.  Collective over the set's transport; runs once, on the cycle thread, right after team creation.
void GpuOps::Calibrate(ProcessSet& ps, SymmTeam& team, int device) {
  Transport* t = ps.transport.get();
  const int n = team.nranks(), me = t->rank();
  if (n < 2) return;
  cudaDeviceProp prop {};
  cudaGetDeviceProperties(&prop, device);
  std::string gpu = prop.name;
  for (auto& c : gpu) if (!isalnum((unsigned char)c)) c = '_';
  const char* home = getenv("HOME");
  const std::string dir = EnvStr("HVD_CACHE_DIR", std::string(home ? home : "/tmp") + "/.cache/horovod_b200");
  const std::string path = dir + "/crossover_v2_" + gpu + "_n" + std::to_string(n) + "_mc" + (team.has_multicast() ? "1" : "0") + ".txt";
  int64_t vals[3] = {0, 0, 0};  // found, oneshot_max_bytes, nvls_min_bytes
  if (me == 0 && EnvBool("HVD_CALIBRATION_CACHE", true)) {
    if (FILE* f = fopen(path.c_str(), "r")) {
      long long a = 0, b = 0;
      if (fscanf(f, "%lld %lld", &a, &b) == 2 && a >= 0 && b >= 0) { vals[0] = 1; vals[1] = a; vals[2] = b; }
      fclose(f);
    }
  }
  t->Bcast(vals, sizeof vals, 0);
  if (!vals[0]) {
    GpuContext& ctx = GpuContext::Get();
    cudaStream_t s = ctx.Stream(device);
    const std::vector<int64_t> sizes = {32 << 10, 128 << 10, 512 << 10, 2 << 20, 8 << 20, 32 << 20};
    const int64_t maxb = std::min<int64_t>(sizes.back(), (int64_t)team.buffer_bytes() / 128 * 128);
    char* buf = nullptr;
    const bool mem_ok = cudaMalloc((void**)&buf, (size_t)maxb) == cudaSuccess;
    uint64_t okw = mem_ok ? 1 : 0;
    t->AllreduceBits(&okw, 1, nullptr, 0);
    if (!okw) { if (buf) cudaFree(buf); cudaGetLastError(); return; }
    cudaMemsetAsync(buf, 0, (size_t)maxb, s);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    const bool nvls_ok = team.has_multicast() && n >= 4;
    const int variants[3] = {kern::kOneShot, kern::kTwoShot, kern::kNvls};
    std::vector<double> us(sizes.size() * 3, 1e30);
    for (size_t si = 0; si < sizes.size(); ++si) {
      const int64_t bytes = std::min(sizes[si], maxb);
      for (int vi = 0; vi < 3; ++vi) {
        if (variants[vi] == kern::kNvls && !nvls_ok) continue;
        kern::AllreduceArgs a {};
        a.ndesc = 1; a.descs = nullptr;
        a.inline_descs[0].in = buf; a.inline_descs[0].out = buf; a.inline_descs[0].offset = 0; a.inline_descs[0].count = bytes / 4;
        a.total_bytes = bytes; a.reduce_lo = 0; a.reduce_hi = bytes;
        a.prescale = 1.0; a.postscale = 1.0; a.op = (int)ReduceOp::SUM; a.dtype = (int)DataType::FLOAT32; a.wire_dtype = (int)DataType::FLOAT32;
        a.variant = variants[vi];
        a.ctas = CtasFor(a.variant, bytes, n, env_.params->comm_ctas, env_.large_msg_ctas);
        const int warm = 2, iters = 6;
        bool ok = true;
        for (int it = 0; it < warm + iters && ok; ++it) {
          if (it == warm) cudaEventRecord(e0, s);
          ok = kern::LaunchAllreduce(team.Params(team.NextSlot()), a, s) == cudaSuccess;
        }
        cudaEventRecord(e1, s);
        if (cudaStreamSynchronize(s) != cudaSuccess || !ok) { cudaGetLastError(); continue; }
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        us[si * 3 + vi] = ms * 1e3 / iters;
      }
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    cudaFree(buf);
    // a barrier that timed out on ANY rank voids the measurement everywhere (collective decision: nobody may skip the
    // broadcast below on its own); the defaults stay and the next real op reports the failure
    uint64_t healthy = team.abort_state() == 0 ? 1 : 0;
    t->AllreduceBits(&healthy, 1, nullptr, 0);
    if (!healthy) return;
    if (me == 0) {
      int64_t oneshot_max = 0, nvls_min = 0;
      bool nvls_found = false;
      std::ostringstream tab;
      for (size_t si = 0; si < sizes.size(); ++si) {
        const double t1 = us[si * 3], t2 = us[si * 3 + 1], t3 = us[si * 3 + 2];
        tab << " " << (sizes[si] >> 10) << "K:" << (int)(t1 + 0.5) << "/" << (int)(t2 + 0.5) << "/" << (t3 > 1e29 ? -1 : (int)(t3 + 0.5));
        if (oneshot_max == (si ? sizes[si - 1] : 0) && t1 <= std::min(t2, t3) * 1.03) oneshot_max = sizes[si];  // contiguous prefix
        if (!nvls_found && t3 < 1e29 && t3 <= t2) { nvls_min = sizes[si]; nvls_found = true; }
      }
      if (!nvls_found) nvls_min = nvls_ok ? (64ll << 20) : (1ll << 60);  // not faster in the measured range / unavailable
      if (oneshot_max == 0) oneshot_max = 4096;
      vals[1] = oneshot_max; vals[2] = nvls_min;
      LOG(INFO) << "allreduce variant calibration on " << n << " x " << prop.name << " (us one-shot/two-shot/NVLS):" << tab.str()
                << " -> one-shot up to " << oneshot_max << " B, NVLS from " << nvls_min << " B";
      if (EnvBool("HVD_CALIBRATION_CACHE", true)) {
        std::string cmd_dir = dir;
        for (size_t i = 1; i <= cmd_dir.size(); ++i)
          if (i == cmd_dir.size() || cmd_dir[i] == '/') { std::string sub = cmd_dir.substr(0, i); mkdir(sub.c_str(), 0755); }
        if (FILE* f = fopen((path + ".tmp").c_str(), "w")) {
          fprintf(f, "%lld %lld\n", (long long)oneshot_max, (long long)nvls_min);
          fclose(f);
          rename((path + ".tmp").c_str(), path.c_str());
        }
      }
    }
    t->Bcast(vals, sizeof vals, 0);
  }
  if (env_.on_calibrated) env_.on_calibrated(vals[1], vals[2]);
}

std::string GpuOps::Describe(ProcessSet& ps) {
  if (!ps.team_tried) return "backend=" + env_.backend + " (no GPU collective issued yet)";
  if (!ps.team && ps.local_team) return "backend=hierarchical intra-host symm=" + ps.local_team->backend() + " cross-host=cpu-transport";
  if (!ps.team) return "backend=host-staged";
  return "backend=" + env_.backend + " symm=" + ps.team->backend() + " buffer=" + std::to_string(ps.team->buffer_bytes());
}

// ---------------------------------------------------------------------------
// allreduce

Status GpuOps::Allreduce(ProcessSet& ps, Entries& es, const Response& r, int device, SharedEvent** done) {
  const int n = ps.set_size();
  HVD_CUDA(cudaSetDevice(device));
  GpuContext& ctx = GpuContext::Get();
  cudaStream_t s = ctx.Stream(device);
  // ---- latency lane: a small response does not queue behind a 256 MiB one.  Responses of at most latency_lane_bytes
  // (decided from the negotiated sizes, i.e. identically on every rank) run on their own stream, barrier channel and
  // reserved tail of the symmetric buffers (the role of the reference's HOROVOD_NUM_NCCL_STREAMS rotation,
  // gpu_operations.cc:138-141, made deterministic across ranks) ----
  bool lat_lane = false;
  if (env_.latency_lane_bytes > 0 && n > 1 && env_.backend == "p2p" && r.symm_key == -1 && r.type == ResponseType::ALLREDUCE) {
    int64_t total = 0;
    for (auto c : r.tensor_sizes) total += Align128(c * (int64_t)DataTypeSize(r.dtype));
    lat_lane = total > 0 && total <= env_.latency_lane_bytes;
  }
  if (lat_lane) s = ctx.LatencyStream(device);
  WaitReady(es, s);
  std::vector<Piece> pieces;
  Status st = BuildPieces(es, r, device, s, &pieces);
  if (!st.ok()) return st;
  const size_t esz = DataTypeSize(r.dtype);

  if (n == 1) {
    const double sc = r.prescale * r.postscale;
    for (auto& p : pieces) {
      if (p.in != p.out || sc != 1.0) HVD_CUDA(kern::LaunchScale(p.in, p.out, p.count, (int)r.dtype, sc, s));
    }
  } else if (env_.backend == "nccl") {
    st = NcclAllreduce(ps, es, r, device, s);
    if (!st.ok()) return st;
  } else {
    std::shared_ptr<SymmTeam> team = env_.backend == "cpu" ? nullptr : EnsureTeam(ps, device);
    if (!team) {
      st = (env_.backend != "cpu" && EnsureHierarchy(ps, device)) ? HierarchicalAllreduce(ps, es, r, device, s)
                                                                   : StagedOnHost(ps, es, r, device, s);
      if (!st.ok()) return st;
    } else {
      // ---- zero-copy path: the tensor lives in registered symmetric memory on EVERY rank (negotiated symm_key) ----
      const int64_t zc_bytes = pieces.size() == 1 ? pieces[0].count * (int64_t)esz : 0;
      if (r.symm_key >= 0 && pieces.size() == 1 && es[0] && zc_bytes > env_.params->oneshot_max_bytes && env_.variant != "oneshot") {
        kern::InplaceArgs ia {};
        if (BuildInplaceArgs(*team, pieces[0].in, zc_bytes, r.dtype, r.reduce_op, r.prescale, r.postscale,
                             (int64_t)(r.symm_key & ((1ll << 44) - 1)), env_.params->comm_ctas, &ia)) {
          kern::CommParams cp = team->Params(team->NextSlot());
          if (env_.timeline && env_.timeline->Initialized())
            env_.timeline->ActivityStartAll(es, ia.use_multicast ? HVD_ACT_P2P_ALLREDUCE_NVLS : HVD_ACT_P2P_ALLREDUCE_TWOSHOT);
          cudaError_t ce = kern::LaunchInplaceAllreduce(cp, ia, s);
          if (ce != cudaSuccess) return Status::UnknownError(std::string("zero-copy allreduce launch failed: ") + cudaGetErrorString(ce));
          ctx.TempFreeAll(device, s);
          return FinishEvent(device, s, es.size(), done);
        }
      }
      // ---- plain tensor, in place, IPC-registrable on every rank (negotiated symm_key == -2): zero-copy P2P two-shot on
      //      the peers' mappings of each other's ordinary allocations ----
      if (r.symm_key == -2 && pieces.size() == 1 && es[0] && pieces[0].in == pieces[0].out && env_.variant != "oneshot") {
        const bool nvls_better = MultimemReduces(r.dtype, r.reduce_op) && team->has_multicast() && n > env_.ipc_max_ranks;
        if (!nvls_better) {
          if (!ps.ipc) ps.ipc = std::make_shared<IpcRegistry>();
          const int64_t bytes = pieces[0].count * (int64_t)esz;
          // fresh response (same on every rank): the collective moment to (re)exchange handles; cached response: no rank's
          // tensor moved since the exchange recorded under this name (a moved tensor invalidates the cache entry)
          const IpcRegistry::Entry* ent = r.from_cache ? ps.ipc->Find(es[0]->name)
                                                       : &ps.ipc->Exchange(ps.transport.get(), es[0]->name, pieces[0].in, (size_t)bytes);
          if (ent && ent->my_ptr != pieces[0].in) ent = nullptr;
          kern::InplaceArgs ia {};
          if (ent && ent->usable &&
              FillInplaceArgs(n, ent->ptr, 0, bytes, r.dtype, r.reduce_op, r.prescale, r.postscale, env_.params->comm_ctas, &ia)) {
            kern::CommParams cp = team->Params(team->NextSlot());
            if (env_.timeline && env_.timeline->Initialized()) env_.timeline->ActivityStartAll(es, HVD_ACT_P2P_ALLREDUCE_TWOSHOT);
            cudaError_t ce = kern::LaunchInplaceAllreduce(cp, ia, s);
            if (ce == cudaSuccess) {
              ipc_launches_.fetch_add(1, std::memory_order_relaxed);
              ctx.TempFreeAll(device, s);
              return FinishEvent(device, s, es.size(), done);
            }
            cudaGetLastError();  // e.g. a dtype the in-place kernel does not implement: fall through to the packed path
          }
        }
      }
      // wire dtype: optional in-kernel compression of fp32 sums
      DataType wire = r.dtype;
      if (r.dtype == DataType::FLOAT32 && (env_.wire_dtype == DataType::BFLOAT16 || env_.wire_dtype == DataType::FLOAT16) &&
          (r.reduce_op == ReduceOp::SUM || r.reduce_op == ReduceOp::AVERAGE))
        wire = env_.wire_dtype;
      // the tail of each buffer slot (reserved when the team was created) belongs to the latency lane
      const int64_t lat_area = (int64_t)team->reserved_tail();
      if (lat_lane && lat_area < env_.latency_lane_bytes) lat_lane = false;  // tiny buffers: no reserved tail (same on every rank)
      std::vector<PlanTensor> ts(pieces.size());
      for (size_t i = 0; i < pieces.size(); ++i) { ts[i].in = pieces[i].in; ts[i].out = pieces[i].out; ts[i].dims = {pieces[i].count}; }
      ReduceParams rp;
      rp.dtype = r.dtype; rp.op = r.reduce_op; rp.prescale = r.prescale; rp.postscale = r.postscale;
      AllreducePolicy pol;
      pol.variant = env_.variant;
      pol.oneshot_max_bytes = env_.params->oneshot_max_bytes;
      pol.multicast = team->has_multicast();
      pol.nvls_min_bytes = env_.params->nvls_min_bytes;
      pol.large_msg_ctas = env_.large_msg_ctas;
      Plan plan;
      st = PlanAllreduce(n, ts, rp, wire, pol, lat_lane ? lat_area : (int64_t)team->buffer_bytes(), env_.params->comm_ctas, &plan);
      if (st.ok()) st = LaunchPlan(*team, device, s, plan, "allreduce", &es, lat_lane);
      if (!st.ok()) return st;
    }
  }
  ctx.TempFreeAll(device, s);
  return FinishEvent(device, s, es.size(), done);
}

Status GpuOps::NcclAllreduce(ProcessSet& ps, Entries& es, const Response& r, int device, cudaStream_t s) {
  if (!ps.nccl_tried) {
    ps.nccl_tried = true;
    std::string why;
    ps.nccl = NcclCreateComm(ps.transport.get(), device, &why);
    if (!ps.nccl) LOG(WARNING) << "NCCL baseline unavailable: " << why;
  }
  if (!ps.nccl || !NcclSupportsDtype(r.dtype)) return StagedOnHost(ps, es, r, device, s);  // e.g. int16: NCCL has no such type
  GpuContext& ctx = GpuContext::Get();
  const size_t esz = DataTypeSize(r.dtype);
  std::vector<Piece> pieces;
  Status st = BuildPieces(es, r, device, s, &pieces);
  if (!st.ok()) return st;
  if (pieces.size() == 1) {
    // unfused: optional prescale kernel, ncclAllReduce(input -> output), optional postscale kernel
    // (reference nccl_operations.cc:238-283)
    const Piece& p = pieces[0];
    const void* in = p.in;
    if (r.prescale != 1.0) { HVD_CUDA(kern::LaunchScale(p.in, p.out, p.count, (int)r.dtype, r.prescale, s)); in = p.out; }
    st = NcclAllReduceCall(*ps.nccl, in, p.out, p.count, r.dtype, r.reduce_op, s);
    if (!st.ok()) return st;
    if (r.postscale != 1.0) HVD_CUDA(kern::LaunchScale(p.out, p.out, p.count, (int)r.dtype, r.postscale, s));
    return Status::OK();
  }
  // fused: scaled pack -> ncclAllReduce in place on the fusion buffer -> scaled unpack
  std::vector<kern::TensorDesc> descs;
  const int64_t total = PackDescs(pieces, (int64_t)esz, &descs);
  char* fusion = (char*)ctx.TempAlloc(device, (size_t)total, false, s);
  if (!fusion) return Status::UnknownError("out of device memory for the NCCL fusion buffer");
  const auto* dtab = (const kern::TensorDesc*)ctx.Stage(device, descs.data(), descs.size() * sizeof(kern::TensorDesc), s);
  if (!dtab) return Status::UnknownError("descriptor table too large");
  HVD_CUDA(kern::LaunchPackUnpack(fusion, dtab, (int)descs.size(), total, (int)r.dtype, (int)r.dtype, r.prescale, 0, 132, s));
  st = NcclAllReduceCall(*ps.nccl, fusion, fusion, total / (int64_t)esz, r.dtype, r.reduce_op, s);
  if (!st.ok()) return st;
  HVD_CUDA(kern::LaunchPackUnpack(fusion, dtab, (int)descs.size(), total, (int)r.dtype, (int)r.dtype, r.postscale, 1, 132, s));
  return Status::OK();
}

// Host-staged fallback (multi-host sets, no peer access): D2H, CPU collective, H2D.
Status GpuOps::StagedOnHost(ProcessSet& ps, Entries& es, const Response& r, int device, cudaStream_t s) {
  const size_t esz = DataTypeSize(r.dtype);
  std::vector<Piece> pieces;
  Status st = BuildPieces(es, r, device, s, &pieces);
  if (!st.ok()) return st;
  int64_t total = 0;
  for (auto& p : pieces) total += p.count;
  std::vector<char> host((size_t)total * esz);
  int64_t off = 0;
  for (auto& p : pieces) { HVD_CUDA(cudaMemcpyAsync(host.data() + off * esz, p.in, (size_t)p.count * esz, cudaMemcpyDeviceToHost, s)); off += p.count; }
  HVD_CUDA(cudaStreamSynchronize(s));
  cpu::ScaleBuffer(host.data(), total, r.dtype, r.prescale);
  cpu::Allreduce(ps.transport.get(), host.data(), total, r.dtype, r.reduce_op);
  cpu::ScaleBuffer(host.data(), total, r.dtype, r.postscale);
  off = 0;
  for (auto& p : pieces) { HVD_CUDA(cudaMemcpyAsync(p.out, host.data() + off * esz, (size_t)p.count * esz, cudaMemcpyHostToDevice, s)); off += p.count; }
  HVD_CUDA(cudaStreamSynchronize(s));  // `host` dies with this frame
  return Status::OK();
}

// ---------------------------------------------------------------------------
// reducescatter: the fused buffer is laid out destination-rank major — region q holds block q of EVERY tensor of the
// (fused) response — so each rank reduces one contiguous range straight into its output tensors: one launch per fused
// response (one-shot P2P loads, or multimem.ld_reduce in the switch).  The reference packs a rank-interleaved fusion
// buffer, calls ncclReduceScatter and unpacks (gpu_operations.cc:655-928, nccl_operations.cc:1221-1346).

Status GpuOps::Reducescatter(ProcessSet& ps, Entries& es, const Response& r, int device, SharedEvent** done) {
  const int me = ps.set_rank(), n = ps.set_size();
  HVD_CUDA(cudaSetDevice(device));
  GpuContext& ctx = GpuContext::Get();
  cudaStream_t s = ctx.Stream(device);
  WaitReady(es, s);
  const int64_t esz = (int64_t)DataTypeSize(r.dtype);
  struct Item { TensorTableEntry* e; std::vector<int64_t> cnt, boff; };  // per-destination block: elements, element offset
  std::vector<Item> items(es.size());
  for (size_t ti = 0; ti < es.size(); ++ti) {
    auto& e = es[ti];
    if (!e) return Status::PreconditionError("Reducescatter is not supported with Join at this time.");
    const int64_t dim0 = e->shape.dim(0);
    int64_t row = 1;
    for (int d = 1; d < e->shape.ndim(); ++d) row *= e->shape.dim(d);
    std::vector<int64_t> rows;
    ReducescatterRows(dim0, n, &rows);
    Item& it = items[ti];
    it.e = e.get(); it.cnt.assign(n, 0); it.boff.assign(n + 1, 0);
    for (int i = 0; i < n; ++i) { it.cnt[i] = rows[i] * row; it.boff[i + 1] = it.boff[i] + it.cnt[i]; }
    if (!e->output) {
      std::vector<int64_t> oshape = e->shape.dims();
      oshape[0] = rows[me];
      e->output = e->alloc_output ? e->alloc_output(oshape) : nullptr;
      if (!e->output && it.cnt[me] > 0) return Status::UnknownError("reducescatter: output allocation failed");
    }
  }
  if (n == 1) {
    const double sc = r.prescale * r.postscale;
    for (auto& it : items)
      if (it.e->input != it.e->output || sc != 1.0) HVD_CUDA(kern::LaunchScale(it.e->input, it.e->output, it.boff[n], (int)r.dtype, sc, s));
    return FinishEvent(device, s, es.size(), done);
  }
  std::shared_ptr<SymmTeam> team = (env_.backend == "cpu") ? nullptr : EnsureTeam(ps, device);
  if (!team) {
    for (auto& it : items) {
      std::vector<char> host((size_t)(it.boff[n] * esz)), out((size_t)(it.cnt[me] * esz));
      HVD_CUDA(cudaMemcpyAsync(host.data(), it.e->input, host.size(), cudaMemcpyDeviceToHost, s));
      HVD_CUDA(cudaStreamSynchronize(s));
      cpu::ScaleBuffer(host.data(), it.boff[n], r.dtype, r.prescale);
      cpu::Reducescatter(ps.transport.get(), host.data(), it.cnt, out.data(), r.dtype, r.reduce_op);
      cpu::ScaleBuffer(out.data(), it.cnt[me], r.dtype, r.postscale);
      HVD_CUDA(cudaMemcpyAsync(it.e->output, out.data(), out.size(), cudaMemcpyHostToDevice, s));
      HVD_CUDA(cudaStreamSynchronize(s));
    }
    return FinishEvent(device, s, es.size(), done);
  }
  std::vector<PlanTensor> ts(items.size());
  for (size_t ti = 0; ti < items.size(); ++ti) {
    auto* e = items[ti].e;
    int64_t row = 1;
    for (int d = 1; d < e->shape.ndim(); ++d) row *= e->shape.dim(d);
    ts[ti].in = e->input; ts[ti].out = e->output; ts[ti].row = row; ts[ti].dims = {e->shape.dim(0)};
  }
  ReduceParams rp;
  rp.dtype = r.dtype; rp.op = r.reduce_op; rp.prescale = r.prescale; rp.postscale = r.postscale;
  rp.nvls = team->has_multicast() && MultimemReduces(r.dtype, r.reduce_op) && n >= 4 && env_.variant != "oneshot" &&
            env_.variant != "twoshot";
  rp.nvls_min_bytes = env_.params->nvls_min_bytes;
  Plan plan;
  Status st = PlanReducescatter(me, n, ts, rp, (int64_t)team->buffer_bytes(), (int)env_.params->comm_ctas, &plan);
  if (st.ok()) st = LaunchPlan(*team, device, s, plan, "reducescatter");
  if (!st.ok()) return st;
  ctx.TempFreeAll(device, s);
  return FinishEvent(device, s, es.size(), done);
}

// ---------------------------------------------------------------------------
// allgather / broadcast / alltoall through the exchange kernel

namespace {
Status StageAndLaunchExchange(SymmTeam& team, GpuContext& ctx, int device, cudaStream_t s, const std::vector<kern::CopyDesc>& sends,
                              const std::vector<kern::CopyDesc>& recvs, int ctas) {
  std::vector<kern::CopyDesc> table(sends);
  table.insert(table.end(), recvs.begin(), recvs.end());
  kern::ExchangeArgs a {};
  const kern::CopyDesc* dt = table.empty() ? nullptr
      : (const kern::CopyDesc*)ctx.Stage(device, table.data(), table.size() * sizeof(kern::CopyDesc), s);
  if (!table.empty() && !dt) return Status::UnknownError("descriptor table too large");
  a.sends = dt; a.nsend = (int)sends.size();
  a.recvs = dt ? dt + sends.size() : nullptr; a.nrecv = (int)recvs.size();
  a.ctas = ctas;
  kern::CommParams cp = team.Params(team.NextSlot());
  cudaError_t ce = kern::LaunchExchange(cp, a, s);
  if (ce != cudaSuccess) return Status::UnknownError(std::string("exchange kernel launch failed: ") + cudaGetErrorString(ce));
  return Status::OK();
}

}  // namespace

Status GpuOps::LaunchPlan(SymmTeam& team, int device, cudaStream_t s, const Plan& plan, const char* what, Entries* es,
                          bool latency_lane) {
  GpuContext& ctx = GpuContext::Get();
  for (const PlanLaunch& l : plan) {
    if (!l.reduce) {
      Status st = StageAndLaunchExchange(team, ctx, device, s, l.sends, l.recvs, l.ctas);
      if (!st.ok()) return st;
      continue;
    }
    kern::AllreduceArgs a = l.args;
    a.ctas = l.ctas;
    if (InlineDescs(a)) {
      memcpy(a.inline_descs, l.table.data(), l.table.size() * sizeof(kern::TensorDesc));  // no staging: small responses are latency bound
    } else {
      const auto* dt = (const kern::TensorDesc*)ctx.Stage(device, l.table.data(), l.table.size() * sizeof(kern::TensorDesc), s);
      if (!dt) return Status::UnknownError("descriptor table too large");
      a.descs = dt;
      a.out_descs = a.nout ? dt + a.ndesc : nullptr;
    }
    kern::CommParams cp = latency_lane ? team.Params(team.NextLatencySlot(), kern::kLatencyChannel, (int64_t)team.buffer_bytes())
                                       : team.Params(team.NextSlot());
    if (es && env_.timeline && env_.timeline->Initialized())
      env_.timeline->ActivityStartAll(*es, a.variant == kern::kOneShot ? HVD_ACT_P2P_ALLREDUCE_ONESHOT
                                           : a.variant == kern::kNvls ? HVD_ACT_P2P_ALLREDUCE_NVLS : HVD_ACT_P2P_ALLREDUCE_TWOSHOT);
    cudaError_t ce = kern::LaunchAllreduce(cp, a, s);
    if (ce != cudaSuccess) return Status::UnknownError(std::string(what) + " kernel launch failed: " + cudaGetErrorString(ce));
  }
  return Status::OK();
}

// A fused allgather response (several tensors, per-rank first dims in r.tensor_sizes) is ONE exchange launch: every rank
// packs its blocks of all tensors back to back into its symmetric buffer and pulls every peer's blocks straight into the
// output tensors.  The reference packs into a fusion buffer, calls ncclAllGather and unpacks (gpu_operations.cc:441-632,
// nccl_operations.cc:906-1133).
Status GpuOps::Allgather(ProcessSet& ps, Entries& es, const Response& r, int device, SharedEvent** done) {
  const int me = ps.set_rank(), n = ps.set_size();
  HVD_CUDA(cudaSetDevice(device));
  GpuContext& ctx = GpuContext::Get();
  cudaStream_t s = ctx.Stream(device);
  WaitReady(es, s);
  const int64_t esz = (int64_t)DataTypeSize(r.dtype);
  struct Item { TensorTableEntry* e; std::vector<int64_t> bytes, displ; };
  std::vector<Item> items(es.size());
  for (size_t ti = 0; ti < es.size(); ++ti) {
    auto& e = es[ti];
    if (!e) return Status::PreconditionError("Allgather is not supported with Join at this time.");
    int64_t row = 1;
    for (int d = 1; d < e->shape.ndim(); ++d) row *= e->shape.dim(d);
    Item& it = items[ti];
    it.e = e.get(); it.bytes.assign(n, 0); it.displ.assign(n + 1, 0);
    int64_t total_rows = 0;
    for (int p = 0; p < n; ++p) {
      int64_t d0 = r.tensor_sizes[ti * n + p];
      it.bytes[p] = d0 * row * esz;
      it.displ[p + 1] = it.displ[p] + it.bytes[p];
      total_rows += d0;
    }
    std::vector<int64_t> oshape = e->shape.dims();
    oshape[0] = total_rows;
    e->output = e->alloc_output ? e->alloc_output(oshape) : e->output;
    if (!e->output && it.displ[n] > 0) return Status::UnknownError("allgather: output allocation failed");
  }
  if (n == 1) {
    for (auto& it : items) if (it.bytes[0]) HVD_CUDA(cudaMemcpyAsync(it.e->output, it.e->input, (size_t)it.bytes[0], cudaMemcpyDeviceToDevice, s));
    return FinishEvent(device, s, es.size(), done);
  }
  std::shared_ptr<SymmTeam> team = (env_.backend == "cpu") ? nullptr : EnsureTeam(ps, device);
  if (!team) {
    for (auto& it : items) {
      std::vector<char> host((size_t)it.displ[n]);
      if (it.bytes[me]) HVD_CUDA(cudaMemcpyAsync(host.data() + it.displ[me], it.e->input, (size_t)it.bytes[me], cudaMemcpyDeviceToHost, s));
      HVD_CUDA(cudaStreamSynchronize(s));
      cpu::Allgatherv(ps.transport.get(), host.data() + it.displ[me], host.data(), it.bytes);
      if (it.displ[n]) HVD_CUDA(cudaMemcpyAsync(it.e->output, host.data(), (size_t)it.displ[n], cudaMemcpyHostToDevice, s));
      HVD_CUDA(cudaStreamSynchronize(s));
    }
    return FinishEvent(device, s, es.size(), done);
  }
  std::vector<PlanTensor> ts(items.size());
  for (size_t ti = 0; ti < items.size(); ++ti) {
    auto* e = items[ti].e;
    int64_t row = 1;
    for (int d = 1; d < e->shape.ndim(); ++d) row *= e->shape.dim(d);
    ts[ti].in = e->input; ts[ti].out = e->output; ts[ti].row = row;
    ts[ti].dims.assign(r.tensor_sizes.begin() + ti * n, r.tensor_sizes.begin() + (ti + 1) * n);
  }
  Plan plan;
  Status st = PlanAllgather(me, n, ts, esz, (int64_t)team->buffer_bytes(), (int)env_.params->comm_ctas, &plan);
  if (st.ok()) st = LaunchPlan(*team, device, s, plan, "allgather");
  if (!st.ok()) return st;
  return FinishEvent(device, s, es.size(), done);
}

// Broadcast responses of one root are fused by the controller; a fused response is ONE launch.  With NVLS the root
// stores through the multicast mapping (multimem.st: one source read, one egress stream, the switch replicates) and
// every rank copies out of its OWN buffer; without it the peers pull from the root's buffer.
Status GpuOps::Broadcast(ProcessSet& ps, Entries& es, const Response& r, int device, SharedEvent** done) {
  const int me = ps.set_rank(), n = ps.set_size();
  HVD_CUDA(cudaSetDevice(device));
  GpuContext& ctx = GpuContext::Get();
  cudaStream_t s = ctx.Stream(device);
  WaitReady(es, s);
  const int root = r.root_rank;
  for (auto& e : es) if (!e) return Status::PreconditionError("Broadcast is not supported with Join at this time.");
  std::shared_ptr<SymmTeam> team = (n == 1 || env_.backend == "cpu") ? nullptr : EnsureTeam(ps, device);
  if (!team) {
    for (auto& e : es) {
      const int64_t bytes = (int64_t)e->bytes();
      if (n == 1 || bytes == 0) {
        if (e->output && e->output != e->input && bytes) HVD_CUDA(cudaMemcpyAsync(e->output, e->input, (size_t)bytes, cudaMemcpyDeviceToDevice, s));
        continue;
      }
      std::vector<char> host((size_t)bytes);
      if (me == root) { HVD_CUDA(cudaMemcpyAsync(host.data(), e->input, (size_t)bytes, cudaMemcpyDeviceToHost, s)); }
      HVD_CUDA(cudaStreamSynchronize(s));
      cpu::Broadcast(ps.transport.get(), host.data(), bytes, root);
      if (me != root || e->output != e->input) HVD_CUDA(cudaMemcpyAsync(e->output, host.data(), (size_t)bytes, cudaMemcpyHostToDevice, s));
      HVD_CUDA(cudaStreamSynchronize(s));
    }
    return FinishEvent(device, s, es.size(), done);
  }
  const bool use_mc = env_.broadcast_multicast && team->has_multicast() && n > 2;
  std::vector<PlanTensor> ts(es.size());
  for (size_t ti = 0; ti < es.size(); ++ti) {
    ts[ti].in = es[ti]->input; ts[ti].out = es[ti]->output; ts[ti].dims = {(int64_t)es[ti]->bytes()};
  }
  Plan plan;
  Status st = PlanBroadcast(me, n, root, ts, use_mc, (int64_t)team->buffer_bytes(), (int)env_.params->comm_ctas, &plan);
  if (st.ok()) st = LaunchPlan(*team, device, s, plan, "broadcast");
  if (!st.ok()) return st;
  return FinishEvent(device, s, es.size(), done);
}

Status GpuOps::Alltoall(ProcessSet& ps, Entries& es, const Response& r, int device, SharedEvent** done) {
  const int me = ps.set_rank(), n = ps.set_size();
  HVD_CUDA(cudaSetDevice(device));
  GpuContext& ctx = GpuContext::Get();
  cudaStream_t s = ctx.Stream(device);
  WaitReady(es, s);
  const int64_t esz = (int64_t)DataTypeSize(r.dtype);
  for (auto& e : es) {
    if (!e) return Status::PreconditionError("Alltoall is not supported with Join at this time.");
    int64_t row = 1;
    for (int d = 1; d < e->shape.ndim(); ++d) row *= e->shape.dim(d);
    // exchange the split matrix through the control plane (reference: AlltoallGetRecvSplits)
    std::vector<int64_t> mine(n), all((size_t)n * n);
    for (int p = 0; p < n; ++p) mine[p] = e->splits[p];
    if (r.root_rank == kUniformSplits) std::fill(all.begin(), all.end(), mine[0]);  // negotiated uniform splits: nothing to exchange
    else ps.transport->AllgatherInts(mine.data(), n, all.data());
    std::vector<int64_t> sbytes(n), rbytes(n), sdisp(n + 1, 0), rdisp(n + 1, 0);
    e->received_splits.assign(n, 0);
    int64_t out_rows = 0;
    for (int p = 0; p < n; ++p) {
      sbytes[p] = mine[p] * row * esz;
      e->received_splits[p] = (int32_t)all[(size_t)p * n + me];
      rbytes[p] = all[(size_t)p * n + me] * row * esz;
      sdisp[p + 1] = sdisp[p] + sbytes[p];
      rdisp[p + 1] = rdisp[p] + rbytes[p];
      out_rows += all[(size_t)p * n + me];
    }
    std::vector<int64_t> oshape = e->shape.dims();
    oshape[0] = out_rows;
    e->output = e->alloc_output ? e->alloc_output(oshape) : e->output;
    if (!e->output && rdisp[n] > 0) return Status::UnknownError("alltoall: output allocation failed");
    if (n == 1) { if (sbytes[0]) HVD_CUDA(cudaMemcpyAsync(e->output, e->input, (size_t)sbytes[0], cudaMemcpyDeviceToDevice, s)); continue; }
    std::shared_ptr<SymmTeam> team = (env_.backend == "cpu") ? nullptr : EnsureTeam(ps, device);
    if (!team) {
      std::vector<char> hin((size_t)sdisp[n]), hout((size_t)rdisp[n]);
      if (sdisp[n]) HVD_CUDA(cudaMemcpyAsync(hin.data(), e->input, (size_t)sdisp[n], cudaMemcpyDeviceToHost, s));
      HVD_CUDA(cudaStreamSynchronize(s));
      cpu::Alltoallv(ps.transport.get(), hin.data(), sbytes, hout.data(), rbytes);
      if (rdisp[n]) HVD_CUDA(cudaMemcpyAsync(e->output, hout.data(), (size_t)rdisp[n], cudaMemcpyHostToDevice, s));
      HVD_CUDA(cudaStreamSynchronize(s));
      continue;
    }
    PlanTensor t;
    t.in = e->input; t.out = e->output; t.row = row; t.dims = all;
    Plan plan;
    Status st = PlanAlltoall(me, n, {t}, esz, (int64_t)team->buffer_bytes(), (int)env_.params->comm_ctas, &plan);
    if (st.ok()) st = LaunchPlan(*team, device, s, plan, "alltoall");
    if (!st.ok()) return st;
  }
  return FinishEvent(device, s, es.size(), done);
}

}  // namespace hvd
