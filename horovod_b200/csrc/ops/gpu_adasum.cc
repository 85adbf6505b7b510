// GPU Adasum.  The reference's "GPU Adasum" on one node is an NCCL sum divided
// by local_size (ops/adasum_gpu_operations.cc:169-275, operations.cc:1459-1466);
// the real pairwise reduction only runs on the CPU across nodes.  Here the true
// VHDD Adasum runs for GPU tensors as well: on a peer-mapped team through the
// sm_90a kernels in kernels/adasum_kernels.cu, otherwise staged through the
// host implementation (cpu::AdasumAllreduce, the numerical oracle).
#include <cstring>
#include "../common/logging.h"
#include "../kernels/p2p_kernels.h"
#include "../symm/symm_memory.h"
#include "cpu_ops.h"
#include "gpu_ops.h"

namespace hvd {

#define HVD_CUDA(call)                                                                      \
  do {                                                                                      \
    cudaError_t _e = (call);                                                                \
    if (_e != cudaSuccess) return Status::UnknownError(std::string(#call) + " failed: " + cudaGetErrorString(_e)); \
  } while (0)

Status GpuOps::Adasum(ProcessSet& ps, Entries& es, const Response& r, int device, SharedEvent** done) {
  const int n = ps.set_size();
  HVD_CUDA(cudaSetDevice(device));
  GpuContext& ctx = GpuContext::Get();
  cudaStream_t s = ctx.Stream(device);
  for (auto& e : es) if (e && e->ready_event) cudaStreamWaitEvent(s, (cudaEvent_t)e->ready_event, 0);
  if (n & (n - 1)) return Status::PreconditionError("Running Adasum with non-power-of-2 ranks is not supported yet.");
  const size_t esz = DataTypeSize(r.dtype);
  std::vector<int64_t> counts(es.size());
  int64_t total = 0;
  for (size_t i = 0; i < es.size(); ++i) { counts[i] = es[i] ? es[i]->shape.num_elements() : r.tensor_sizes[i]; total += counts[i]; }

  if (n == 1) {
    const double sc = r.prescale * r.postscale;
    for (auto& e : es) if (e && (e->input != e->output || sc != 1.0))
      HVD_CUDA(kern::LaunchScale(e->input, e->output, e->shape.num_elements(), (int)r.dtype, sc, s));
  } else {
    std::shared_ptr<SymmTeam> team = env_.backend == "cpu" ? nullptr : EnsureTeam(ps, device);
    Status st = team ? AdasumP2P(ps, *team, es, r, counts, device, s) : Status::InProgress();
    if (!team || st.in_progress()) {
      // host-staged VHDD
      std::vector<char> host((size_t)total * esz);
      int64_t off = 0;
      for (size_t i = 0; i < es.size(); ++i) {
        if (es[i]) HVD_CUDA(cudaMemcpyAsync(host.data() + off * esz, es[i]->input, (size_t)counts[i] * esz, cudaMemcpyDeviceToHost, s));
        else memset(host.data() + off * esz, 0, (size_t)counts[i] * esz);
        off += counts[i];
      }
      HVD_CUDA(cudaStreamSynchronize(s));
      cpu::ScaleBuffer(host.data(), total, r.dtype, r.prescale);
      Status cs = cpu::AdasumAllreduce(ps.transport.get(), host.data(), counts, r.dtype);
      if (!cs.ok()) return cs;
      cpu::ScaleBuffer(host.data(), total, r.dtype, r.postscale);
      off = 0;
      for (size_t i = 0; i < es.size(); ++i) {
        if (es[i]) HVD_CUDA(cudaMemcpyAsync(es[i]->output, host.data() + off * esz, (size_t)counts[i] * esz, cudaMemcpyHostToDevice, s));
        off += counts[i];
      }
      HVD_CUDA(cudaStreamSynchronize(s));
    } else if (!st.ok()) {
      return st;
    }
  }
  SharedEvent* ev = ctx.NewEvent(device, (int)std::max<size_t>(es.size(), 1));
  HVD_CUDA(cudaEventRecord(ev->ev, s));
  *done = ev;
  return Status::OK();
}

// Peer-to-peer kernel path: see kernels/adasum_kernels.cu. Returns InProgress when not applicable.
Status GpuOps::AdasumP2P(ProcessSet& ps, SymmTeam& team, Entries& es, const Response& r, const std::vector<int64_t>& counts,
                         int device, cudaStream_t s) {
  (void)ps;
  if (!(r.dtype == DataType::FLOAT32 || r.dtype == DataType::FLOAT16 || r.dtype == DataType::BFLOAT16)) return Status::InProgress();
  if ((int)es.size() > kern::kAdasumMaxTensors) return Status::InProgress();
  GpuContext& ctx = GpuContext::Get();
  const size_t esz = DataTypeSize(r.dtype);
  std::vector<kern::TensorDesc> descs(es.size());
  int64_t total = 0;
  for (size_t i = 0; i < es.size(); ++i) {
    if (es[i]) { descs[i].in = es[i]->input; descs[i].out = es[i]->output; }
    else {
      void* z = ctx.TempAlloc(device, (size_t)counts[i] * esz, true, s);
      if (!z) return Status::UnknownError("out of device memory for join placeholder");
      descs[i].in = z; descs[i].out = z;
    }
    descs[i].offset = total;
    descs[i].count = counts[i];
    total += (counts[i] * 4 + 127) / 128 * 128;
  }
  if (total > (int64_t)team.buffer_bytes()) {
    // larger than the symmetric buffer: the host implementation takes over (D2H, CPU VHDD, H2D) — correct but slow, so say so
    static bool warned = false;
    if (!warned) {
      warned = true;
      LOG(WARNING) << "Adasum: a fused response of " << (total >> 20) << " MiB (fp32) does not fit the " << (team.buffer_bytes() >> 20)
                   << " MiB symmetric buffer and is reduced on the host; raise HVD_SYMM_BUFFER_BYTES or lower HOROVOD_FUSION_THRESHOLD";
    }
    return Status::InProgress();
  }
  const auto* dt = (const kern::TensorDesc*)ctx.Stage(device, descs.data(), descs.size() * sizeof(kern::TensorDesc), s);
  if (!dt) return Status::InProgress();
  kern::AdasumArgs a {};
  a.descs = dt; a.ndesc = (int)descs.size(); a.total_bytes = total; a.dtype = (int)r.dtype;
  a.ctas = (int)std::max<int64_t>(1, std::min<int64_t>(env_.params->comm_ctas, (total + 16383) / 16384));
  a.scratch_stride_bytes = kern::kAdasumScratchStride;
  if (env_.adasum_persistent) {
    // one resident kernel for the whole reduction (grid barriers inside): its CTAs must fit on the device together
    a.ctas = std::min(a.ctas, 128);
    a.persist_scratch = ctx.TempAlloc(device, kern::AdasumPersistentScratchBytes(a.ctas, a.ndesc), false, s);
    a.persist_sync = ctx.GridSyncBlock(device);
    if (!a.persist_scratch || !a.persist_sync) { a.persist_scratch = nullptr; a.persist_sync = nullptr; }
  }
  kern::CommParams cp = team.Params(team.NextSlot());
  if (env_.timeline && env_.timeline->Initialized()) env_.timeline->ActivityStartAll(es, HVD_ACT_P2P_ADASUM);
  cudaError_t e = kern::LaunchAdasum(cp, a, r.prescale, r.postscale, s);
  if (e != cudaSuccess) return Status::UnknownError(std::string("adasum kernel launch failed: ") + cudaGetErrorString(e));
  ctx.TempFreeAll(device, s);
  return Status::OK();
}

}  // namespace hvd
