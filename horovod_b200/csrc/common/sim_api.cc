// Single-GPU simulation harness for the P2P kernels: N "ranks" are N plain
// allocations on one device and N concurrently launched kernels on N streams.
// The cross-"GPU" flag protocol, chunk ownership and descriptor walking are
// exactly what runs across NVLink; only the address mapping differs.  Lets the
// kernels be validated (and run under compute-sanitizer) on one GPU.
#include <cuda_runtime.h>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <vector>
#include "../kernels/p2p_kernels.h"
#include "../ops/gpu_ops.h"
#include "../symm/symm_memory.h"

using namespace hvd;

namespace {
struct Sim {
  std::vector<std::shared_ptr<SymmTeam>> teams;
  std::vector<cudaStream_t> streams;
  size_t bytes = 0;
};
std::map<int, Sim> g_sims;  // by nranks

Sim* GetSim(int nranks, int device, size_t buffer_bytes) {
  Sim& s = g_sims[nranks];
  if (s.teams.empty() || s.bytes < buffer_bytes) {
    s.teams = SymmTeam::CreateSimulated(nranks, device, buffer_bytes);
    s.bytes = buffer_bytes;
    if (s.teams.empty()) return nullptr;
    for (auto st : s.streams) cudaStreamDestroy(st);
    s.streams.assign(nranks, nullptr);
    for (int r = 0; r < nranks; ++r) cudaStreamCreateWithFlags(&s.streams[r], cudaStreamNonBlocking);
    // a scheduling deadlock of the simulation must surface as an error, not as a hung test
    const char* to = getenv("HVD_KERNEL_TIMEOUT_SECONDS");
    for (auto& t : s.teams) t->set_timeout_seconds(to ? atof(to) : 20.0);
  }
  return &s;
}
int64_t Align128(int64_t b) { return (b + 127) / 128 * 128; }

// Every simulated rank's parameters for the next collective, taken before any launch: NextSlot() flips a rank's
// ping-pong buffer, so a launch that is rejected (bad arguments are rejected on every rank alike) must not leave the
// ranks on different buffers, where every later collective of this rank count would read stale peer data.
std::vector<kern::CommParams> NextParams(Sim* sim) {
  std::vector<kern::CommParams> cps;
  for (auto& t : sim->teams) cps.push_back(t->Params(t->NextSlot()));
  return cps;
}

// After the device drained: a barrier that timed out (scheduling deadlock of the simulation) is an error, and the team is
// thrown away so that the next call starts from clean flags / epochs.
int Finish(int nranks, cudaError_t sync_result) {
  if (sync_result != cudaSuccess) return (int)sync_result;
  auto it = g_sims.find(nranks);
  if (it == g_sims.end()) return 0;
  for (auto& t : it->second.teams) {
    if (t->abort_state() != 0) {
      for (auto st : it->second.streams) cudaStreamDestroy(st);
      g_sims.erase(it);
      return -3;
    }
  }
  return 0;
}
}  // namespace

extern "C" {

// in_ptrs/out_ptrs: [nranks][ntensors] device pointers. Returns 0 on success, else a cudaError_t (or -1).
int hvd_sim_allreduce(int nranks, int device, int ntensors, const int64_t* counts, const uint64_t* in_ptrs,
                      const uint64_t* out_ptrs, int dtype, int wire_dtype, int op, int variant, int ctas, double prescale,
                      double postscale, int repeats, float* ms_out) {
  if (cudaSetDevice(device) != cudaSuccess) return -1;
  const int64_t wsz = (int64_t)DataTypeSize((DataType)wire_dtype);
  int64_t total = 0;
  std::vector<int64_t> offs(ntensors);
  for (int i = 0; i < ntensors; ++i) { offs[i] = total; total += Align128(counts[i] * wsz); }
  Sim* sim = GetSim(nranks, device, (size_t)std::max<int64_t>(total, 1 << 20));
  if (!sim) return -1;
  std::vector<const kern::TensorDesc*> dtabs(nranks);
  for (int r = 0; r < nranks; ++r) {
    std::vector<kern::TensorDesc> d(ntensors);
    for (int i = 0; i < ntensors; ++i) {
      d[i].in = (const void*)in_ptrs[(size_t)r * ntensors + i];
      d[i].out = (void*)out_ptrs[(size_t)r * ntensors + i];
      d[i].offset = offs[i];
      d[i].count = counts[i];
    }
    dtabs[r] = (const kern::TensorDesc*)GpuContext::Get().Stage(device, d.data(), d.size() * sizeof(kern::TensorDesc), sim->streams[r]);
    if (!dtabs[r]) return -2;
  }
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaDeviceSynchronize();
  cudaEventRecord(e0, sim->streams[0]);
  for (int it = 0; it < repeats; ++it) {
    const std::vector<kern::CommParams> cps = NextParams(sim);
    for (int r = 0; r < nranks; ++r) {
      kern::AllreduceArgs a {};
      a.descs = dtabs[r]; a.ndesc = ntensors; a.total_bytes = total; a.reduce_lo = 0; a.reduce_hi = total;
      a.prescale = prescale; a.postscale = postscale; a.op = op; a.dtype = dtype; a.wire_dtype = wire_dtype;
      a.variant = variant; a.ctas = ctas;
      if (variant == kern::kPipelined) {  // small chunks so that a modest test message exercises ring reuse
        const char* cb = getenv("HVD_PIPE_CHUNK_BYTES");
        a.pipe_chunk_bytes = cb ? atoll(cb) / 4096 * 4096 : 65536;
        if (a.pipe_chunk_bytes < 4096) a.pipe_chunk_bytes = 4096;
        a.pipe_slots = (int)std::min<int64_t>(kern::kPipeMaxSlots, std::max<int64_t>(2, (int64_t)sim->bytes / a.pipe_chunk_bytes));
        const char* sl = getenv("HVD_PIPE_SLOTS");
        if (sl && atoi(sl) >= 2) a.pipe_slots = std::min(a.pipe_slots, atoi(sl));
        a.pipe_base = sim->teams[r]->NextPipeBase((uint32_t)((total + a.pipe_chunk_bytes - 1) / a.pipe_chunk_bytes));
        a.pipe_use_nvls = 0;
        a.pipe_rblock_bytes = 8192;
      }
      cudaError_t e = kern::LaunchAllreduce(cps[r], a, sim->streams[r]);
      if (e != cudaSuccess) return (int)e;
    }
  }
  cudaEventRecord(e1, sim->streams[0]);
  cudaError_t e = cudaDeviceSynchronize();
  if (ms_out) cudaEventElapsedTime(ms_out, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  return Finish(nranks, e);
}

// Allgather-style exchange: every rank contributes `bytes` from in_ptrs[r]; out_ptrs[r] receives nranks*bytes.
int hvd_sim_allgather(int nranks, int device, int64_t bytes, const uint64_t* in_ptrs, const uint64_t* out_ptrs, int ctas) {
  if (cudaSetDevice(device) != cudaSuccess) return -1;
  Sim* sim = GetSim(nranks, device, (size_t)std::max<int64_t>(bytes, 1 << 20));
  if (!sim) return -1;
  const std::vector<kern::CommParams> cps = NextParams(sim);
  for (int r = 0; r < nranks; ++r) {
    std::vector<kern::CopyDesc> t;
    t.push_back({(const void*)in_ptrs[r], nullptr, 0, bytes, r, 0});
    for (int k = 0; k < nranks; ++k) {
      int p = (r + k) % nranks;
      t.push_back({nullptr, (char*)out_ptrs[r] + (int64_t)p * bytes, 0, bytes, p, 0});
    }
    const auto* dt = (const kern::CopyDesc*)GpuContext::Get().Stage(device, t.data(), t.size() * sizeof(kern::CopyDesc), sim->streams[r]);
    if (!dt) return -2;
    kern::ExchangeArgs a {};
    a.sends = dt; a.nsend = 1; a.recvs = dt + 1; a.nrecv = nranks; a.ctas = ctas;
    cudaError_t e = kern::LaunchExchange(cps[r], a, sim->streams[r]);
    if (e != cudaSuccess) return (int)e;
  }
  return Finish(nranks, cudaDeviceSynchronize());
}

// Adasum over N simulated ranks: in_ptrs/out_ptrs [nranks][ntensors]; dtype fp32/fp16/bf16.
int hvd_sim_adasum(int nranks, int device, int ntensors, const int64_t* counts, const uint64_t* in_ptrs, const uint64_t* out_ptrs,
                   int dtype, int ctas, double prescale, double postscale) {
  if (cudaSetDevice(device) != cudaSuccess) return -1;
  int64_t total = 0;
  std::vector<int64_t> offs(ntensors);
  for (int i = 0; i < ntensors; ++i) { offs[i] = total; total += Align128(counts[i] * 4); }
  Sim* sim = GetSim(nranks, device, (size_t)std::max<int64_t>(total, 1 << 20));
  if (!sim) return -1;
  // Step-major launch order (step k of EVERY rank before step k+1 of any rank): the streams of the simulated ranks may
  // share a hardware queue, and a rank-major order would park rank 1's kernels behind rank 0's spinning ones.
  std::vector<const kern::TensorDesc*> dtabs(nranks);
  const std::vector<kern::CommParams> cps = NextParams(sim);
  for (int r = 0; r < nranks; ++r) {
    std::vector<kern::TensorDesc> d(ntensors);
    for (int i = 0; i < ntensors; ++i) {
      d[i].in = (const void*)in_ptrs[(size_t)r * ntensors + i];
      d[i].out = (void*)out_ptrs[(size_t)r * ntensors + i];
      d[i].offset = offs[i];
      d[i].count = counts[i];
    }
    dtabs[r] = (const kern::TensorDesc*)GpuContext::Get().Stage(device, d.data(), d.size() * sizeof(kern::TensorDesc), sim->streams[r]);
    if (!dtabs[r]) return -2;
  }
  // HVD_ADASUM_PERSISTENT (default 1): the single-launch kernel; every simulated rank gets its own scratch + grid-sync block
  const char* pe = getenv("HVD_ADASUM_PERSISTENT");
  const bool persistent = !(pe && atoi(pe) == 0);
  std::vector<void*> pscratch(nranks, nullptr), psync(nranks, nullptr);
  if (persistent) {
    for (int r = 0; r < nranks; ++r) {
      cudaMalloc(&pscratch[r], kern::AdasumPersistentScratchBytes(ctas, ntensors));
      cudaMalloc(&psync[r], 256);
      cudaMemset(psync[r], 0, 256);
    }
  }
  auto free_persist = [&]() { for (int r = 0; r < nranks; ++r) { if (pscratch[r]) cudaFree(pscratch[r]); if (psync[r]) cudaFree(psync[r]); } };
  const int steps = persistent ? 1 : kern::AdasumNumLaunches(nranks);
  for (int k = 0; k < steps; ++k) {
    for (int r = 0; r < nranks; ++r) {
      kern::AdasumArgs a {};
      a.descs = dtabs[r]; a.ndesc = ntensors; a.total_bytes = total; a.dtype = dtype; a.ctas = ctas;
      a.scratch_stride_bytes = kern::kAdasumScratchStride;
      a.persist_scratch = pscratch[r]; a.persist_sync = psync[r];
      cudaError_t e = kern::LaunchAdasumStep(cps[r], a, prescale, postscale, sim->streams[r], persistent ? -1 : k);
      if (e != cudaSuccess) { free_persist(); return (int)e; }
    }
  }
  const cudaError_t sync = cudaDeviceSynchronize();
  free_persist();
  return Finish(nranks, sync);
}

// Zero-copy in-place allreduce over N simulated ranks: ptrs[r] = rank r's tensor (plain device memory here).
int hvd_sim_inplace(int nranks, int device, int64_t bytes, const uint64_t* ptrs, int dtype, int op, int ctas, double scale,
                    int repeats, float* ms_out) {
  if (cudaSetDevice(device) != cudaSuccess) return -1;
  Sim* sim = GetSim(nranks, device, 1 << 20);
  if (!sim) return -1;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaDeviceSynchronize();
  cudaEventRecord(e0, sim->streams[0]);
  for (int it = 0; it < repeats; ++it) {
    const std::vector<kern::CommParams> cps = NextParams(sim);
    for (int r = 0; r < nranks; ++r) {
      kern::InplaceArgs a {};
      for (int p = 0; p < nranks; ++p) a.ptr[p] = (void*)ptrs[p];
      a.mc = nullptr; a.bytes = bytes; a.scale = scale; a.op = op; a.dtype = dtype; a.use_multicast = 0; a.ctas = ctas;
      cudaError_t e = kern::LaunchInplaceAllreduce(cps[r], a, sim->streams[r]);
      if (e != cudaSuccess) return (int)e;
    }
  }
  cudaEventRecord(e1, sim->streams[0]);
  cudaError_t e = cudaDeviceSynchronize();
  if (ms_out) cudaEventElapsedTime(ms_out, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  return Finish(nranks, e);
}

// The two halves of a sharded optimizer step over N simulated ranks: ptrs[r] = rank r's registered range (plain device
// memory here), rank r owns the contiguous slice [r * bytes / n, (r + 1) * bytes / n).  `reducescatter` != 0 runs the
// in-place reduce-scatter (dtype, op, scale as hvd_sim_inplace), else the in-place allgather (bytes only).
static int hvd_sim_inplace_sharded(int nranks, int device, int64_t bytes, const uint64_t* ptrs, int dtype, int op, int ctas, double scale,
                            int repeats, int reducescatter) {
  if (cudaSetDevice(device) != cudaSuccess) return -1;
  Sim* sim = GetSim(nranks, device, 1 << 20);
  if (!sim) return -1;
  cudaDeviceSynchronize();
  for (int it = 0; it < repeats; ++it) {
    const std::vector<kern::CommParams> cps = NextParams(sim);
    for (int r = 0; r < nranks; ++r) {
      kern::InplaceArgs a {};
      for (int p = 0; p < nranks; ++p) a.ptr[p] = (void*)ptrs[p];
      a.mc = nullptr; a.bytes = bytes; a.scale = scale; a.op = op; a.dtype = dtype; a.use_multicast = 0; a.ctas = ctas;
      cudaError_t e = reducescatter ? kern::LaunchInplaceReducescatter(cps[r], a, sim->streams[r])
                                    : kern::LaunchInplaceAllgather(cps[r], a, sim->streams[r]);
      if (e != cudaSuccess) return (int)e;
    }
  }
  return Finish(nranks, cudaDeviceSynchronize());
}

int hvd_sim_inplace_reducescatter(int nranks, int device, int64_t bytes, const uint64_t* ptrs, int dtype, int op, int ctas,
                                  double scale, int repeats) {
  return hvd_sim_inplace_sharded(nranks, device, bytes, ptrs, dtype, op, ctas, scale, repeats, 1);
}

int hvd_sim_inplace_allgather(int nranks, int device, int64_t bytes, const uint64_t* ptrs, int ctas, int repeats) {
  return hvd_sim_inplace_sharded(nranks, device, bytes, ptrs, 0, 1, ctas, 1.0, repeats, 0);
}

void hvd_sim_reset() {
  for (auto& kv : g_sims) for (auto st : kv.second.streams) cudaStreamDestroy(st);
  g_sims.clear();
}

}  // extern "C"
