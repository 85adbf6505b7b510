// Single-GPU simulation harness for the P2P kernels: N "ranks" are N plain
// allocations on one device and N concurrently launched kernels on N streams.
// The cross-"GPU" flag protocol, chunk ownership and descriptor walking are
// exactly what runs across NVLink; only the address mapping differs.  Lets the
// kernels be validated (and run under compute-sanitizer) on one GPU.
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <string>
#include <map>
#include <memory>
#include <vector>
#include "../kernels/p2p_kernels.h"
#include "../ops/collective_plan.h"
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

// ---------------------------------------------------------------------------
// The launch plans of reducescatter / allgather(v) / broadcast / alltoall(v) (ops/collective_plan.h) for all N ranks.

enum PlanKind { kPlanReducescatter = 0, kPlanAllgather = 1, kPlanBroadcast = 2, kPlanAlltoall = 3 };

// dims per tensor i: reducescatter dims[i] = dim0; allgather dims[i*n .. i*n+n) = every rank's dim0; broadcast dims[i] =
// bytes; alltoall dims[i*n*n ..) = the split matrix (rows rank p sends to rank q at p*n+q).  rows[i]: elements per row
// (not used by broadcast).  in_ptrs / out_ptrs: [nranks][ntensors].
struct PlanRequest {
  int kind, n, ntensors;
  const int64_t* dims;
  const int64_t* rows;
  int dtype, op;
  double prescale, postscale;
  int root;
  const uint64_t* in_ptrs;
  const uint64_t* out_ptrs;
  int64_t cap;
  int ctas;
  int grid = 0;  // > 0: every launch of every rank runs this many CTAs instead of the grid the planner sized to the data
};

// Every rank's plan and the byte ranges of its outputs (what the engine allocates for that rank).
Status BuildPlans(const PlanRequest& q, std::vector<Plan>* plans, std::vector<std::vector<OutSpan>>* outs) {
  const int n = q.n, t = q.ntensors;
  if (n < 2 || n > kern::kMaxPeers || t < 0 || q.kind < 0 || q.kind > kPlanAlltoall || (q.kind == kPlanBroadcast && (q.root < 0 || q.root >= n)))
    return Status::InvalidArgument("bad plan request");
  const int64_t esz = q.kind == kPlanBroadcast ? 1 : (int64_t)DataTypeSize((DataType)q.dtype);
  plans->assign(n, Plan());
  outs->assign(n, {});
  for (int r = 0; r < n; ++r) {
    std::vector<PlanTensor> ts(t);
    for (int i = 0; i < t; ++i) {
      PlanTensor& pt = ts[i];
      pt.in = (const void*)q.in_ptrs[(size_t)r * t + i];
      pt.out = (void*)q.out_ptrs[(size_t)r * t + i];
      pt.row = q.kind == kPlanBroadcast ? 1 : q.rows[i];
      int64_t out_rows = 0;
      if (q.kind == kPlanReducescatter) {
        pt.dims = {q.dims[i]};
        std::vector<int64_t> rows;
        ReducescatterRows(q.dims[i], n, &rows);
        out_rows = rows[r];
      } else if (q.kind == kPlanAllgather) {
        pt.dims.assign(q.dims + (size_t)i * n, q.dims + (size_t)(i + 1) * n);
        for (int p = 0; p < n; ++p) out_rows += pt.dims[p];
      } else if (q.kind == kPlanBroadcast) {
        pt.dims = {q.dims[i]};
        out_rows = (r == q.root && pt.out == pt.in) ? 0 : q.dims[i];
      } else {
        pt.dims.assign(q.dims + (size_t)i * n * n, q.dims + (size_t)(i + 1) * n * n);
        for (int p = 0; p < n; ++p) out_rows += pt.dims[(size_t)p * n + r];
      }
      (*outs)[r].push_back({pt.out, out_rows * pt.row * esz});
    }
    Status st;
    Plan& plan = (*plans)[r];
    if (q.kind == kPlanReducescatter) {
      ReduceParams rp;
      rp.dtype = (DataType)q.dtype; rp.op = (ReduceOp)q.op; rp.prescale = q.prescale; rp.postscale = q.postscale;
      st = PlanReducescatter(r, n, ts, rp, q.cap, q.ctas, &plan);  // the simulated team has no multicast object: rp.nvls false
    } else if (q.kind == kPlanAllgather) {
      st = PlanAllgather(r, n, ts, esz, q.cap, q.ctas, &plan);
    } else if (q.kind == kPlanBroadcast) {
      st = PlanBroadcast(r, n, q.root, ts, false, q.cap, q.ctas, &plan);
    } else {
      st = PlanAlltoall(r, n, ts, esz, q.cap, q.ctas, &plan);
    }
    if (!st.ok()) return st;
  }
  return Status::OK();
}

void CopyMessage(const std::string& m, char* err, int err_len) {
  if (err && err_len > 0) { strncpy(err, m.c_str(), (size_t)err_len - 1); err[err_len - 1] = 0; }
}

// Plans all N ranks, checks them (CheckPlans) and only then launches, step-major: launch k of every rank before launch k+1
// of any rank.  -5: no plan (the buffer is too small), -4: the ranks' plans disagree (nothing was launched).  The tables
// of all launches go to the device in one copy before the first launch.
int SimCollective(const PlanRequest& q, int device) {
  if (cudaSetDevice(device) != cudaSuccess) return -1;
  std::vector<Plan> plans;
  std::vector<std::vector<OutSpan>> outs;
  if (!BuildPlans(q, &plans, &outs).ok()) return -5;
  if (q.grid > 0)
    for (auto& plan : plans) for (auto& l : plan) l.ctas = q.grid;
  if (!CheckPlans(plans, outs, q.cap, q.kind == kPlanBroadcast ? q.root : -1).ok()) return -4;
  Sim* sim = GetSim(q.n, device, (size_t)std::max<int64_t>(q.cap, 1 << 20));
  if (!sim) return -1;
  if ((int64_t)sim->teams[0]->buffer_bytes() < q.cap) return -1;
  const size_t nl = plans[0].size();
  std::vector<char> host;
  std::vector<size_t> at((size_t)q.n * nl);
  for (size_t k = 0; k < nl; ++k) {
    for (int r = 0; r < q.n; ++r) {
      const PlanLaunch& l = plans[r][k];
      at[k * q.n + r] = host.size();
      if (l.reduce) {
        const char* b = (const char*)l.table.data();
        host.insert(host.end(), b, b + l.table.size() * sizeof(kern::TensorDesc));
      } else {
        const char* b = (const char*)l.sends.data();
        host.insert(host.end(), b, b + l.sends.size() * sizeof(kern::CopyDesc));
        b = (const char*)l.recvs.data();
        host.insert(host.end(), b, b + l.recvs.size() * sizeof(kern::CopyDesc));
      }
      host.resize((host.size() + 255) / 256 * 256);
    }
  }
  cudaDeviceSynchronize();
  char* dev = nullptr;
  if (!host.empty()) {
    if (cudaMalloc(&dev, host.size()) != cudaSuccess) return -1;
    if (cudaMemcpy(dev, host.data(), host.size(), cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(dev); return -1; }
  }
  cudaError_t launch_error = cudaSuccess;
  for (size_t k = 0; k < nl && launch_error == cudaSuccess; ++k) {
    const std::vector<kern::CommParams> cps = NextParams(sim);
    for (int r = 0; r < q.n && launch_error == cudaSuccess; ++r) {
      const PlanLaunch& l = plans[r][k];
      char* t = dev + at[k * q.n + r];
      if (l.reduce) {
        kern::AllreduceArgs a = l.args;
        a.descs = (const kern::TensorDesc*)t; a.out_descs = a.descs + a.ndesc; a.ctas = l.ctas;
        launch_error = kern::LaunchAllreduce(cps[r], a, sim->streams[r]);
      } else {
        kern::ExchangeArgs a {};
        a.sends = l.sends.empty() ? nullptr : (const kern::CopyDesc*)t; a.nsend = (int)l.sends.size();
        a.recvs = l.recvs.empty() ? nullptr : (const kern::CopyDesc*)t + l.sends.size(); a.nrecv = (int)l.recvs.size();
        a.ctas = l.ctas;
        launch_error = kern::LaunchExchange(cps[r], a, sim->streams[r]);
      }
    }
  }
  const cudaError_t sync = cudaDeviceSynchronize();
  if (dev) cudaFree(dev);
  if (launch_error != cudaSuccess) return (int)launch_error;
  return Finish(q.n, sync);
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

// Allgather-style exchange: every rank contributes `bytes` from in_ptrs[r]; out_ptrs[r] receives nranks*bytes.  The
// tables are the engine's allgather plan of one uint8 tensor, but the grid is `ctas` CTAs whatever the size (the engine
// sizes it to the data), so that a small message also runs with CTAs that own no chunk and only take part in the barrier.
int hvd_sim_allgather(int nranks, int device, int64_t bytes, const uint64_t* in_ptrs, const uint64_t* out_ptrs, int ctas) {
  std::vector<int64_t> dims(nranks, bytes);
  const int64_t row = 1;
  PlanRequest q {kPlanAllgather, nranks, 1, dims.data(), &row, (int)DataType::UINT8, 0, 1.0, 1.0, -1, in_ptrs, out_ptrs,
                 std::max<int64_t>(bytes, 1 << 20), ctas};
  q.grid = ctas;
  return SimCollective(q, device);
}

// Reducescatter over N simulated ranks as the engine plans it: dim0s[t] / rows[t] (elements per first-dim row) of every
// tensor, in_ptrs / out_ptrs [nranks][ntensors]; `cap` bytes of symmetric buffer per launch.  Returns 0, a cudaError_t,
// -3 (simulated barrier timed out), -4 (the ranks' plans disagree; nothing launched) or -5 (no plan fits `cap`).
int hvd_sim_reducescatter(int nranks, int device, int ntensors, const int64_t* dim0s, const int64_t* rows, const uint64_t* in_ptrs,
                          const uint64_t* out_ptrs, int dtype, int op, double prescale, double postscale, int64_t cap, int ctas) {
  PlanRequest q {kPlanReducescatter, nranks, ntensors, dim0s, rows, dtype, op, prescale, postscale, -1, in_ptrs, out_ptrs, cap, ctas};
  return SimCollective(q, device);
}

// Allgatherv: dims[t][nranks] = every rank's first dim of tensor t; element size `esz`.  Return codes as above.
int hvd_sim_allgatherv(int nranks, int device, int ntensors, const int64_t* dims, const int64_t* rows, int dtype,
                       const uint64_t* in_ptrs, const uint64_t* out_ptrs, int64_t cap, int ctas) {
  PlanRequest q {kPlanAllgather, nranks, ntensors, dims, rows, dtype, 0, 1.0, 1.0, -1, in_ptrs, out_ptrs, cap, ctas};
  return SimCollective(q, device);
}

// Broadcast of ntensors tensors of bytes[t] bytes from `root`; out_ptrs == in_ptrs on the root is in place.
int hvd_sim_broadcast(int nranks, int device, int ntensors, const int64_t* bytes, int root, const uint64_t* in_ptrs,
                      const uint64_t* out_ptrs, int64_t cap, int ctas) {
  PlanRequest q {kPlanBroadcast, nranks, ntensors, bytes, nullptr, (int)DataType::UINT8, 0, 1.0, 1.0, root, in_ptrs, out_ptrs, cap, ctas};
  return SimCollective(q, device);
}

// Alltoallv: splits[t][nranks][nranks] = rows rank p sends to rank q (p * nranks + q) of tensor t.
int hvd_sim_alltoallv(int nranks, int device, int ntensors, const int64_t* splits, const int64_t* rows, int dtype,
                      const uint64_t* in_ptrs, const uint64_t* out_ptrs, int64_t cap, int ctas) {
  PlanRequest q {kPlanAlltoall, nranks, ntensors, splits, rows, dtype, 0, 1.0, 1.0, -1, in_ptrs, out_ptrs, cap, ctas};
  return SimCollective(q, device);
}

// The same plans on the host only (no GPU needed; the pointers are never dereferenced): `kind` 0 reducescatter,
// 1 allgatherv, 2 broadcast, 3 alltoallv, arguments as the hvd_sim_* entries.  Runs CheckPlans and writes *nlaunch and
// one row of 6 int64 per byte range the plans move: {0, rank, dst, src_rank, src, bytes} for every range rank `rank`
// receives into an output (`src_rank`'s input bytes at `src`; a reduce range once per contributing rank) and
// {1, rank, buffer offset, rank, src, bytes} for every input range rank `rank` packs.  Returns the number of rows, -5 (no
// plan), -4 (CheckPlans failed) or -6 (more than max_rows), with the reason in `err`.
int64_t hvd_plan_collective(int kind, int nranks, int ntensors, const int64_t* dims, const int64_t* rows, int dtype, int op,
                            int root, const uint64_t* in_ptrs, const uint64_t* out_ptrs, int64_t cap, int ctas, int* nlaunch,
                            int64_t* out_rows, int64_t max_rows, char* err, int err_len) {
  PlanRequest q {kind, nranks, ntensors, dims, rows, dtype, op, 1.0, 1.0, root, in_ptrs, out_ptrs, cap, ctas};
  std::vector<Plan> plans;
  std::vector<std::vector<OutSpan>> outs;
  Status st = BuildPlans(q, &plans, &outs);
  if (!st.ok()) { CopyMessage(st.reason(), err, err_len); return -5; }
  st = CheckPlans(plans, outs, cap, kind == kPlanBroadcast ? root : -1);
  if (!st.ok()) { CopyMessage(st.reason(), err, err_len); return -4; }
  *nlaunch = (int)plans[0].size();
  int64_t m = 0;
  auto emit = [&](int64_t a, int64_t b, int64_t c, int64_t d, int64_t e, int64_t f) {
    if (m < max_rows) { int64_t* o = out_rows + 6 * m; o[0] = a; o[1] = b; o[2] = c; o[3] = d; o[4] = e; o[5] = f; }
    ++m;
  };
  for (int r = 0; r < nranks; ++r) {
    for (size_t k = 0; k < plans[r].size(); ++k) {
      const PlanLaunch& l = plans[r][k];
      if (l.reduce) {
        const int per = l.args.ndesc / nranks;
        const int64_t esz = (int64_t)DataTypeSize((DataType)l.args.dtype);
        for (int i = 0; i < l.args.ndesc; ++i)
          if (l.table[i].count > 0) emit(1, r, l.table[i].offset, r, (int64_t)(uintptr_t)l.table[i].in, l.table[i].count * esz);
        for (int j = 0; j < l.args.nout; ++j) {
          const kern::TensorDesc& o = l.table[l.args.ndesc + j];
          if (o.count > 0)
            for (int p = 0; p < nranks; ++p)
              emit(0, r, (int64_t)(uintptr_t)o.out, p, (int64_t)(uintptr_t)plans[p][k].table[(size_t)r * per + j].in, o.count * esz);
        }
        continue;
      }
      for (const kern::CopyDesc& s : l.sends) emit(1, r, s.offset, r, (int64_t)(uintptr_t)s.src, s.bytes);
      for (const kern::CopyDesc& d : l.recvs) {
        for (const kern::CopyDesc& s : plans[d.peer][k].sends) {  // CheckPlans found exactly this send
          if (s.offset <= d.offset && d.offset + d.bytes <= s.offset + s.bytes) {
            emit(0, r, (int64_t)(uintptr_t)d.dst, d.peer, (int64_t)(uintptr_t)s.src + (d.offset - s.offset), d.bytes);
            break;
          }
        }
      }
    }
  }
  if (m > max_rows) { CopyMessage("more than max_rows ranges", err, err_len); return -6; }
  return m;
}

// PlanAllreduce of one rank on the host only (the pointers are never dereferenced): pieces counts[t] / in_ptrs[t] /
// out_ptrs[t], the wire dtype the engine chose, HVD_ALLREDUCE_VARIANT `variant` and the rest of the AllreducePolicy.  Writes
// one row of 15 int64 per launch, {reduce, variant, ctas, total_bytes, reduce_lo, reduce_hi, dtype, wire_dtype, op, the bits
// of prescale and of postscale, InlineDescs, nout, oneshot_nvls, ndesc}, and the launches' descriptors in order, one row
// {in, out, offset, count} each.  Returns the number of launches, -5 (no plan) with the reason in `err`, or -6 (more than
// max_launches or max_descs).
int64_t hvd_plan_allreduce(int nranks, int ntensors, const int64_t* counts, const uint64_t* in_ptrs, const uint64_t* out_ptrs,
                           int dtype, int wire_dtype, int op, double prescale, double postscale, const char* variant,
                           int64_t oneshot_max_bytes, int multicast, int64_t nvls_min_bytes, int64_t cap, int comm_ctas,
                           int64_t large_msg_ctas, int64_t* launch_rows, int64_t max_launches, int64_t* desc_rows, int64_t max_descs,
                           char* err, int err_len) {
  std::vector<PlanTensor> ts(ntensors);
  for (int i = 0; i < ntensors; ++i) {
    ts[i].in = (const void*)in_ptrs[i]; ts[i].out = (void*)out_ptrs[i]; ts[i].dims = {counts[i]};
  }
  ReduceParams rp;
  rp.dtype = (DataType)dtype; rp.op = (ReduceOp)op; rp.prescale = prescale; rp.postscale = postscale;
  AllreducePolicy pol;
  pol.variant = variant;
  pol.oneshot_max_bytes = oneshot_max_bytes;
  pol.multicast = multicast != 0;
  pol.nvls_min_bytes = nvls_min_bytes;
  pol.large_msg_ctas = large_msg_ctas;
  Plan plan;
  Status st = PlanAllreduce(nranks, ts, rp, (DataType)wire_dtype, pol, cap, comm_ctas, &plan);
  if (!st.ok()) { CopyMessage(st.reason(), err, err_len); return -5; }
  int64_t nd = 0;
  for (const PlanLaunch& l : plan) nd += (int64_t)l.table.size();
  if ((int64_t)plan.size() > max_launches || nd > max_descs) { CopyMessage("more than max_launches or max_descs", err, err_len); return -6; }
  int64_t* o = launch_rows;
  int64_t* d = desc_rows;
  for (const PlanLaunch& l : plan) {
    const kern::AllreduceArgs& a = l.args;
    int64_t pre, post;
    memcpy(&pre, &a.prescale, sizeof pre);
    memcpy(&post, &a.postscale, sizeof post);
    const int64_t row[15] = {l.reduce, a.variant, l.ctas, a.total_bytes, a.reduce_lo, a.reduce_hi, a.dtype, a.wire_dtype, a.op, pre, post,
                             InlineDescs(a), a.nout, a.oneshot_nvls, a.ndesc};
    o = std::copy(row, row + 15, o);
    for (const kern::TensorDesc& t : l.table) {
      const int64_t drow[4] = {(int64_t)(uintptr_t)t.in, (int64_t)(uintptr_t)t.out, t.offset, t.count};
      d = std::copy(drow, drow + 4, d);
    }
  }
  return (int64_t)plan.size();
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

// The captured alltoall over N simulated ranks, every rank's arguments indexed by rank: in_ptrs / rows / row_bytes its
// input, split_ptrs its n splits on the device (int64 with splits_int64, else int32), out_ptrs / capacity its output,
// recv_ptrs (int64, n) and status_ptrs (int32, 1).  Without `streams` the N kernels run on the harness's streams and the
// call waits for them (returns 0, a cudaError_t, -1 or -3 as hvd_sim_inplace).  With `streams` (N cudaStream_t) it only
// launches rank r's kernel on streams[r] and returns, so that a caller can order the launches after device work of its
// own or capture all N ranks into one CUDA graph; the harness of this rank count must exist by then (one call without
// `streams`), and must not be reset while such a graph may still run.
int hvd_sim_captured_alltoall(int nranks, int device, const uint64_t* in_ptrs, const int64_t* rows, const int64_t* row_bytes,
                              const uint64_t* split_ptrs, int splits_int64, const uint64_t* out_ptrs, const int64_t* capacity,
                              const uint64_t* recv_ptrs, const uint64_t* status_ptrs, int ctas, const uint64_t* streams) {
  if (nranks < 2 || nranks > kern::kMaxPeers || cudaSetDevice(device) != cudaSuccess) return -1;
  Sim* sim = streams ? (g_sims.count(nranks) ? &g_sims[nranks] : nullptr) : GetSim(nranks, device, 1 << 20);
  if (!sim) return -1;
  // rejected on every rank or on none: a rank launched alone would wait at its barrier for peers that never come
  if (ctas < 1 || ctas > kern::kMaxCtas) return (int)cudaErrorInvalidValue;
  for (int r = 0; r < nranks; ++r)
    if (rows[r] < 0 || capacity[r] < 0 || row_bytes[r] < 0) return (int)cudaErrorInvalidValue;
  if (!streams) cudaDeviceSynchronize();
  for (int r = 0; r < nranks; ++r) {
    kern::CapturedAlltoallArgs a {};
    for (int p = 0; p < nranks; ++p) { a.in[p] = (const void*)in_ptrs[p]; a.counts[p] = sim->teams[r]->CountRegion(p); }
    a.in_offset = 0; a.rows = rows[r]; a.capacity = capacity[r]; a.row_bytes = row_bytes[r];
    a.splits = (const void*)split_ptrs[r]; a.splits_int64 = splits_int64;
    a.out = (void*)out_ptrs[r]; a.recv_splits = (int64_t*)recv_ptrs[r]; a.status = (int*)status_ptrs[r];
    a.ctas = ctas;
    cudaError_t e = kern::LaunchCapturedAlltoall(sim->teams[r]->Params(0, kern::kAlltoallChannel), a,
                                                 streams ? (cudaStream_t)streams[r] : sim->streams[r]);
    if (e != cudaSuccess) return (int)e;
  }
  return streams ? 0 : Finish(nranks, cudaDeviceSynchronize());
}

void hvd_sim_reset() {
  for (auto& kv : g_sims) for (auto st : kv.second.streams) cudaStreamDestroy(st);
  g_sims.clear();
}

}  // extern "C"
