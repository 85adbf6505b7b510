// C ABI loaded with ctypes by horovod_b200/common/basics.py.
// Parity: the extern "C" block of horovod/common/operations.{h,cc}
// (operations.h:35-183): init / shutdown / rank & size queries / build
// capability queries / process-set management / timeline control.
#include <cstring>
#include <string>
#include <vector>
#include "../kernels/p2p_kernels.h"
#include "../symm/symm_memory.h"
#include "../ops/cpu_ops.h"
#include "engine.h"
#include "env.h"
#include "logging.h"

using namespace hvd;

namespace {
thread_local std::string g_err;
int Fail(const std::string& m) { g_err = m; return -1; }
}  // namespace

extern "C" {

const char* hvd_last_error() { return g_err.c_str(); }

// process_sets: flat rank list + per-set sizes
int hvd_init(int rank, int size, int local_rank, int local_size, int cross_rank, int cross_size, const char* rdzv_addr,
             int rdzv_port, const char* scope, const int* ps_ranks, const int* ps_sizes, int n_ps) {
  InitConfig cfg;
  cfg.rank = rank; cfg.size = size; cfg.local_rank = local_rank; cfg.local_size = local_size;
  cfg.cross_rank = cross_rank; cfg.cross_size = cross_size;
  cfg.rendezvous_addr = rdzv_addr ? rdzv_addr : "";
  cfg.rendezvous_port = rdzv_port;
  cfg.scope = scope && *scope ? scope : "hvd";
  cfg.hostname = EnvStr(HOROVOD_HOSTNAME);
  int off = 0;
  for (int i = 0; i < n_ps; ++i) {
    cfg.process_sets.emplace_back(ps_ranks + off, ps_ranks + off + ps_sizes[i]);
    off += ps_sizes[i];
  }
  Status st = Engine::Get().Init(cfg);
  if (!st.ok()) return Fail(st.reason());
  return 0;
}

void hvd_shutdown() { Engine::Get().Shutdown(); }
int hvd_is_initialized() { return Engine::Get().initialized() ? 1 : 0; }
int hvd_is_running() { return Engine::Get().running() ? 1 : 0; }  // false once the loop ended (peer shutdown / failure)
int hvd_rank() { return Engine::Get().initialized() ? Engine::Get().rank() : -1; }
int hvd_size() { return Engine::Get().initialized() ? Engine::Get().size() : -1; }
int hvd_local_rank() { return Engine::Get().initialized() ? Engine::Get().local_rank() : -1; }
int hvd_local_size() { return Engine::Get().initialized() ? Engine::Get().local_size() : -1; }
int hvd_cross_rank() { return Engine::Get().initialized() ? Engine::Get().cross_rank() : -1; }
int hvd_cross_size() { return Engine::Get().initialized() ? Engine::Get().cross_size() : -1; }
int hvd_is_homogeneous() { return Engine::Get().is_homogeneous() ? 1 : 0; }

// capability queries (reference: horovod_mpi_built, horovod_gloo_built, horovod_nccl_built, ...)
int hvd_mpi_built() { return 0; }
int hvd_mpi_enabled() { return 0; }
int hvd_mpi_threads_supported() { return 0; }
int hvd_gloo_built() { return 1; }    // the native TCP/shm transport fills gloo's role
int hvd_gloo_enabled() { return 1; }
int hvd_nccl_built() { return 1; }    // NCCL baseline op is always compiled (dlopen at runtime)
int hvd_ddl_built() { return 0; }
int hvd_ccl_built() { return 0; }
int hvd_cuda_built() { return 1; }
int hvd_rocm_built() { return 0; }
int hvd_p2p_built() { return 1; }     // sm_90a NVLink kernels
int hvd_cuda_available() { return GpuContext::Get().Available() ? 1 : 0; }

int hvd_add_process_set(const int* ranks, int n) {
  std::string err;
  int id = Engine::Get().AddProcessSet(std::vector<int>(ranks, ranks + n), &err);
  if (id < 0) return Fail(err);
  return id;
}
int hvd_remove_process_set(int id) {
  std::string err;
  int r = Engine::Get().RemoveProcessSet(id, &err);
  if (r < 0) return Fail(err);
  return r;
}
int hvd_number_of_process_sets() { return (int)Engine::Get().process_sets().Ids().size(); }
void hvd_process_set_ids(int* out) {
  auto ids = Engine::Get().process_sets().Ids();
  for (size_t i = 0; i < ids.size(); ++i) out[i] = ids[i];
}
int hvd_process_set_size(int id) {
  auto ps = Engine::Get().process_sets().Get(id);
  return ps ? ps->set_size() : Fail("Process set with id " + std::to_string(id) + " does not exist.");
}
int hvd_process_set_rank(int id) {
  auto ps = Engine::Get().process_sets().Get(id);
  if (!ps) return Fail("Process set with id " + std::to_string(id) + " does not exist.");
  return ps->set_rank();
}
int hvd_process_set_included(int id) {
  auto ps = Engine::Get().process_sets().Get(id);
  if (!ps) return Fail("Process set with id " + std::to_string(id) + " does not exist.");
  return ps->member() ? 1 : 0;
}
int hvd_process_set_ranks(int id, int* out) {
  auto ps = Engine::Get().process_sets().Get(id);
  if (!ps) return Fail("Process set with id " + std::to_string(id) + " does not exist.");
  for (size_t i = 0; i < ps->ranks.size(); ++i) out[i] = ps->ranks[i];
  return (int)ps->ranks.size();
}

int hvd_start_timeline(const char* file, int mark_cycles) {
  Status st = Engine::Get().StartTimeline(file, mark_cycles != 0);
  return st.ok() ? 0 : Fail(st.reason());
}
int hvd_stop_timeline() {
  Status st = Engine::Get().StopTimeline();
  return st.ok() ? 0 : Fail(st.reason());
}

// introspection
int hvd_topology_string(char* buf, int len) {
  std::string s = Engine::Get().TopologyString();
  strncpy(buf, s.c_str(), len > 0 ? len - 1 : 0);
  if (len > 0) buf[len - 1] = 0;
  return (int)s.size();
}
int hvd_gpu_backend_string(int process_set_id, char* buf, int len) {
  auto ps = Engine::Get().process_sets().Get(process_set_id);
  std::string s = ps ? Engine::Get().gpu_ops().Describe(*ps) : "unknown process set";
  strncpy(buf, s.c_str(), len > 0 ? len - 1 : 0);
  if (len > 0) buf[len - 1] = 0;
  return (int)s.size();
}
unsigned long long hvd_stat(int which) {
  Engine& e = Engine::Get();
  switch (which) {
    case 0: return e.cycles();
    case 1: return e.fast_path_cycles();
    case 2: return e.responses_executed();
    case 3: return kern::KernelLaunchCount();
    case 4: return e.captured_launches();
    case 5: return e.gpu_ops().ipc_launches();
    case 10: case 11: case 12: case 13: return e.latency_sum_ns(which - 10);
    case 20: case 21: case 22: case 23: return e.latency_count(which - 20);
    default: return 0;
  }
}
int hvd_control_plane_string(int process_set_id, char* out, int cap) {
  if (cap <= 0) return -1;
  snprintf(out, (size_t)cap, "%s", Engine::Get().ControlPlaneString(process_set_id).c_str());
  return 0;
}
unsigned long long hvd_host_path_count(int which) { return cpu::HostPathCount(which); }
// named counters: hvd_metric(type, field) with type = ResponseType value, field = Engine::MetricField
unsigned long long hvd_metric(int type, int field) {
  if (type < 0 || type >= Engine::kMetricTypes || field < 0 || field >= Engine::kPerType) return 0;
  return Engine::Get().metric(type, field);
}
int hvd_metric_type_name(int type, char* out, int cap) {
  if (type < 0 || type >= Engine::kMetricTypes || cap <= 0) return -1;
  const char* n = ResponseTypeName((ResponseType)type);
  snprintf(out, (size_t)cap, "%s", n ? n : "");
  return 0;
}
// tunables (read back what the autotuner / env decided)
long long hvd_param(int which) {
  const TunableParams& p = Engine::Get().parameter_manager().params();
  switch (which) {
    case 0: return p.fusion_threshold_bytes;
    case 1: return (long long)(p.cycle_time_ms * 1000.0);
    case 2: return p.cache_enabled;
    case 3: return p.oneshot_max_bytes;
    case 4: return p.nvls_min_bytes;
    case 5: return p.comm_ctas;
    case 6: return p.active;
    default: return -1;
  }
}

}  // extern "C"
