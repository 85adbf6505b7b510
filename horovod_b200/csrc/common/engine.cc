#include "engine.h"
#include <arpa/inet.h>
#include <ifaddrs.h>
#include <netinet/in.h>
#include <pthread.h>
#include <sched.h>
#include <unistd.h>
#include <algorithm>
#include <chrono>
#include <cstring>
#include <future>
#include <sstream>
#include "../ops/cpu_ops.h"
#include "../ops/nccl_baseline.h"
#include "../symm/symm_memory.h"
#include "../ops/ipc_registry.h"
#include "env.h"
#include "logging.h"
#include "nvtx_op_range.h"

namespace hvd {

// IPv4 address of the first interface named in `ifaces` (comma separated) that has one; "" when none matches.
static std::string InterfaceAddress(const std::string& ifaces) {
  if (ifaces.empty()) return "";
  struct ifaddrs* list = nullptr;
  if (getifaddrs(&list) != 0) return "";
  std::string found;
  size_t start = 0;
  while (found.empty() && start <= ifaces.size()) {
    size_t end = ifaces.find(',', start);
    if (end == std::string::npos) end = ifaces.size();
    const std::string want = ifaces.substr(start, end - start);
    for (struct ifaddrs* it = list; it && found.empty(); it = it->ifa_next) {
      if (!it->ifa_addr || it->ifa_addr->sa_family != AF_INET || want != it->ifa_name) continue;
      char buf[INET_ADDRSTRLEN];
      if (inet_ntop(AF_INET, &((struct sockaddr_in*)it->ifa_addr)->sin_addr, buf, sizeof buf)) found = buf;
    }
    start = end + 1;
  }
  freeifaddrs(list);
  if (found.empty()) LOG(WARNING) << "HOROVOD_GLOO_IFACE=" << ifaces << ": no such interface with an IPv4 address; using the default route";
  return found;
}

namespace {
// NVTX range from enqueue until the entry dies (after its completion callback)
void AttachNvtx(const std::shared_ptr<TensorTableEntry>& e) {
  if (!NvtxEnabled()) return;
  NvtxOp op = NvtxOp::ALLREDUCE;
  const bool grouped = e->group_id >= 0;
  switch (e->type) {
    case RequestType::ALLREDUCE: op = grouped ? NvtxOp::GROUPED_ALLREDUCE : NvtxOp::ALLREDUCE; break;
    case RequestType::ADASUM: op = NvtxOp::ADASUM; break;
    case RequestType::ALLGATHER: op = grouped ? NvtxOp::GROUPED_ALLGATHER : NvtxOp::ALLGATHER; break;
    case RequestType::BROADCAST: op = NvtxOp::BROADCAST; break;
    case RequestType::ALLTOALL: op = NvtxOp::ALLTOALL; break;
    case RequestType::REDUCESCATTER: op = grouped ? NvtxOp::GROUPED_REDUCESCATTER : NvtxOp::REDUCESCATTER; break;
    default: break;
  }
  auto r = std::make_shared<NvtxOpRange>();
  r->Start(op, (int64_t)e->bytes());
  e->nvtx_range = r;
}

struct DeviceClockBase { cudaEvent_t ev = nullptr; uint64_t host_ns = 0; uint64_t session_ns = 0; };
// One (CUDA event, host timestamp) pair per device and timeline session: device-side offsets of later events are
// measured against it with cudaEventElapsedTime, which places GPU spans on the host-clocked timeline.
DeviceClockBase* DeviceBaseFor(int device, uint64_t session_ns) {
  static std::mutex mu;
  static std::map<int, DeviceClockBase> bases;
  std::lock_guard<std::mutex> l(mu);
  DeviceClockBase& b = bases[device];
  if (b.ev && b.session_ns == session_ns) return &b;
  if (!b.ev && cudaEventCreate(&b.ev) != cudaSuccess) { cudaGetLastError(); b.ev = nullptr; return nullptr; }
  cudaStream_t s = GpuContext::Get().Stream(device);
  if (cudaEventRecord(b.ev, s) != cudaSuccess || cudaEventSynchronize(b.ev) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  b.host_ns = NowNs();
  b.session_ns = session_ns;
  return &b;
}


std::string JoinInts(const std::vector<int>& v) {
  std::ostringstream os;
  for (size_t i = 0; i < v.size(); ++i) os << (i ? "," : "") << v[i];
  return os.str();
}

void SetAffinityFromEnv(int local_rank) {
  std::string spec = EnvStr(HOROVOD_THREAD_AFFINITY);
  if (spec.empty()) return;
  std::vector<int> cores;
  std::stringstream ss(spec);
  std::string tok;
  while (std::getline(ss, tok, ',')) if (!tok.empty()) cores.push_back(atoi(tok.c_str()));
  if (local_rank >= (int)cores.size()) { LOG(WARNING) << "HOROVOD_THREAD_AFFINITY has fewer entries than local ranks"; return; }
  cpu_set_t set;
  CPU_ZERO(&set);
  CPU_SET(cores[local_rank], &set);
  if (pthread_setaffinity_np(pthread_self(), sizeof set, &set) != 0) LOG(WARNING) << "could not pin the background thread to core " << cores[local_rank];
}
}  // namespace

Engine::Engine() = default;
Engine::~Engine() { Shutdown(); }
Engine& Engine::Get() { static Engine* e = new Engine(); return *e; }  // leaked on purpose: no static-destruction races with CUDA

// ---------------------------------------------------------------------------
// init / shutdown

Status Engine::Init(const InitConfig& cfg) {
  // already running -> no-op.  A loop that ended on its own (a peer shut the job down, or it failed) leaves the rank /
  // size queries valid until the local shutdown, like the reference; a new init() then starts a fresh runtime.
  if (initialized_.load() && !loop_exited_.load()) return Status::OK();
  if (thread_.joinable()) thread_.join();
  cfg_ = cfg;
  init_done_ = false; init_failed_ = false; shutdown_requested_ = false; loop_exited_ = false;
  cycles_ = 0; fast_cycles_ = 0; responses_ = 0;
  for (auto& m : op_metrics_) m = 0;
  ResetLogLevelFromEnv();
  SetLogRank(cfg.rank);
  thread_ = std::thread(&Engine::BackgroundThread, this);
  while (!init_done_.load() && !init_failed_.load()) std::this_thread::sleep_for(std::chrono::microseconds(200));
  if (init_failed_.load()) {
    if (thread_.joinable()) thread_.join();
    return Status::UnknownError("Horovod initialization failed: " + last_error());
  }
  initialized_ = true;
  return Status::OK();
}

void Engine::Shutdown() {
  if (!thread_.joinable()) { initialized_ = false; return; }
  shutdown_requested_ = true;
  Wake();
  thread_.join();
  initialized_ = false;
}

void Engine::Wake() {
  { std::lock_guard<std::mutex> l(wake_mu_); wake_flag_ = true; }
  wake_cv_.notify_one();
}

void Engine::NotePending(int64_t bytes) {
  if (pending_bytes_.fetch_add(bytes > 0 ? bytes : 1) == 0) first_pending_ns_ = NowNs();
}
void Engine::RequestFlush() { flush_ = true; Wake(); }
void Engine::BeginWait() { waiters_.fetch_add(1); Wake(); }
void Engine::EndWait() { waiters_.fetch_sub(1); }

std::string Engine::ControlPlaneString(int process_set_id) {
  if (!transport_) return "not initialised";
  if (process_set_id == 0) return transport_->Describe();
  auto ps = sets_.Get(process_set_id);
  if (!ps) return "no such process set";
  return ps->transport ? ps->transport->Describe() : std::string("not a member of this process set");
}

std::shared_ptr<ProcessSet> Engine::MakeProcessSet(const std::vector<int>& ranks) {
  auto ps = std::make_shared<ProcessSet>();
  ps->ranks = ranks;
  // the set of ALL ranks talks through the root transport itself, so that it keeps the shared-memory control and data
  // planes of a single-host job (a Split view only forwards point-to-point traffic)
  bool everyone = (int)ranks.size() == transport_->size();
  for (size_t i = 0; everyone && i < ranks.size(); ++i) everyone = ranks[i] == (int)i;
  ps->transport = everyone ? transport_ : transport_->Split(ranks);
  if (ps->transport) {
    ps->cache.set_capacity((uint32_t)EnvInt(HOROVOD_CACHE_CAPACITY, 1024));
    ps->controller.reset(new Controller(ps->transport, &ps->queue, &ps->cache, cfg_.rank == ranks[0] ? &timeline_ : nullptr));
    ps->controller->set_disable_group_fusion(EnvBool(HOROVOD_DISABLE_GROUP_FUSION, false));
  }
  return ps;
}

void Engine::FailAll(const Status& s) {
  for (int32_t id : sets_.Ids()) {
    auto ps = sets_.Get(id);
    if (!ps) continue;
    if (ps->team) ps->team->Abort();
    if (ps->local_team) ps->local_team->Abort();
    ps->queue.FinalizeTensorQueue(s);
  }
}

void Engine::BackgroundThread() {
  try {
    SetAffinityFromEnv(cfg_.local_rank);
    elastic_ = EnvBool(HOROVOD_ELASTIC, false);
    // ---- transport ----
    if (cfg_.transport) {
      transport_ = cfg_.transport;
    } else if (cfg_.size == 1) {
      transport_ = CreateTcpTransport(0, 1, nullptr, cfg_.scope, "127.0.0.1", 1.0);
    } else {
      if (cfg_.rendezvous_addr.empty() || cfg_.rendezvous_port <= 0)
        throw TransportError("no rendezvous server configured (HOROVOD_GLOO_RENDEZVOUS_ADDR/PORT); launch with hvdrun or torchrun");
      HttpKVStore store(cfg_.rendezvous_addr, cfg_.rendezvous_port);
      double timeout = EnvDouble(HOROVOD_TIMEOUT_SECONDS, 60.0);
      // address peers connect to: HVD_HOST_ADDR, else the IPv4 address of the interface the launcher selected
      // (--network-interfaces -> HOROVOD_GLOO_IFACE), else the local address of the route to the rendezvous server
      std::string adv = EnvStr("HVD_HOST_ADDR", "");
      if (adv.empty()) adv = InterfaceAddress(EnvStr("HOROVOD_GLOO_IFACE", ""));
      if (adv.empty()) adv = store.LocalAddress();
      char hn[256] = "localhost";
      gethostname(hn, sizeof hn);
      std::string host = cfg_.hostname.empty() ? std::string(hn) : cfg_.hostname;
      // test-only: the elastic fault-injection tests present one machine as several launcher "hosts" (localhost /
      // 127.0.0.1); with this knob the RUNTIME still sees one host, i.e. one NVLink team over all ranks
      if (EnvBool("HVD_TEST_ONE_HOST", false)) host = "hvd-test-one-host";
      store.Set(cfg_.scope, "host." + std::to_string(cfg_.rank), host);
      std::vector<std::string> hosts(cfg_.size);
      for (int r = 0; r < cfg_.size; ++r) hosts[r] = r == cfg_.rank ? host : store.Get(cfg_.scope, "host." + std::to_string(r), timeout);
      transport_ = CreateTcpTransport(cfg_.rank, cfg_.size, &store, cfg_.scope, adv, timeout, hosts);
      std::string cp = EnvStr(HVD_CONTROL_PLANE, "auto");
      if (cp != "tcp") {
        std::string seg = "hvd-" + std::to_string(cfg_.rendezvous_port) + "-";
        for (char c : cfg_.scope) seg.push_back(isalnum((unsigned char)c) ? c : '_');
        transport_ = transport_->single_host() ? WrapWithShmControl(transport_, seg) : WrapWithHierarchicalControl(transport_, seg);
      }
      // local / cross topology when the launcher did not provide it
      if (cfg_.local_size <= 0) {
        int lr = 0, ls = 0;
        for (int r = 0; r < cfg_.size; ++r) if (hosts[r] == host) { if (r < cfg_.rank) ++lr; ++ls; }
        cfg_.local_rank = lr; cfg_.local_size = ls;
        std::vector<std::string> uniq;
        for (auto& h : hosts) if (std::find(uniq.begin(), uniq.end(), h) == uniq.end()) uniq.push_back(h);
        cfg_.cross_size = (int)uniq.size();
        cfg_.cross_rank = (int)(std::find(uniq.begin(), uniq.end(), host) - uniq.begin());
      }
      std::vector<int64_t> ls(cfg_.size);
      int64_t mine = cfg_.local_size;
      transport_->AllgatherInts(&mine, 1, ls.data());
      homogeneous_ = true;
      for (auto v : ls) if (v != mine) homogeneous_ = false;
    }

    // ---- knobs ----
    params_.ConfigureFromEnv();
    if (EnvIsSet(HOROVOD_FUSION_THRESHOLD)) params_.SetFusionThresholdBytes(EnvInt(HOROVOD_FUSION_THRESHOLD, 128 << 20), true);
    if (EnvIsSet(HOROVOD_CYCLE_TIME)) params_.SetCycleTimeMs(EnvDouble(HOROVOD_CYCLE_TIME, 1.0), true);
    if (EnvIsSet(HOROVOD_CACHE_CAPACITY)) params_.SetCacheEnabled(EnvInt(HOROVOD_CACHE_CAPACITY, 1024) > 0, true);
    if (EnvIsSet(HVD_ONESHOT_MAX_BYTES)) params_.SetOneshotMaxBytes(EnvInt(HVD_ONESHOT_MAX_BYTES, 512 << 10), true);
    if (EnvIsSet(HVD_NVLS_MIN_BYTES)) params_.SetNvlsMinBytes(EnvInt(HVD_NVLS_MIN_BYTES, 1 << 20), true);
    if (EnvIsSet(HVD_COMM_CTAS)) params_.SetCommCtas((int32_t)EnvInt(HVD_COMM_CTAS, 128), true);
    params_.Initialize(cfg_.rank, EnvStr(HOROVOD_AUTOTUNE_LOG));
    params_.SetAutoTuning(EnvBool(HOROVOD_AUTOTUNE, false));

    GpuOpEnv genv;
    genv.params = &params_.params();
    genv.timeline = &timeline_;
    genv.backend = EnvStr(HVD_GPU_BACKEND, "p2p");
    genv.variant = EnvStr(HVD_ALLREDUCE_VARIANT, "auto");
    std::string wire = EnvStr(HVD_WIRE_DTYPE, "none");
    genv.wire_dtype = wire == "bf16" ? DataType::BFLOAT16 : wire == "fp16" ? DataType::FLOAT16 : DataType::FLOAT32;
    genv.symm_buffer_bytes = (size_t)EnvInt(HVD_SYMM_BUFFER_BYTES, 128ll << 20);
    genv.want_multicast = EnvBool("HVD_ENABLE_NVLS", true);
    genv.large_msg_ctas = std::min<int64_t>(kern::kMaxCtas, std::max<int64_t>(4, EnvInt("HVD_LARGE_MSG_CTAS", 256)));
    genv.broadcast_multicast = EnvBool("HVD_BROADCAST_MULTICAST", true);
    // on-the-fly IPC registration of plain in-place tensors (ops/ipc_registry.h); 0 disables
    ipc_min_bytes_ = (genv.backend == "p2p" && EnvBool("HVD_IPC_REGISTRATION", true) && GpuContext::Get().Available())
                         ? std::max<int64_t>(16, EnvInt("HVD_IPC_MIN_BYTES", 4 << 20)) : 0;
    genv.ipc_max_ranks = (int)EnvInt("HVD_IPC_MAX_RANKS", 4);
    genv.latency_lane_bytes = std::min<int64_t>(1 << 20, std::max<int64_t>(0, EnvInt("HVD_LATENCY_LANE_BYTES", 256 << 10)));
    // the reference's knob for concurrent responses (operations.cc:465): 1 = a single stream, i.e. no latency lane
    if (EnvIsSet(HOROVOD_NUM_STREAMS) && EnvInt(HOROVOD_NUM_STREAMS, 1) <= 1 && !EnvIsSet("HVD_LATENCY_LANE_BYTES")) genv.latency_lane_bytes = 0;
    genv.adasum_persistent = EnvBool("HVD_ADASUM_PERSISTENT", true);
    genv.zero_copy_nvls_min_bytes = EnvInt("HVD_ZERO_COPY_NVLS_MIN_BYTES", 1 << 20);
    genv.calibrate = EnvBool("HVD_CALIBRATE", true) && !EnvBool(HOROVOD_AUTOTUNE, false);
    genv.on_calibrated = [this](int64_t oneshot_max, int64_t nvls_min) {
      // measured crossovers replace the built-in defaults unless the user pinned a value
      if (!EnvIsSet(HVD_ONESHOT_MAX_BYTES)) params_.SetOneshotMaxBytes(oneshot_max);
      if (!EnvIsSet(HVD_NVLS_MIN_BYTES)) params_.SetNvlsMinBytes(nvls_min);
    };
    gpu_ops_.reset(new GpuOps(genv));

    // ---- GPU / NVLink topology discovery (new relative to the reference, SURVEY 3.1) ----
    if (GpuContext::Get().Available()) {
      int dev = cfg_.local_rank % GpuContext::Get().DeviceCount();
      GpuTopology topo = DiscoverGpuTopology(dev);
      topology_str_ = topo.DebugString();
      LOG(INFO) << "GPU topology: " << topology_str_;
    } else {
      topology_str_ = "no CUDA device";
    }

    // ---- process sets ----
    sets_.Clear();
    std::vector<int> all(cfg_.size);
    for (int i = 0; i < cfg_.size; ++i) all[i] = i;
    sets_.Insert(MakeProcessSet(all));
    for (auto& r : cfg_.process_sets) {
      std::vector<int> sorted = r;
      std::sort(sorted.begin(), sorted.end());
      sets_.Insert(MakeProcessSet(sorted));
    }
    {  // registration consistency check across ranks (reference process_set.cc:95-134)
      int64_t sig = (int64_t)cfg_.process_sets.size();
      for (auto& r : cfg_.process_sets) for (int v : r) sig = sig * 1000003 + v + 1;
      std::vector<int64_t> sigs(cfg_.size);
      transport_->AllgatherInts(&sig, 1, sigs.data());
      for (auto v : sigs) if (v != sig) throw TransportError("process sets passed to hvd.init() differ between ranks");
    }

    // ---- timeline ----
    std::string tl = EnvStr(HOROVOD_TIMELINE);
    if (!tl.empty() && tl != "DYNAMIC" && cfg_.rank == 0) {
      timeline_.Initialize(tl, cfg_.size);
      timeline_.SetMarkCycles(EnvBool(HOROVOD_TIMELINE_MARK_CYCLES, false));
    }
    finalizers_.Create(1);

    init_done_ = true;
    LOG(DEBUG) << "background thread running: size " << cfg_.size << ", local " << cfg_.local_rank << "/" << cfg_.local_size;
    while (RunLoopOnce()) {}
    FailAll(Status::Aborted(SHUT_DOWN_ERROR_MSG));
  } catch (const std::exception& ex) {
    SetError(ex.what());
    if (!init_done_.load()) {
      LOG(ERROR) << "initialization failed: " << ex.what();
      init_failed_ = true;
    } else {
      LOG(ERROR) << "background loop failed: " << ex.what();
      FailAll(Status::UnknownError(std::string("Horovod background loop failed: ") + ex.what()));
    }
  }
  // teardown
  finalizers_.Reset();
  timeline_.Shutdown();
  for (int32_t id : sets_.Ids()) {
    auto ps = sets_.Get(id);
    if (ps && ps->nccl && elastic_) NcclAbort(*ps->nccl);
  }
  sets_.Clear();
  transport_.reset();
  loop_exited_ = true;
}

// ---------------------------------------------------------------------------
// the cycle

// When does a negotiation cycle start?  (The reference sleeps a fixed HOROVOD_CYCLE_TIME between cycles.)
//   * immediately when a framework thread is WAITING on a handle (synchronize / poll -> RequestFlush)
//   * as soon as HVD_BATCH_BYTES of tensors are queued (enough to amortise one fused NVLink kernel)
//   * when the oldest queued tensor is HVD_BATCH_DELAY_MS old
//   * every cycle_time when idle, so this rank still takes part in rounds other ranks start.
// Each fused response costs one kernel launch whose CTAs rendezvous with the peer GPUs; fewer, larger responses keep
// SMs for the overlapping backward pass (49 launches per ResNet-50 step doubled the step time).
bool Engine::RunLoopOnce() {
  static const int64_t batch_bytes = EnvInt("HVD_BATCH_BYTES", 16ll << 20);
  static const double batch_delay_ms = EnvDouble("HVD_BATCH_DELAY_MS", 2.0);
  static const double spin_us = EnvDouble("HVD_SPIN_US", 50.0);
  {
    const auto idle_deadline = std::chrono::steady_clock::now() + std::chrono::duration<double, std::milli>(params_.params().cycle_time_ms);
    // short spin first: a blocking allreduce in a tight loop re-enqueues within microseconds
    const auto spin_end = std::chrono::steady_clock::now() + std::chrono::duration<double, std::micro>(spin_us);
    while (!flush_.load(std::memory_order_acquire) && waiters_.load(std::memory_order_acquire) == 0 && pending_bytes_.load(std::memory_order_acquire) < batch_bytes &&
           std::chrono::steady_clock::now() < spin_end) {
#if defined(__x86_64__)
      __builtin_ia32_pause();
#endif
    }
    std::unique_lock<std::mutex> l(wake_mu_);
    while (true) {
      const int64_t pb = pending_bytes_.load();
      const bool flush = flush_.load() || waiters_.load() > 0 || shutdown_requested_.load();
      auto now = std::chrono::steady_clock::now();
      if (flush || pb >= batch_bytes) break;
      if (pb > 0 && (double)(NowNs() - first_pending_ns_.load()) >= batch_delay_ms * 1e6) break;
      if (now >= idle_deadline) break;
      auto until = idle_deadline;
      if (pb > 0) {
        auto d = std::chrono::steady_clock::now() + std::chrono::duration_cast<std::chrono::steady_clock::duration>(
                     std::chrono::duration<double, std::milli>(std::max(0.0, batch_delay_ms - (double)(NowNs() - first_pending_ns_.load()) / 1e6)));
        if (d < until) until = d;
      }
      wake_flag_ = false;
      wake_cv_.wait_until(l, until, [&] { return wake_flag_; });
    }
    wake_flag_ = false;
    pending_bytes_ = 0;
    flush_ = false;
  }
  ++cycles_;
  cycle_start_ns_ = NowNs();
  timeline_.MarkCycleStart();
  {  // runtime timeline start / stop requests
    std::lock_guard<std::mutex> l(tl_mu_);
    if (tl_pending_stop_) { timeline_.Shutdown(); tl_pending_stop_ = false; }
    if (tl_pending_start_) {
      if (cfg_.rank == 0) { timeline_.Initialize(tl_pending_file_, cfg_.size); timeline_.SetMarkCycles(tl_pending_mark_); }
      tl_pending_start_ = false;
    }
  }
  bool keep_going = true;
  const TunableParams tp = params_.params();
  for (int32_t id : sets_.Ids()) {
    auto ps = sets_.Get(id);
    if (!ps || !ps->member()) continue;
    ps->controller->set_fusion_threshold(tp.fusion_threshold_bytes);
    ps->controller->set_cache_enabled(tp.cache_enabled);
    // only the GLOBAL set decides when the engine stops: the members of a sub-set may all have asked for shutdown while
    // another rank has not yet, and leaving early would cut that rank's connections in the middle of a negotiation
    const uint64_t t_neg = NowNs();
    ResponseList rl = ps->controller->ComputeResponseList(id == 0 && shutdown_requested_.load());
    if (rl.responses.empty()) ++fast_cycles_;
    else NoteLatency(1, NowNs() - t_neg);
    for (auto& r : rl.responses) PerformOperation(*ps, r);
    if (id == 0 && rl.shutdown) keep_going = false;
    else if (rl.shutdown) shutdown_requested_ = true;  // a sub-set's stall inspector gave up: take the job down through the global set
  }
  if (params_.IsAutoTuning() || tp.active) {
    auto g = sets_.Get(0);
    TunableParams p = params_.params();
    g->controller->SynchronizeParameters(&p);
    if (cfg_.rank != 0) params_.SetParams(p);
  }
  return keep_going;
}

void Engine::PerformOperation(ProcessSet& ps, Response& r) {
  Entries es;
  ps.queue.GetTensorEntriesFromResponse(r, es);
  ++responses_;
  const uint64_t t_exec = NowNs();
  struct Probe {  // latency probes: one sample per response, taken when the function returns (callbacks have run)
    Engine* eng; uint64_t t0; uint64_t first_enqueue;
    ~Probe() {
      const uint64_t now = NowNs();
      eng->NoteLatency(2, now - t0);
      if (first_enqueue) {
        if (eng->cycle_start_ns_ > first_enqueue) eng->NoteLatency(0, eng->cycle_start_ns_ - first_enqueue);
        eng->NoteLatency(3, now - first_enqueue);
      }
    }
  } probe{this, t_exec, 0};
  for (auto& e : es) if (e && e->enqueue_ns && (probe.first_enqueue == 0 || e->enqueue_ns < probe.first_enqueue)) probe.first_enqueue = e->enqueue_ns;
  auto finish_all = [&](const Status& st) {
    for (auto& e : es) if (e && e->callback) { Completion c; c.status = st; c.received_splits = e->received_splits; e->callback(c); }
  };
  for (auto& e : es) if (e && e->group_id >= 0) ps.groups.DeregisterGroup(e->group_id);

  switch (r.type) {
    case ResponseType::ERROR:
      op_metrics_[(int)ResponseType::ERROR * kPerType + kResponses].fetch_add(1, std::memory_order_relaxed);
      op_metrics_[(int)ResponseType::ERROR * kPerType + kTensors].fetch_add(r.tensor_names.size(), std::memory_order_relaxed);
      finish_all(Status::PreconditionError(r.error_message));
      return;
    case ResponseType::JOIN:
      for (auto& e : es) if (e && e->callback) { Completion c; c.last_joined_rank = ps.ranks[std::max(0, r.last_joined_rank)]; e->callback(c); }
      return;
    case ResponseType::BARRIER: finish_all(Status::OK()); return;
    case ResponseType::PROCESS_SET_ADD: {
      std::vector<int> ranks(r.tensor_sizes.begin(), r.tensor_sizes.end());
      Completion c;
      if (sets_.Find(ranks) >= 0) c.status = Status::InvalidArgument("A process set with these ranks has already been added.");
      else c.last_joined_rank = sets_.Insert(MakeProcessSet(ranks));
      for (auto& e : es) if (e && e->callback) e->callback(c);
      return;
    }
    case ResponseType::SYMM_ALLOC: {
      // collective allocation of a registered region on this set's peer-mapped team
      Completion c;
      int dev = -1;
      for (auto& e : es) if (e) dev = e->device;
      const size_t bytes = r.tensor_sizes.empty() ? 0 : (size_t)r.tensor_sizes[0];
      std::shared_ptr<SymmTeam> team = dev >= 0 && ps.set_size() > 1 ? gpu_ops_->EnsureTeam(ps, dev) : nullptr;
      uint64_t have = team ? 1 : 0;
      ps.transport->AllreduceBits(&have, 1, nullptr, 0);
      if (!have) {
        c.status = Status::PreconditionError("symmetric memory is not available for this process set (single rank, "
                                             "several hosts, or no peer access)");
      } else {
        std::string why;
        int idx = team->AllocRegion(ps.transport.get(), bytes, cfg_.scope + "-" + std::to_string(cfg_.rendezvous_port) +
                                                                    "-ps" + std::to_string(ps.id) + "-" + r.tensor_names[0], &why);
        if (idx < 0) c.status = Status::UnknownError("symmetric allocation failed: " + why);
        else c.aux_ptr = team->RegionPtr(idx);
      }
      for (auto& e : es) if (e && e->callback) e->callback(c);
      return;
    }
    case ResponseType::PROCESS_SET_REMOVE: {
      int32_t id = r.tensor_sizes.empty() ? -1 : (int32_t)r.tensor_sizes[0];
      Completion c;
      auto victim = sets_.Get(id);
      if (!victim || id == 0) c.status = Status::InvalidArgument("Process set " + std::to_string(id) + " does not exist or cannot be removed.");
      else { victim->queue.FinalizeTensorQueue(Status::Aborted("process set removed")); sets_.Remove(id); c.last_joined_rank = id; }
      for (auto& e : es) if (e && e->callback) e->callback(c);
      return;
    }
    default: break;
  }

  // The device is a LOCAL property: take it from an entry this rank submitted; a joined rank (no entries) uses the
  // device it passed to hvd.join() — the coordinator cannot know it (response.devices only tells CPU vs GPU).
  int device = r.devices.empty() ? CPU_DEVICE_ID : r.devices[ps.set_rank()];
  if (device != CPU_DEVICE_ID) {
    int local = -2;
    for (auto& e : es) if (e) { local = e->device; break; }
    if (local == -2) local = join_device_.load();
    if (local >= 0) device = local;
  }
  int64_t bytes = 0;
  for (auto n : r.tensor_sizes) bytes += n * (int64_t)DataTypeSize(r.dtype);
  if (timeline_.Initialized()) for (auto& e : es) if (e) timeline_.Start(e->name, r.type, e->bytes());

  Status st;
  SharedEvent* done = nullptr;
  // device-timed timeline row: CUDA events (timing enabled) around the kernels of this response on the hvd stream
  cudaEvent_t tl_t0 = nullptr, tl_t1 = nullptr;
  DeviceClockBase* tl_base = nullptr;
  if (device != CPU_DEVICE_ID && timeline_.Initialized()) {
    tl_base = DeviceBaseFor(device, timeline_.session_start_ns());
    if (tl_base && cudaEventCreate(&tl_t0) == cudaSuccess && cudaEventCreate(&tl_t1) == cudaSuccess) {
      cudaEventRecord(tl_t0, GpuContext::Get().Stream(device));
    } else {
      if (tl_t0) cudaEventDestroy(tl_t0);
      tl_t0 = tl_t1 = nullptr; cudaGetLastError();
    }
  }
  try {
    if (device == CPU_DEVICE_ID) {
      st = ExecuteCpu(ps, es, r);
    } else {
      switch (r.type) {
        case ResponseType::ALLREDUCE: st = gpu_ops_->Allreduce(ps, es, r, device, &done); break;
        case ResponseType::ADASUM: st = gpu_ops_->Adasum(ps, es, r, device, &done); break;
        case ResponseType::ALLGATHER: st = gpu_ops_->Allgather(ps, es, r, device, &done); break;
        case ResponseType::BROADCAST: st = gpu_ops_->Broadcast(ps, es, r, device, &done); break;
        case ResponseType::ALLTOALL: st = gpu_ops_->Alltoall(ps, es, r, device, &done); break;
        case ResponseType::REDUCESCATTER: st = gpu_ops_->Reducescatter(ps, es, r, device, &done); break;
        default: st = Status::InvalidArgument("unsupported GPU response type"); break;
      }
    }
  } catch (const TransportError& ex) {
    if (done) { for (size_t i = 0; i < es.size(); ++i) GpuContext::Get().Release(done); }
    finish_all(Status::UnknownError(ex.what()));
    throw;
  }

  if (ps.set_rank() == 0 && ps.id == 0 && params_.IsAutoTuning()) params_.Update(r.tensor_names, bytes);
  {
    const int ty = (int)r.type;
    if (ty >= 0 && ty < kMetricTypes) {
      auto* m = &op_metrics_[ty * kPerType];
      m[kResponses].fetch_add(1, std::memory_order_relaxed);
      m[kTensors].fetch_add(r.tensor_names.size(), std::memory_order_relaxed);
      int64_t payload = 0;   // bytes this rank contributed (allgather / alltoall sizes are per rank, the entries know them)
      for (auto& e : es) if (e) payload += (int64_t)e->bytes();
      m[kBytes].fetch_add((uint64_t)(payload > 0 ? payload : bytes), std::memory_order_relaxed);
      if (device != CPU_DEVICE_ID) m[kOnGpu].fetch_add(1, std::memory_order_relaxed);
      if (!st.ok()) m[kErrors].fetch_add(1, std::memory_order_relaxed);
    }
  }

  if (tl_t1) cudaEventRecord(tl_t1, GpuContext::Get().Stream(device));
  if (done) {
    if (timeline_.Initialized()) {
      done->refs.fetch_add(1);
      std::vector<std::string> names;
      for (auto& e : es) if (e) names.push_back(e->name);
      const std::string act = std::string("GPU ") + ResponseTypeName(r.type);
      const uint64_t launched_ns = NowNs();
      finalizers_.Execute([this, done, names, tl_t0, tl_t1, tl_base, act, launched_ns] {
        cudaSetDevice(done->device);
        cudaEventSynchronize(done->ev);
        if (tl_t0 && tl_t1 && tl_base && cudaEventSynchronize(tl_t1) == cudaSuccess) {
          float off_ms = 0, dur_ms = 0;
          if (cudaEventElapsedTime(&off_ms, tl_base->ev, tl_t0) == cudaSuccess && cudaEventElapsedTime(&dur_ms, tl_t0, tl_t1) == cudaSuccess) {
            const int64_t start_us = timeline_.ToTimelineUs(tl_base->host_ns) + (int64_t)(off_ms * 1e3);
            // QUEUE (reference activity name, common.h:80-114): launched on the host, not yet running on the device — the
            // stream was still busy or waiting for the tensors' ready events
            const int64_t launched_us = timeline_.ToTimelineUs(launched_ns);
            if (start_us > launched_us + 1) timeline_.DeviceSpan(names, HVD_ACT_QUEUE, launched_us, start_us - launched_us);
            timeline_.DeviceSpan(names, act, start_us, (int64_t)(dur_ms * 1e3));
          }
        }
        if (tl_t0) cudaEventDestroy(tl_t0);
        if (tl_t1) cudaEventDestroy(tl_t1);
        cudaGetLastError();
        for (auto& n : names) timeline_.End(n);
        GpuContext::Get().Release(done);
      });
      tl_t0 = tl_t1 = nullptr;
    }
    for (auto& e : es) {
      if (e && e->callback) {
        Completion c; c.status = st; c.done_event = st.ok() ? done : nullptr; c.received_splits = e->received_splits;
        if (!st.ok()) GpuContext::Get().Release(done);
        e->callback(c);
      } else {
        GpuContext::Get().Release(done);  // joined placeholder: nobody will wait on it
      }
    }
  } else {
    if (timeline_.Initialized()) for (auto& e : es) if (e) timeline_.End(e->name);
    finish_all(st);
  }
  if (tl_t0) cudaEventDestroy(tl_t0);
  if (tl_t1) cudaEventDestroy(tl_t1);
}

// ---------------------------------------------------------------------------
// CPU execution

Status Engine::ExecuteCpu(ProcessSet& ps, Entries& es, const Response& r) {
  Transport* t = ps.transport.get();
  const int n = ps.set_size(), me = ps.set_rank();
  const size_t esz = DataTypeSize(r.dtype);
  switch (r.type) {
    case ResponseType::ALLREDUCE:
    case ResponseType::ADASUM: {
      const bool adasum = r.type == ResponseType::ADASUM;
      std::vector<int64_t> counts(es.size());
      int64_t total = 0;
      for (size_t i = 0; i < es.size(); ++i) { counts[i] = es[i] ? es[i]->shape.num_elements() : r.tensor_sizes[i]; total += counts[i]; }
      char* buf;
      const bool single = es.size() == 1 && es[0];
      if (single) {
        if (es[0]->output != es[0]->input) memcpy(es[0]->output, es[0]->input, (size_t)total * esz);
        buf = (char*)es[0]->output;
      } else {
        if (timeline_.Initialized()) timeline_.ActivityStartAll(es, HVD_ACT_MEMCPY_IN_FUSION_BUFFER);
        fusion_host_.resize((size_t)total * esz);
        buf = fusion_host_.data();
        int64_t off = 0;
        for (size_t i = 0; i < es.size(); ++i) {
          if (es[i]) memcpy(buf + off * esz, es[i]->input, (size_t)counts[i] * esz);
          else memset(buf + off * esz, 0, (size_t)counts[i] * esz);
          off += counts[i];
        }
      }
      cpu::ScaleBuffer(buf, total, r.dtype, r.prescale);
      if (timeline_.Initialized()) timeline_.ActivityStartAll(es, adasum ? HVD_ACT_CPU_ADASUM : HVD_ACT_CPU_ALLREDUCE);
      if (adasum) {
        Status st = cpu::AdasumAllreduce(t, buf, counts, r.dtype);
        if (!st.ok()) return st;
      } else {
        cpu::Allreduce(t, buf, total, r.dtype, r.reduce_op);
      }
      cpu::ScaleBuffer(buf, total, r.dtype, r.postscale);
      if (!single) {
        if (timeline_.Initialized()) timeline_.ActivityStartAll(es, HVD_ACT_MEMCPY_OUT_FUSION_BUFFER);
        int64_t off = 0;
        for (size_t i = 0; i < es.size(); ++i) {
          if (es[i]) memcpy(es[i]->output, buf + off * esz, (size_t)counts[i] * esz);
          off += counts[i];
        }
      }
      return Status::OK();
    }
    case ResponseType::ALLGATHER: {
      for (size_t ti = 0; ti < es.size(); ++ti) {
        auto& e = es[ti];
        if (!e) return Status::PreconditionError("Allgather is not supported with Join at this time.");
        int64_t row = 1;
        for (int d = 1; d < e->shape.ndim(); ++d) row *= e->shape.dim(d);
        std::vector<int64_t> bytes(n);
        int64_t rows = 0;
        for (int p = 0; p < n; ++p) { bytes[p] = r.tensor_sizes[ti * n + p] * row * (int64_t)esz; rows += r.tensor_sizes[ti * n + p]; }
        std::vector<int64_t> oshape = e->shape.dims();
        oshape[0] = rows;
        if (e->alloc_output) e->output = e->alloc_output(oshape);
        if (!e->output && rows * row > 0) return Status::UnknownError("allgather: output allocation failed");
        if (timeline_.Initialized()) timeline_.ActivityStart(e->name, HVD_ACT_CPU_ALLGATHER);
        cpu::Allgatherv(t, e->input, e->output, bytes);
      }
      return Status::OK();
    }
    case ResponseType::BROADCAST: {
      for (auto& e : es) {
        if (!e) return Status::PreconditionError("Broadcast is not supported with Join at this time.");
        if (me == r.root_rank && e->output != e->input && e->output) memcpy(e->output, e->input, e->bytes());
        if (timeline_.Initialized()) timeline_.ActivityStart(e->name, HVD_ACT_CPU_BROADCAST);
        cpu::Broadcast(t, e->output ? e->output : const_cast<void*>(e->input), (int64_t)e->bytes(), r.root_rank);
      }
      return Status::OK();
    }
    case ResponseType::ALLTOALL: {
      for (auto& e : es) {
        if (!e) return Status::PreconditionError("Alltoall is not supported with Join at this time.");
        int64_t row = 1;
        for (int d = 1; d < e->shape.ndim(); ++d) row *= e->shape.dim(d);
        std::vector<int64_t> mine(n), all((size_t)n * n);
        for (int p = 0; p < n; ++p) mine[p] = e->splits[p];
        if (r.root_rank == kUniformSplits) std::fill(all.begin(), all.end(), mine[0]);  // negotiated: same shape, no explicit splits anywhere
        else t->AllgatherInts(mine.data(), n, all.data());
        std::vector<int64_t> sb(n), rb(n);
        int64_t out_rows = 0;
        e->received_splits.assign(n, 0);
        for (int p = 0; p < n; ++p) {
          sb[p] = mine[p] * row * (int64_t)esz;
          rb[p] = all[(size_t)p * n + me] * row * (int64_t)esz;
          e->received_splits[p] = (int32_t)all[(size_t)p * n + me];
          out_rows += all[(size_t)p * n + me];
        }
        std::vector<int64_t> oshape = e->shape.dims();
        oshape[0] = out_rows;
        if (e->alloc_output) e->output = e->alloc_output(oshape);
        if (!e->output && out_rows * row > 0) return Status::UnknownError("alltoall: output allocation failed");
        if (timeline_.Initialized()) timeline_.ActivityStart(e->name, HVD_ACT_CPU_ALLTOALL);
        cpu::Alltoallv(t, e->input, sb, e->output, rb);
      }
      return Status::OK();
    }
    case ResponseType::REDUCESCATTER: {
      for (auto& e : es) {
        if (!e) return Status::PreconditionError("Reducescatter is not supported with Join at this time.");
        int64_t row = 1;
        for (int d = 1; d < e->shape.ndim(); ++d) row *= e->shape.dim(d);
        std::vector<int64_t> rows;
        ReducescatterRows(e->shape.dim(0), n, &rows);
        std::vector<int64_t> counts(n);
        for (int p = 0; p < n; ++p) counts[p] = rows[p] * row;
        std::vector<int64_t> oshape = e->shape.dims();
        oshape[0] = rows[me];
        if (!e->output && e->alloc_output) e->output = e->alloc_output(oshape);
        if (!e->output && counts[me] > 0) return Status::UnknownError("reducescatter: output allocation failed");
        const int64_t total = e->shape.num_elements();
        fusion_host_.resize((size_t)total * esz);
        memcpy(fusion_host_.data(), e->input, (size_t)total * esz);
        cpu::ScaleBuffer(fusion_host_.data(), total, r.dtype, r.prescale);
        if (timeline_.Initialized()) timeline_.ActivityStart(e->name, HVD_ACT_CPU_REDUCESCATTER);
        cpu::Reducescatter(t, fusion_host_.data(), counts, e->output, r.dtype, r.reduce_op);
        cpu::ScaleBuffer(e->output, counts[me], r.dtype, r.postscale);
      }
      return Status::OK();
    }
    default: return Status::InvalidArgument("unsupported response type");
  }
}

// ---------------------------------------------------------------------------
// enqueue API

Status Engine::CheckSet(int32_t id, std::shared_ptr<ProcessSet>* out) {
  if (!initialized_.load() || loop_exited_.load()) return Status::PreconditionError(loop_exited_.load() ? SHUT_DOWN_ERROR_MSG : NOT_INITIALIZED_ERROR_MSG);
  auto ps = sets_.Get(id);
  if (!ps) return Status::InvalidArgument("Process set with id " + std::to_string(id) + " does not exist.");
  if (!ps->member()) return Status::InvalidArgument("This rank (" + std::to_string(cfg_.rank) + ") is not a member of process set " + std::to_string(id) + ".");
  *out = ps;
  return Status::OK();
}

namespace {
Request MakeRequest(const TensorTableEntry& e, int set_rank, RequestType type) {
  Request q;
  q.request_rank = set_rank; q.type = type; q.dtype = e.dtype; q.name = e.name; q.root_rank = e.root_rank;
  q.device = e.device; q.shape = e.shape.dims(); q.prescale = e.prescale; q.postscale = e.postscale;
  q.reduce_op = e.reduce_op; q.group_id = e.group_id;
  return q;
}
}  // namespace

Status Engine::EnqueueAllreduces(std::vector<std::shared_ptr<TensorTableEntry>>& es, int32_t psid) {
  std::shared_ptr<ProcessSet> ps;
  Status st = CheckSet(psid, &ps);
  if (!st.ok()) return st;
  std::vector<Request> msgs;
  int32_t gid = -1;
  if (es.size() > 1) {
    std::vector<std::string> names;
    for (auto& e : es) names.push_back(e->name);
    gid = ps->groups.RegisterGroup(names);
  }
  for (auto& e : es) {
    e->process_set_id = psid;
    e->enqueue_ns = NowNs(); AttachNvtx(e);
    e->group_id = gid;
    RequestType type = RequestType::ALLREDUCE;
    if (e->reduce_op == ReduceOp::ADASUM) {
      type = RequestType::ADASUM;
    } else if (e->reduce_op == ReduceOp::AVERAGE) {
      // Average = Sum with the divisor folded into postscale; the divisor stays the full set
      // size even when ranks have joined (reference test_torch.py:2979-3050)
      e->reduce_op = ReduceOp::SUM;
      e->postscale /= (double)ps->set_size();
    }
    e->type = type;
    Request q = MakeRequest(*e, ps->set_rank(), type);
    q.group_size = gid >= 0 ? (int32_t)es.size() : 0;
    if (type == RequestType::ALLREDUCE && e->device >= 0 && e->input == e->output && es.size() == 1) {
      // in-place tensor inside a registered symmetric region -> candidate for the zero-copy kernel
      std::shared_ptr<SymmTeam> team;
      { std::lock_guard<std::mutex> l(ps->team_mu); team = ps->team; }
      int64_t off = 0;
      int idx = -1;
      if (team && (e->bytes() % 16) == 0 && team->FindRegion(e->input, e->bytes(), nullptr, &off, &idx) && (off % 16) == 0)
        q.symm_key = ((int64_t)idx << 44) | off;
      else if (ipc_min_bytes_ > 0 && (int64_t)e->bytes() >= ipc_min_bytes_ && (e->bytes() % 16) == 0 && ((uintptr_t)e->input % 16) == 0 &&
               ps->set_size() > 1)
        q.symm_key = IpcKeyFor(e->input);  // plain allocation: candidate for on-the-fly IPC registration (<= -2, or -1)
    }
    msgs.push_back(std::move(q));
  }
  st = ps->queue.AddToTensorQueueMulti(es, msgs);
  if (!st.ok()) { if (gid >= 0) ps->groups.DeregisterGroup(gid); return st; }
  { int64_t b = 0; for (auto& e : es) b += (int64_t)e->bytes(); NotePending(b); }
  Wake();
  return Status::OK();
}

Status Engine::EnqueueAllgathers(std::vector<std::shared_ptr<TensorTableEntry>>& es, int32_t psid) {
  std::shared_ptr<ProcessSet> ps;
  Status st = CheckSet(psid, &ps);
  if (!st.ok()) return st;
  std::vector<Request> msgs;
  int32_t gid = -1;
  if (es.size() > 1) {
    std::vector<std::string> names;
    for (auto& e : es) names.push_back(e->name);
    gid = ps->groups.RegisterGroup(names);
  }
  for (auto& e : es) {
    e->process_set_id = psid; e->type = RequestType::ALLGATHER; e->group_id = gid; e->enqueue_ns = NowNs(); AttachNvtx(e);
    Request q = MakeRequest(*e, ps->set_rank(), RequestType::ALLGATHER);
    q.group_size = gid >= 0 ? (int32_t)es.size() : 0;
    msgs.push_back(std::move(q));
  }
  st = ps->queue.AddToTensorQueueMulti(es, msgs);
  if (!st.ok()) { if (gid >= 0) ps->groups.DeregisterGroup(gid); return st; }
  { int64_t b = 0; for (auto& e : es) b += (int64_t)e->bytes(); NotePending(b); }
  Wake();
  return Status::OK();
}

Status Engine::EnqueueBroadcast(std::shared_ptr<TensorTableEntry> e, int32_t psid) {
  std::shared_ptr<ProcessSet> ps;
  Status st = CheckSet(psid, &ps);
  if (!st.ok()) return st;
  // root_rank arrives as a GLOBAL rank (reference operations.cc:1702-1710)
  auto it = std::find(ps->ranks.begin(), ps->ranks.end(), e->root_rank);
  if (it == ps->ranks.end())
    return Status::InvalidArgument("broadcast received invalid root rank " + std::to_string(e->root_rank) + " for provided process set");
  e->root_rank = (int)(it - ps->ranks.begin());
  e->process_set_id = psid; e->type = RequestType::BROADCAST; e->enqueue_ns = NowNs(); AttachNvtx(e);
  st = ps->queue.AddToTensorQueue(e, MakeRequest(*e, ps->set_rank(), RequestType::BROADCAST));
  if (!st.ok()) return st;
  NotePending((int64_t)e->bytes());
  Wake();
  return Status::OK();
}

Status Engine::EnqueueAlltoall(std::shared_ptr<TensorTableEntry> e, int32_t psid) {
  std::shared_ptr<ProcessSet> ps;
  Status st = CheckSet(psid, &ps);
  if (!st.ok()) return st;
  const int n = ps->set_size();
  if (e->shape.ndim() < 1) return Status::InvalidArgument("alltoall requires a tensor with at least one dimension");
  const bool implicit_splits = e->splits.empty();
  if (implicit_splits) {
    if (e->shape.dim(0) % n != 0)
      return Status::InvalidArgument("tensor must have first dimension divisible by the number of workers when no splits are specified.");
    e->splits.assign(n, (int32_t)(e->shape.dim(0) / n));
  } else {
    if ((int)e->splits.size() != n) return Status::InvalidArgument("Number of entries in splits does not equal number of workers.");
    int64_t sum = 0;
    for (auto s : e->splits) { if (s < 0) return Status::InvalidArgument("splits must be non-negative"); sum += s; }
    if (sum > e->shape.dim(0)) return Status::InvalidArgument("Sum of splits entries is greater than the first dimension of tensor.");
  }
  e->process_set_id = psid; e->type = RequestType::ALLTOALL; e->enqueue_ns = NowNs(); AttachNvtx(e);
  Request q = MakeRequest(*e, ps->set_rank(), RequestType::ALLTOALL);
  // root_rank is unused by alltoall: kUniformSplits marks "no splits given" — when every rank says so with the same shape the
  // split matrix is known everywhere and the per-call exchange through the control plane (the reference's
  // AlltoallGetRecvSplits, mpi_controller.cc:243) is skipped
  q.root_rank = implicit_splits ? kUniformSplits : 0;
  st = ps->queue.AddToTensorQueue(e, q);
  if (!st.ok()) return st;
  NotePending((int64_t)e->bytes());
  Wake();
  return Status::OK();
}

Status Engine::EnqueueReducescatters(std::vector<std::shared_ptr<TensorTableEntry>>& es, int32_t psid) {
  std::shared_ptr<ProcessSet> ps;
  Status st = CheckSet(psid, &ps);
  if (!st.ok()) return st;
  std::vector<Request> msgs;
  int32_t gid = -1;
  if (es.size() > 1) {
    std::vector<std::string> names;
    for (auto& e : es) names.push_back(e->name);
    gid = ps->groups.RegisterGroup(names);
  }
  for (auto& e : es) {
    if (e->reduce_op == ReduceOp::AVERAGE) { e->reduce_op = ReduceOp::SUM; e->postscale /= (double)ps->set_size(); }
    e->process_set_id = psid; e->type = RequestType::REDUCESCATTER; e->group_id = gid; e->enqueue_ns = NowNs(); AttachNvtx(e);
    Request q = MakeRequest(*e, ps->set_rank(), RequestType::REDUCESCATTER);
    q.group_size = gid >= 0 ? (int32_t)es.size() : 0;
    msgs.push_back(std::move(q));
  }
  st = ps->queue.AddToTensorQueueMulti(es, msgs);
  if (!st.ok()) { if (gid >= 0) ps->groups.DeregisterGroup(gid); return st; }
  { int64_t b = 0; for (auto& e : es) b += (int64_t)e->bytes(); NotePending(b); }
  Wake();
  return Status::OK();
}

Status Engine::EnqueueJoin(std::shared_ptr<TensorTableEntry> e, int32_t psid) {
  std::shared_ptr<ProcessSet> ps;
  Status st = CheckSet(psid, &ps);
  if (!st.ok()) return st;
  e->name = JOIN_TENSOR_NAME; e->process_set_id = psid; e->type = RequestType::JOIN;
  if (e->device >= 0) join_device_ = e->device;
  st = ps->queue.AddToTensorQueue(e, MakeRequest(*e, ps->set_rank(), RequestType::JOIN));
  if (!st.ok()) return st;
  RequestFlush();
  return Status::OK();
}

Status Engine::EnqueueBarrier(std::shared_ptr<TensorTableEntry> e, int32_t psid) {
  std::shared_ptr<ProcessSet> ps;
  Status st = CheckSet(psid, &ps);
  if (!st.ok()) return st;
  e->name = BARRIER_TENSOR_NAME; e->process_set_id = psid; e->type = RequestType::BARRIER;
  st = ps->queue.AddToTensorQueue(e, MakeRequest(*e, ps->set_rank(), RequestType::BARRIER));
  if (!st.ok()) return st;
  RequestFlush();
  return Status::OK();
}

// ---------------------------------------------------------------------------
// dynamic process sets: negotiated like a tensor on the global set, so every
// rank applies the change at the same point of the response stream.

int32_t Engine::AddProcessSet(const std::vector<int>& ranks_in, std::string* err) {
  std::vector<int> ranks = ranks_in;
  std::sort(ranks.begin(), ranks.end());
  ranks.erase(std::unique(ranks.begin(), ranks.end()), ranks.end());
  for (int r : ranks) if (r < 0 || r >= cfg_.size) { if (err) *err = "process set rank out of range"; return -1; }
  if (ranks.empty()) { if (err) *err = "empty process set"; return -1; }
  std::shared_ptr<ProcessSet> g;
  Status st = CheckSet(0, &g);
  if (!st.ok()) { if (err) *err = st.reason(); return -1; }
  auto e = std::make_shared<TensorTableEntry>();
  e->name = PS_ADD_PREFIX + JoinInts(ranks);
  e->type = RequestType::PROCESS_SET_ADD;
  std::promise<Completion> prom;
  auto fut = prom.get_future();
  e->callback = [&prom](const Completion& c) { prom.set_value(c); };
  Request q = MakeRequest(*e, g->set_rank(), RequestType::PROCESS_SET_ADD);
  q.shape.assign(ranks.begin(), ranks.end());
  st = g->queue.AddToTensorQueue(e, q);
  if (!st.ok()) { if (err) *err = st.reason(); return -1; }
  RequestFlush();
  Completion c = fut.get();
  if (!c.status.ok()) { if (err) *err = c.status.reason(); return -1; }
  return c.last_joined_rank;
}

int32_t Engine::RemoveProcessSet(int32_t id, std::string* err) {
  std::shared_ptr<ProcessSet> g;
  Status st = CheckSet(0, &g);
  if (!st.ok()) { if (err) *err = st.reason(); return -1; }
  auto e = std::make_shared<TensorTableEntry>();
  e->name = PS_REMOVE_PREFIX + std::to_string(id);
  e->type = RequestType::PROCESS_SET_REMOVE;
  std::promise<Completion> prom;
  auto fut = prom.get_future();
  e->callback = [&prom](const Completion& c) { prom.set_value(c); };
  Request q = MakeRequest(*e, g->set_rank(), RequestType::PROCESS_SET_REMOVE);
  q.shape = {id};
  st = g->queue.AddToTensorQueue(e, q);
  if (!st.ok()) { if (err) *err = st.reason(); return -1; }
  RequestFlush();
  Completion c = fut.get();
  if (!c.status.ok()) { if (err) *err = c.status.reason(); return -1; }
  return c.last_joined_rank;
}

// Collective (every member of the set must call it with the same size): allocates `bytes` of peer-mapped memory on
// `device` and returns its local address. Tensors placed there take the zero-copy allreduce path.
void* Engine::AllocSymmetric(size_t bytes, int device, int32_t psid, std::string* err, std::shared_ptr<void>* keep_alive) {
  std::shared_ptr<ProcessSet> ps;
  Status st = CheckSet(psid, &ps);
  if (!st.ok()) { if (err) *err = st.reason(); return nullptr; }
  auto e = std::make_shared<TensorTableEntry>();
  e->name = SYMM_ALLOC_PREFIX + std::to_string(symm_alloc_counter_++);
  e->type = RequestType::SYMM_ALLOC;
  e->device = device;
  std::promise<Completion> prom;
  auto fut = prom.get_future();
  e->callback = [&prom](const Completion& c) { prom.set_value(c); };
  Request q = MakeRequest(*e, ps->set_rank(), RequestType::SYMM_ALLOC);
  q.shape = {(int64_t)bytes};
  st = ps->queue.AddToTensorQueue(e, q);
  if (!st.ok()) { if (err) *err = st.reason(); return nullptr; }
  RequestFlush();
  Completion c = fut.get();
  if (!c.status.ok()) { if (err) *err = c.status.reason(); return nullptr; }
  if (keep_alive) {
    std::lock_guard<std::mutex> l(ps->team_mu);
    if (ps->team) *keep_alive = ps->team->KeepAlive();
  }
  return c.aux_ptr;
}

Status Engine::CapturedAllreduce(void* ptr, int64_t bytes, DataType dtype, ReduceOp op, double prescale, double postscale,
                                 int32_t psid, int max_ctas, void* stream, int channel) {
  std::shared_ptr<ProcessSet> ps;
  Status st = CheckSet(psid, &ps);
  if (!st.ok()) return st;
  if (op == ReduceOp::ADASUM) return Status::InvalidArgument("captured allreduce does not support Adasum");
  if (op == ReduceOp::AVERAGE) { op = ReduceOp::SUM; postscale /= (double)ps->set_size(); }
  if (ps->set_size() == 1) return Status::OK();
  captured_launches_.fetch_add(1, std::memory_order_relaxed);
  return gpu_ops_->CapturedAllreduce(*ps, ptr, bytes, dtype, op, prescale, postscale, max_ctas, (cudaStream_t)stream,
                                     channel);
}

Status Engine::CapturedReducescatter(void* ptr, int64_t bytes, DataType dtype, ReduceOp op, double prescale, double postscale,
                                     int32_t psid, int max_ctas, void* stream) {
  std::shared_ptr<ProcessSet> ps;
  Status st = CheckSet(psid, &ps);
  if (!st.ok()) return st;
  if (op == ReduceOp::ADASUM) return Status::InvalidArgument("captured reducescatter does not support Adasum");
  if (op == ReduceOp::AVERAGE) { op = ReduceOp::SUM; postscale /= (double)ps->set_size(); }
  if (ps->set_size() == 1) return Status::OK();
  captured_launches_.fetch_add(1, std::memory_order_relaxed);
  return gpu_ops_->CapturedReducescatter(*ps, ptr, bytes, dtype, op, prescale, postscale, max_ctas, (cudaStream_t)stream);
}

Status Engine::CapturedAllgather(void* ptr, int64_t bytes, int32_t psid, int max_ctas, void* stream, int channel) {
  std::shared_ptr<ProcessSet> ps;
  Status st = CheckSet(psid, &ps);
  if (!st.ok()) return st;
  if (ps->set_size() == 1) return Status::OK();
  captured_launches_.fetch_add(1, std::memory_order_relaxed);
  return gpu_ops_->CapturedAllgather(*ps, ptr, bytes, max_ctas, (cudaStream_t)stream, channel);
}

Status Engine::CapturedAlltoall(const void* in, int64_t rows, int64_t row_bytes, const void* splits, int64_t nsplits,
                                bool splits_int64, void* out, int64_t capacity, int64_t* recv_splits, int* status, int32_t psid,
                                int max_ctas, void* stream) {
  std::shared_ptr<ProcessSet> ps;
  Status st = CheckSet(psid, &ps);
  if (!st.ok()) return st;
  if (nsplits != ps->set_size())
    return Status::InvalidArgument("captured alltoall: splits has " + std::to_string(nsplits) + " entries, the process set " +
                                   std::to_string(ps->set_size()) + " ranks");
  // unlike the in-place collectives, a one-rank alltoall still has to move rows: there is no kernel without a team
  if (ps->set_size() < 2) return Status::PreconditionError("captured alltoall needs a peer-mapped process set of at least 2 ranks");
  captured_launches_.fetch_add(1, std::memory_order_relaxed);
  return gpu_ops_->CapturedAlltoall(*ps, in, rows, row_bytes, splits, nsplits, splits_int64, out, capacity, recv_splits, status,
                                    max_ctas, (cudaStream_t)stream);
}

Status Engine::StartTimeline(const std::string& file, bool mark_cycles) {
  if (!initialized_.load()) return Status::PreconditionError(NOT_INITIALIZED_ERROR_MSG);
  std::lock_guard<std::mutex> l(tl_mu_);
  tl_pending_file_ = file; tl_pending_mark_ = mark_cycles; tl_pending_start_ = true;
  Wake();
  return Status::OK();
}
Status Engine::StopTimeline() {
  if (!initialized_.load()) return Status::PreconditionError(NOT_INITIALIZED_ERROR_MSG);
  std::lock_guard<std::mutex> l(tl_mu_);
  tl_pending_stop_ = true;
  Wake();
  return Status::OK();
}

}  // namespace hvd
