#include "symm_memory.h"
#include <cuda.h>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <sys/socket.h>
#include <sys/un.h>
#include <unistd.h>
#include <poll.h>
#include <cstring>
#include <fstream>
#include <mutex>
#include <sstream>
#include "../common/logging.h"

namespace hvd {

#define HVD_STR2(x) #x
#define HVD_STR(x) HVD_STR2(x)

namespace {

// ---- lazily loaded driver API (libcuda is not linked: the CPU-only test box
// must be able to load this library) ----------------------------------------
struct Driver {
  void* lib = nullptr;
  bool ok = false;
#define HVD_DRV(name) decltype(&name) p_##name = nullptr;
  HVD_DRV(cuDeviceGet) HVD_DRV(cuDeviceGetAttribute) HVD_DRV(cuGetErrorString)
  HVD_DRV(cuMemGetAllocationGranularity) HVD_DRV(cuMemCreate) HVD_DRV(cuMemExportToShareableHandle)
  HVD_DRV(cuMemImportFromShareableHandle) HVD_DRV(cuMemAddressReserve) HVD_DRV(cuMemMap) HVD_DRV(cuMemSetAccess)
  HVD_DRV(cuMemUnmap) HVD_DRV(cuMemRelease) HVD_DRV(cuMemAddressFree)
  HVD_DRV(cuMulticastCreate) HVD_DRV(cuMulticastAddDevice) HVD_DRV(cuMulticastBindMem)
  HVD_DRV(cuMulticastGetGranularity) HVD_DRV(cuMulticastUnbind)
#undef HVD_DRV
  Driver() {
    lib = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) lib = dlopen("libcuda.so", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) return;
    bool all = true;
#define HVD_LOAD(name) p_##name = (decltype(&name))dlsym(lib, HVD_STR(name)); if (!p_##name) all = false;
    HVD_LOAD(cuDeviceGet) HVD_LOAD(cuDeviceGetAttribute) HVD_LOAD(cuGetErrorString)
    HVD_LOAD(cuMemGetAllocationGranularity) HVD_LOAD(cuMemCreate) HVD_LOAD(cuMemExportToShareableHandle)
    HVD_LOAD(cuMemImportFromShareableHandle) HVD_LOAD(cuMemAddressReserve) HVD_LOAD(cuMemMap) HVD_LOAD(cuMemSetAccess)
    HVD_LOAD(cuMemUnmap) HVD_LOAD(cuMemRelease) HVD_LOAD(cuMemAddressFree)
    bool base = all;
    HVD_LOAD(cuMulticastCreate) HVD_LOAD(cuMulticastAddDevice) HVD_LOAD(cuMulticastBindMem)
    HVD_LOAD(cuMulticastGetGranularity) HVD_LOAD(cuMulticastUnbind)
#undef HVD_LOAD
    ok = base;
    mc_ok = all;
  }
  bool mc_ok = false;
  std::string Err(CUresult r) {
    const char* s = nullptr;
    if (p_cuGetErrorString) p_cuGetErrorString(r, &s);
    return s ? s : ("CUresult " + std::to_string((int)r));
  }
};
Driver& Drv() { static Driver d; return d; }

size_t RoundUp(size_t v, size_t g) { return (v + g - 1) / g * g; }

// ---- fd passing over abstract unix datagram sockets -------------------------
struct FdChannel {
  int fd = -1;
  std::string prefix;
  bool Open(const std::string& pfx, int rank) {
    prefix = pfx;
    fd = socket(AF_UNIX, SOCK_DGRAM, 0);
    if (fd < 0) return false;
    sockaddr_un a = Addr(rank);
    socklen_t len = (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + strlen(a.sun_path + 1));
    return bind(fd, (sockaddr*)&a, len) == 0;
  }
  sockaddr_un Addr(int rank) const {
    sockaddr_un a {};
    a.sun_family = AF_UNIX;
    std::string name = prefix + "-" + std::to_string(rank);
    a.sun_path[0] = '\0';  // abstract namespace: no filesystem entry, vanishes with the process
    strncpy(a.sun_path + 1, name.c_str(), sizeof(a.sun_path) - 2);
    return a;
  }
  bool SendFd(int to_rank, int payload_fd, int32_t kind, int32_t from_rank) {
    sockaddr_un a = Addr(to_rank);
    socklen_t len = (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + strlen(a.sun_path + 1));
    int32_t msg[2] = {kind, from_rank};
    iovec iov {msg, sizeof msg};
    char ctrl[CMSG_SPACE(sizeof(int))] = {};
    msghdr mh {};
    mh.msg_name = &a; mh.msg_namelen = len; mh.msg_iov = &iov; mh.msg_iovlen = 1;
    mh.msg_control = ctrl; mh.msg_controllen = sizeof ctrl;
    cmsghdr* c = CMSG_FIRSTHDR(&mh);
    c->cmsg_level = SOL_SOCKET; c->cmsg_type = SCM_RIGHTS; c->cmsg_len = CMSG_LEN(sizeof(int));
    memcpy(CMSG_DATA(c), &payload_fd, sizeof(int));
    for (int attempt = 0; attempt < 200; ++attempt) {
      if (sendmsg(fd, &mh, 0) >= 0) return true;
      usleep(10000);  // peer socket may not be bound yet / buffer full
    }
    return false;
  }
  bool RecvFd(int* out_fd, int32_t* kind, int32_t* from_rank, int timeout_ms) {
    pollfd pf {fd, POLLIN, 0};
    if (poll(&pf, 1, timeout_ms) <= 0) return false;
    int32_t msg[2] = {0, 0};
    iovec iov {msg, sizeof msg};
    char ctrl[CMSG_SPACE(sizeof(int))] = {};
    msghdr mh {};
    mh.msg_iov = &iov; mh.msg_iovlen = 1; mh.msg_control = ctrl; mh.msg_controllen = sizeof ctrl;
    if (recvmsg(fd, &mh, 0) < 0) return false;
    cmsghdr* c = CMSG_FIRSTHDR(&mh);
    if (!c || c->cmsg_type != SCM_RIGHTS) return false;
    memcpy(out_fd, CMSG_DATA(c), sizeof(int));
    *kind = msg[0]; *from_rank = msg[1];
    return true;
  }
  ~FdChannel() { if (fd >= 0) close(fd); }
};

bool AllAgree(Transport* t, bool ok) {
  uint64_t w = ok ? 1 : 0;
  t->AllreduceBits(&w, 1, nullptr, 0);
  return w != 0;
}

}  // namespace

// ---------------------------------------------------------------------------

std::string GpuTopology::DebugString() const {
  std::ostringstream os;
  os << "device " << device << "/" << device_count << " '" << name << "' sm_" << cc_major << cc_minor << " SMs=" << sm_count
     << " mem=" << (total_mem >> 20) << "MiB vmm=" << vmm_supported << " fd_export=" << fd_handles_supported
     << " multicast(NVLS)=" << multicast_supported << " numa=" << numa_node << " peer_access=[";
  for (size_t i = 0; i < peer_access.size(); ++i) os << (i ? "," : "") << peer_access[i];
  os << "]";
  return os.str();
}

GpuTopology DiscoverGpuTopology(int device) {
  GpuTopology t;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0 || device < 0 || device >= n) { cudaGetLastError(); return t; }
  t.device = device;
  t.device_count = n;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) {
    t.name = prop.name; t.sm_count = prop.multiProcessorCount; t.cc_major = prop.major; t.cc_minor = prop.minor;
    t.total_mem = prop.totalGlobalMem;
    char path[128];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%04x:%02x:%02x.0/numa_node", prop.pciDomainID, prop.pciBusID, prop.pciDeviceID);
    std::ifstream f(path);
    if (f.good()) f >> t.numa_node;
  }
  t.peer_access.assign(n, 0);
  t.p2p_native_atomics.assign(n, 0);
  for (int j = 0; j < n; ++j) {
    if (j == device) { t.peer_access[j] = 1; t.p2p_native_atomics[j] = 1; continue; }
    int can = 0;
    cudaDeviceCanAccessPeer(&can, device, j);
    t.peer_access[j] = can;
    int at = 0;
    cudaDeviceGetP2PAttribute(&at, cudaDevP2PAttrNativeAtomicSupported, device, j);
    t.p2p_native_atomics[j] = at;
  }
  Driver& d = Drv();
  if (d.ok) {
    CUdevice dev;
    if (d.p_cuDeviceGet(&dev, device) == CUDA_SUCCESS) {
      int v = 0;
      if (d.p_cuDeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_VIRTUAL_MEMORY_MANAGEMENT_SUPPORTED, dev) == CUDA_SUCCESS) t.vmm_supported = v;
      v = 0;
      if (d.p_cuDeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, dev) == CUDA_SUCCESS) t.fd_handles_supported = v;
      v = 0;
      if (d.mc_ok && d.p_cuDeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev) == CUDA_SUCCESS) t.multicast_supported = v;
    }
  }
  cudaGetLastError();
  return t;
}

// ---------------------------------------------------------------------------

struct SymmTeam::Impl {
  enum class Kind { VMM, IPC, SIM } kind = Kind::SIM;
  int nranks = 0, rank = 0;
  size_t alloc_bytes = 0;
  // VMM
  std::vector<CUmemGenericAllocationHandle> handles;  // [nranks]; [rank] = own
  std::vector<CUdeviceptr> vas;                       // [nranks]
  CUmemGenericAllocationHandle mc_handle = 0;
  CUdeviceptr mc_va = 0;
  bool mc_bound = false;
  int device = 0;
  // IPC / SIM
  std::vector<void*> ptrs;  // [nranks]; own = cudaMalloc, peers = ipc-opened
  std::vector<void*> sim_all;  // SIM: allocations owned by rank 0's impl
  void* epochs = nullptr;
  int* abort_host = nullptr;
  // registered (zero-copy) regions: user tensors that live in peer-mapped memory
  struct Region {
    size_t bytes = 0;
    std::vector<CUmemGenericAllocationHandle> handles;  // VMM
    std::vector<CUdeviceptr> vas;
    CUmemGenericAllocationHandle mc_handle = 0;
    CUdeviceptr mc_va = 0;
    bool mc_bound = false;
    std::vector<void*> ptrs;                             // IPC: [rank] own cudaMalloc, others ipc-opened
  };
  std::vector<Region> regions;
  std::mutex region_mu;
  void FreeRegion(Region& r) {
    Driver& d = Drv();
    if (kind == Kind::VMM) {
      if (r.mc_va) { d.p_cuMemUnmap(r.mc_va, r.bytes); d.p_cuMemAddressFree(r.mc_va, r.bytes); }
      if (r.mc_bound && r.mc_handle) { CUdevice dev; d.p_cuDeviceGet(&dev, device); d.p_cuMulticastUnbind(r.mc_handle, dev, 0, r.bytes); }
      if (r.mc_handle) d.p_cuMemRelease(r.mc_handle);
      for (size_t i = 0; i < r.vas.size(); ++i) {
        if (r.vas[i]) { d.p_cuMemUnmap(r.vas[i], r.bytes); d.p_cuMemAddressFree(r.vas[i], r.bytes); }
        if (r.handles[i]) d.p_cuMemRelease(r.handles[i]);
      }
    } else {
      for (int i = 0; i < (int)r.ptrs.size(); ++i) {
        if (!r.ptrs[i]) continue;
        if (kind == Kind::SIM || i == rank) cudaFree(r.ptrs[i]); else cudaIpcCloseMemHandle(r.ptrs[i]);
      }
    }
    r = Region();
  }

  ~Impl() {
    // may run very late (a symm_empty tensor that outlived hvd.shutdown() dies at interpreter exit): when the runtime is
    // already unloading there is nothing left to unmap, the process's address space goes away with it
    if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return; }
    cudaDeviceSynchronize();
    for (auto& r : regions) FreeRegion(r);
    Driver& d = Drv();
    if (kind == Kind::VMM) {
      if (mc_va) { d.p_cuMemUnmap(mc_va, alloc_bytes); d.p_cuMemAddressFree(mc_va, alloc_bytes); }
      if (mc_bound && mc_handle) {
        CUdevice dev; d.p_cuDeviceGet(&dev, device);
        d.p_cuMulticastUnbind(mc_handle, dev, 0, alloc_bytes);
      }
      if (mc_handle) d.p_cuMemRelease(mc_handle);
      for (size_t i = 0; i < vas.size(); ++i) {
        if (vas[i]) { d.p_cuMemUnmap(vas[i], alloc_bytes); d.p_cuMemAddressFree(vas[i], alloc_bytes); }
        if (handles[i]) d.p_cuMemRelease(handles[i]);
      }
    } else if (kind == Kind::IPC) {
      for (int i = 0; i < (int)ptrs.size(); ++i) {
        if (!ptrs[i]) continue;
        if (i == rank) cudaFree(ptrs[i]); else cudaIpcCloseMemHandle(ptrs[i]);
      }
    } else {
      for (void* p : sim_all) cudaFree(p);
    }
    if (epochs) cudaFree(epochs);
    if (abort_host) cudaFreeHost(abort_host);
    cudaGetLastError();
  }
};

SymmTeam::~SymmTeam() = default;

std::shared_ptr<void> SymmTeam::KeepAlive() const { return std::static_pointer_cast<void>(impl_); }

kern::CommParams SymmTeam::Params(int which, int channel, int64_t byte_offset) const {
  kern::CommParams cp {};
  cp.nranks = nranks_;
  cp.rank = rank_;
  // channel 0 = the cycle thread's flag words at the start of the region; channels >= 1 own kFlagWords each further up
  const size_t foff = channel == 0 ? 0 : (kern::kChannelFlagsOffset / 4 + (size_t)(channel - 1) * kern::kFlagWords);
  for (int i = 0; i < nranks_; ++i) { cp.buf[i] = (char*)buf_[which][i] + byte_offset; cp.flags[i] = flags_[i] + foff; }
  cp.mc_buf = mc_va_[which] ? (char*)mc_va_[which] + byte_offset : nullptr;
  cp.epochs = epochs_ + (size_t)channel * kern::kMaxCtas;
  cp.abort_flag = abort_dev_;
  cp.timeout_ns = timeout_ns_;
  return cp;
}

namespace {
// flag words (kFlagWords * 4 = 8 KiB) followed by the two Adasum partial-dot tables (2 x kAdasumScratchStride)
constexpr size_t kFlagRegionBytes = 256 * 1024;
static_assert(kern::kFlagWords * 4 + 2 * kern::kAdasumScratchStride <= (long long)kern::kChannelFlagsOffset, "Adasum scratch overlaps the channel flags");
static_assert(kern::kChannelFlagsOffset + (kern::kNumChannels - 1) * kern::kFlagWords * 4 <= (long long)kFlagRegionBytes, "flag region too small");
}

std::shared_ptr<SymmTeam> SymmTeam::Create(Transport* t, int device, size_t buffer_bytes, bool want_mc,
                                           const std::string& tag, std::string* why) {
  const int n = t->size(), me = t->rank();
  auto fail = [&](const std::string& m) { if (why) *why = m; return std::shared_ptr<SymmTeam>(); };
  if (n > kern::kMaxPeers) return fail("team larger than kMaxPeers");
  if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); AllAgree(t, false); return fail("cudaSetDevice failed"); }
  cudaFree(0);
  GpuTopology topo = DiscoverGpuTopology(device);

  // every rank must use a distinct device that can reach all others
  std::vector<int64_t> devs(n);
  int64_t mine = device;
  t->AllgatherInts(&mine, 1, devs.data());
  bool ok = true;
  for (int i = 0; i < n; ++i) {
    if (i == me) continue;
    if (devs[i] == device) ok = false;
    else if (devs[i] < 0 || devs[i] >= (int64_t)topo.peer_access.size() || !topo.peer_access[devs[i]]) ok = false;
  }
  if (!AllAgree(t, ok)) return fail("ranks share a GPU or lack peer access");

  std::shared_ptr<SymmTeam> team(new SymmTeam());
  team->nranks_ = n; team->rank_ = me; team->device_ = device;
  auto impl = std::make_shared<Impl>();
  team->impl_ = impl;
  impl->nranks = n; impl->rank = me; impl->device = device;

  Driver& d = Drv();
  bool use_vmm = d.ok && topo.vmm_supported && topo.fd_handles_supported && getenv("HVD_SYMM_FORCE_IPC") == nullptr;
  use_vmm = AllAgree(t, use_vmm);
  bool use_mc = use_vmm && want_mc && d.mc_ok && topo.multicast_supported && n > 1;
  use_mc = AllAgree(t, use_mc);

  size_t gran = 2 << 20;
  CUmemAllocationProp prop {};
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device;
  prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  if (use_vmm) {
    size_t g = 0;
    if (d.p_cuMemGetAllocationGranularity(&g, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS && g) gran = g;
  }
  CUmulticastObjectProp mcprop {};
  if (use_mc) {
    mcprop.numDevices = n;
    mcprop.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    mcprop.size = 0;
    size_t g = 0;
    mcprop.size = RoundUp(2 * buffer_bytes + kFlagRegionBytes, gran);
    if (d.p_cuMulticastGetGranularity(&g, &mcprop, CU_MULTICAST_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS && g > gran) gran = g;
  }
  const size_t buf_bytes = RoundUp(buffer_bytes, 4096);
  const size_t alloc = RoundUp(2 * buf_bytes + kFlagRegionBytes, gran);
  impl->alloc_bytes = alloc;
  team->buffer_bytes_ = buf_bytes;
  std::vector<char*> base(n, nullptr);

  if (use_vmm) {
    impl->kind = Impl::Kind::VMM;
    impl->handles.assign(n, 0);
    impl->vas.assign(n, 0);
    CUresult r = d.p_cuMemCreate(&impl->handles[me], alloc, &prop, 0);
    bool good = r == CUDA_SUCCESS;
    int myfd = -1;
    if (good) good = d.p_cuMemExportToShareableHandle(&myfd, impl->handles[me], CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0) == CUDA_SUCCESS;
    FdChannel ch;
    if (good) good = ch.Open("hvd-symm-" + tag, me);
    if (!AllAgree(t, good)) { if (myfd >= 0) close(myfd); return fail("VMM allocation / fd export failed: " + d.Err(r)); }
    // sockets are bound on every rank (the AllAgree above is the barrier): exchange
    std::vector<int> fds(n, -1);
    for (int p = 0; p < n && good; ++p) if (p != me) good = ch.SendFd(p, myfd, 0, me);
    for (int k = 0; k < n - 1 && good; ++k) {
      int fd = -1; int32_t kind = 0, from = -1;
      good = ch.RecvFd(&fd, &kind, &from, 30000) && kind == 0 && from >= 0 && from < n && from != me;
      if (good) fds[from] = fd;
    }
    close(myfd);
    for (int p = 0; p < n && good; ++p) {
      if (p == me) continue;
      good = d.p_cuMemImportFromShareableHandle(&impl->handles[p], (void*)(uintptr_t)fds[p], CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR) == CUDA_SUCCESS;
    }
    for (int fd : fds) if (fd >= 0) close(fd);
    CUmemAccessDesc acc {};
    acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    acc.location.id = device;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    for (int p = 0; p < n && good; ++p) {
      good = d.p_cuMemAddressReserve(&impl->vas[p], alloc, gran, 0, 0) == CUDA_SUCCESS &&
             d.p_cuMemMap(impl->vas[p], alloc, 0, impl->handles[p], 0) == CUDA_SUCCESS &&
             d.p_cuMemSetAccess(impl->vas[p], alloc, &acc, 1) == CUDA_SUCCESS;
      base[p] = (char*)impl->vas[p];
    }
    if (!AllAgree(t, good)) return fail("importing / mapping peer allocations failed");

    if (use_mc) {
      bool mg = true;
      int mcfd = -1;
      CUdevice cudev;
      d.p_cuDeviceGet(&cudev, device);
      mcprop.size = alloc;
      if (me == 0) {
        mg = d.p_cuMulticastCreate(&impl->mc_handle, &mcprop) == CUDA_SUCCESS &&
             d.p_cuMemExportToShareableHandle(&mcfd, impl->mc_handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0) == CUDA_SUCCESS;
        for (int p = 1; p < n && mg; ++p) mg = ch.SendFd(p, mcfd, 1, 0);
        if (mcfd >= 0) close(mcfd);
      }
      mg = AllAgree(t, mg);
      if (mg && me != 0) {
        int fd = -1; int32_t kind = 0, from = -1;
        mg = ch.RecvFd(&fd, &kind, &from, 30000) && kind == 1;
        if (mg) mg = d.p_cuMemImportFromShareableHandle(&impl->mc_handle, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR) == CUDA_SUCCESS;
        if (fd >= 0) close(fd);
      }
      if (mg) mg = d.p_cuMulticastAddDevice(impl->mc_handle, cudev) == CUDA_SUCCESS;
      mg = AllAgree(t, mg);  // every device added before anyone binds
      if (mg) {
        mg = d.p_cuMulticastBindMem(impl->mc_handle, 0, impl->handles[me], 0, alloc, 0) == CUDA_SUCCESS;
        impl->mc_bound = mg;
      }
      if (mg) mg = d.p_cuMemAddressReserve(&impl->mc_va, alloc, gran, 0, 0) == CUDA_SUCCESS &&
                   d.p_cuMemMap(impl->mc_va, alloc, 0, impl->mc_handle, 0) == CUDA_SUCCESS &&
                   d.p_cuMemSetAccess(impl->mc_va, alloc, &acc, 1) == CUDA_SUCCESS;
      mg = AllAgree(t, mg);
      if (mg) {
        team->mc_va_[0] = (void*)impl->mc_va;
        team->mc_va_[1] = (void*)(impl->mc_va + buf_bytes);
      } else {
        LOG(INFO) << "NVLS multicast setup failed; continuing with plain peer mappings";
        if (impl->mc_va) { d.p_cuMemUnmap(impl->mc_va, alloc); d.p_cuMemAddressFree(impl->mc_va, alloc); impl->mc_va = 0; }
      }
    }
    team->backend_ = team->mc_va_[0] ? "vmm+mc" : "vmm";
  } else {
    // ---- cudaIpc fallback ----
    impl->kind = Impl::Kind::IPC;
    impl->ptrs.assign(n, nullptr);
    bool good = cudaMalloc(&impl->ptrs[me], alloc) == cudaSuccess;
    cudaIpcMemHandle_t h {};
    if (good) good = cudaIpcGetMemHandle(&h, impl->ptrs[me]) == cudaSuccess;
    if (!AllAgree(t, good)) { cudaGetLastError(); return fail("cudaMalloc / cudaIpcGetMemHandle failed"); }
    std::vector<uint8_t> mineb((uint8_t*)&h, (uint8_t*)&h + sizeof h);
    std::vector<std::vector<uint8_t>> all;
    t->GatherBytes(mineb, &all, 0);
    std::vector<uint8_t> cat;
    if (me == 0) for (auto& v : all) cat.insert(cat.end(), v.begin(), v.end());
    t->BcastBytes(&cat, 0);
    for (int p = 0; p < n && good; ++p) {
      if (p == me) continue;
      cudaIpcMemHandle_t ph;
      memcpy(&ph, cat.data() + (size_t)p * sizeof ph, sizeof ph);
      good = cudaIpcOpenMemHandle(&impl->ptrs[p], ph, cudaIpcMemLazyEnablePeerAccess) == cudaSuccess;
    }
    if (!AllAgree(t, good)) { cudaGetLastError(); return fail("cudaIpcOpenMemHandle failed"); }
    for (int p = 0; p < n; ++p) base[p] = (char*)impl->ptrs[p];
    team->backend_ = "ipc";
  }

  for (int p = 0; p < n; ++p) {
    team->buf_[0][p] = base[p];
    team->buf_[1][p] = base[p] + buf_bytes;
    team->flags_[p] = (uint32_t*)(base[p] + 2 * buf_bytes);
  }
  bool good = cudaMemset(base[me] + 2 * buf_bytes, 0, kFlagRegionBytes) == cudaSuccess;
  good = good && cudaMalloc(&impl->epochs, kern::kNumChannels * kern::kMaxCtas * sizeof(uint32_t)) == cudaSuccess &&
         cudaMemset(impl->epochs, 0, kern::kNumChannels * kern::kMaxCtas * sizeof(uint32_t)) == cudaSuccess;
  good = good && cudaHostAlloc((void**)&impl->abort_host, sizeof(int), cudaHostAllocMapped) == cudaSuccess;
  if (good) { *impl->abort_host = 0; good = cudaHostGetDevicePointer((void**)&team->abort_dev_, impl->abort_host, 0) == cudaSuccess; }
  good = good && cudaDeviceSynchronize() == cudaSuccess;
  team->epochs_ = (uint32_t*)impl->epochs;
  team->abort_host_ = impl->abort_host;
  if (!AllAgree(t, good)) { cudaGetLastError(); return fail("flag / epoch initialisation failed"); }
  return team;
}

// ---------------------------------------------------------------------------
// registered regions

int SymmTeam::AllocRegion(Transport* t, size_t bytes, const std::string& tag, std::string* why) {
  auto fail = [&](const std::string& m) { if (why) *why = m; return -1; };
  Impl& im = *impl_;
  if (im.kind == Impl::Kind::SIM) return fail("simulated teams use AllocRegionSim");
  cudaSetDevice(device_);
  const int n = nranks_, me = rank_;
  Driver& d = Drv();
  Impl::Region reg;
  std::vector<void*> ptr(n, nullptr);
  void* mc_ptr = nullptr;
  if (im.kind == Impl::Kind::VMM) {
    CUmemAllocationProp prop {};
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = device_;
    prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t gran = 2 << 20, g = 0;
    if (d.p_cuMemGetAllocationGranularity(&g, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS && g) gran = g;
    const bool use_mc = has_multicast();
    CUmulticastObjectProp mcprop {};
    if (use_mc) {
      mcprop.numDevices = n; mcprop.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR; mcprop.size = RoundUp(bytes, gran);
      if (d.p_cuMulticastGetGranularity(&g, &mcprop, CU_MULTICAST_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS && g > gran) gran = g;
    }
    const size_t alloc = RoundUp(bytes, gran);
    reg.bytes = alloc;
    reg.handles.assign(n, 0);
    reg.vas.assign(n, 0);
    bool good = d.p_cuMemCreate(&reg.handles[me], alloc, &prop, 0) == CUDA_SUCCESS;
    int myfd = -1;
    if (good) good = d.p_cuMemExportToShareableHandle(&myfd, reg.handles[me], CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0) == CUDA_SUCCESS;
    FdChannel ch;
    if (good) good = ch.Open("hvd-symm-" + tag, me);
    if (!AllAgree(t, good)) { if (myfd >= 0) close(myfd); im.FreeRegion(reg); return fail("region allocation / fd export failed (out of memory?)"); }
    std::vector<int> fds(n, -1);
    for (int p = 0; p < n && good; ++p) if (p != me) good = ch.SendFd(p, myfd, 0, me);
    for (int k = 0; k < n - 1 && good; ++k) {
      int fd = -1; int32_t kind = 0, from = -1;
      good = ch.RecvFd(&fd, &kind, &from, 30000) && kind == 0 && from >= 0 && from < n && from != me;
      if (good) fds[from] = fd;
    }
    close(myfd);
    for (int p = 0; p < n && good; ++p) {
      if (p == me) continue;
      good = d.p_cuMemImportFromShareableHandle(&reg.handles[p], (void*)(uintptr_t)fds[p], CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR) == CUDA_SUCCESS;
    }
    for (int fd : fds) if (fd >= 0) close(fd);
    CUmemAccessDesc acc {};
    acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE; acc.location.id = device_; acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    for (int p = 0; p < n && good; ++p) {
      good = d.p_cuMemAddressReserve(&reg.vas[p], alloc, gran, 0, 0) == CUDA_SUCCESS &&
             d.p_cuMemMap(reg.vas[p], alloc, 0, reg.handles[p], 0) == CUDA_SUCCESS &&
             d.p_cuMemSetAccess(reg.vas[p], alloc, &acc, 1) == CUDA_SUCCESS;
      ptr[p] = (void*)reg.vas[p];
    }
    if (!AllAgree(t, good)) { im.FreeRegion(reg); return fail("mapping the peers' region failed"); }
    if (use_mc) {
      bool mg = true;
      int mcfd = -1;
      CUdevice cudev;
      d.p_cuDeviceGet(&cudev, device_);
      mcprop.size = alloc;
      if (me == 0) {
        mg = d.p_cuMulticastCreate(&reg.mc_handle, &mcprop) == CUDA_SUCCESS &&
             d.p_cuMemExportToShareableHandle(&mcfd, reg.mc_handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0) == CUDA_SUCCESS;
        for (int p = 1; p < n && mg; ++p) mg = ch.SendFd(p, mcfd, 1, 0);
        if (mcfd >= 0) close(mcfd);
      }
      mg = AllAgree(t, mg);
      if (mg && me != 0) {
        int fd = -1; int32_t kind = 0, from = -1;
        mg = ch.RecvFd(&fd, &kind, &from, 30000) && kind == 1;
        if (mg) mg = d.p_cuMemImportFromShareableHandle(&reg.mc_handle, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR) == CUDA_SUCCESS;
        if (fd >= 0) close(fd);
      }
      if (mg) mg = d.p_cuMulticastAddDevice(reg.mc_handle, cudev) == CUDA_SUCCESS;
      mg = AllAgree(t, mg);
      if (mg) { mg = d.p_cuMulticastBindMem(reg.mc_handle, 0, reg.handles[me], 0, alloc, 0) == CUDA_SUCCESS; reg.mc_bound = mg; }
      if (mg) mg = d.p_cuMemAddressReserve(&reg.mc_va, alloc, gran, 0, 0) == CUDA_SUCCESS &&
                   d.p_cuMemMap(reg.mc_va, alloc, 0, reg.mc_handle, 0) == CUDA_SUCCESS &&
                   d.p_cuMemSetAccess(reg.mc_va, alloc, &acc, 1) == CUDA_SUCCESS;
      mg = AllAgree(t, mg);
      if (mg) mc_ptr = (void*)reg.mc_va;
      else if (reg.mc_va) { d.p_cuMemUnmap(reg.mc_va, alloc); d.p_cuMemAddressFree(reg.mc_va, alloc); reg.mc_va = 0; }
    }
  } else {  // IPC
    reg.bytes = RoundUp(bytes, 2 << 20);
    reg.ptrs.assign(n, nullptr);
    bool good = cudaMalloc(&reg.ptrs[me], reg.bytes) == cudaSuccess;
    cudaIpcMemHandle_t h {};
    if (good) good = cudaIpcGetMemHandle(&h, reg.ptrs[me]) == cudaSuccess;
    if (!AllAgree(t, good)) { cudaGetLastError(); im.FreeRegion(reg); return fail("cudaMalloc / cudaIpcGetMemHandle failed"); }
    std::vector<uint8_t> mineb((uint8_t*)&h, (uint8_t*)&h + sizeof h);
    std::vector<std::vector<uint8_t>> all;
    t->GatherBytes(mineb, &all, 0);
    std::vector<uint8_t> cat;
    if (me == 0) for (auto& v : all) cat.insert(cat.end(), v.begin(), v.end());
    t->BcastBytes(&cat, 0);
    for (int p = 0; p < n && good; ++p) {
      if (p == me) continue;
      cudaIpcMemHandle_t ph;
      memcpy(&ph, cat.data() + (size_t)p * sizeof ph, sizeof ph);
      good = cudaIpcOpenMemHandle(&reg.ptrs[p], ph, cudaIpcMemLazyEnablePeerAccess) == cudaSuccess;
    }
    if (!AllAgree(t, good)) { cudaGetLastError(); im.FreeRegion(reg); return fail("cudaIpcOpenMemHandle failed"); }
    for (int p = 0; p < n; ++p) ptr[p] = reg.ptrs[p];
  }
  cudaMemset(ptr[me], 0, reg.bytes);
  cudaDeviceSynchronize();
  AllAgree(t, true);  // nobody touches a peer's region before it is zero-filled
  std::lock_guard<std::mutex> l(im.region_mu);
  RegionView v;
  v.bytes = reg.bytes; v.mc = mc_ptr;
  for (int p = 0; p < n; ++p) v.ptr[p] = ptr[p];
  regions_.push_back(v);
  im.regions.push_back(std::move(reg));
  return (int)regions_.size() - 1;
}

bool SymmTeam::FindRegion(const void* p, size_t len, RegionView* view, int64_t* offset, int* index) const {
  std::lock_guard<std::mutex> l(impl_->region_mu);
  const char* c = (const char*)p;
  for (size_t i = 0; i < regions_.size(); ++i) {
    const char* base = (const char*)regions_[i].ptr[rank_];
    if (c >= base && c + len <= base + regions_[i].bytes) {
      if (view) *view = regions_[i];
      if (offset) *offset = c - base;
      if (index) *index = (int)i;
      return true;
    }
  }
  return false;
}

void* SymmTeam::RegionPtr(int index) const {
  std::lock_guard<std::mutex> l(impl_->region_mu);
  return index >= 0 && index < (int)regions_.size() ? regions_[index].ptr[rank_] : nullptr;
}

std::vector<std::shared_ptr<SymmTeam>> SymmTeam::CreateSimulated(int n, int device, size_t buffer_bytes) {
  std::vector<std::shared_ptr<SymmTeam>> out;
  if (n > kern::kMaxPeers || cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return out; }
  const size_t buf_bytes = RoundUp(buffer_bytes, 4096);
  const size_t alloc = 2 * buf_bytes + kFlagRegionBytes;
  std::vector<char*> base(n);
  auto shared_allocs = std::make_shared<std::vector<void*>>();
  for (int r = 0; r < n; ++r) {
    void* p = nullptr;
    if (cudaMalloc(&p, alloc) != cudaSuccess) { for (void* q : *shared_allocs) cudaFree(q); cudaGetLastError(); return {}; }
    cudaMemset((char*)p + 2 * buf_bytes, 0, kFlagRegionBytes);
    base[r] = (char*)p;
    shared_allocs->push_back(p);
  }
  for (int r = 0; r < n; ++r) {
    std::shared_ptr<SymmTeam> team(new SymmTeam());
    auto impl = std::make_shared<Impl>();
    impl->kind = Impl::Kind::SIM; impl->nranks = n; impl->rank = r; impl->device = device; impl->alloc_bytes = alloc;
    if (r == 0) impl->sim_all = *shared_allocs;
    team->impl_ = impl;
    team->nranks_ = n; team->rank_ = r; team->device_ = device; team->buffer_bytes_ = buf_bytes; team->backend_ = "sim";
    for (int p = 0; p < n; ++p) {
      team->buf_[0][p] = base[p]; team->buf_[1][p] = base[p] + buf_bytes; team->flags_[p] = (uint32_t*)(base[p] + 2 * buf_bytes);
    }
    cudaMalloc(&impl->epochs, kern::kNumChannels * kern::kMaxCtas * sizeof(uint32_t));
    cudaMemset(impl->epochs, 0, kern::kNumChannels * kern::kMaxCtas * sizeof(uint32_t));
    cudaHostAlloc((void**)&impl->abort_host, sizeof(int), cudaHostAllocMapped);
    *impl->abort_host = 0;
    cudaHostGetDevicePointer((void**)&team->abort_dev_, impl->abort_host, 0);
    team->epochs_ = (uint32_t*)impl->epochs;
    team->abort_host_ = impl->abort_host;
    out.push_back(team);
  }
  cudaDeviceSynchronize();
  return out;
}

}  // namespace hvd
