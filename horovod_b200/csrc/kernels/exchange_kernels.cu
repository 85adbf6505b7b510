// "pack -> flag barrier -> pull" byte-moving kernel behind allgather(v),
// broadcast and alltoall(v) on peer-mapped symmetric buffers (sm_90a).
//
// Every rank copies what it sends into its own symmetric buffer (send descs),
// the CTAs rendezvous with the same-index CTAs of all peers, then every rank
// pulls the pieces addressed to it straight out of the peers' buffers over
// NVLink into the final output tensor (recv descs) — no staging on the
// receive side, one launch per collective.
//
// Replaces the reference's ncclAllGather / grouped ncclBroadcast /
// ncclSend+ncclRecv call sites (ops/nccl_operations.cc:880,1071,1083-1095,
// 1174-1199) and the allgather fusion memcpy kernels around them.
#include <cstdlib>
#include "p2p_common.cuh"

namespace hvd {
namespace kern {
namespace {

constexpr int kRow = kThreads * 16;
constexpr int kXChunk = 32768;  // chunk -> CTA mapping granularity inside the symmetric buffer (one 8-deep trip of the CTA)

__device__ __forceinline__ void copy_bytes_vec(const char* src, char* dst, int64_t n) {
  // 16 B vectors, 8 in flight per thread (all loads of a trip are issued before the first store: an NVLink round trip is
  // ~2 us) when both sides are 16 B aligned, bytes otherwise
  if ((((uintptr_t)src | (uintptr_t)dst) & 15) == 0) {
    const int64_t nv = n / 16;
    constexpr int U = 8;
    for (int64_t i0 = threadIdx.x; i0 < nv; i0 += (int64_t)U * kThreads) {
      uint4 v[U];
#pragma unroll
      for (int j = 0; j < U; ++j) { int64_t i = i0 + (int64_t)j * kThreads; if (i < nv) v[j] = ld_stream(src + i * 16); }
#pragma unroll
      for (int j = 0; j < U; ++j) { int64_t i = i0 + (int64_t)j * kThreads; if (i < nv) st_stream(dst + i * 16, v[j]); }
    }
    for (int64_t i = nv * 16 + threadIdx.x; i < n; i += kThreads) dst[i] = src[i];
  } else {
    for (int64_t i = threadIdx.x; i < n; i += kThreads) dst[i] = src[i];
  }
}

// Root side of a multicast broadcast: local source -> multimem.st on the team's multicast mapping, i.e. ONE read of the
// source and one NVLink egress stream that the switch replicates into every rank's symmetric buffer (a pull-style
// broadcast makes the root serve N-1 readers).  `src` and `mc` are 16 B aligned; a tail shorter than 16 B is zero-padded
// (the host pads the buffer window to 16 B).
__device__ __forceinline__ void mc_copy_vec(const char* src, char* mc, int64_t n) {
  const int64_t nv = n / 16;
  if ((uintptr_t)src & 15) {  // unaligned source (a view into a larger tensor): assemble each vector from bytes
    for (int64_t i = threadIdx.x; i < nv; i += kThreads) {
      uint4 v;
      char* b = reinterpret_cast<char*>(&v);
#pragma unroll
      for (int k = 0; k < 16; ++k) b[k] = src[i * 16 + k];
      asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc + i * 16), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
    }
  } else
  for (int64_t i0 = threadIdx.x; i0 < nv; i0 += 4 * kThreads) {
    uint4 v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { int64_t i = i0 + (int64_t)j * kThreads; if (i < nv) v[j] = ld_stream(src + i * 16); }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int64_t i = i0 + (int64_t)j * kThreads;
      if (i < nv) asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc + i * 16), "r"(v[j].x), "r"(v[j].y), "r"(v[j].z), "r"(v[j].w) : "memory");
    }
  }
  if ((n & 15) && threadIdx.x == 0) {
    uint4 v = make_uint4(0, 0, 0, 0);
    char* b = reinterpret_cast<char*>(&v);
    for (int64_t i = nv * 16; i < n; ++i) b[i - nv * 16] = src[i];
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc + nv * 16), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
  }
}

// Processes the part of [offset, offset+bytes) of a symmetric buffer that
// falls into chunks owned by this CTA (chunk c -> CTA c % grid).
template <typename F>
__device__ __forceinline__ void for_my_chunks(int64_t offset, int64_t bytes, int cta, int grid, F f) {
  const int64_t end = offset + bytes;
  const int64_t c0 = offset / kXChunk;
  // first chunk >= c0 that belongs to this CTA, then every grid-th one
  int64_t c = c0 + ((cta - (int)(c0 % grid) + grid) % grid);
  for (; c * kXChunk < end; c += grid) {
    int64_t lo = c * kXChunk, hi = lo + kXChunk;
    if (lo < offset) lo = offset;
    if (hi > end) hi = end;
    if (lo < hi) f(lo, hi);
  }
}

__global__ void __launch_bounds__(kThreads, 2)
exchange_kernel(const __grid_constant__ CommParams cp, const __grid_constant__ ExchangeArgs a) {
  const int cta = blockIdx.x, grid = gridDim.x;
  uint32_t epoch = cp.epochs[cta];
  char* mybuf = reinterpret_cast<char*>(cp.buf[cp.rank]);
  for (int s = 0; s < a.nsend; ++s) {
    const CopyDesc d = a.sends[s];
    if (d.pad == kSendMulticast && cp.mc_buf) {
      char* mc = reinterpret_cast<char*>(cp.mc_buf);
      for_my_chunks(d.offset, d.bytes, cta, grid, [&](int64_t lo, int64_t hi) {
        mc_copy_vec(reinterpret_cast<const char*>(d.src) + (lo - d.offset), mc + lo, hi - lo);
      });
      continue;
    }
    for_my_chunks(d.offset, d.bytes, cta, grid, [&](int64_t lo, int64_t hi) {
      copy_bytes_vec(reinterpret_cast<const char*>(d.src) + (lo - d.offset), mybuf + lo, hi - lo);
    });
  }
  bool alive = true;
  if (cp.nranks > 1) alive = peer_barrier(cp, epoch, cta); else __syncthreads();
  for (int r = 0; r < a.nrecv && alive; ++r) {
    const CopyDesc d = a.recvs[r];
    const char* peer = reinterpret_cast<const char*>(cp.buf[d.peer]);
    for_my_chunks(d.offset, d.bytes, cta, grid, [&](int64_t lo, int64_t hi) {
      copy_bytes_vec(peer + lo, reinterpret_cast<char*>(d.dst) + (lo - d.offset), hi - lo);
    });
  }
  if (threadIdx.x == 0) cp.epochs[cta] = epoch;
}

// ---------------------------------------------------------------------------
// TMA variant (opt-in, HVD_EXCHANGE_TMA=1): the same pack -> barrier -> pull protocol, but the bytes move as bulk
// asynchronous copies (cp.async.bulk, SASS UBLKCP) through a ring of shared-memory stages driven by ONE thread per CTA:
// global (local HBM or a peer over NVLink) -> smem stage -> global.  No registers or LSU slots are spent on the payload
// and (kTmaStages - 1) x 16 KiB per CTA are in flight regardless of occupancy, which is what a pure copy collective
// (allgather / broadcast / alltoall) wants on an H100.
constexpr int kTmaStages = 3;  // 3 x 32 KiB: two CTAs per SM still fit in 227 KB of shared memory
constexpr int kTmaStageBytes = kXChunk;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }

struct TmaRing {
  char* stage;      // kTmaStages x kTmaStageBytes of dynamic shared memory (128 B aligned)
  uint64_t* full;   // one mbarrier per stage
  uint32_t issued;  // loads issued so far by the driver thread (stage = issued % S, parity = (issued / S) & 1)
};

// Driver thread only.  Copies the 16 B-aligned part of this CTA's chunks of [offset, offset + bytes): src_of(lo) and
// dst_of(lo) give the addresses of buffer offset `lo` on the source and destination side.
template <typename SrcOf, typename DstOf>
__device__ __forceinline__ void tma_copy_my_chunks(TmaRing& ring, int64_t offset, int64_t bytes, int cta, int grid, SrcOf src_of,
                                                   DstOf dst_of) {
  const int64_t end = offset + (bytes & ~(int64_t)15);
  if (end <= offset) return;  // fewer than 16 bytes: the byte tail of the caller covers it
  // chunk walker shared by the load side (`lc`) and the store side (`sc`)
  auto next_mine = [&](int64_t c) { return c + ((cta - (int)(c % grid) + grid) % grid); };  // first chunk >= c of this CTA
  auto bounds = [&](int64_t c, int64_t& lo, int64_t& hi) {
    lo = c * kXChunk; hi = lo + kXChunk;
    if (lo < offset) lo = offset;
    if (hi > end) hi = end;
  };
  int64_t lc = next_mine(offset / kXChunk), sc = lc;
  uint32_t loaded = 0, stored = 0;
  const uint32_t first = ring.issued;
  auto issue_load = [&]() {
    int64_t lo, hi;
    bounds(lc, lo, hi);
    const uint32_t n = (uint32_t)(hi - lo);
    const uint32_t s = ring.issued % kTmaStages;
    mbar_expect_tx(&ring.full[s], n);
    bulk_g2s(ring.stage + (size_t)s * kTmaStageBytes, src_of(lo), n, &ring.full[s]);
    ++ring.issued; ++loaded;
    lc = next_mine(lc + 1);
  };
  while (loaded < kTmaStages && lc * kXChunk < end) issue_load();
  while (sc * kXChunk < end) {
    int64_t lo, hi;
    bounds(sc, lo, hi);
    const uint32_t idx = first + stored;
    const uint32_t s = idx % kTmaStages;
    mbar_wait(&ring.full[s], (idx / kTmaStages) & 1);
    bulk_s2g(dst_of(lo), ring.stage + (size_t)s * kTmaStageBytes, (uint32_t)(hi - lo));
    ++stored;
    sc = next_mine(sc + 1);
    if (lc * kXChunk < end) {
      bulk_wait_read_all();  // the stage just stored from is about to be overwritten by the next load
      issue_load();
    }
  }
  bulk_wait_read_all();
}

__global__ void __launch_bounds__(kThreads, 2)
exchange_tma_kernel(const __grid_constant__ CommParams cp, const __grid_constant__ ExchangeArgs a) {
  extern __shared__ __align__(128) char tma_smem[];
  __shared__ __align__(8) uint64_t full_bar[kTmaStages];
  const int cta = blockIdx.x, grid = gridDim.x;
  uint32_t epoch = cp.epochs[cta];
  TmaRing ring {tma_smem, full_bar, 0};
  if (threadIdx.x == 0) {
    for (int s = 0; s < kTmaStages; ++s) mbar_init(&full_bar[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  char* mybuf = reinterpret_cast<char*>(cp.buf[cp.rank]);
  for (int s = 0; s < a.nsend; ++s) {
    const CopyDesc d = a.sends[s];
    const char* src = reinterpret_cast<const char*>(d.src);
    if (d.pad == kSendMulticast && cp.mc_buf) {
      char* mc = reinterpret_cast<char*>(cp.mc_buf);
      for_my_chunks(d.offset, d.bytes, cta, grid, [&](int64_t lo, int64_t hi) { mc_copy_vec(src + (lo - d.offset), mc + lo, hi - lo); });
    } else if (((((uintptr_t)src) | (uintptr_t)d.offset) & 15) == 0) {
      if (threadIdx.x == 0)
        tma_copy_my_chunks(ring, d.offset, d.bytes, cta, grid, [&](int64_t lo) { return src + (lo - d.offset); },
                           [&](int64_t lo) { return mybuf + lo; });
      const int64_t tail = d.bytes & 15;  // < 16 B at the very end: the CTA that owns the last chunk copies it bytewise
      if (tail && (int)(((d.offset + d.bytes - 1) / kXChunk) % grid) == cta && (int)threadIdx.x < tail) {
        const int64_t o = d.bytes - tail + threadIdx.x;
        mybuf[d.offset + o] = src[o];
      }
    } else {
      for_my_chunks(d.offset, d.bytes, cta, grid, [&](int64_t lo, int64_t hi) { copy_bytes_vec(src + (lo - d.offset), mybuf + lo, hi - lo); });
    }
  }
  if (threadIdx.x == 0) { bulk_wait_all(); fence_proxy_async(); }  // my pack is complete before the flags are released
  bool alive = true;
  if (cp.nranks > 1) alive = peer_barrier(cp, epoch, cta); else __syncthreads();
  if (threadIdx.x == 0) fence_proxy_async();  // generic-proxy acquire -> async-proxy reads of the peers' buffers
  for (int r = 0; r < a.nrecv && alive; ++r) {
    const CopyDesc d = a.recvs[r];
    const char* peer = reinterpret_cast<const char*>(cp.buf[d.peer]);
    char* dst = reinterpret_cast<char*>(d.dst);
    if (((((uintptr_t)dst) | (uintptr_t)d.offset) & 15) == 0) {
      if (threadIdx.x == 0)
        tma_copy_my_chunks(ring, d.offset, d.bytes, cta, grid, [&](int64_t lo) { return peer + lo; },
                           [&](int64_t lo) { return dst + (lo - d.offset); });
      const int64_t tail = d.bytes & 15;
      if (tail && (int)(((d.offset + d.bytes - 1) / kXChunk) % grid) == cta && (int)threadIdx.x < tail) {
        const int64_t o = d.bytes - tail + threadIdx.x;
        dst[o] = peer[d.offset + o];
      }
    } else {
      for_my_chunks(d.offset, d.bytes, cta, grid, [&](int64_t lo, int64_t hi) { copy_bytes_vec(peer + lo, dst + (lo - d.offset), hi - lo); });
    }
  }
  if (threadIdx.x == 0) { bulk_wait_all(); cp.epochs[cta] = epoch; }
}

}  // namespace

cudaError_t LaunchExchange(const CommParams& cp, const ExchangeArgs& args, cudaStream_t stream) {
  if (args.ctas < 1 || args.ctas > kMaxCtas) return cudaErrorInvalidValue;
  static const bool use_tma = [] { const char* e = getenv("HVD_EXCHANGE_TMA"); return e && atoi(e) > 0; }();
  if (use_tma) {
    constexpr int smem = kTmaStages * kTmaStageBytes;
    static const cudaError_t attr = cudaFuncSetAttribute(exchange_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (attr != cudaSuccess) return attr;
    exchange_tma_kernel<<<args.ctas, kThreads, smem, stream>>>(cp, args);
  } else {
    exchange_kernel<<<args.ctas, kThreads, 0, stream>>>(cp, args);
  }
  CountKernelLaunch();
  return cudaGetLastError();
}

}  // namespace kern
}  // namespace hvd
