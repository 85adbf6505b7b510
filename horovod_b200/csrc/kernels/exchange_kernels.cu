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
#include "p2p_common.cuh"

namespace hvd {
namespace kern {
namespace {

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

}  // namespace

cudaError_t LaunchExchange(const CommParams& cp, const ExchangeArgs& args, cudaStream_t stream) {
  if (args.ctas < 1 || args.ctas > kMaxCtas) return cudaErrorInvalidValue;
  exchange_kernel<<<args.ctas, kThreads, 0, stream>>>(cp, args);
  CountKernelLaunch();
  return cudaGetLastError();
}

}  // namespace kern
}  // namespace hvd
