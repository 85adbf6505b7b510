// Fused allreduce / reducescatter over peer-mapped symmetric buffers (sm_90a).
//
// One launch per fused response:
//   pack     every tensor -> my symmetric buffer   (prescale, cast T -> wire W)
//   barrier  CTA b of all ranks (release/acquire flags written into peer memory)
//   one-shot : each rank loads the same 16 B vector from all N peers over
//              NVLink, reduces in fp32/int32/fp64 registers, applies
//              postscale (Average), casts W -> T and stores straight into the
//              output tensors.                                  [(N-1)·S in]
//   two-shot : rank r reduces the chunks it owns and stores the result into
//              every peer's buffer, barrier, every rank unpacks its own buffer
//              into the output tensors.                         [2(N-1)/N·S]
//   NVLS     : same as two-shot but the reduction is one
//              multimem.ld_reduce (the NVSwitch adds) and the broadcast one
//              multimem.st on the multicast mapping.            [~S/N in+out]
// The chunk -> CTA mapping is the same in all phases (chunk c belongs to CTA
// c % grid on every rank), so CTA b only ever needs to synchronise with CTA b
// of its peers: no grid-wide barrier, no cooperative launch.
//
// Replaces: batched_scaled_memcpy_k + ncclAllReduce + batched_scaled_memcpy_k
// (reference ops/cuda/cuda_kernels.cu:259-324, ops/nccl_operations.cc:231-283).
#include <cstdlib>
#include "p2p_common.cuh"

namespace hvd {
namespace kern {

static unsigned long long g_launches = 0;
unsigned long long KernelLaunchCount() { return __atomic_load_n(&g_launches, __ATOMIC_RELAXED); }
void CountKernelLaunch() { __atomic_fetch_add(&g_launches, 1ull, __ATOMIC_RELAXED); }

namespace {

constexpr int kRowBytes = kThreads * 16;  // one 16 B vector per thread

template <typename W> struct Nvls { static constexpr bool ok = false; };
template <> struct Nvls<float> {
  static constexpr bool ok = true;
  static __device__ __forceinline__ uint4 ld_reduce(const void* p) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
  }
};
template <> struct Nvls<__nv_bfloat16> {
  static constexpr bool ok = true;
  static __device__ __forceinline__ uint4 ld_reduce(const void* p) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
  }
};
template <> struct Nvls<__half> {
  static constexpr bool ok = true;
  static __device__ __forceinline__ uint4 ld_reduce(const void* p) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
  }
};
__device__ __forceinline__ void multimem_st(void* p, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ---- phase bodies ----------------------------------------------------------
// Every loop handles U rows (U * 8 KiB) per trip: all loads of a trip are issued
// before the first dependent store so each thread keeps U (x N peers) 16 B
// requests in flight — NVLink round trips are ~2 us, HBM ~0.7 us.

template <typename T, typename W, int U>
__device__ __forceinline__ void pack_range(const TensorDesc* descs, int nd, int64_t total, char* buf, int64_t lo, int64_t hi,
                                           typename ScaleOf<typename Traits<W>::Acc>::type scale) {
  using A = typename Traits<W>::Acc;
  constexpr int NW = 16 / (int)sizeof(W);
  constexpr int64_t kSrcRow = (int64_t)kRowBytes / (int)sizeof(W) * (int)sizeof(T);  // source bytes per wire row
  DescCursor cur;
  cur.init(descs, nd, total);
  for (int64_t o0 = lo + (int64_t)threadIdx.x * 16; o0 < hi; o0 += (int64_t)U * kRowBytes) {
    A a[U][NW];
    cur.seek(o0);
    const int64_t olast = o0 + (int64_t)(U - 1) * kRowBytes;
    const int64_t e0 = (o0 - cur.lo) / (int64_t)sizeof(W);
    const char* src = cur.in + e0 * (int64_t)sizeof(T);
    // fast path: all U vectors of this trip are full vectors of ONE tensor and the source is 16 B aligned (the row
    // stride is a multiple of 16 B, so one check covers the trip): no cursor work, no bounds checks
    if (olast < hi && olast + 16 <= cur.lo + cur.count * (int64_t)sizeof(W) && ((reinterpret_cast<uintptr_t>(src) & 15) == 0)) {
#pragma unroll
      for (int j = 0; j < U; ++j) load_elems_fast<T, NW, A>(reinterpret_cast<const T*>(src + j * kSrcRow), a[j]);
#pragma unroll
      for (int j = 0; j < U; ++j) {
#pragma unroll
        for (int i = 0; i < NW; ++i) a[j][i] = apply_scale<A>(a[j][i], scale);
        st_stream(buf + o0 + (int64_t)j * kRowBytes, pack_vec<W, NW>(a[j]));
      }
      continue;
    }
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const int64_t o = o0 + (int64_t)j * kRowBytes;
      if (o < hi) {
        cur.seek(o);
        const int64_t e = (o - cur.lo) / (int64_t)sizeof(W);
        load_elems<T, NW, A>(reinterpret_cast<const T*>(cur.in) + e, cur.count - e, a[j]);
      }
    }
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const int64_t o = o0 + (int64_t)j * kRowBytes;
      if (o < hi) {
#pragma unroll
        for (int i = 0; i < NW; ++i) a[j][i] = apply_scale<A>(a[j][i], scale);
        st_stream(buf + o, pack_vec<W, NW>(a[j]));
      }
    }
  }
}

template <typename T, typename W, int U>
__device__ __forceinline__ void unpack_range(const TensorDesc* descs, int nd, int64_t total, const char* buf, int64_t lo,
                                             int64_t hi) {
  using A = typename Traits<W>::Acc;
  constexpr int NW = 16 / (int)sizeof(W);
  constexpr int64_t kDstRow = (int64_t)kRowBytes / (int)sizeof(W) * (int)sizeof(T);
  DescCursor cur;
  cur.init(descs, nd, total);
  for (int64_t o0 = lo + (int64_t)threadIdx.x * 16; o0 < hi; o0 += (int64_t)U * kRowBytes) {
    uint4 v[U];
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const int64_t o = o0 + (int64_t)j * kRowBytes;
      if (o < hi) v[j] = ld_stream(buf + o);
    }
    cur.seek(o0);
    const int64_t olast = o0 + (int64_t)(U - 1) * kRowBytes;
    const int64_t e0 = (o0 - cur.lo) / (int64_t)sizeof(W);
    char* dst = cur.out + e0 * (int64_t)sizeof(T);
    if (olast < hi && olast + 16 <= cur.lo + cur.count * (int64_t)sizeof(W) && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
#pragma unroll
      for (int j = 0; j < U; ++j) {
        A a[NW];
        unpack_vec<W, NW>(v[j], a);
        store_elems_fast<T, NW, A>(reinterpret_cast<T*>(dst + j * kDstRow), a);
      }
      continue;
    }
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const int64_t o = o0 + (int64_t)j * kRowBytes;
      if (o < hi) {
        cur.seek(o);
        const int64_t e = (o - cur.lo) / (int64_t)sizeof(W);
        if (e < cur.count) {
          A a[NW];
          unpack_vec<W, NW>(v[j], a);
          store_elems<T, NW, A>(reinterpret_cast<T*>(cur.out) + e, cur.count - e, a);
        }
      }
    }
  }
}

// Issues the loads of one trip, the U rows at byte offsets o0 + j * kRowBytes below `hi`, from all N peers (base[p] + o)
// into v[j][p].  Every rank starts at its own buffer and rotates, so that at any instant the N ranks pull from N
// different peers; v[j][] is indexed by peer, so that peer_combine adds in rank order.  One uniform dispatch on (nranks,
// rank) per trip makes every index a compile-time constant (v[] stays in registers).  A kernel instantiated for NR peers
// runs nranks in (NR/2, NR], and 1 .. 2 for NR = 2.
template <int NR, int U, int N, int R>
__device__ __forceinline__ void peer_loads_from(void* const* base, int64_t o0, int64_t hi, uint4 (*v)[NR]) {
#pragma unroll
  for (int j = 0; j < U; ++j) {
    const int64_t o = o0 + (int64_t)j * kRowBytes;
    if (j == 0 || o < hi) {  // (callers loop while o0 < hi)
#pragma unroll
      for (int k = 0; k < N; ++k) {
        const int p = (R + k) % N;
        v[j][p] = ld_stream(reinterpret_cast<const char*>(base[p]) + o);
      }
    }
  }
}
template <int NR, int U, int N, int R = 0>
__device__ __forceinline__ void peer_loads_rank(int rank, void* const* base, int64_t o0, int64_t hi, uint4 (*v)[NR]) {
  if constexpr (R + 1 < N) {
    if (rank != R) { peer_loads_rank<NR, U, N, R + 1>(rank, base, o0, hi, v); return; }
  }
  peer_loads_from<NR, U, N, R>(base, o0, hi, v);
}
template <int NR, int U, int N = NR>
__device__ __forceinline__ void peer_loads(const CommParams& cp, void* const* base, int64_t o0, int64_t hi, uint4 (*v)[NR]) {
  if constexpr (N > (NR == 2 ? 1 : NR / 2 + 1)) {
    if (cp.nranks != N) { peer_loads<NR, U, N - 1>(cp, base, o0, hi, v); return; }
  }
  peer_loads_rank<NR, U, N>(cp.rank, base, o0, hi, v);
}
// Combines the N contributions in rank order 0 .. N-1 (v[p] = peer p): floating-point sums and products are not
// associative and MIN / MAX keep the first of two NaN-unordered operands, so only one fixed order gives every rank, and
// every variant, the same bits.
template <typename W, int NR>
__device__ __forceinline__ void peer_combine(const CommParams& cp, const uint4* v, int op, typename Traits<W>::Acc* acc) {
  using A = typename Traits<W>::Acc;
  constexpr int NW = 16 / (int)sizeof(W);
  unpack_vec<W, NW>(v[0], acc);
#pragma unroll
  for (int k = 1; k < NR; ++k) {
    if (k < cp.nranks) {
      A b[NW];
      unpack_vec<W, NW>(v[k], b);
#pragma unroll
      for (int i = 0; i < NW; ++i) acc[i] = combine<A>(acc[i], b[i], op);
    }
  }
}

template <typename T, typename W, int NR>
__global__ void __launch_bounds__(kThreads, 2)
allreduce_kernel(const __grid_constant__ CommParams cp, const __grid_constant__ AllreduceArgs a, const int chunk_bytes) {
  using A = typename Traits<W>::Acc;
  using S = typename ScaleOf<A>::type;
  constexpr int NW = 16 / (int)sizeof(W);
  constexpr int U = 8 / NR;  // rows per trip in the peer phases
  constexpr int UP = NW >= 16 ? 4 : 8;  // rows per trip in the local pack / unpack phases (8 x 16 B loads in flight per thread)
  const int cta = blockIdx.x, grid = gridDim.x;
  const TensorDesc* descs = a.descs ? a.descs : a.inline_descs;
  const TensorDesc* odescs = a.out_descs ? a.out_descs : descs;
  const int nout = a.out_descs ? a.nout : a.ndesc;
  uint32_t epoch = cp.epochs[cta];
  char* mybuf = reinterpret_cast<char*>(cp.buf[cp.rank]);
  const int64_t total = a.total_bytes;
  const int64_t nchunks = (total + chunk_bytes - 1) / chunk_bytes;
  const S prescale = (S)a.prescale, postscale = (S)a.postscale;
  bool alive = true;

  // ---- pack ----
  for (int64_t c = cta; c < nchunks; c += grid) {
    const int64_t lo = c * chunk_bytes;
    const int64_t hi = lo + chunk_bytes < total ? lo + chunk_bytes : total;
    pack_range<T, W, UP>(descs, a.ndesc, total, mybuf, lo, hi, prescale);
  }
  if (cp.nranks > 1) alive = peer_barrier(cp, epoch, cta); else __syncthreads();

  if (a.variant == kOneShot) {
    // ---- reduce straight into the outputs ----
    DescCursor cur;
    cur.init(odescs, nout, total);
    for (int64_t c = cta; c < nchunks && alive; c += grid) {
      int64_t lo = c * chunk_bytes;
      int64_t hi = lo + chunk_bytes < total ? lo + chunk_bytes : total;
      if (lo < a.reduce_lo) lo = a.reduce_lo;
      if (hi > a.reduce_hi) hi = a.reduce_hi;
      if (a.oneshot_nvls) {
        // reduce-scatter through the switch: one multimem.ld_reduce per vector instead of N peer loads
        if constexpr (Nvls<W>::ok) {
          constexpr int UN = 4;
          for (int64_t o0 = lo + (int64_t)threadIdx.x * 16; o0 < hi; o0 += (int64_t)UN * kRowBytes) {
            uint4 v[UN];
#pragma unroll
            for (int j = 0; j < UN; ++j) {
              const int64_t o = o0 + (int64_t)j * kRowBytes;
              if (o < hi) v[j] = Nvls<W>::ld_reduce(reinterpret_cast<const char*>(cp.mc_buf) + o);
            }
#pragma unroll
            for (int j = 0; j < UN; ++j) {
              const int64_t o = o0 + (int64_t)j * kRowBytes;
              if (o < hi) {
                A acc[NW];
                unpack_vec<W, NW>(v[j], acc);
                cur.seek(o);
                const int64_t e = (o - cur.lo) / (int64_t)sizeof(W);
                if (e < cur.count) {
#pragma unroll
                  for (int i = 0; i < NW; ++i) acc[i] = apply_scale<A>(acc[i], postscale);
                  store_elems<T, NW, A>(reinterpret_cast<T*>(cur.out) + e, cur.count - e, acc);
                }
              }
            }
          }
        }
        continue;
      }
      for (int64_t o0 = lo + (int64_t)threadIdx.x * 16; o0 < hi; o0 += (int64_t)U * kRowBytes) {
        uint4 v[U][NR];
        peer_loads<NR, U>(cp, cp.buf, o0, hi, v);
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const int64_t o = o0 + (int64_t)j * kRowBytes;
          if (o < hi) {
            A acc[NW];
            peer_combine<W, NR>(cp, v[j], a.op, acc);
            cur.seek(o);
            const int64_t e = (o - cur.lo) / (int64_t)sizeof(W);
            if (e < cur.count) {
#pragma unroll
              for (int i = 0; i < NW; ++i) acc[i] = apply_scale<A>(acc[i], postscale);
              store_elems<T, NW, A>(reinterpret_cast<T*>(cur.out) + e, cur.count - e, acc);
            }
          }
        }
      }
    }
  } else {
    // ---- reduce the chunks I own, publish to every peer ----
    for (int64_t c = cta, k = 0; c < nchunks && alive; c += grid, ++k) {
      int owner = (int)((k + cta) % cp.nranks);
      if (owner != cp.rank) continue;
      const int64_t lo = c * chunk_bytes;
      const int64_t hi = lo + chunk_bytes < total ? lo + chunk_bytes : total;
      if (a.variant == kNvls) {
        if constexpr (Nvls<W>::ok) {
          constexpr int UN = 4;
          for (int64_t o0 = lo + (int64_t)threadIdx.x * 16; o0 < hi; o0 += (int64_t)UN * kRowBytes) {
            uint4 v[UN];
#pragma unroll
            for (int j = 0; j < UN; ++j) {
              const int64_t o = o0 + (int64_t)j * kRowBytes;
              if (o < hi) v[j] = Nvls<W>::ld_reduce(reinterpret_cast<const char*>(cp.mc_buf) + o);
            }
#pragma unroll
            for (int j = 0; j < UN; ++j) {
              const int64_t o = o0 + (int64_t)j * kRowBytes;
              if (o < hi) {
                if (postscale != (S)1) {
                  A acc[NW];
                  unpack_vec<W, NW>(v[j], acc);
#pragma unroll
                  for (int i = 0; i < NW; ++i) acc[i] = apply_scale<A>(acc[i], postscale);
                  v[j] = pack_vec<W, NW>(acc);
                }
                multimem_st(reinterpret_cast<char*>(cp.mc_buf) + o, v[j]);
              }
            }
          }
        }
      } else {
        for (int64_t o0 = lo + (int64_t)threadIdx.x * 16; o0 < hi; o0 += (int64_t)U * kRowBytes) {
          uint4 v[U][NR];
          peer_loads<NR, U>(cp, cp.buf, o0, hi, v);
#pragma unroll
          for (int j = 0; j < U; ++j) {
            const int64_t o = o0 + (int64_t)j * kRowBytes;
            if (o < hi) {
              A acc[NW];
              peer_combine<W, NR>(cp, v[j], a.op, acc);
#pragma unroll
              for (int i = 0; i < NW; ++i) acc[i] = apply_scale<A>(acc[i], postscale);
              const uint4 r = pack_vec<W, NW>(acc);
#pragma unroll
              for (int p = 0; p < NR; ++p) {
                int q = cp.rank + p; if (q >= cp.nranks) q -= cp.nranks;
                if (p < cp.nranks) st_stream(reinterpret_cast<char*>(cp.buf[q]) + o, r);
              }
            }
          }
        }
      }
    }
    if (alive) alive = peer_barrier(cp, epoch, cta);
    // ---- unpack my buffer ----
    for (int64_t c = cta; c < nchunks && alive; c += grid) {
      int64_t lo = c * chunk_bytes;
      int64_t hi = lo + chunk_bytes < total ? lo + chunk_bytes : total;
      if (lo < a.reduce_lo) lo = a.reduce_lo;
      if (hi > a.reduce_hi) hi = a.reduce_hi;
      if (lo < hi) unpack_range<T, W, UP>(odescs, nout, total, mybuf, lo, hi);
    }
  }
  if (threadIdx.x == 0) cp.epochs[cta] = epoch;
}

// One chunk of the in-switch allreduce: UN independent multimem.ld_reduce per thread are issued before the first
// multimem.st so UN x 16 B per thread are in flight through the NVSwitch.
template <typename W, int UN>
__device__ __forceinline__ void nvls_inplace_rows(char* mc, int64_t lo, int64_t hi, typename ScaleOf<typename Traits<W>::Acc>::type scale) {
  using A = typename Traits<W>::Acc;
  using S = typename ScaleOf<A>::type;
  constexpr int NW = 16 / (int)sizeof(W);
  for (int64_t o0 = lo + (int64_t)threadIdx.x * 16; o0 < hi; o0 += (int64_t)UN * kRowBytes) {
    uint4 v[UN];
#pragma unroll
    for (int j = 0; j < UN; ++j) { const int64_t o = o0 + (int64_t)j * kRowBytes; if (o < hi) v[j] = Nvls<W>::ld_reduce(mc + o); }
#pragma unroll
    for (int j = 0; j < UN; ++j) {
      const int64_t o = o0 + (int64_t)j * kRowBytes;
      if (o < hi) {
        if (scale != (S)1) {
          A acc[NW];
          unpack_vec<W, NW>(v[j], acc);
#pragma unroll
          for (int i = 0; i < NW; ++i) acc[i] = apply_scale<A>(acc[i], scale);
          v[j] = pack_vec<W, NW>(acc);
        }
        multimem_st(mc + o, v[j]);
      }
    }
  }
}

// ---------------------------------------------------------------------------
// Zero-copy allreduce on REGISTERED tensors (memory allocated with hvd.symm_empty / the bucketed DistributedOptimizer):
// the user tensor itself is peer-mapped, so there is no pack and no unpack — the kernel is only the NVLink phase.
//   barrier A   every rank's data is final (the kernel was ordered after the producer's ready event)
//   reduce      rank r sums the chunks it owns out of all N tensors and stores the result into all N tensors
//               (multimem.ld_reduce + multimem.st when the region is multicast-bound: the NVSwitch does the add
//               and the broadcast); a chunk has exactly one reader — its owner — so writing in place is safe
//   barrier B   every result landed
template <typename W, int NR>
__global__ void __launch_bounds__(kThreads, 2)
inplace_allreduce_kernel(const __grid_constant__ CommParams cp, const __grid_constant__ InplaceArgs a) {
  using A = typename Traits<W>::Acc;
  using S = typename ScaleOf<A>::type;
  constexpr int NW = 16 / (int)sizeof(W);
  constexpr int U = 8 / NR;
  const int cta = blockIdx.x, grid = gridDim.x;
  uint32_t epoch = cp.epochs[cta];
  const int64_t total = a.bytes;  // multiple of 16
  const int chunk_bytes = a.chunk_bytes;
  const int64_t nchunks = (total + chunk_bytes - 1) / chunk_bytes;
  const S scale = (S)a.scale;
  bool alive = peer_barrier(cp, epoch, cta);
  for (int64_t c = cta, k = 0; c < nchunks && alive; c += grid, ++k) {
    if ((int)((k + cta) % cp.nranks) != cp.rank) continue;
    const int64_t lo = c * chunk_bytes;
    const int64_t hi = lo + chunk_bytes < total ? lo + chunk_bytes : total;
    if (a.use_multicast) {
      if constexpr (Nvls<W>::ok) {
        char* mc = reinterpret_cast<char*>(a.mc);
        if (a.nvls_unroll == 8) nvls_inplace_rows<W, 8>(mc, lo, hi, scale);
        else nvls_inplace_rows<W, 4>(mc, lo, hi, scale);
      }
    } else {
      for (int64_t o0 = lo + (int64_t)threadIdx.x * 16; o0 < hi; o0 += (int64_t)U * kRowBytes) {
        uint4 v[U][NR];
        peer_loads<NR, U>(cp, a.ptr, o0, hi, v);
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const int64_t o = o0 + (int64_t)j * kRowBytes;
          if (o < hi) {
            A acc[NW];
            peer_combine<W, NR>(cp, v[j], a.op, acc);
#pragma unroll
            for (int i = 0; i < NW; ++i) acc[i] = apply_scale<A>(acc[i], scale);
            const uint4 r = pack_vec<W, NW>(acc);
#pragma unroll
            for (int p = 0; p < NR; ++p) {
              int q = cp.rank + p; if (q >= cp.nranks) q -= cp.nranks;
              if (p < cp.nranks) st_stream(reinterpret_cast<char*>(a.ptr[q]) + o, r);
            }
          }
        }
      }
    }
  }
  if (alive) peer_barrier(cp, epoch, cta);
  if (threadIdx.x == 0) cp.epochs[cta] = epoch;
}

// ---------------------------------------------------------------------------
// Zero-copy reduce-scatter / allgather on REGISTERED tensors, the two halves of a sharded optimizer step (ZeRO-1).
// Contiguous ownership, not the interleaved chunks of the allreduce above: for a range of `bytes` (a multiple of
// 16 * nranks) rank r owns [r*S, (r+1)*S) with S = bytes / nranks, so that its shard is one slice it can update.
// CTA b of every rank covers the same chunks of every shard and only synchronises with CTA b of its peers; a launch on
// rank q completes only after all of its CTAs passed barrier B, i.e. after every CTA of every peer did its last access.

// In-switch reduction of [lo, hi) stored to `dst` only (a plain local store instead of multimem.st).
template <typename W, int UN>
__device__ __forceinline__ void nvls_reduce_rows(const char* mc, char* dst, int64_t lo, int64_t hi,
                                                 typename ScaleOf<typename Traits<W>::Acc>::type scale) {
  using A = typename Traits<W>::Acc;
  using S = typename ScaleOf<A>::type;
  constexpr int NW = 16 / (int)sizeof(W);
  for (int64_t o0 = lo + (int64_t)threadIdx.x * 16; o0 < hi; o0 += (int64_t)UN * kRowBytes) {
    uint4 v[UN];
#pragma unroll
    for (int j = 0; j < UN; ++j) { const int64_t o = o0 + (int64_t)j * kRowBytes; if (o < hi) v[j] = Nvls<W>::ld_reduce(mc + o); }
#pragma unroll
    for (int j = 0; j < UN; ++j) {
      const int64_t o = o0 + (int64_t)j * kRowBytes;
      if (o < hi) {
        if (scale != (S)1) {
          A acc[NW];
          unpack_vec<W, NW>(v[j], acc);
#pragma unroll
          for (int i = 0; i < NW; ++i) acc[i] = apply_scale<A>(acc[i], scale);
          v[j] = pack_vec<W, NW>(acc);
        }
        st_stream(dst + o, v[j]);
      }
    }
  }
}

//   barrier A   every rank's gradients are final
//   reduce      rank r loads its shard out of all N tensors (or one multimem.ld_reduce), combines, scales and stores the
//               result into ITS OWN tensor only; bytes outside the shard are neither reduced nor written
//   barrier B   no peer may overwrite its gradients (next zero_grad / backward) while a reader still loads them
template <typename W, int NR>
__global__ void __launch_bounds__(kThreads, 2)
inplace_reducescatter_kernel(const __grid_constant__ CommParams cp, const __grid_constant__ InplaceArgs a) {
  using A = typename Traits<W>::Acc;
  using S = typename ScaleOf<A>::type;
  constexpr int NW = 16 / (int)sizeof(W);
  constexpr int U = 8 / NR;
  const int cta = blockIdx.x, grid = gridDim.x;
  uint32_t epoch = cp.epochs[cta];
  const int64_t shard = a.bytes / cp.nranks, base = shard * cp.rank;
  const int chunk_bytes = a.chunk_bytes;
  const int64_t nchunks = (shard + chunk_bytes - 1) / chunk_bytes;
  const S scale = (S)a.scale;
  char* mine = reinterpret_cast<char*>(a.ptr[cp.rank]);
  bool alive = peer_barrier(cp, epoch, cta);
  for (int64_t c = cta; c < nchunks && alive; c += grid) {
    const int64_t lo = base + c * chunk_bytes;
    const int64_t hi = lo + chunk_bytes < base + shard ? lo + chunk_bytes : base + shard;
    if (a.use_multicast) {
      if constexpr (Nvls<W>::ok) {
        const char* mc = reinterpret_cast<const char*>(a.mc);
        if (a.nvls_unroll == 8) nvls_reduce_rows<W, 8>(mc, mine, lo, hi, scale);
        else nvls_reduce_rows<W, 4>(mc, mine, lo, hi, scale);
      }
    } else {
      for (int64_t o0 = lo + (int64_t)threadIdx.x * 16; o0 < hi; o0 += (int64_t)U * kRowBytes) {
        uint4 v[U][NR];
        peer_loads<NR, U>(cp, a.ptr, o0, hi, v);
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const int64_t o = o0 + (int64_t)j * kRowBytes;
          if (o < hi) {
            A acc[NW];
            peer_combine<W, NR>(cp, v[j], a.op, acc);
#pragma unroll
            for (int i = 0; i < NW; ++i) acc[i] = apply_scale<A>(acc[i], scale);
            st_stream(mine + o, pack_vec<W, NW>(acc));
          }
        }
      }
    }
  }
  if (alive) peer_barrier(cp, epoch, cta);
  if (threadIdx.x == 0) cp.epochs[cta] = epoch;
}

//   barrier A   every owner's update of its shard is final and every peer finished reading its own copy (backward)
//   store       the owner reads its shard locally and writes it into every peer's copy (16 B stores per peer, or one
//               multimem.st through the multicast alias); bytes only, the dtype does not matter
//   barrier B   every shard landed before any rank's launch completes
template <int NR>
__global__ void __launch_bounds__(kThreads, 2)
inplace_allgather_kernel(const __grid_constant__ CommParams cp, const __grid_constant__ InplaceArgs a) {
  constexpr int U = 8;
  const int cta = blockIdx.x, grid = gridDim.x;
  uint32_t epoch = cp.epochs[cta];
  const int64_t shard = a.bytes / cp.nranks, base = shard * cp.rank;
  const int chunk_bytes = a.chunk_bytes;
  const int64_t nchunks = (shard + chunk_bytes - 1) / chunk_bytes;
  const char* mine = reinterpret_cast<const char*>(a.ptr[cp.rank]);
  bool alive = peer_barrier(cp, epoch, cta);
  for (int64_t c = cta; c < nchunks && alive; c += grid) {
    const int64_t lo = base + c * chunk_bytes;
    const int64_t hi = lo + chunk_bytes < base + shard ? lo + chunk_bytes : base + shard;
    for (int64_t o0 = lo + (int64_t)threadIdx.x * 16; o0 < hi; o0 += (int64_t)U * kRowBytes) {
      uint4 v[U];
#pragma unroll
      for (int j = 0; j < U; ++j) { const int64_t o = o0 + (int64_t)j * kRowBytes; if (o < hi) v[j] = ld_stream(mine + o); }
#pragma unroll
      for (int j = 0; j < U; ++j) {
        const int64_t o = o0 + (int64_t)j * kRowBytes;
        if (o < hi) {
          if (a.use_multicast) {
            multimem_st(reinterpret_cast<char*>(a.mc) + o, v[j]);
          } else {
#pragma unroll
            for (int p = 1; p < NR; ++p) {  // p = 0 is my own copy, which already holds the shard
              int q = cp.rank + p; if (q >= cp.nranks) q -= cp.nranks;
              if (p < cp.nranks) st_stream(reinterpret_cast<char*>(a.ptr[q]) + o, v[j]);
            }
          }
        }
      }
    }
  }
  if (alive) peer_barrier(cp, epoch, cta);
  if (threadIdx.x == 0) cp.epochs[cta] = epoch;
}

template <typename W>
cudaError_t launch_inplace(const CommParams& cp, const InplaceArgs& a, cudaStream_t s) {
  if (cp.nranks <= 2) inplace_allreduce_kernel<W, 2><<<a.ctas, kThreads, 0, s>>>(cp, a);
  else if (cp.nranks <= 4) inplace_allreduce_kernel<W, 4><<<a.ctas, kThreads, 0, s>>>(cp, a);
  else inplace_allreduce_kernel<W, 8><<<a.ctas, kThreads, 0, s>>>(cp, a);
  CountKernelLaunch();
  return cudaGetLastError();
}

template <typename W>
cudaError_t launch_reducescatter(const CommParams& cp, const InplaceArgs& a, cudaStream_t s) {
  if (cp.nranks <= 2) inplace_reducescatter_kernel<W, 2><<<a.ctas, kThreads, 0, s>>>(cp, a);
  else if (cp.nranks <= 4) inplace_reducescatter_kernel<W, 4><<<a.ctas, kThreads, 0, s>>>(cp, a);
  else inplace_reducescatter_kernel<W, 8><<<a.ctas, kThreads, 0, s>>>(cp, a);
  CountKernelLaunch();
  return cudaGetLastError();
}

// Checks shared by the sharded launchers and the chunk size / NVLS unroll they pick (as LaunchInplaceAllreduce does).
bool prepare_sharded(const CommParams& cp, InplaceArgs* a) {
  if (a->ctas < 1 || a->ctas > kMaxCtas || cp.nranks < 1 || cp.nranks > kMaxPeers || a->bytes <= 0 ||
      a->bytes % (16 * (int64_t)cp.nranks))
    return false;
  int64_t want = a->bytes / ((int64_t)a->ctas * cp.nranks);
  int chunk = (int)((want / kRowBytes) * kRowBytes);
  if (chunk < kRowBytes) chunk = kRowBytes;
  const int max_chunk = [] { const char* e = getenv("HVD_INPLACE_CHUNK_BYTES"); int v = e ? atoi(e) : kChunkBytes;
                                    return v < kRowBytes ? kRowBytes : (v / kRowBytes) * kRowBytes; }();
  if (chunk > max_chunk) chunk = max_chunk;
  a->chunk_bytes = chunk;
  a->nvls_unroll = [] { const char* e = getenv("HVD_NVLS_UNROLL"); return e && atoi(e) == 8 ? 8 : 4; }();
  return true;
}

// Stand-alone pack / unpack (NCCL baseline path): whole grid strides over rows.
template <typename T, typename W>
__global__ void __launch_bounds__(kThreads)
pack_unpack_kernel(char* buffer, const TensorDesc* descs, int nd, int64_t total, double scale, int direction) {
  using A = typename Traits<W>::Acc;
  using S = typename ScaleOf<A>::type;
  constexpr int NW = 16 / (int)sizeof(W);
  DescCursor cur;
  cur.init(descs, nd, total);
  for (int64_t o = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * 16; o < total; o += (int64_t)gridDim.x * kRowBytes) {
    cur.seek(o);
    const int64_t e = (o - cur.lo) / (int64_t)sizeof(W);
    A acc[NW];
    if (direction == 0) {
      load_elems<T, NW, A>(reinterpret_cast<const T*>(cur.in) + e, cur.count - e, acc);
#pragma unroll
      for (int i = 0; i < NW; ++i) acc[i] = apply_scale<A>(acc[i], (S)scale);
      st_stream(buffer + o, pack_vec<W, NW>(acc));
    } else {
      if (e >= cur.count) continue;
      unpack_vec<W, NW>(ld_stream(buffer + o), acc);
#pragma unroll
      for (int i = 0; i < NW; ++i) acc[i] = apply_scale<A>(acc[i], (S)scale);
      store_elems<T, NW, A>(reinterpret_cast<T*>(cur.out) + e, cur.count - e, acc);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) scale_kernel(const T* in, T* out, int64_t n, double scale) {
  using A = typename Traits<T>::Acc;
  using S = typename ScaleOf<A>::type;
  constexpr int N = 16 / (int)sizeof(T);
  for (int64_t e = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * N; e < n; e += (int64_t)gridDim.x * kThreads * N) {
    A a[N];
    load_elems<T, N, A>(in + e, n - e, a);
#pragma unroll
    for (int i = 0; i < N; ++i) a[i] = apply_scale<A>(a[i], (S)scale);
    store_elems<T, N, A>(out + e, n - e, a);
  }
}

template <typename T, typename W>
cudaError_t launch_tw(const CommParams& cp, const AllreduceArgs& a, int chunk_bytes, cudaStream_t s) {
  dim3 grid(a.ctas), block(kThreads);
  if (cp.nranks <= 2) allreduce_kernel<T, W, 2><<<grid, block, 0, s>>>(cp, a, chunk_bytes);
  else if (cp.nranks <= 4) allreduce_kernel<T, W, 4><<<grid, block, 0, s>>>(cp, a, chunk_bytes);
  else allreduce_kernel<T, W, 8><<<grid, block, 0, s>>>(cp, a, chunk_bytes);
  CountKernelLaunch();
  return cudaGetLastError();
}

template <typename T, typename W>
cudaError_t launch_pu(char* buffer, const TensorDesc* descs, int nd, int64_t total, double scale, int dir, int ctas,
                      cudaStream_t s) {
  pack_unpack_kernel<T, W><<<ctas, kThreads, 0, s>>>(buffer, descs, nd, total, scale, dir);
  CountKernelLaunch();
  return cudaGetLastError();
}

}  // namespace

// dtype codes: hvd::DataType
#define HVD_DISPATCH(dtype, wire, FN, ...)                                                         \
  switch (dtype) {                                                                                 \
    case 0: return FN<uint8_t, uint8_t>(__VA_ARGS__);                                               \
    case 9: return FN<uint8_t, uint8_t>(__VA_ARGS__);                                               \
    case 1: return FN<int8_t, int8_t>(__VA_ARGS__);                                                 \
    case 2: case 3: return FN<int16_t, int16_t>(__VA_ARGS__);                                       \
    case 4: return FN<int32_t, int32_t>(__VA_ARGS__);                                               \
    case 5: return FN<int64_t, int64_t>(__VA_ARGS__);                                               \
    case 6: return FN<__half, __half>(__VA_ARGS__);                                                 \
    case 7:                                                                                        \
      if (wire == 10) return FN<float, __nv_bfloat16>(__VA_ARGS__);                                 \
      if (wire == 6) return FN<float, __half>(__VA_ARGS__);                                         \
      return FN<float, float>(__VA_ARGS__);                                                         \
    case 8: return FN<double, double>(__VA_ARGS__);                                                 \
    case 10: return FN<__nv_bfloat16, __nv_bfloat16>(__VA_ARGS__);                                  \
    default: return cudaErrorInvalidValue;                                                         \
  }

cudaError_t LaunchAllreduce(const CommParams& cp, const AllreduceArgs& args, cudaStream_t stream) {
  if (args.ctas < 1 || args.ctas > kMaxCtas || cp.nranks < 1 || cp.nranks > kMaxPeers) return cudaErrorInvalidValue;
  if (args.variant != kOneShot && args.variant != kTwoShot && args.variant != kNvls) return cudaErrorInvalidValue;
  if (args.total_bytes <= 0) return cudaSuccess;
  if (args.variant == kNvls) {
    const int w = args.dtype == 7 ? (args.wire_dtype == 10 || args.wire_dtype == 6 ? args.wire_dtype : 7) : args.dtype;
    if (!(w == 7 || w == 6 || w == 10) || args.op != 1 || cp.mc_buf == nullptr) return cudaErrorInvalidValue;
  }
  if (args.oneshot_nvls) {
    const int w = args.dtype == 7 ? (args.wire_dtype == 10 || args.wire_dtype == 6 ? args.wire_dtype : 7) : args.dtype;
    if (args.variant != kOneShot || !(w == 7 || w == 6 || w == 10) || args.op != 1 || cp.mc_buf == nullptr) return cudaErrorInvalidValue;
  }
  // chunk size: enough chunks that every (rank, CTA) pair owns work, bounded by [8 KiB, 32 KiB]
  int64_t want = args.total_bytes / ((int64_t)args.ctas * cp.nranks);
  int chunk = (int)((want / kRowBytes) * kRowBytes);
  if (chunk < kRowBytes) chunk = kRowBytes;
  if (chunk > kChunkBytes) chunk = kChunkBytes;
  HVD_DISPATCH(args.dtype, args.wire_dtype, launch_tw, cp, args, chunk, stream)
}

cudaError_t LaunchInplaceAllreduce(const CommParams& cp, const InplaceArgs& args, cudaStream_t stream) {
  if (args.ctas < 1 || args.ctas > kMaxCtas || args.bytes <= 0 || (args.bytes & 15)) return cudaErrorInvalidValue;
  InplaceArgs a = args;
  int64_t want = a.bytes / ((int64_t)a.ctas * cp.nranks);
  int chunk = (int)((want / kRowBytes) * kRowBytes);
  if (chunk < kRowBytes) chunk = kRowBytes;
  const int max_chunk = [] { const char* e = getenv("HVD_INPLACE_CHUNK_BYTES"); int v = e ? atoi(e) : kChunkBytes;
                                    return v < kRowBytes ? kRowBytes : (v / kRowBytes) * kRowBytes; }();
  const int unroll = [] { const char* e = getenv("HVD_NVLS_UNROLL"); return e && atoi(e) == 8 ? 8 : 4; }();
  if (chunk > max_chunk) chunk = max_chunk;
  a.chunk_bytes = chunk;
  a.nvls_unroll = unroll;
  switch (a.dtype) {
    case 7: return launch_inplace<float>(cp, a, stream);
    case 6: return launch_inplace<__half>(cp, a, stream);
    case 10: return launch_inplace<__nv_bfloat16>(cp, a, stream);
    case 8: if (a.use_multicast) return cudaErrorInvalidValue; return launch_inplace<double>(cp, a, stream);
    case 4: if (a.use_multicast) return cudaErrorInvalidValue; return launch_inplace<int32_t>(cp, a, stream);
    case 5: if (a.use_multicast) return cudaErrorInvalidValue; return launch_inplace<int64_t>(cp, a, stream);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t LaunchInplaceReducescatter(const CommParams& cp, const InplaceArgs& args, cudaStream_t stream) {
  InplaceArgs a = args;
  if (!prepare_sharded(cp, &a)) return cudaErrorInvalidValue;
  const bool sum_like = a.op == 1;
  if (a.use_multicast && (!sum_like || a.mc == nullptr)) return cudaErrorInvalidValue;
  switch (a.dtype) {
    case 7: return launch_reducescatter<float>(cp, a, stream);
    case 6: return launch_reducescatter<__half>(cp, a, stream);
    case 10: return launch_reducescatter<__nv_bfloat16>(cp, a, stream);
    case 8: if (a.use_multicast) return cudaErrorInvalidValue; return launch_reducescatter<double>(cp, a, stream);
    case 4: if (a.use_multicast) return cudaErrorInvalidValue; return launch_reducescatter<int32_t>(cp, a, stream);
    case 5: if (a.use_multicast) return cudaErrorInvalidValue; return launch_reducescatter<int64_t>(cp, a, stream);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t LaunchInplaceAllgather(const CommParams& cp, const InplaceArgs& args, cudaStream_t stream) {
  InplaceArgs a = args;
  if (!prepare_sharded(cp, &a)) return cudaErrorInvalidValue;
  if (a.use_multicast && a.mc == nullptr) return cudaErrorInvalidValue;
  if (cp.nranks <= 2) inplace_allgather_kernel<2><<<a.ctas, kThreads, 0, stream>>>(cp, a);
  else if (cp.nranks <= 4) inplace_allgather_kernel<4><<<a.ctas, kThreads, 0, stream>>>(cp, a);
  else inplace_allgather_kernel<8><<<a.ctas, kThreads, 0, stream>>>(cp, a);
  CountKernelLaunch();
  return cudaGetLastError();
}

cudaError_t LaunchPackUnpack(void* buffer, const TensorDesc* descs, int ndesc, int64_t total_bytes, int dtype,
                             int wire_dtype, double scale, int direction, int ctas, cudaStream_t stream) {
  if (total_bytes <= 0) return cudaSuccess;
  HVD_DISPATCH(dtype, wire_dtype, launch_pu, (char*)buffer, descs, ndesc, total_bytes, scale, direction, ctas, stream)
}

namespace {
template <typename T, typename W> cudaError_t launch_scale(const void* in, void* out, int64_t n, double scale, cudaStream_t s) {
  int64_t per = (int64_t)kThreads * (16 / sizeof(T));
  int64_t blocks = (n + per - 1) / per;
  if (blocks > 132 * 8) blocks = 132 * 8;
  if (blocks < 1) blocks = 1;
  scale_kernel<T><<<(int)blocks, kThreads, 0, s>>>((const T*)in, (T*)out, n, scale);
  CountKernelLaunch();
  return cudaGetLastError();
}
}  // namespace

cudaError_t LaunchScale(const void* in, void* out, int64_t count, int dtype, double scale, cudaStream_t stream) {
  if (count <= 0) return cudaSuccess;
  const int wire = dtype;
  HVD_DISPATCH(dtype, wire, launch_scale, in, out, count, scale, stream)
}

}  // namespace kern
}  // namespace hvd
