// Device-side building blocks shared by the P2P collective kernels:
// dtype traits, 128-bit streaming loads/stores, fused-buffer descriptor cursor
// and the cross-GPU flag barrier.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>
#include "p2p_kernels.h"

namespace hvd {
namespace kern {

// ---------------------------------------------------------------------------
// dtype traits: accumulate type + conversions

template <typename T> struct Traits;
template <> struct Traits<float> { using Acc = float; static __device__ __forceinline__ float to_acc(float v) { return v; } static __device__ __forceinline__ float from_acc(float v) { return v; } };
template <> struct Traits<double> { using Acc = double; static __device__ __forceinline__ double to_acc(double v) { return v; } static __device__ __forceinline__ double from_acc(double v) { return v; } };
template <> struct Traits<__half> { using Acc = float; static __device__ __forceinline__ float to_acc(__half v) { return __half2float(v); } static __device__ __forceinline__ __half from_acc(float v) { return __float2half_rn(v); } };
template <> struct Traits<__nv_bfloat16> { using Acc = float; static __device__ __forceinline__ float to_acc(__nv_bfloat16 v) { return __bfloat162float(v); } static __device__ __forceinline__ __nv_bfloat16 from_acc(float v) { return __float2bfloat16_rn(v); } };
template <> struct Traits<int32_t> { using Acc = int32_t; static __device__ __forceinline__ int32_t to_acc(int32_t v) { return v; } static __device__ __forceinline__ int32_t from_acc(int32_t v) { return v; } };
template <> struct Traits<int64_t> { using Acc = int64_t; static __device__ __forceinline__ int64_t to_acc(int64_t v) { return v; } static __device__ __forceinline__ int64_t from_acc(int64_t v) { return v; } };
template <> struct Traits<uint8_t> { using Acc = int32_t; static __device__ __forceinline__ int32_t to_acc(uint8_t v) { return v; } static __device__ __forceinline__ uint8_t from_acc(int32_t v) { return (uint8_t)v; } };
template <> struct Traits<int8_t> { using Acc = int32_t; static __device__ __forceinline__ int32_t to_acc(int8_t v) { return v; } static __device__ __forceinline__ int8_t from_acc(int32_t v) { return (int8_t)v; } };
template <> struct Traits<int16_t> { using Acc = int32_t; static __device__ __forceinline__ int32_t to_acc(int16_t v) { return v; } static __device__ __forceinline__ int16_t from_acc(int32_t v) { return (int16_t)v; } };

template <typename A> __device__ __forceinline__ A combine(A a, A b, int op) {
  switch (op) {
    case 3: return b < a ? b : a;   // MIN
    case 4: return b > a ? b : a;   // MAX
    case 5: return a * b;           // PRODUCT
    default: return a + b;          // SUM / AVERAGE / ADASUM-local
  }
}
template <typename A> struct ScaleOf { using type = double; };
template <> struct ScaleOf<float> { using type = float; };
template <typename A> __device__ __forceinline__ A apply_scale(A a, typename ScaleOf<A>::type s) { return (A)(a * s); }
template <> __device__ __forceinline__ int32_t apply_scale<int32_t>(int32_t a, double s) { return s == 1.0 ? a : (int32_t)((double)a * s); }
template <> __device__ __forceinline__ int64_t apply_scale<int64_t>(int64_t a, double s) { return s == 1.0 ? a : (int64_t)((double)a * s); }

// ---------------------------------------------------------------------------
// 128-bit streaming accesses (no L1 allocation: every byte is touched once)

__device__ __forceinline__ uint4 ld_stream(const void* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_stream(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

template <typename W, int NW> __device__ __forceinline__ void unpack_vec(const uint4& v, typename Traits<W>::Acc* a) {
  const W* p = reinterpret_cast<const W*>(&v);
#pragma unroll
  for (int i = 0; i < NW; ++i) a[i] = Traits<W>::to_acc(p[i]);
}
template <typename W, int NW> __device__ __forceinline__ uint4 pack_vec(const typename Traits<W>::Acc* a) {
  uint4 v;
  W* p = reinterpret_cast<W*>(&v);
#pragma unroll
  for (int i = 0; i < NW; ++i) p[i] = Traits<W>::from_acc(a[i]);
  return v;
}

// Loads N consecutive elements of T (vector path when 16 B aligned and fully
// in range, guarded scalar path with zero fill otherwise) into accumulators.
template <typename T, int N, typename A> __device__ __forceinline__ void load_elems(const T* p, int64_t remaining, A* a) {
  constexpr int kBytes = N * (int)sizeof(T);
  static_assert(kBytes >= 16 ? kBytes % 16 == 0 : (kBytes == 8 || kBytes == 4), "unsupported vector width");
  constexpr int kAlign = kBytes >= 16 ? 16 : kBytes;
  if (remaining >= N && ((reinterpret_cast<uintptr_t>(p) & (kAlign - 1)) == 0)) {
    if constexpr (kBytes >= 16) {
#pragma unroll
      for (int k = 0; k < kBytes / 16; ++k) {
        uint4 v = ld_stream(reinterpret_cast<const char*>(p) + 16 * k);
        const T* q = reinterpret_cast<const T*>(&v);
#pragma unroll
        for (int i = 0; i < 16 / (int)sizeof(T); ++i) a[k * (16 / (int)sizeof(T)) + i] = (A)Traits<T>::to_acc(q[i]);
      }
    } else if constexpr (kBytes == 8) {  // e.g. 4 x bf16 feeding an fp32 wire vector (Adasum pack)
      const uint2 v = *reinterpret_cast<const uint2*>(p);
      const T* q = reinterpret_cast<const T*>(&v);
#pragma unroll
      for (int i = 0; i < N; ++i) a[i] = (A)Traits<T>::to_acc(q[i]);
    } else {
      const uint32_t v = *reinterpret_cast<const uint32_t*>(p);
      const T* q = reinterpret_cast<const T*>(&v);
#pragma unroll
      for (int i = 0; i < N; ++i) a[i] = (A)Traits<T>::to_acc(q[i]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i) a[i] = i < remaining ? (A)Traits<T>::to_acc(p[i]) : (A)0;
  }
}
template <typename T, int N, typename A> __device__ __forceinline__ void store_elems(T* p, int64_t remaining, const A* a) {
  constexpr int kBytes = N * (int)sizeof(T);
  static_assert(kBytes >= 16 ? kBytes % 16 == 0 : (kBytes == 8 || kBytes == 4), "unsupported vector width");
  constexpr int kAlign = kBytes >= 16 ? 16 : kBytes;
  if (remaining >= N && ((reinterpret_cast<uintptr_t>(p) & (kAlign - 1)) == 0)) {
    if constexpr (kBytes >= 16) {
#pragma unroll
      for (int k = 0; k < kBytes / 16; ++k) {
        uint4 v;
        T* q = reinterpret_cast<T*>(&v);
#pragma unroll
        for (int i = 0; i < 16 / (int)sizeof(T); ++i) q[i] = Traits<T>::from_acc((typename Traits<T>::Acc)a[k * (16 / (int)sizeof(T)) + i]);
        st_stream(reinterpret_cast<char*>(p) + 16 * k, v);
      }
    } else if constexpr (kBytes == 8) {
      uint2 v;
      T* q = reinterpret_cast<T*>(&v);
#pragma unroll
      for (int i = 0; i < N; ++i) q[i] = Traits<T>::from_acc((typename Traits<T>::Acc)a[i]);
      *reinterpret_cast<uint2*>(p) = v;
    } else {
      uint32_t v;
      T* q = reinterpret_cast<T*>(&v);
#pragma unroll
      for (int i = 0; i < N; ++i) q[i] = Traits<T>::from_acc((typename Traits<T>::Acc)a[i]);
      *reinterpret_cast<uint32_t*>(p) = v;
    }
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i) if (i < remaining) p[i] = Traits<T>::from_acc((typename Traits<T>::Acc)a[i]);
  }
}

// ---------------------------------------------------------------------------
// Cursor over the fused-buffer descriptor table: maps a wire byte offset to the
// tensor that owns it.  Offsets seen by one thread grow monotonically inside a
// phase, so after the first binary search it only walks forward.

struct DescCursor {
  const TensorDesc* d;
  int n;
  int i;
  int64_t lo, hi, total;
  // the current descriptor, held in registers: the table is read again only when the cursor crosses a tensor boundary
  // (ncu of the round-1 kernel: the per-vector descriptor reload + 64-bit compares were ~40 % of the stall samples)
  const char* in;
  char* out;
  int64_t count;
  __device__ __forceinline__ void init(const TensorDesc* descs, int ndesc, int64_t total_bytes) {
    d = descs; n = ndesc; i = -1; lo = 0; hi = 0; total = total_bytes; in = nullptr; out = nullptr; count = 0;
  }
  __device__ __forceinline__ int64_t end_of(int k) const { return k + 1 < n ? d[k + 1].offset : total; }
  __device__ __forceinline__ void load() { in = reinterpret_cast<const char*>(d[i].in); out = reinterpret_cast<char*>(d[i].out); count = d[i].count; }
  __device__ __forceinline__ void seek(int64_t o) {
    if (i >= 0 && o >= lo && o < hi) return;
    if (i < 0 || o < lo) {
      int a = 0, b = n - 1;
      while (a < b) {
        int m = (a + b + 1) >> 1;
        if (d[m].offset <= o) a = m; else b = m - 1;
      }
      i = a; lo = d[i].offset; hi = end_of(i);
    } else {
      while (o >= hi && i + 1 < n) { ++i; lo = hi; hi = end_of(i); }
    }
    load();
  }
};

// N consecutive elements, caller guarantees a 16 B aligned address and N elements in range.
template <typename T, int N, typename A> __device__ __forceinline__ void load_elems_fast(const T* p, A* a) {
  constexpr int kBytes = N * (int)sizeof(T);
  if constexpr (kBytes >= 16) {
#pragma unroll
    for (int k = 0; k < kBytes / 16; ++k) {
      uint4 v = ld_stream(reinterpret_cast<const char*>(p) + 16 * k);
      const T* q = reinterpret_cast<const T*>(&v);
#pragma unroll
      for (int i = 0; i < 16 / (int)sizeof(T); ++i) a[k * (16 / (int)sizeof(T)) + i] = (A)Traits<T>::to_acc(q[i]);
    }
  } else {
    load_elems<T, N, A>(p, N, a);
  }
}
template <typename T, int N, typename A> __device__ __forceinline__ void store_elems_fast(T* p, const A* a) {
  constexpr int kBytes = N * (int)sizeof(T);
  if constexpr (kBytes >= 16) {
#pragma unroll
    for (int k = 0; k < kBytes / 16; ++k) {
      uint4 v;
      T* q = reinterpret_cast<T*>(&v);
#pragma unroll
      for (int i = 0; i < 16 / (int)sizeof(T); ++i) q[i] = Traits<T>::from_acc((typename Traits<T>::Acc)a[k * (16 / (int)sizeof(T)) + i]);
      st_stream(reinterpret_cast<char*>(p) + 16 * k, v);
    }
  } else {
    store_elems<T, N, A>(p, N, a);
  }
}

// Byte copy by the whole CTA (exchange and alltoall kernels).
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

// ---------------------------------------------------------------------------
// Cross-GPU barrier between CTA `cta` of every rank.  Flags hold monotonically
// increasing epochs (never reset), one word per (cta, source rank) in the
// destination rank's memory; a rank can be at most one barrier ahead of a peer.

__device__ __forceinline__ bool peer_barrier(const CommParams& cp, uint32_t& epoch, int cta) {
  __shared__ int s_abort;
  if (threadIdx.x == 0) s_abort = 0;
  __syncthreads();
  ++epoch;
  if ((int)threadIdx.x < cp.nranks) {
    const int peer = threadIdx.x;
    st_release_sys(cp.flags[peer] + cta * kMaxPeers + cp.rank, epoch);
    const uint32_t* mine = cp.flags[cp.rank] + cta * kMaxPeers + peer;
    uint32_t spins = 0;
    unsigned long long t0 = 0;
    while ((int32_t)(ld_relaxed_sys(mine) - epoch) < 0) {
      if ((++spins & 0x3fff) == 0 && cp.abort_flag) {
        if (*reinterpret_cast<volatile int*>(cp.abort_flag)) { s_abort = 1; break; }
        if (cp.timeout_ns) {
          unsigned long long now;
          asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
          if (t0 == 0) t0 = now;
          else if (now - t0 > cp.timeout_ns) { *reinterpret_cast<volatile int*>(cp.abort_flag) = 2; s_abort = 1; break; }
        }
      }
    }
    (void)ld_acquire_sys(mine);  // acquire + L1 invalidate once, after the relaxed spin
  }
  __syncthreads();
  const int aborted = s_abort;
  __syncthreads();  // every thread has read the verdict before thread 0 of the next barrier may reset it
  return aborted == 0;
}

}  // namespace kern
}  // namespace hvd
