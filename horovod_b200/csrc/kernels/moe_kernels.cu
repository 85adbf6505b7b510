// Local data movement of expert-parallel dispatch and combine (hvd.ExpertDispatcher) for sm_90a.
//
// Around the captured alltoall (alltoall_kernels.cu), which moves rows between ranks, these kernels move rows within a
// rank:
//   route_count + route_pos  the stable order of the [T * k] (token, slot) assignments by expert: per-expert counts,
//                            per-rank splits and pos[a], the send-buffer row of assignment a = t * k + j.  The order is
//                            expert ascending, then a ascending (a stable argsort of the expert ids).
//   scatter                  dst[pos[t, j]] = src[t], or round(gates[t, j] * src[t]); optionally also the fp32 dot of
//                            src[t] with rows[pos[t, j]] of a second buffer (the gate gradient of the combine).
//   gather                   y[t] = sum_j gates[t, j] * src[pos[t, j]] in fp32, j ascending, rounded once (unit gates:
//                            a plain sum in j order).
//   regroup                  received rows, grouped by source rank, to rows grouped by local expert (zero-filled past the
//                            received total, with the group ends `offsets`), and the reverse, which also writes the
//                            return splits.
//
// Determinism: every output element is computed by one thread in a fixed order.  The counts use shared-memory integer
// atomics, whose result does not depend on their order; the tile bases are scanned by the last CTA (a ticket that it
// resets for the next launch, as in grad_shard_stats_kernel).  The gate dot is a per-lane sum over a fixed set of
// 16-byte chunks followed by a butterfly over the warp, so it depends on the row length only.  Results do not depend on
// the grid.  No state is kept between launches.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <type_traits>
#include "p2p_kernels.h"

namespace hvd {
namespace kern {
namespace {

constexpr int kMoeThreads = 256;
constexpr int kMoeWarps = kMoeThreads / 32;
constexpr int kRouteTile = 2048;                         // assignments per route CTA
constexpr int kRouteWarpSpan = kRouteTile / kMoeWarps;  // contiguous assignments per warp of route_pos
constexpr int kMoeUnroll = 4;                            // 16 B chunks in flight per lane
constexpr int kDtF32 = 7, kDtBf16 = 10, kDtF16 = 6;      // hvd::DataType codes

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

__device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Chunk c of a row of h elements: elements [c * V, c * V + V) that are < h, V = 16 / sizeof(T).  One 16 B access when the
// row is 16 B aligned (`vec`) and the chunk is whole, element by element otherwise; missing elements read as 0.
template <typename T> __device__ __forceinline__ void ld_chunk(const T* row, int64_t c, int64_t h, bool vec, float* f) {
  constexpr int V = 16 / sizeof(T);
  const int64_t e0 = c * V;
  if (vec && e0 + V <= h) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + e0);
    const T* q = reinterpret_cast<const T*>(&u);
#pragma unroll
    for (int i = 0; i < V; ++i) f[i] = to_f(q[i]);
  } else {
#pragma unroll
    for (int i = 0; i < V; ++i) f[i] = e0 + i < h ? to_f(row[e0 + i]) : 0.f;
  }
}
template <typename T> __device__ __forceinline__ void st_chunk(T* row, int64_t c, int64_t h, bool vec, const float* f) {
  constexpr int V = 16 / sizeof(T);
  const int64_t e0 = c * V;
  if (vec && e0 + V <= h) {
    uint4 u;
    T* q = reinterpret_cast<T*>(&u);
#pragma unroll
    for (int i = 0; i < V; ++i) q[i] = from_f<T>(f[i]);
    *reinterpret_cast<uint4*>(row + e0) = u;
  } else {
#pragma unroll
    for (int i = 0; i < V; ++i) if (e0 + i < h) row[e0 + i] = from_f<T>(f[i]);
  }
}

// Copies `bytes` from src to dst with one warp: 16 B vectors when both are 16 B aligned, bytes otherwise.  src == nullptr
// zero-fills.
__device__ __forceinline__ void warp_copy_bytes(const char* src, char* dst, int64_t bytes, int lane) {
  const bool vec = aligned16(dst) && (!src || aligned16(src));
  int64_t done = 0;
  if (vec) {
    const int64_t nv = bytes / 16;
    for (int64_t i0 = lane; i0 < nv; i0 += 32 * kMoeUnroll) {
      uint4 v[kMoeUnroll];
#pragma unroll
      for (int u = 0; u < kMoeUnroll; ++u) {
        const int64_t i = i0 + 32 * u;
        if (i < nv) v[u] = src ? reinterpret_cast<const uint4*>(src)[i] : make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int u = 0; u < kMoeUnroll; ++u) {
        const int64_t i = i0 + 32 * u;
        if (i < nv) reinterpret_cast<uint4*>(dst)[i] = v[u];
      }
    }
    done = nv * 16;
  }
  for (int64_t i = done + lane; i < bytes; i += 32) dst[i] = src ? src[i] : 0;
}

// Exclusive prefix sum over the block of one value per thread (kMoeThreads threads); *total receives the sum.
__device__ __forceinline__ int64_t block_exclusive_scan(int64_t v, int64_t* s_warp, int64_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  int64_t before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < kMoeWarps; ++w) {
    if (w < warp) before += s_warp[w];
    all += s_warp[w];
  }
  __syncthreads();
  *total = all;
  return before + inc - v;
}

// ---- route_count: per-tile expert histograms, then (last CTA) the bases, counts and splits ----------------------------
// hist[b * E + e]: assignments of tile b with expert e; bad[b]: whether tile b holds an id outside [0, E).  The last CTA
// turns hist into the first send-buffer row of each (tile, expert): start[e] + the assignments of expert e in earlier
// tiles.  counts[e] (int64) and splits[q] (int32, rank q holds experts [q * el, q * el + el)) are the totals; with a bad
// id anywhere every split is -1 and every count 0, so the exchange reports a negative split on every rank.
template <typename I>
__global__ void __launch_bounds__(kMoeThreads)
moe_route_count_kernel(const I* __restrict__ idx, int64_t A, int E, int n, int el, int* hist, int* bad, unsigned* ticket,
                       int64_t* counts, int* splits) {
  __shared__ int s_cnt[kMoeMaxExperts];
  __shared__ int s_bad;
  __shared__ bool s_last;
  __shared__ int64_t s_warp[kMoeWarps];
  const int b = blockIdx.x, tiles = gridDim.x, tid = threadIdx.x;
  for (int e = tid; e < E; e += kMoeThreads) s_cnt[e] = 0;
  if (tid == 0) s_bad = 0;
  __syncthreads();
  const int64_t lo = (int64_t)b * kRouteTile, hi = lo + kRouteTile < A ? lo + kRouteTile : A;
  for (int64_t a = lo + tid; a < hi; a += kMoeThreads) {
    const int64_t e = (int64_t)idx[a];
    if (e < 0 || e >= E) s_bad = 1;
    else atomicAdd(&s_cnt[e], 1);
  }
  __syncthreads();
  for (int e = tid; e < E; e += kMoeThreads) hist[(int64_t)b * E + e] = s_cnt[e];
  if (tid == 0) bad[b] = s_bad;
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(ticket, 1u) == (unsigned)tiles - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // ---- last CTA: totals per expert, then the tile bases ----
  int any_bad = 0;
  for (int t = tid; t < tiles; t += kMoeThreads) any_bad |= __ldcg(bad + t);
  any_bad = __syncthreads_or(any_bad);
  // thread `tid` owns experts [4 tid, 4 tid + 4) (E <= 4 * kMoeThreads)
  int64_t tot[4], sum = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int e = 4 * tid + i;
    int64_t run = 0;
    if (e < E)
      for (int t = 0; t < tiles; ++t) {
        int* h = hist + (int64_t)t * E + e;
        const int c = __ldcg(h);
        *h = (int)run;
        run += c;
      }
    tot[i] = run;
    sum += run;
  }
  int64_t total;
  int64_t start = block_exclusive_scan(sum, s_warp, &total);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int e = 4 * tid + i;
    if (e < E) {
      s_cnt[e] = (int)start;
      for (int t = 0; t < tiles; ++t) hist[(int64_t)t * E + e] += (int)start;
      counts[e] = any_bad ? 0 : tot[i];
    }
    start += tot[i];
  }
  __syncthreads();
  for (int q = tid; q < n; q += kMoeThreads) {
    const int b0 = s_cnt[q * el], b1 = q + 1 < n ? s_cnt[(q + 1) * el] : (int)total;
    splits[q] = any_bad ? -1 : b1 - b0;
  }
  if (tid == 0) *ticket = 0u;  // ready for the next launch on this stream
}

// ---- route_pos: pos[a] = base[tile][e] + the assignments of expert e before a in the tile ----------------------------
// Warp w of CTA b owns assignments [b * kRouteTile + w * kRouteWarpSpan, + kRouteWarpSpan), walked 32 at a time: first
// counted per (warp, expert), then those counts are turned into per-warp bases in warp order, then each lane's rank
// among the lanes with the same expert (__match_any_sync) gives its row.  An id outside [0, E) gets pos -1.
template <typename I>
__global__ void __launch_bounds__(kMoeThreads)
moe_route_pos_kernel(const I* __restrict__ idx, int64_t A, int E, const int* __restrict__ base, int* __restrict__ pos) {
  __shared__ int s_w[kMoeWarps][kMoeMaxExperts];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < kMoeWarps * E; i += kMoeThreads) s_w[i / E][i % E] = 0;
  __syncthreads();
  const int64_t lo = (int64_t)b * kRouteTile + (int64_t)warp * kRouteWarpSpan;
  const unsigned lt = (1u << lane) - 1u;
  for (int pass = 0; pass < 2; ++pass) {
    for (int c = 0; c < kRouteWarpSpan; c += 32) {
      const int64_t a = lo + c + lane;
      int e = -1;
      if (a < A) {
        const int64_t v = (int64_t)idx[a];
        e = v >= 0 && v < E ? (int)v : -1;
      }
      const int key = e >= 0 ? e : E + lane;  // lanes without a valid expert each form their own group
      const unsigned grp = __match_any_sync(0xffffffffu, key);
      const int leader = __ffs(grp) - 1;
      if (pass == 0) {
        if (e >= 0 && lane == leader) s_w[warp][e] += __popc(grp);
      } else {
        if (a < A) pos[a] = e >= 0 ? s_w[warp][e] + __popc(grp & lt) : -1;
        __syncwarp();
        if (e >= 0 && lane == leader) s_w[warp][e] += __popc(grp);
      }
      __syncwarp();
    }
    if (pass == 0) {
      __syncthreads();
      for (int e = tid; e < E; e += kMoeThreads) {
        int run = base[(int64_t)b * E + e];
#pragma unroll
        for (int w = 0; w < kMoeWarps; ++w) { const int c = s_w[w][e]; s_w[w][e] = run; run += c; }
      }
      __syncthreads();
    }
  }
}

// ---- scatter --------------------------------------------------------------------------------------------------------
// One warp per token t: for j < k with 0 <= p = pos[t * k + j] < dst_rows, dst[p] = src[t] (gates == nullptr: the bytes
// as they are) or round(gates[t * k + j] * src[t]).  With dot_rows, grad_gates[t * k + j] = sum_i src[t][i] *
// dot_rows[p][i] in fp32.  A non-zero *status writes nothing but zero gate gradients.
template <typename T, typename G>
__global__ void __launch_bounds__(kMoeThreads)
moe_scatter_kernel(const T* __restrict__ src, int64_t ntok, int k, int64_t h, const int* __restrict__ pos, T* dst,
                   int64_t dst_rows, const G* __restrict__ gates, const T* __restrict__ dot_rows, G* __restrict__ grad_gates,
                   const int* __restrict__ status) {
  constexpr int V = 16 / sizeof(T);
  const int lane = threadIdx.x & 31;
  const int64_t nch = (h + V - 1) / V;
  const bool dead = status && *status != 0;
  for (int64_t t = (int64_t)blockIdx.x * kMoeWarps + (threadIdx.x >> 5); t < ntok; t += (int64_t)gridDim.x * kMoeWarps) {
    if (dead) {
      if (grad_gates && lane < k) grad_gates[t * k + lane] = from_f<G>(0.f);
      continue;
    }
    const T* s = src + t * h;
    for (int j = 0; j < k; ++j) {
      const int p = pos[t * k + j];
      if (p < 0 || p >= dst_rows) {
        if (grad_gates && lane == 0) grad_gates[t * k + j] = from_f<G>(0.f);
        continue;
      }
      T* d = dst + (int64_t)p * h;
      if (!gates) {
        warp_copy_bytes(reinterpret_cast<const char*>(s), reinterpret_cast<char*>(d), h * (int64_t)sizeof(T), lane);
        continue;
      }
      const float g = to_f(gates[t * k + j]);
      const T* r = dot_rows ? dot_rows + (int64_t)p * h : nullptr;
      const bool vs = aligned16(s), vd = aligned16(d), vr = r && aligned16(r);
      float dot = 0.f;
      for (int64_t c0 = lane; c0 < nch; c0 += 32 * kMoeUnroll) {
        float f[kMoeUnroll][V];
#pragma unroll
        for (int u = 0; u < kMoeUnroll; ++u)
          if (c0 + 32 * u < nch) ld_chunk(s, c0 + 32 * u, h, vs, f[u]);
        if (r) {
#pragma unroll
          for (int u = 0; u < kMoeUnroll; ++u) {
            if (c0 + 32 * u < nch) {
              float v[V];
              ld_chunk(r, c0 + 32 * u, h, vr, v);
#pragma unroll
              for (int i = 0; i < V; ++i) dot = fmaf(f[u][i], v[i], dot);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < kMoeUnroll; ++u) {
          if (c0 + 32 * u < nch) {
#pragma unroll
            for (int i = 0; i < V; ++i) f[u][i] = __fmul_rn(g, f[u][i]);
            st_chunk(d, c0 + 32 * u, h, vd, f[u]);
          }
        }
      }
      if (r) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
        if (lane == 0) grad_gates[t * k + j] = from_f<G>(dot);
      }
    }
  }
}

// ---- gather ---------------------------------------------------------------------------------------------------------
// One warp per token t: y[t] = round(sum_j g_j * src[pos[t * k + j]]) with the sum in fp32, j ascending (g_j = 1 without
// gates: a plain sum).  Positions outside [0, src_rows) add nothing; a non-zero *status gives y = 0.
template <typename T, typename G>
__global__ void __launch_bounds__(kMoeThreads)
moe_gather_kernel(const T* __restrict__ src, int64_t src_rows, const int* __restrict__ pos, int k, int64_t ntok, int64_t h,
                  const G* __restrict__ gates, const int* __restrict__ status, T* __restrict__ y) {
  constexpr int V = 16 / sizeof(T);
  const int lane = threadIdx.x & 31;
  const int64_t nch = (h + V - 1) / V;
  const bool dead = status && *status != 0;
  for (int64_t t = (int64_t)blockIdx.x * kMoeWarps + (threadIdx.x >> 5); t < ntok; t += (int64_t)gridDim.x * kMoeWarps) {
    T* yr = y + t * h;
    const bool vy = aligned16(yr);
    for (int64_t c0 = lane; c0 < nch; c0 += 32 * kMoeUnroll) {
      float acc[kMoeUnroll][V];
#pragma unroll
      for (int u = 0; u < kMoeUnroll; ++u)
#pragma unroll
        for (int i = 0; i < V; ++i) acc[u][i] = dead ? 0.f : -0.f;  // -0 + x == x for every x: the sum starts at term 0
      if (!dead) {
        for (int j = 0; j < k; ++j) {
          const int p = pos[t * k + j];
          if (p < 0 || p >= src_rows) continue;
          const T* r = src + (int64_t)p * h;
          const bool vr = aligned16(r);
          const float g = gates ? to_f(gates[t * k + j]) : 1.f;
          float v[kMoeUnroll][V];
#pragma unroll
          for (int u = 0; u < kMoeUnroll; ++u)
            if (c0 + 32 * u < nch) ld_chunk(r, c0 + 32 * u, h, vr, v[u]);
#pragma unroll
          for (int u = 0; u < kMoeUnroll; ++u)
#pragma unroll
            for (int i = 0; i < V; ++i) acc[u][i] = __fadd_rn(acc[u][i], gates ? __fmul_rn(g, v[u][i]) : v[u][i]);
        }
      }
#pragma unroll
      for (int u = 0; u < kMoeUnroll; ++u)
        if (c0 + 32 * u < nch) st_chunk(yr, c0 + 32 * u, h, vy, acc[u]);
    }
  }
}

// ---- regroup --------------------------------------------------------------------------------------------------------
// counts[p * el + e]: rows rank p sent for local expert e.  Source-major order (what the alltoall delivers) is p, then e;
// expert-major order is e, then p; within a (p, e) segment the sender's order is kept.  Every CTA derives both segment
// starts from counts (all zero when *status is non-zero).  Forward: dst (expert-major, rows rows) row r = src row of r,
// zero past the total; offsets[e] = the end of group e.  Reverse: src (expert-major) rows below the total go to their
// source-major rows of dst; ret_splits[p] = the rows of rank p.  In place (src == dst) only when el == 1, where both
// orders are the same and nothing is copied.
__global__ void __launch_bounds__(kMoeThreads)
moe_regroup_kernel(const char* src, char* dst, int64_t row_bytes, int64_t rows, const int64_t* __restrict__ counts, int n,
                   int el, const int* __restrict__ status, int reverse, int* __restrict__ offsets, int* __restrict__ ret_splits) {
  __shared__ int64_t s_em[kMoeMaxExperts + 1];  // expert-major start of segment (e, p), at e * n + p; [S] = total
  __shared__ int64_t s_sm[kMoeMaxExperts];      // source-major start of segment (p, e), at e * n + p
  __shared__ int64_t s_warp[kMoeWarps];
  const int tid = threadIdx.x, lane = tid & 31, S = n * el;
  const bool dead = status && *status != 0;
  int64_t total = 0;
  for (int order = 0; order < 2; ++order) {
    // thread tid owns positions [4 tid, 4 tid + 4) of the order: source-major i = p * el + e, expert-major i = e * n + p
    int64_t c[4], sum = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int x = 4 * tid + i;
      int seg = 0;
      if (x < S) seg = order == 0 ? x : (x % n) * el + x / n;
      c[i] = x < S && !dead ? counts[seg] : 0;
      sum += c[i];
    }
    int64_t at = block_exclusive_scan(sum, s_warp, &total);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int x = 4 * tid + i;
      if (x < S) {
        if (order == 0) s_sm[(x % el) * n + x / el] = at;
        else s_em[x] = at;
      }
      at += c[i];
    }
  }
  if (tid == 0) s_em[S] = total;
  __syncthreads();
  if (blockIdx.x == 0) {
    if (!reverse && offsets)
      for (int e = tid; e < el; e += kMoeThreads) offsets[e] = (int)s_em[(e + 1) * n];
    if (reverse && ret_splits)
      for (int p = tid; p < n; p += kMoeThreads) ret_splits[p] = (int)((p + 1 < n ? s_sm[p + 1] : total) - s_sm[p]);
  }
  const bool identity = el == 1 && src == dst;
  const int64_t end = reverse ? (total < rows ? total : rows) : rows;
  for (int64_t r = (int64_t)blockIdx.x * kMoeWarps + (tid >> 5); r < end; r += (int64_t)gridDim.x * kMoeWarps) {
    const char* from = nullptr;
    char* to = nullptr;
    if (r < total) {
      int lo = 0, hi = S;  // the last segment whose start is <= r
      while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (s_em[mid] <= r) lo = mid; else hi = mid; }
      const int64_t q = s_sm[lo] + (r - s_em[lo]);
      if (q >= rows || identity) continue;
      from = reverse ? src + r * row_bytes : src + q * row_bytes;
      to = reverse ? dst + q * row_bytes : dst + r * row_bytes;
    } else {
      to = dst + r * row_bytes;  // forward only: the zero tail
    }
    warp_copy_bytes(from, to, row_bytes, lane);
  }
}

int MoeGrid(int64_t warps_of_work, int ctas) {
  const int64_t need = (warps_of_work + kMoeWarps - 1) / kMoeWarps;
  const int64_t cap = ctas > 0 ? ctas : 2048;
  return (int)(need < 1 ? 1 : (need < cap ? need : cap));
}

template <typename I>
cudaError_t LaunchRoute(const I* idx, int64_t A, int E, int n, int el, int* hist, unsigned* ticket, int64_t* counts,
                        int* splits, int* pos, cudaStream_t stream) {
  const int64_t tiles = MoeRouteTiles(A);
  int* bad = hist + tiles * E;
  moe_route_count_kernel<I><<<(unsigned)tiles, kMoeThreads, 0, stream>>>(idx, A, E, n, el, hist, bad, ticket, counts, splits);
  CountKernelLaunch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || A == 0) return e;
  moe_route_pos_kernel<I><<<(unsigned)tiles, kMoeThreads, 0, stream>>>(idx, A, E, hist, pos);
  CountKernelLaunch();
  return cudaGetLastError();
}

template <typename T, typename G>
void ScatterT(const MoeRows& a, cudaStream_t s) {
  moe_scatter_kernel<T, G><<<MoeGrid(a.ntok, a.ctas), kMoeThreads, 0, s>>>(
      (const T*)a.src, a.ntok, a.k, a.h, a.pos, (T*)a.dst, a.dst_rows, (const G*)a.gates, (const T*)a.dot_rows,
      (G*)a.grad_gates, a.status);
}
template <typename T, typename G>
void GatherT(const MoeRows& a, cudaStream_t s) {
  moe_gather_kernel<T, G><<<MoeGrid(a.ntok, a.ctas), kMoeThreads, 0, s>>>(
      (const T*)a.src, a.src_rows, a.pos, a.k, a.ntok, a.h, (const G*)a.gates, a.status, (T*)a.dst);
}

// calls F<T, G>(a, s) for the row dtype T and the gate dtype G (fp32 or T); false for another combination
template <template <typename, typename> class F, typename T>
bool ByGate(const MoeRows& a, cudaStream_t s) {
  if (a.gate_dtype == kDtF32) { F<T, float>()(a, s); return true; }
  if constexpr (std::is_same<T, __nv_bfloat16>::value) if (a.gate_dtype == kDtBf16) { F<T, T>()(a, s); return true; }
  if constexpr (std::is_same<T, __half>::value) if (a.gate_dtype == kDtF16) { F<T, T>()(a, s); return true; }
  return false;
}
template <template <typename, typename> class F>
bool ByDtype(const MoeRows& a, cudaStream_t s) {
  if (a.dtype == kDtF32) return ByGate<F, float>(a, s);
  if (a.dtype == kDtBf16) return ByGate<F, __nv_bfloat16>(a, s);
  if (a.dtype == kDtF16) return ByGate<F, __half>(a, s);
  return false;
}
template <typename T, typename G> struct ScatterF { void operator()(const MoeRows& a, cudaStream_t s) { ScatterT<T, G>(a, s); } };
template <typename T, typename G> struct GatherF { void operator()(const MoeRows& a, cudaStream_t s) { GatherT<T, G>(a, s); } };

}  // namespace

int64_t MoeRouteTiles(int64_t assignments) {
  const int64_t t = (assignments + kRouteTile - 1) / kRouteTile;
  return t < 1 ? 1 : t;
}

cudaError_t LaunchMoeRoute(const void* idx, bool idx_int64, int64_t assignments, int num_experts, int nranks, int* hist,
                           unsigned* ticket, int64_t* counts, int* splits, int* pos, cudaStream_t stream) {
  if (num_experts < 1 || num_experts > kMoeMaxExperts || nranks < 1 || num_experts % nranks != 0 || assignments < 0 ||
      MoeRouteTiles(assignments) > 0x7fffffff || !hist || !ticket || !counts || !splits || (assignments > 0 && (!idx || !pos)))
    return cudaErrorInvalidValue;
  const int el = num_experts / nranks;
  return idx_int64 ? LaunchRoute((const int64_t*)idx, assignments, num_experts, nranks, el, hist, ticket, counts, splits, pos, stream)
                   : LaunchRoute((const int32_t*)idx, assignments, num_experts, nranks, el, hist, ticket, counts, splits, pos, stream);
}

cudaError_t LaunchMoeScatter(const MoeRows& a, cudaStream_t stream) {
  if (a.ntok < 0 || a.k < 1 || a.k > kMoeMaxTopK || a.h < 1) return cudaErrorInvalidValue;
  if (a.ntok == 0) return cudaSuccess;  // (empty tensors may have no data pointer)
  if (a.dot_rows && (!a.gates || !a.grad_gates)) return cudaErrorInvalidValue;
  if (!a.gates) {  // the copy ignores the gate dtype
    MoeRows c = a;
    c.gate_dtype = kDtF32;
    if (!ByDtype<ScatterF>(c, stream)) return cudaErrorInvalidValue;
  } else if (!ByDtype<ScatterF>(a, stream)) {
    return cudaErrorInvalidValue;
  }
  CountKernelLaunch();
  return cudaGetLastError();
}

cudaError_t LaunchMoeGather(const MoeRows& a, cudaStream_t stream) {
  if (a.ntok < 0 || a.k < 1 || a.k > kMoeMaxTopK || a.h < 1) return cudaErrorInvalidValue;
  if (a.ntok == 0) return cudaSuccess;
  MoeRows c = a;
  if (!a.gates) c.gate_dtype = kDtF32;
  if (!ByDtype<GatherF>(c, stream)) return cudaErrorInvalidValue;
  CountKernelLaunch();
  return cudaGetLastError();
}

cudaError_t LaunchMoeRegroup(const void* src, void* dst, int64_t row_bytes, int64_t rows, const int64_t* counts, int nranks,
                             int experts_per_rank, const int* status, bool reverse, int* offsets, int* ret_splits, int ctas,
                             cudaStream_t stream) {
  if (row_bytes < 1 || rows < 0 || nranks < 1 || experts_per_rank < 1 || (int64_t)nranks * experts_per_rank > kMoeMaxExperts ||
      !counts || (src == dst && experts_per_rank != 1))
    return cudaErrorInvalidValue;
  moe_regroup_kernel<<<MoeGrid(rows, ctas), kMoeThreads, 0, stream>>>(
      (const char*)src, (char*)dst, row_bytes, rows, counts, nranks, experts_per_rank, status, reverse ? 1 : 0, offsets,
      ret_splits);
  CountKernelLaunch();
  return cudaGetLastError();
}

}  // namespace kern
}  // namespace hvd
