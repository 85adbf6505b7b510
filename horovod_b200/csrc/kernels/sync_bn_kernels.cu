// Batch normalization over the global batch of a process set (hvd.SyncBatchNorm) for sm_90a.
//
// An input with channels at dim 1 is read in one of two views, both in the caller's layout:
//   rows   [M, C], C innermost: channels_last / channels_last_3d, [N, C], and any input whose spatial size is 1;
//   planes [N, C, L]: contiguous NCHW / NCL / NCDHW.
// Per layer and step: bn_stats (this rank's count / mean / M2 per channel into its slot of the registered buffer), the
// captured allgather of the slots, bn_combine (rank-order merge, running stats), bn_elemt; backward: bn_backward_reduce
// (sum dy, sum dy * (x - mean) into the registered buffer), the captured allreduce, bn_backward_elemt.
//
// All arithmetic is fp32; partials of different CTAs are combined in fp64 by the last CTA of a channel tile (a ticket
// that it resets for the next launch, as in grad_shard_stats_kernel), always in the same order.  No atomic decides a
// result, so the same input gives the same bits on every call.  Statistics are Welford / Chan (count, mean, M2), never
// sum x and sum x^2, which cancel catastrophically when the mean is large compared with the spread.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include "p2p_kernels.h"
#include "sync_bn_kernels.h"

namespace hvd {
namespace kern {
namespace {

constexpr int kBnThreads = 256;
constexpr int kDtF32 = 7, kDtBf16 = 10, kDtF16 = 6;  // hvd::DataType codes

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

// one 16-byte vector of T: V consecutive elements
template <typename T> struct alignas(16) Pack { T v[16 / sizeof(T)]; };

__device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// `valid` (1..V) elements from p; a 16-byte load when `vec` (the caller checked the alignment) and the group is whole.
// Elements past `valid` read as 0.
template <typename T, int V> __device__ __forceinline__ void ld(const T* p, int valid, bool vec, float* o) {
  if (vec && valid == V) {
    const Pack<T> q = *reinterpret_cast<const Pack<T>*>(p);
#pragma unroll
    for (int k = 0; k < V; ++k) o[k] = to_f<T>(q.v[k]);
  } else {
#pragma unroll
    for (int k = 0; k < V; ++k) o[k] = k < valid ? to_f<T>(p[k]) : 0.f;
  }
}
template <typename T, int V> __device__ __forceinline__ void st(T* p, int valid, bool vec, const float* o) {
  if (vec && valid == V) {
    Pack<T> q;
#pragma unroll
    for (int k = 0; k < V; ++k) q.v[k] = from_f<T>(o[k]);
    *reinterpret_cast<Pack<T>*>(p) = q;
  } else {
#pragma unroll
    for (int k = 0; k < V; ++k) if (k < valid) p[k] = from_f<T>(o[k]);
  }
}

// weight / bias / running statistics / parameter gradients: fp32 or the input dtype, chosen at run time (read once per
// channel, so the switch costs nothing)
__device__ __forceinline__ float ld_any(const void* p, int dt, int64_t i) {
  if (dt == kDtBf16) return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]);
  if (dt == kDtF16) return __half2float(static_cast<const __half*>(p)[i]);
  return static_cast<const float*>(p)[i];
}
__device__ __forceinline__ void st_any(void* p, int dt, int64_t i, double v) {
  if (dt == kDtBf16) static_cast<__nv_bfloat16*>(p)[i] = __double2bfloat16(v);
  else if (dt == kDtF16) static_cast<__half*>(p)[i] = __double2half(v);
  else static_cast<float*>(p)[i] = (float)v;
}

// A CTA's statistics of one channel.
struct BnPart { double n; float mean, m2; };

// Chan's merge of (nb, mb, m2b) into (n, mean, m2)
__device__ __forceinline__ void chan(float& n, float& mean, float& m2, float nb, float mb, float m2b) {
  if (nb == 0.f) return;
  const float nab = n + nb, f = nb / nab, d = mb - mean;
  mean = fmaf(d, f, mean);
  m2 += m2b + d * d * n * f;
  n = nab;
}

// Every thread accumulates x - s_c, where the shift s_c is the channel's first element (x[0, c] / x[0, c, 0]): the
// fp32 running mean then stays small, so its rounding does not grow with the data's offset.
//
// The last CTA of a channel tile [t0, t0 + tc): combines the `splits` CTA partials of every channel in fp64 and writes
// the channel's {count, mean + s_c, M2} to slot[3c .. 3c+2] (the shift s_c = shift[c * shift_stride]).  g = kBnThreads / tc threads share a channel, each taking a fixed
// strided subset, then a fixed tree.  The partials are merged as shifted sums about the first partial's mean K:
// N = sum n_j, S1 = sum n_j (m_j - K), S2 = sum (M2_j + n_j (m_j - K)^2), then mean = K + S1 / N and
// M2 = S2 - S1^2 / N -- Chan's formula applied to all partials at once, without a division per step.
template <typename T>
__device__ void finalize_stats(const BnPart* part, int64_t C, int64_t t0, int tc, unsigned splits, double* slot,
                               const T* shift, int64_t shift_stride, double (*red)[kBnThreads]) {
  const int g = kBnThreads / tc, ch = threadIdx.x / g, sub = threadIdx.x % g;
  const int64_t c = t0 + ch;
  double n = 0.0, s1 = 0.0, s2 = 0.0, K = 0.0;
  if (c < C) {
    K = (double)__ldcg(&part[c].mean);
    for (unsigned j = sub; j < splits; j += g) {
      const BnPart* p = part + (int64_t)j * C + c;
      const double nj = __ldcg(&p->n), d = (double)__ldcg(&p->mean) - K;
      n += nj;
      s1 = fma(nj, d, s1);
      s2 += (double)__ldcg(&p->m2) + nj * d * d;
    }
  }
  red[0][threadIdx.x] = n; red[1][threadIdx.x] = s1; red[2][threadIdx.x] = s2;
  __syncthreads();
  for (int h = g / 2; h > 0; h >>= 1) {
    if (sub < h) {
      red[0][threadIdx.x] += red[0][threadIdx.x + h];
      red[1][threadIdx.x] += red[1][threadIdx.x + h];
      red[2][threadIdx.x] += red[2][threadIdx.x + h];
    }
    __syncthreads();
  }
  if (sub == 0 && c < C) {
    n = red[0][threadIdx.x]; s1 = red[1][threadIdx.x]; s2 = red[2][threadIdx.x];
    slot[3 * c] = n;
    slot[3 * c + 1] = n > 0.0 ? (double)to_f<T>(shift[c * shift_stride]) + (K + s1 / n) : 0.0;
    slot[3 * c + 2] = n > 0.0 ? fmax(s2 - s1 * s1 / n, 0.0) : 0.0;
  }
}

// The last CTA of a channel tile: sums the `splits` (sum dy, sum dy * (x - mean)) partials of every channel in fp64 in a
// fixed order; writes them to sums[2c], sums[2c+1] and the local parameter gradients.
__device__ void finalize_sums(const float2* part, int64_t C, int64_t t0, int tc, unsigned splits, const float* invstd,
                              double* sums, void* grad_w, void* grad_b, int wdt, double (*red)[kBnThreads]) {
  const int g = kBnThreads / tc, ch = threadIdx.x / g, sub = threadIdx.x % g;
  const int64_t c = t0 + ch;
  double a = 0.0, b = 0.0;
  if (c < C) {
    for (unsigned j = sub; j < splits; j += g) {
      const float2* p = part + (int64_t)j * C + c;
      a += (double)__ldcg(&p->x);
      b += (double)__ldcg(&p->y);
    }
  }
  red[0][threadIdx.x] = a; red[1][threadIdx.x] = b;
  __syncthreads();
  for (int h = g / 2; h > 0; h >>= 1) {
    if (sub < h) {
      red[0][threadIdx.x] += red[0][threadIdx.x + h];
      red[1][threadIdx.x] += red[1][threadIdx.x + h];
    }
    __syncthreads();
  }
  if (sub == 0 && c < C) {
    a = red[0][threadIdx.x]; b = red[1][threadIdx.x];
    sums[2 * c] = a;
    sums[2 * c + 1] = b;
    if (grad_b) st_any(grad_b, wdt, c, a);
    if (grad_w) st_any(grad_w, wdt, c, b * (double)invstd[c]);
  }
}

// Rows view: a thread owns V consecutive channels (one 16-byte vector) of column `col` and walks rows; `cols` threads
// cover a tile of cols * V channels, kBnThreads / cols lanes split its rows.
struct RowsIdx {
  int lane, lanes, valid;
  int64_t c0;
};
template <int V> __device__ __forceinline__ RowsIdx rows_idx(int64_t C, int cols) {
  RowsIdx r;
  r.lane = threadIdx.x / cols;
  r.lanes = kBnThreads / cols;
  r.c0 = ((int64_t)blockIdx.x * cols + threadIdx.x % cols) * V;
  r.valid = r.c0 < C ? (int)min((int64_t)V, C - r.c0) : 0;
  return r;
}

template <typename T>
__global__ void __launch_bounds__(kBnThreads)
bn_stats_rows_kernel(const T* __restrict__ x, int64_t M, int64_t C, int cols, BnPart* __restrict__ part,
                     unsigned* __restrict__ tickets, double* __restrict__ slot) {
  constexpr int V = 16 / sizeof(T);
  __shared__ float s_n[kBnThreads];
  __shared__ float s_mean[V][kBnThreads];
  __shared__ float s_m2[V][kBnThreads];
  __shared__ double red[3][kBnThreads];
  __shared__ bool last;
  const RowsIdx r = rows_idx<V>(C, cols);
  const int tid = threadIdx.x;
  const bool vec = aligned16(x) && C % V == 0;
  float n = 0.f, mean[V], m2[V], sh[V];
#pragma unroll
  for (int k = 0; k < V; ++k) mean[k] = m2[k] = 0.f;
  if (r.valid > 0 && M > 0) {
    ld<T, V>(x + r.c0, r.valid, false, sh);
    for (int64_t m = (int64_t)blockIdx.y * r.lanes + r.lane; m < M; m += (int64_t)gridDim.y * r.lanes) {
      float v[V];
      ld<T, V>(x + m * C + r.c0, r.valid, vec, v);
#pragma unroll
      for (int k = 0; k < V; ++k) v[k] -= sh[k];
      n += 1.f;
      const float inv = 1.f / n;  // one division per row, shared by the thread's V channels
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const float d = v[k] - mean[k];
        mean[k] = fmaf(d, inv, mean[k]);
        m2[k] = fmaf(d, v[k] - mean[k], m2[k]);
      }
    }
  }
  s_n[tid] = n;
#pragma unroll
  for (int k = 0; k < V; ++k) { s_mean[k][tid] = mean[k]; s_m2[k][tid] = m2[k]; }
  __syncthreads();
  for (int h = r.lanes / 2; h > 0; h >>= 1) {  // fixed tree over the lanes of each column
    if (r.lane < h) {
      const int o = tid + h * cols;
      const float na = s_n[tid];
#pragma unroll
      for (int k = 0; k < V; ++k) {
        float nk = na, mk = s_mean[k][tid], qk = s_m2[k][tid];
        chan(nk, mk, qk, s_n[o], s_mean[k][o], s_m2[k][o]);
        s_mean[k][tid] = mk; s_m2[k][tid] = qk;
      }
      s_n[tid] = na + s_n[o];
    }
    __syncthreads();
  }
  if (r.lane == 0) {
#pragma unroll
    for (int k = 0; k < V; ++k)
      if (k < r.valid) part[(int64_t)blockIdx.y * C + r.c0 + k] = BnPart{(double)s_n[tid], s_mean[k][tid], s_m2[k][tid]};
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) last = atomicAdd(tickets + blockIdx.x, 1u) == gridDim.y - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  finalize_stats<T>(part, C, (int64_t)blockIdx.x * cols * V, cols * V, gridDim.y, slot, x, 1, red);
  if (tid == 0) tickets[blockIdx.x] = 0u;  // ready for the next launch on this stream
}

// Planes view: CTA (c, y) takes chunks y, y + gridDim.y, ... of the N * ceil(L / chunk) chunks of channel c.
template <typename T>
__global__ void __launch_bounds__(kBnThreads)
bn_stats_planes_kernel(const T* __restrict__ x, int64_t N, int64_t C, int64_t L, BnPart* __restrict__ part,
                       unsigned* __restrict__ tickets, double* __restrict__ slot) {
  constexpr int V = 16 / sizeof(T);
  constexpr int64_t kChunk = (int64_t)kBnThreads * V;
  __shared__ float s_n[kBnThreads], s_mean[kBnThreads], s_m2[kBnThreads];
  __shared__ double red[3][kBnThreads];
  __shared__ bool last;
  const int tid = threadIdx.x;
  const int64_t c = blockIdx.x, cpp = (L + kChunk - 1) / kChunk, Q = N * cpp;
  const bool vec = aligned16(x) && L % V == 0;
  float n = 0.f, mean = 0.f, m2 = 0.f;
  const float sh = Q > 0 ? to_f<T>(x[c * L]) : 0.f;
  for (int64_t q = blockIdx.y; q < Q; q += gridDim.y) {
    const int64_t pn = q / cpp, l = (q % cpp) * kChunk + (int64_t)tid * V;
    if (l >= L) continue;
    const int valid = (int)min((int64_t)V, L - l);
    float v[V];
    ld<T, V>(x + (pn * C + c) * L + l, valid, vec, v);
    // the vector's own mean and M2, then one Chan merge (one division per vector)
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < V; ++k) { v[k] = k < valid ? v[k] - sh : 0.f; s += v[k]; }
    const float nb = (float)valid, mb = s / nb;
    float qb = 0.f;
#pragma unroll
    for (int k = 0; k < V; ++k) if (k < valid) { const float d = v[k] - mb; qb = fmaf(d, d, qb); }
    chan(n, mean, m2, nb, mb, qb);
  }
  s_n[tid] = n; s_mean[tid] = mean; s_m2[tid] = m2;
  __syncthreads();
  for (int h = kBnThreads / 2; h > 0; h >>= 1) {
    if (tid < h) {
      float na = s_n[tid], ma = s_mean[tid], qa = s_m2[tid];
      chan(na, ma, qa, s_n[tid + h], s_mean[tid + h], s_m2[tid + h]);
      s_n[tid] = na; s_mean[tid] = ma; s_m2[tid] = qa;
    }
    __syncthreads();
  }
  if (tid == 0) {
    part[(int64_t)blockIdx.y * C + c] = BnPart{(double)s_n[0], s_mean[0], s_m2[0]};
    __threadfence();
    last = atomicAdd(tickets + c, 1u) == gridDim.y - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  finalize_stats<T>(part, C, c, 1, gridDim.y, slot, x, L, red);
  if (tid == 0) tickets[c] = 0u;
}

// Merges the nranks slots of every channel in rank order 0 .. N-1 in fp64 (Chan), so every rank computes the same bits.
__global__ void __launch_bounds__(kBnThreads)
bn_combine_kernel(const double* __restrict__ slots, int nranks, int64_t stride, int64_t C, double eps, double momentum,
                  const int64_t* __restrict__ nbt, float* __restrict__ mean_out, float* __restrict__ invstd_out,
                  float* __restrict__ count_out, void* rm, void* rv, int sdt) {
  const int64_t c = (int64_t)blockIdx.x * kBnThreads + threadIdx.x;
  if (c >= C) return;
  // reciprocals (__drcp_rn) instead of divisions: the division's slow path is a call that spills
  double n = 0.0, mean = 0.0, m2 = 0.0;
  for (int r = 0; r < nranks; ++r) {
    const double* s = slots + r * stride + 3 * c;
    const double nb = s[0];
    if (nb == 0.0) continue;
    const double nab = n + nb, f = nb * __drcp_rn(nab), d = s[1] - mean;
    mean = fma(d, f, mean);
    m2 += s[2] + d * d * n * f;
    n = nab;
  }
  const double var = m2 * __drcp_rn(n);
  mean_out[c] = (float)mean;
  invstd_out[c] = (float)rsqrt(var + eps);
  if (c == 0) *count_out = (float)n;
  if (rm) {
    // torch's update; momentum=None is the cumulative average 1 / num_batches_tracked, read here so the host never waits
    const double f = nbt ? __drcp_rn((double)*nbt) : momentum;
    const double unbiased = n > 1.0 ? m2 * __drcp_rn(n - 1.0) : var;
    st_any(rm, sdt, c, (1.0 - f) * (double)ld_any(rm, sdt, c) + f * mean);
    st_any(rv, sdt, c, (1.0 - f) * (double)ld_any(rv, sdt, c) + f * unbiased);
  }
}

// y = (x - mean) * invstd * w + b
template <typename T>
__global__ void __launch_bounds__(kBnThreads)
bn_elemt_rows_kernel(const T* __restrict__ x, T* __restrict__ y, int64_t M, int64_t C, int cols,
                     const float* __restrict__ mean, const float* __restrict__ invstd, const void* w, const void* b,
                     int wdt) {
  constexpr int V = 16 / sizeof(T);
  const RowsIdx r = rows_idx<V>(C, cols);
  if (r.valid == 0) return;
  const bool vx = aligned16(x) && C % V == 0, vy = aligned16(y) && C % V == 0;
  float mu[V], a[V], sh[V];
#pragma unroll
  for (int k = 0; k < V; ++k) {
    const int64_t c = r.c0 + (k < r.valid ? k : 0);
    mu[k] = mean[c];
    a[k] = invstd[c] * (w ? ld_any(w, wdt, c) : 1.f);
    sh[k] = b ? ld_any(b, wdt, c) : 0.f;
  }
  for (int64_t m = (int64_t)blockIdx.y * r.lanes + r.lane; m < M; m += (int64_t)gridDim.y * r.lanes) {
    float v[V];
    ld<T, V>(x + m * C + r.c0, r.valid, vx, v);
#pragma unroll
    for (int k = 0; k < V; ++k) v[k] = fmaf(v[k] - mu[k], a[k], sh[k]);
    st<T, V>(y + m * C + r.c0, r.valid, vy, v);
  }
}

template <typename T>
__global__ void __launch_bounds__(kBnThreads)
bn_elemt_planes_kernel(const T* __restrict__ x, T* __restrict__ y, int64_t N, int64_t C, int64_t L,
                       const float* __restrict__ mean, const float* __restrict__ invstd, const void* w, const void* b,
                       int wdt) {
  constexpr int V = 16 / sizeof(T);
  const bool vx = aligned16(x) && L % V == 0, vy = aligned16(y) && L % V == 0;
  for (int64_t p = blockIdx.y; p < N * C; p += gridDim.y) {
    const int64_t c = p % C;
    const float mu = mean[c], a = invstd[c] * (w ? ld_any(w, wdt, c) : 1.f), sh = b ? ld_any(b, wdt, c) : 0.f;
    for (int64_t l = ((int64_t)blockIdx.x * kBnThreads + threadIdx.x) * V; l < L; l += (int64_t)gridDim.x * kBnThreads * V) {
      const int valid = (int)min((int64_t)V, L - l);
      float v[V];
      ld<T, V>(x + p * L + l, valid, vx, v);
#pragma unroll
      for (int k = 0; k < V; ++k) v[k] = fmaf(v[k] - mu, a, sh);
      st<T, V>(y + p * L + l, valid, vy, v);
    }
  }
}

// sum dy and sum dy * (x - mean) per channel
template <typename T>
__global__ void __launch_bounds__(kBnThreads)
bn_backward_reduce_rows_kernel(const T* __restrict__ dy, const T* __restrict__ x, int64_t M, int64_t C, int cols,
                               const float* __restrict__ mean, const float* __restrict__ invstd,
                               float2* __restrict__ part, unsigned* __restrict__ tickets, double* __restrict__ sums,
                               void* grad_w, void* grad_b, int wdt) {
  constexpr int V = 16 / sizeof(T);
  __shared__ float s_a[V][kBnThreads];
  __shared__ float s_b[V][kBnThreads];
  __shared__ double red[3][kBnThreads];
  __shared__ bool last;
  const RowsIdx r = rows_idx<V>(C, cols);
  const int tid = threadIdx.x;
  const bool vd = aligned16(dy) && C % V == 0, vx = aligned16(x) && C % V == 0;
  float mu[V], a[V], bb[V];
#pragma unroll
  for (int k = 0; k < V; ++k) { a[k] = bb[k] = 0.f; mu[k] = r.valid > 0 ? mean[r.c0 + (k < r.valid ? k : 0)] : 0.f; }
  if (r.valid > 0) {
    for (int64_t m = (int64_t)blockIdx.y * r.lanes + r.lane; m < M; m += (int64_t)gridDim.y * r.lanes) {
      float g[V], v[V];
      ld<T, V>(dy + m * C + r.c0, r.valid, vd, g);
      ld<T, V>(x + m * C + r.c0, r.valid, vx, v);
#pragma unroll
      for (int k = 0; k < V; ++k) { a[k] += g[k]; bb[k] = fmaf(g[k], v[k] - mu[k], bb[k]); }
    }
  }
#pragma unroll
  for (int k = 0; k < V; ++k) { s_a[k][tid] = a[k]; s_b[k][tid] = bb[k]; }
  __syncthreads();
  for (int h = r.lanes / 2; h > 0; h >>= 1) {
    if (r.lane < h) {
#pragma unroll
      for (int k = 0; k < V; ++k) { s_a[k][tid] += s_a[k][tid + h * cols]; s_b[k][tid] += s_b[k][tid + h * cols]; }
    }
    __syncthreads();
  }
  if (r.lane == 0) {
#pragma unroll
    for (int k = 0; k < V; ++k)
      if (k < r.valid) part[(int64_t)blockIdx.y * C + r.c0 + k] = make_float2(s_a[k][tid], s_b[k][tid]);
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) last = atomicAdd(tickets + blockIdx.x, 1u) == gridDim.y - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  finalize_sums(part, C, (int64_t)blockIdx.x * cols * V, cols * V, gridDim.y, invstd, sums, grad_w, grad_b, wdt, red);
  if (tid == 0) tickets[blockIdx.x] = 0u;
}

template <typename T>
__global__ void __launch_bounds__(kBnThreads)
bn_backward_reduce_planes_kernel(const T* __restrict__ dy, const T* __restrict__ x, int64_t N, int64_t C, int64_t L,
                                 const float* __restrict__ mean, const float* __restrict__ invstd,
                                 float2* __restrict__ part, unsigned* __restrict__ tickets, double* __restrict__ sums,
                                 void* grad_w, void* grad_b, int wdt) {
  constexpr int V = 16 / sizeof(T);
  constexpr int64_t kChunk = (int64_t)kBnThreads * V;
  __shared__ float s_a[kBnThreads], s_b[kBnThreads];
  __shared__ double red[3][kBnThreads];
  __shared__ bool last;
  const int tid = threadIdx.x;
  const int64_t c = blockIdx.x, cpp = (L + kChunk - 1) / kChunk, Q = N * cpp;
  const bool vd = aligned16(dy) && L % V == 0, vx = aligned16(x) && L % V == 0;
  const float mu = mean[c];
  float a = 0.f, bb = 0.f;
  for (int64_t q = blockIdx.y; q < Q; q += gridDim.y) {
    const int64_t pn = q / cpp, l = (q % cpp) * kChunk + (int64_t)tid * V;
    if (l >= L) continue;
    const int valid = (int)min((int64_t)V, L - l);
    float g[V], v[V];
    ld<T, V>(dy + (pn * C + c) * L + l, valid, vd, g);
    ld<T, V>(x + (pn * C + c) * L + l, valid, vx, v);
#pragma unroll
    for (int k = 0; k < V; ++k) { a += g[k]; bb = fmaf(g[k], k < valid ? v[k] - mu : 0.f, bb); }
  }
  s_a[tid] = a; s_b[tid] = bb;
  __syncthreads();
  for (int h = kBnThreads / 2; h > 0; h >>= 1) {
    if (tid < h) { s_a[tid] += s_a[tid + h]; s_b[tid] += s_b[tid + h]; }
    __syncthreads();
  }
  if (tid == 0) {
    part[(int64_t)blockIdx.y * C + c] = make_float2(s_a[0], s_b[0]);
    __threadfence();
    last = atomicAdd(tickets + c, 1u) == gridDim.y - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  finalize_sums(part, C, c, 1, gridDim.y, invstd, sums, grad_w, grad_b, wdt, red);
  if (tid == 0) tickets[c] = 0u;
}

// dx = (dy - sum_dy / n - (x - mean) * invstd^2 * sum_dy_xmu / n) * invstd * w, with the sums over every rank
struct BwdCoef { float mu, mdy, k, s; };
__device__ __forceinline__ BwdCoef bwd_coef(int64_t c, const float* mean, const float* invstd, const void* w, int wdt,
                                            const double* sums, float n) {
  const float is = invstd[c];
  return BwdCoef{mean[c], (float)sums[2 * c] / n, (float)sums[2 * c + 1] / n * is * is,
                 is * (w ? ld_any(w, wdt, c) : 1.f)};
}

template <typename T>
__global__ void __launch_bounds__(kBnThreads)
bn_backward_elemt_rows_kernel(const T* __restrict__ dy, const T* __restrict__ x, T* __restrict__ dx, int64_t M,
                              int64_t C, int cols, const float* __restrict__ mean, const float* __restrict__ invstd,
                              const void* w, int wdt, const double* __restrict__ sums, const float* __restrict__ count) {
  constexpr int V = 16 / sizeof(T);
  const RowsIdx r = rows_idx<V>(C, cols);
  if (r.valid == 0) return;
  const bool vd = aligned16(dy) && C % V == 0, vx = aligned16(x) && C % V == 0, vo = aligned16(dx) && C % V == 0;
  const float n = *count;
  BwdCoef cf[V];
#pragma unroll
  for (int k = 0; k < V; ++k) cf[k] = bwd_coef(r.c0 + (k < r.valid ? k : 0), mean, invstd, w, wdt, sums, n);
  for (int64_t m = (int64_t)blockIdx.y * r.lanes + r.lane; m < M; m += (int64_t)gridDim.y * r.lanes) {
    float g[V], v[V];
    ld<T, V>(dy + m * C + r.c0, r.valid, vd, g);
    ld<T, V>(x + m * C + r.c0, r.valid, vx, v);
#pragma unroll
    for (int k = 0; k < V; ++k) g[k] = (g[k] - cf[k].mdy - (v[k] - cf[k].mu) * cf[k].k) * cf[k].s;
    st<T, V>(dx + m * C + r.c0, r.valid, vo, g);
  }
}

template <typename T>
__global__ void __launch_bounds__(kBnThreads)
bn_backward_elemt_planes_kernel(const T* __restrict__ dy, const T* __restrict__ x, T* __restrict__ dx, int64_t N,
                                int64_t C, int64_t L, const float* __restrict__ mean, const float* __restrict__ invstd,
                                const void* w, int wdt, const double* __restrict__ sums, const float* __restrict__ count) {
  constexpr int V = 16 / sizeof(T);
  const bool vd = aligned16(dy) && L % V == 0, vx = aligned16(x) && L % V == 0, vo = aligned16(dx) && L % V == 0;
  const float n = *count;
  for (int64_t p = blockIdx.y; p < N * C; p += gridDim.y) {
    const BwdCoef cf = bwd_coef(p % C, mean, invstd, w, wdt, sums, n);
    for (int64_t l = ((int64_t)blockIdx.x * kBnThreads + threadIdx.x) * V; l < L; l += (int64_t)gridDim.x * kBnThreads * V) {
      const int valid = (int)min((int64_t)V, L - l);
      float g[V], v[V];
      ld<T, V>(dy + p * L + l, valid, vd, g);
      ld<T, V>(x + p * L + l, valid, vx, v);
#pragma unroll
      for (int k = 0; k < V; ++k) g[k] = (g[k] - cf.mdy - (v[k] - cf.mu) * cf.k) * cf.s;
      st<T, V>(dx + p * L + l, valid, vo, g);
    }
  }
}

int VecOf(int dtype) { return dtype == kDtF32 ? 4 : 8; }

int NumSms() {
  static const int sms = [] {
    int d = 0, v = 132;
    if (cudaGetDevice(&d) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d) != cudaSuccess) v = 132;
    return v;
  }();
  return sms;
}

int RowsCols(int64_t C, int dtype) {
  const int64_t vecs = (C + VecOf(dtype) - 1) / VecOf(dtype);
  int cols = 1;
  while (cols < 32 && cols < vecs) cols *= 2;
  return cols;
}

// grid of the element-wise kernels
dim3 ElemtGrid(const BnGeom& g, int dtype, int* cols) {
  const int V = VecOf(dtype);
  if (g.layout == kBnRows) {
    *cols = RowsCols(g.C, dtype);
    const int64_t tile = (int64_t)*cols * V, lanes = kBnThreads / *cols;
    const int64_t splits = std::min<int64_t>(65535, std::max<int64_t>(1, (g.M + lanes * 8 - 1) / (lanes * 8)));
    return dim3((unsigned)((g.C + tile - 1) / tile), (unsigned)splits);
  }
  *cols = 0;
  const int64_t chunk = (int64_t)kBnThreads * V;
  return dim3((unsigned)std::min<int64_t>(65535, std::max<int64_t>(1, (g.L + chunk - 1) / chunk)),
              (unsigned)std::min<int64_t>(65535, std::max<int64_t>(1, g.M * g.C)));
}

}  // namespace

BnPlan BnReducePlan(const BnGeom& g, int dtype) {
  const int V = VecOf(dtype);
  const int64_t target = 2 * (int64_t)NumSms();  // CTAs in flight; more would only lengthen the last CTA's merge
  BnPlan p {};
  if (g.layout == kBnRows) {
    p.cols = RowsCols(g.C, dtype);
    const int64_t tile = (int64_t)p.cols * V, lanes = kBnThreads / p.cols;
    p.tiles = (g.C + tile - 1) / tile;
    const int64_t want = (target + p.tiles - 1) / p.tiles, rows = (g.M + lanes * 8 - 1) / (lanes * 8);
    p.splits = std::max<int64_t>(1, std::min(want, rows));
  } else {
    p.cols = 0;
    p.tiles = g.C;
    const int64_t chunk = (int64_t)kBnThreads * V, q = g.M * ((g.L + chunk - 1) / chunk);
    p.splits = std::max<int64_t>(1, std::min((target + g.C - 1) / g.C, q));
  }
  p.splits = std::min<int64_t>(p.splits, 65535);
  return p;
}

cudaError_t LaunchBnStats(const void* x, const BnGeom& g, int dtype, void* partial, unsigned* tickets, double* slot,
                          cudaStream_t stream) {
  const BnPlan p = BnReducePlan(g, dtype);
  dim3 grid((unsigned)p.tiles, (unsigned)p.splits);
  if (p.tiles <= 0) return cudaSuccess;
  BnPart* part = static_cast<BnPart*>(partial);
  if (g.layout == kBnRows) {
    if (dtype == kDtF32) bn_stats_rows_kernel<float><<<grid, kBnThreads, 0, stream>>>((const float*)x, g.M, g.C, p.cols, part, tickets, slot);
    else if (dtype == kDtBf16) bn_stats_rows_kernel<__nv_bfloat16><<<grid, kBnThreads, 0, stream>>>((const __nv_bfloat16*)x, g.M, g.C, p.cols, part, tickets, slot);
    else if (dtype == kDtF16) bn_stats_rows_kernel<__half><<<grid, kBnThreads, 0, stream>>>((const __half*)x, g.M, g.C, p.cols, part, tickets, slot);
    else return cudaErrorInvalidValue;
  } else {
    if (dtype == kDtF32) bn_stats_planes_kernel<float><<<grid, kBnThreads, 0, stream>>>((const float*)x, g.M, g.C, g.L, part, tickets, slot);
    else if (dtype == kDtBf16) bn_stats_planes_kernel<__nv_bfloat16><<<grid, kBnThreads, 0, stream>>>((const __nv_bfloat16*)x, g.M, g.C, g.L, part, tickets, slot);
    else if (dtype == kDtF16) bn_stats_planes_kernel<__half><<<grid, kBnThreads, 0, stream>>>((const __half*)x, g.M, g.C, g.L, part, tickets, slot);
    else return cudaErrorInvalidValue;
  }
  CountKernelLaunch();
  return cudaGetLastError();
}

cudaError_t LaunchBnCombine(const double* slots, int nranks, int64_t slot_stride, int64_t C, double eps, double momentum,
                            const int64_t* num_batches_tracked, float* mean, float* invstd, float* count, void* running_mean,
                            void* running_var, int stat_dtype, cudaStream_t stream) {
  if (C <= 0) return cudaSuccess;
  bn_combine_kernel<<<(unsigned)((C + kBnThreads - 1) / kBnThreads), kBnThreads, 0, stream>>>(
      slots, nranks, slot_stride, C, eps, momentum, num_batches_tracked, mean, invstd, count, running_mean, running_var,
      stat_dtype);
  CountKernelLaunch();
  return cudaGetLastError();
}

cudaError_t LaunchBnElemt(const void* x, void* y, const BnGeom& g, int dtype, const float* mean, const float* invstd,
                          const void* weight, const void* bias, int wdtype, cudaStream_t stream) {
  if (g.M * g.C * g.L == 0) return cudaSuccess;
  int cols = 0;
  const dim3 grid = ElemtGrid(g, dtype, &cols);
  if (g.layout == kBnRows) {
    if (dtype == kDtF32) bn_elemt_rows_kernel<float><<<grid, kBnThreads, 0, stream>>>((const float*)x, (float*)y, g.M, g.C, cols, mean, invstd, weight, bias, wdtype);
    else if (dtype == kDtBf16) bn_elemt_rows_kernel<__nv_bfloat16><<<grid, kBnThreads, 0, stream>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, g.M, g.C, cols, mean, invstd, weight, bias, wdtype);
    else if (dtype == kDtF16) bn_elemt_rows_kernel<__half><<<grid, kBnThreads, 0, stream>>>((const __half*)x, (__half*)y, g.M, g.C, cols, mean, invstd, weight, bias, wdtype);
    else return cudaErrorInvalidValue;
  } else {
    if (dtype == kDtF32) bn_elemt_planes_kernel<float><<<grid, kBnThreads, 0, stream>>>((const float*)x, (float*)y, g.M, g.C, g.L, mean, invstd, weight, bias, wdtype);
    else if (dtype == kDtBf16) bn_elemt_planes_kernel<__nv_bfloat16><<<grid, kBnThreads, 0, stream>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, g.M, g.C, g.L, mean, invstd, weight, bias, wdtype);
    else if (dtype == kDtF16) bn_elemt_planes_kernel<__half><<<grid, kBnThreads, 0, stream>>>((const __half*)x, (__half*)y, g.M, g.C, g.L, mean, invstd, weight, bias, wdtype);
    else return cudaErrorInvalidValue;
  }
  CountKernelLaunch();
  return cudaGetLastError();
}

cudaError_t LaunchBnBackwardReduce(const void* dy, const void* x, const BnGeom& g, int dtype, const float* mean,
                                   const float* invstd, void* partial, unsigned* tickets, double* sums, void* grad_weight,
                                   void* grad_bias, int wdtype, cudaStream_t stream) {
  const BnPlan p = BnReducePlan(g, dtype);
  if (p.tiles <= 0) return cudaSuccess;
  dim3 grid((unsigned)p.tiles, (unsigned)p.splits);
  float2* part = static_cast<float2*>(partial);
  if (g.layout == kBnRows) {
    if (dtype == kDtF32) bn_backward_reduce_rows_kernel<float><<<grid, kBnThreads, 0, stream>>>((const float*)dy, (const float*)x, g.M, g.C, p.cols, mean, invstd, part, tickets, sums, grad_weight, grad_bias, wdtype);
    else if (dtype == kDtBf16) bn_backward_reduce_rows_kernel<__nv_bfloat16><<<grid, kBnThreads, 0, stream>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, g.M, g.C, p.cols, mean, invstd, part, tickets, sums, grad_weight, grad_bias, wdtype);
    else if (dtype == kDtF16) bn_backward_reduce_rows_kernel<__half><<<grid, kBnThreads, 0, stream>>>((const __half*)dy, (const __half*)x, g.M, g.C, p.cols, mean, invstd, part, tickets, sums, grad_weight, grad_bias, wdtype);
    else return cudaErrorInvalidValue;
  } else {
    if (dtype == kDtF32) bn_backward_reduce_planes_kernel<float><<<grid, kBnThreads, 0, stream>>>((const float*)dy, (const float*)x, g.M, g.C, g.L, mean, invstd, part, tickets, sums, grad_weight, grad_bias, wdtype);
    else if (dtype == kDtBf16) bn_backward_reduce_planes_kernel<__nv_bfloat16><<<grid, kBnThreads, 0, stream>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, g.M, g.C, g.L, mean, invstd, part, tickets, sums, grad_weight, grad_bias, wdtype);
    else if (dtype == kDtF16) bn_backward_reduce_planes_kernel<__half><<<grid, kBnThreads, 0, stream>>>((const __half*)dy, (const __half*)x, g.M, g.C, g.L, mean, invstd, part, tickets, sums, grad_weight, grad_bias, wdtype);
    else return cudaErrorInvalidValue;
  }
  CountKernelLaunch();
  return cudaGetLastError();
}

cudaError_t LaunchBnBackwardElemt(const void* dy, const void* x, void* dx, const BnGeom& g, int dtype, const float* mean,
                                  const float* invstd, const void* weight, int wdtype, const double* sums,
                                  const float* count, cudaStream_t stream) {
  if (g.M * g.C * g.L == 0) return cudaSuccess;
  int cols = 0;
  const dim3 grid = ElemtGrid(g, dtype, &cols);
  if (g.layout == kBnRows) {
    if (dtype == kDtF32) bn_backward_elemt_rows_kernel<float><<<grid, kBnThreads, 0, stream>>>((const float*)dy, (const float*)x, (float*)dx, g.M, g.C, cols, mean, invstd, weight, wdtype, sums, count);
    else if (dtype == kDtBf16) bn_backward_elemt_rows_kernel<__nv_bfloat16><<<grid, kBnThreads, 0, stream>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, (__nv_bfloat16*)dx, g.M, g.C, cols, mean, invstd, weight, wdtype, sums, count);
    else if (dtype == kDtF16) bn_backward_elemt_rows_kernel<__half><<<grid, kBnThreads, 0, stream>>>((const __half*)dy, (const __half*)x, (__half*)dx, g.M, g.C, cols, mean, invstd, weight, wdtype, sums, count);
    else return cudaErrorInvalidValue;
  } else {
    if (dtype == kDtF32) bn_backward_elemt_planes_kernel<float><<<grid, kBnThreads, 0, stream>>>((const float*)dy, (const float*)x, (float*)dx, g.M, g.C, g.L, mean, invstd, weight, wdtype, sums, count);
    else if (dtype == kDtBf16) bn_backward_elemt_planes_kernel<__nv_bfloat16><<<grid, kBnThreads, 0, stream>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, (__nv_bfloat16*)dx, g.M, g.C, g.L, mean, invstd, weight, wdtype, sums, count);
    else if (dtype == kDtF16) bn_backward_elemt_planes_kernel<__half><<<grid, kBnThreads, 0, stream>>>((const __half*)dy, (const __half*)x, (__half*)dx, g.M, g.C, g.L, mean, invstd, weight, wdtype, sums, count);
    else return cudaErrorInvalidValue;
  }
  CountKernelLaunch();
  return cudaGetLastError();
}

}  // namespace kern
}  // namespace hvd
