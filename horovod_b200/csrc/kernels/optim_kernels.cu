// Multi-tensor fused optimizer updates (SGD+momentum, Adam/AdamW) for sm_90a.
// One launch updates every parameter of the model: blockIdx.y selects the
// tensor from a device table, blockIdx.x strides over it with 16 B vectors.
// The reference leaves the optimizer to the framework (one or several kernels
// per parameter); SURVEY 2.5b lists "the optimizer update" as un-fused headroom.
// `grad_scale` lets DistributedOptimizer fold gradient post-division into the
// update instead of a separate elementwise pass.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <algorithm>
#include <cstring>
#include <type_traits>
#include "optim_kernels.h"
#include "p2p_kernels.h"

namespace hvd {
namespace kern {
namespace {

constexpr int kOptThreads = 256;
constexpr int kOptVec = 4;
constexpr int kOptIters = 4;
constexpr int kOptPerBlock = kOptThreads * kOptVec * kOptIters;

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

template <typename T> struct alignas(sizeof(T) * kOptVec) Vec4 { T v[kOptVec]; };

// max that keeps a NaN once it has seen one (fmaxf drops it), as torch's clamp and max do: an inf-norm of NaN gradients
// is NaN, and so is an Adafactor v clamped from a NaN
__device__ __forceinline__ float nan_max(float a, float b) { return (a > b || a != a) ? a : b; }
__device__ __forceinline__ double nan_max(double a, double b) { return (a > b || a != a) ? a : b; }

template <typename T> __device__ __forceinline__ void load4(const T* p, int64_t i, int64_t n, bool aligned, float* o) {
  if (aligned && i + kOptVec <= n) {
    Vec4<T> v = *reinterpret_cast<const Vec4<T>*>(p + i);
#pragma unroll
    for (int k = 0; k < kOptVec; ++k) o[k] = to_f<T>(v.v[k]);
  } else {
#pragma unroll
    for (int k = 0; k < kOptVec; ++k) o[k] = i + k < n ? to_f<T>(p[i + k]) : 0.f;
  }
}
template <typename T> __device__ __forceinline__ void store4(T* p, int64_t i, int64_t n, bool aligned, const float* o) {
  if (aligned && i + kOptVec <= n) {
    Vec4<T> v;
#pragma unroll
    for (int k = 0; k < kOptVec; ++k) v.v[k] = from_f<T>(o[k]);
    *reinterpret_cast<Vec4<T>*>(p + i) = v;
  } else {
#pragma unroll
    for (int k = 0; k < kOptVec; ++k) if (i + k < n) p[i + k] = from_f<T>(o[k]);
  }
}
template <typename T> __device__ __forceinline__ bool is_aligned(const void* p) { return (reinterpret_cast<uintptr_t>(p) % (sizeof(T) * kOptVec)) == 0; }

// fp32 master weights (kMaster): P is bf16 / fp16 and every table entry carries `master`, an fp32 copy of its parameter.
// The update runs on the master with exactly the arithmetic of the fp32-parameter instantiation, then the master is
// stored and the parameter receives it rounded to nearest-even.  Reconcile: where the stored bits of the parameter are
// not those of round(master) -- a write from outside the optimizer (load_state_dict, broadcast_parameters, an in-place
// edit) or a zero-filled master -- the master restarts from the parameter.  pv holds the parameter on entry and the
// value the update starts from on return.
template <typename P> __device__ __forceinline__ void reconcile4(float* pv, const float* wv) {
#pragma unroll
  for (int k = 0; k < kOptVec; ++k)
    if (__float_as_uint(to_f<P>(from_f<P>(wv[k]))) == __float_as_uint(pv[k])) pv[k] = wv[k];
}

// Exponential moving average epilogue (kEma): after the update, e = fmaf(w, x - e, e) with w = 1 - decay, where x is
// the fp32 master (kMaster) or the value stored into the parameter, rounded to P.  With `start` set the EMA begins now:
// e = x, and the old e is not read (zero is a valid EMA, so no value of e can mean "absent").  pv holds the updated
// fp32 value.  The EMA has its own alignment flag, so it works on unaligned views like the other state.
template <typename P, bool kMaster>
__device__ __forceinline__ void ema4(float* e, int64_t i, int64_t n, bool ea, const float* pv, float w, int start) {
  float ev[kOptVec];
  if (!start) load4<float>(e, i, n, ea, ev);
#pragma unroll
  for (int k = 0; k < kOptVec; ++k) {
    const float x = kMaster ? pv[k] : to_f<P>(from_f<P>(pv[k]));
    ev[k] = start ? x : fmaf(w, x - ev[k], ev[k]);
  }
  store4<float>(e, i, n, ea, ev);
}

// `grad_scale_dev` (nullptr: 1) is a factor that lives on the device, e.g. a clip coefficient computed by earlier kernels:
// it reaches the update without a host synchronisation.  Multiplying by 1.f is exact, so nullptr changes no result.
// Momentum is stored in the parameter dtype, or in fp32 with a master.
template <typename P, typename G, bool kMaster, bool kEma>
__global__ void __launch_bounds__(kOptThreads)
fused_sgd_kernel(const OptTensor* __restrict__ table, float lr, float momentum, float dampening, float wd, int nesterov,
                 float grad_scale, const float* __restrict__ grad_scale_dev, int first_step, float ema_w, int ema_start) {
  using M = std::conditional_t<kMaster, float, P>;
  const OptTensor t = table[blockIdx.y];
  const int64_t n = t.count;
  const int64_t base = (int64_t)blockIdx.x * kOptPerBlock;
  if (base >= n) return;
  grad_scale *= grad_scale_dev ? *grad_scale_dev : 1.f;
  P* p = reinterpret_cast<P*>(t.param);
  const G* g = reinterpret_cast<const G*>(t.grad);
  M* mbuf = reinterpret_cast<M*>(t.state0);
  float* w = kMaster ? reinterpret_cast<float*>(t.master) : nullptr;
  // pa: the parameter (and, without a master, the momentum); wa: the fp32 master and momentum
  const bool pa = is_aligned<P>(p) && (kMaster || !mbuf || is_aligned<M>(mbuf)), ga = is_aligned<G>(g);
  const bool wa = kMaster && is_aligned<float>(w) && (!mbuf || is_aligned<M>(mbuf));
  const bool ma = kMaster ? wa : pa;
  float* e = kEma ? reinterpret_cast<float*>(t.ema) : nullptr;
  const bool ea = kEma && is_aligned<float>(e);
#pragma unroll
  for (int it = 0; it < kOptIters; ++it) {
    const int64_t i = base + ((int64_t)it * kOptThreads + threadIdx.x) * kOptVec;
    if (i >= n) break;
    float pv[kOptVec], gv[kOptVec], mv[kOptVec];
    load4<P>(p, i, n, pa, pv);
    load4<G>(g, i, n, ga, gv);
    if (mbuf && !first_step) load4<M>(mbuf, i, n, ma, mv);
    if constexpr (kMaster) {
      float wv[kOptVec];
      load4<float>(w, i, n, wa, wv);
      reconcile4<P>(pv, wv);
    }
#pragma unroll
    for (int k = 0; k < kOptVec; ++k) {
      float d = gv[k] * grad_scale;
      if (wd != 0.f) d = fmaf(wd, pv[k], d);
      if (mbuf) {
        float b = first_step ? d : fmaf(momentum, mv[k], (1.f - dampening) * d);
        mv[k] = b;
        d = nesterov ? fmaf(momentum, b, d) : b;
      }
      pv[k] = fmaf(-lr, d, pv[k]);
    }
    if constexpr (kMaster) store4<float>(w, i, n, wa, pv);
    store4<P>(p, i, n, pa, pv);
    if (mbuf) store4<M>(mbuf, i, n, ma, mv);
    if constexpr (kEma) ema4<P, kMaster>(e, i, n, ea, pv, ema_w, ema_start);
  }
}

template <typename P, typename G, bool kMaster, bool kEma>
__global__ void __launch_bounds__(kOptThreads)
fused_adam_kernel(const OptTensor* __restrict__ table, float lr, float b1, float b2, float eps, float wd, float c1, float c2,
                  float grad_scale, const float* __restrict__ grad_scale_dev, int adamw, float ema_w, int ema_start) {
  const OptTensor t = table[blockIdx.y];
  const int64_t n = t.count;
  const int64_t base = (int64_t)blockIdx.x * kOptPerBlock;
  if (base >= n) return;
  grad_scale *= grad_scale_dev ? *grad_scale_dev : 1.f;
  P* p = reinterpret_cast<P*>(t.param);
  const G* g = reinterpret_cast<const G*>(t.grad);
  float* m = reinterpret_cast<float*>(t.state0);
  float* v = reinterpret_cast<float*>(t.state1);
  float* w = kMaster ? reinterpret_cast<float*>(t.master) : nullptr;
  const bool pa = is_aligned<P>(p), ga = is_aligned<G>(g),
             sa = is_aligned<float>(m) && is_aligned<float>(v) && (!kMaster || is_aligned<float>(w));
  const float rsc2 = rsqrtf(c2), step = lr / c1;
  float* e = kEma ? reinterpret_cast<float*>(t.ema) : nullptr;
  const bool ea = kEma && is_aligned<float>(e);
#pragma unroll
  for (int it = 0; it < kOptIters; ++it) {
    const int64_t i = base + ((int64_t)it * kOptThreads + threadIdx.x) * kOptVec;
    if (i >= n) break;
    float pv[kOptVec], gv[kOptVec], mv[kOptVec], vv[kOptVec];
    load4<P>(p, i, n, pa, pv);
    load4<G>(g, i, n, ga, gv);
    load4<float>(m, i, n, sa, mv);
    load4<float>(v, i, n, sa, vv);
    if constexpr (kMaster) {
      float wv[kOptVec];
      load4<float>(w, i, n, sa, wv);
      reconcile4<P>(pv, wv);
    }
#pragma unroll
    for (int k = 0; k < kOptVec; ++k) {
      float d = gv[k] * grad_scale;
      if (adamw) pv[k] *= (1.f - lr * wd); else if (wd != 0.f) d = fmaf(wd, pv[k], d);
      mv[k] = fmaf(b1, mv[k], (1.f - b1) * d);
      vv[k] = fmaf(b2, vv[k], (1.f - b2) * d * d);
      const float denom = sqrtf(vv[k]) * rsc2 + eps;
      pv[k] -= step * mv[k] / denom;
    }
    if constexpr (kMaster) store4<float>(w, i, n, sa, pv);
    store4<P>(p, i, n, pa, pv);
    store4<float>(m, i, n, sa, mv);
    store4<float>(v, i, n, sa, vv);
    if constexpr (kEma) ema4<P, kMaster>(e, i, n, ea, pv, ema_w, ema_start);
  }
}

// LAMB (You et al., "Large Batch Optimization for Deep Learning"): the bias-corrected Adam direction plus decoupled weight
// decay, u = (m / c1) / (sqrt(v / c2) + eps) + wd * w, applied as w -= lr * r * u with the per-tensor trust ratio
// r = ||w|| / ||u|| (1 if either norm is 0, or if the caller does not adapt).  The norms cover whole tensors, which may be
// split over several table entries (and ranks) sharing one `slot`, so the step is three launches: stage 1 updates the
// moments and writes one (sum w^2, sum u^2) partial per CTA, the finalize kernel adds each entry's partials in fp64 in a
// fixed order into norms[2 * slot], norms[2 * slot + 1], and stage 2 recomputes u from the stored moments and applies it.
// Deterministic, no atomics, nothing left behind between launches.  Only stage 1 reads the gradient.
__device__ __forceinline__ float lamb_u(float m, float v, float w, float c1, float c2, float eps, float wd) {
  return fmaf(wd, w, (m / c1) / (sqrtf(v / c2) + eps));
}

template <typename P, typename G, bool kMaster>
__global__ void __launch_bounds__(kOptThreads)
fused_lamb_norms_kernel(const OptTensor* __restrict__ table, float b1, float b2, float eps, float wd, float c1, float c2,
                        float grad_scale, const float* __restrict__ grad_scale_dev, float2* __restrict__ partial) {
  __shared__ float2 red[kOptThreads / 32];
  const OptTensor t = table[blockIdx.y];
  const int64_t n = t.count;
  const int64_t base = (int64_t)blockIdx.x * kOptPerBlock;
  if (base >= n) return;
  grad_scale *= grad_scale_dev ? *grad_scale_dev : 1.f;
  const P* p = reinterpret_cast<const P*>(t.param);
  const G* g = reinterpret_cast<const G*>(t.grad);
  float* m = reinterpret_cast<float*>(t.state0);
  float* v = reinterpret_cast<float*>(t.state1);
  const float* w = kMaster ? reinterpret_cast<const float*>(t.master) : nullptr;
  const bool pa = is_aligned<P>(p), ga = is_aligned<G>(g),
             sa = is_aligned<float>(m) && is_aligned<float>(v) && (!kMaster || is_aligned<float>(w));
  float sw = 0.f, su = 0.f;
#pragma unroll
  for (int it = 0; it < kOptIters; ++it) {
    const int64_t i = base + ((int64_t)it * kOptThreads + threadIdx.x) * kOptVec;
    if (i >= n) break;
    float pv[kOptVec], gv[kOptVec], mv[kOptVec], vv[kOptVec];
    load4<P>(p, i, n, pa, pv);
    load4<G>(g, i, n, ga, gv);
    load4<float>(m, i, n, sa, mv);
    load4<float>(v, i, n, sa, vv);
    if constexpr (kMaster) {
      float wv[kOptVec];
      load4<float>(w, i, n, sa, wv);
      reconcile4<P>(pv, wv);
    }
#pragma unroll
    for (int k = 0; k < kOptVec; ++k) {
      const float d = gv[k] * grad_scale;
      mv[k] = fmaf(b1, mv[k], (1.f - b1) * d);
      vv[k] = fmaf(b2, vv[k], (1.f - b2) * d * d);
      if (i + k < n) {  // past the end u would be 0 / eps, NaN for eps = 0
        const float u = lamb_u(mv[k], vv[k], pv[k], c1, c2, eps, wd);
        sw = fmaf(pv[k], pv[k], sw);
        su = fmaf(u, u, su);
      }
    }
    store4<float>(m, i, n, sa, mv);
    store4<float>(v, i, n, sa, vv);
  }
  // CTA partial: a fixed shuffle tree per warp, then the warps in order
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sw += __shfl_xor_sync(0xffffffffu, sw, o);
    su += __shfl_xor_sync(0xffffffffu, su, o);
  }
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = make_float2(sw, su);
  __syncthreads();
  if (threadIdx.x == 0) {
    float2 a = red[0];
    for (int k = 1; k < kOptThreads / 32; ++k) { a.x += red[k].x; a.y += red[k].y; }
    partial[t.partial + blockIdx.x] = a;
  }
}

// One CTA per entry: its partials in fp64, a fixed strided subset per thread, then a fixed tree; added into its slot.
// Every slot appears at most once per launch (checked by the host), so the read-modify-write does not race.
__global__ void __launch_bounds__(kOptThreads)
lamb_finalize_kernel(const OptTensor* __restrict__ table, const float2* __restrict__ partial, float* __restrict__ norms) {
  __shared__ double rw[kOptThreads], ru[kOptThreads];
  const OptTensor t = table[blockIdx.x];
  const int64_t nb = (t.count + kOptPerBlock - 1) / kOptPerBlock;
  double a = 0.0, b = 0.0;
  for (int64_t j = threadIdx.x; j < nb; j += kOptThreads) {
    const float2 x = partial[t.partial + j];
    a += (double)x.x;
    b += (double)x.y;
  }
  rw[threadIdx.x] = a;
  ru[threadIdx.x] = b;
  __syncthreads();
#pragma unroll
  for (int h = kOptThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) { rw[threadIdx.x] += rw[threadIdx.x + h]; ru[threadIdx.x] += ru[threadIdx.x + h]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    norms[2 * t.slot] = (float)((double)norms[2 * t.slot] + rw[0]);
    norms[2 * t.slot + 1] = (float)((double)norms[2 * t.slot + 1] + ru[0]);
  }
}

template <typename P, bool kMaster, bool kEma>
__global__ void __launch_bounds__(kOptThreads)
fused_lamb_apply_kernel(const OptTensor* __restrict__ table, float lr, float eps, float wd, float c1, float c2, int adapt,
                        const float* __restrict__ norms, float ema_w, int ema_start) {
  const OptTensor t = table[blockIdx.y];
  const int64_t n = t.count;
  const int64_t base = (int64_t)blockIdx.x * kOptPerBlock;
  if (base >= n) return;
  float r = 1.f;
  if (adapt) {
    const float wn = sqrtf(norms[2 * t.slot]), un = sqrtf(norms[2 * t.slot + 1]);
    if (wn > 0.f && un > 0.f) r = wn / un;
  }
  const float step = lr * r;
  P* p = reinterpret_cast<P*>(t.param);
  const float* m = reinterpret_cast<const float*>(t.state0);
  const float* v = reinterpret_cast<const float*>(t.state1);
  float* w = kMaster ? reinterpret_cast<float*>(t.master) : nullptr;
  const bool pa = is_aligned<P>(p), sa = is_aligned<float>(m) && is_aligned<float>(v) && (!kMaster || is_aligned<float>(w));
  float* e = kEma ? reinterpret_cast<float*>(t.ema) : nullptr;
  const bool ea = kEma && is_aligned<float>(e);
#pragma unroll
  for (int it = 0; it < kOptIters; ++it) {
    const int64_t i = base + ((int64_t)it * kOptThreads + threadIdx.x) * kOptVec;
    if (i >= n) break;
    float pv[kOptVec], mv[kOptVec], vv[kOptVec];
    load4<P>(p, i, n, pa, pv);
    load4<float>(m, i, n, sa, mv);
    load4<float>(v, i, n, sa, vv);
    if constexpr (kMaster) {
      float wv[kOptVec];
      load4<float>(w, i, n, sa, wv);
      reconcile4<P>(pv, wv);  // the same value stage 1 started from: nothing wrote p or the master in between
    }
#pragma unroll
    for (int k = 0; k < kOptVec; ++k) pv[k] = fmaf(-step, lamb_u(mv[k], vv[k], pv[k], c1, c2, eps, wd), pv[k]);
    if constexpr (kMaster) store4<float>(w, i, n, sa, pv);
    store4<P>(p, i, n, pa, pv);
    if constexpr (kEma) ema4<P, kMaster>(e, i, n, ea, pv, ema_w, ema_start);
  }
}

// LARS (You, Gitman, Ginsburg, "Large Batch Training of Convolutional Networks"; the MLPerf ResNet-50 optimizer): with
// g the scaled gradient, d = g + wd * w, the per-tensor trust ratio r = tc * ||w|| / (||g|| + wd * ||w|| + eps) (1 if
// either norm is 0, or if the caller does not adapt), v = momentum * v + lr * r * d, w -= v.  LAMB's three launches and
// table, with the fp32 momentum buffer in `state0` (`state1` is not read): stage 1 writes one (sum w^2, sum g^2)
// partial per CTA, lamb_finalize_kernel adds them into norms[2 * slot], norms[2 * slot + 1], and stage 2 reads the
// gradient again and applies the update.  Both stages scale the gradient alike.
template <typename P, typename G, bool kMaster>
__global__ void __launch_bounds__(kOptThreads)
fused_lars_norms_kernel(const OptTensor* __restrict__ table, float grad_scale, const float* __restrict__ grad_scale_dev,
                        float2* __restrict__ partial) {
  __shared__ float2 red[kOptThreads / 32];
  const OptTensor t = table[blockIdx.y];
  const int64_t n = t.count;
  const int64_t base = (int64_t)blockIdx.x * kOptPerBlock;
  if (base >= n) return;
  grad_scale *= grad_scale_dev ? *grad_scale_dev : 1.f;
  const P* p = reinterpret_cast<const P*>(t.param);
  const G* g = reinterpret_cast<const G*>(t.grad);
  const float* w = kMaster ? reinterpret_cast<const float*>(t.master) : nullptr;
  const bool pa = is_aligned<P>(p), ga = is_aligned<G>(g), wa = kMaster && is_aligned<float>(w);
  float sw = 0.f, sg = 0.f;
#pragma unroll
  for (int it = 0; it < kOptIters; ++it) {
    const int64_t i = base + ((int64_t)it * kOptThreads + threadIdx.x) * kOptVec;
    if (i >= n) break;
    float pv[kOptVec], gv[kOptVec];
    load4<P>(p, i, n, pa, pv);
    load4<G>(g, i, n, ga, gv);
    if constexpr (kMaster) {
      float wv[kOptVec];
      load4<float>(w, i, n, wa, wv);
      reconcile4<P>(pv, wv);
    }
#pragma unroll
    for (int k = 0; k < kOptVec; ++k) {
      if (i + k < n) {  // past the end g reads as 0, and 0 * grad_scale is NaN for an infinite scale
        const float d = gv[k] * grad_scale;
        sw = fmaf(pv[k], pv[k], sw);
        sg = fmaf(d, d, sg);
      }
    }
  }
  // CTA partial: the tree of fused_lamb_norms_kernel
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sw += __shfl_xor_sync(0xffffffffu, sw, o);
    sg += __shfl_xor_sync(0xffffffffu, sg, o);
  }
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = make_float2(sw, sg);
  __syncthreads();
  if (threadIdx.x == 0) {
    float2 a = red[0];
    for (int k = 1; k < kOptThreads / 32; ++k) { a.x += red[k].x; a.y += red[k].y; }
    partial[t.partial + blockIdx.x] = a;
  }
}

template <typename P, typename G, bool kMaster, bool kEma>
__global__ void __launch_bounds__(kOptThreads)
fused_lars_apply_kernel(const OptTensor* __restrict__ table, float lr, float momentum, float wd, float tc, float eps,
                        int adapt, float grad_scale, const float* __restrict__ grad_scale_dev, const float* __restrict__ norms,
                        float ema_w, int ema_start) {
  const OptTensor t = table[blockIdx.y];
  const int64_t n = t.count;
  const int64_t base = (int64_t)blockIdx.x * kOptPerBlock;
  if (base >= n) return;
  grad_scale *= grad_scale_dev ? *grad_scale_dev : 1.f;
  float r = 1.f;
  if (adapt) {
    const float wn = sqrtf(norms[2 * t.slot]), gn = sqrtf(norms[2 * t.slot + 1]);
    if (wn > 0.f && gn > 0.f) r = tc * wn / (fmaf(wd, wn, gn) + eps);
  }
  const float step = lr * r;
  P* p = reinterpret_cast<P*>(t.param);
  const G* g = reinterpret_cast<const G*>(t.grad);
  float* v = reinterpret_cast<float*>(t.state0);
  float* w = kMaster ? reinterpret_cast<float*>(t.master) : nullptr;
  const bool pa = is_aligned<P>(p), ga = is_aligned<G>(g), sa = is_aligned<float>(v) && (!kMaster || is_aligned<float>(w));
  float* e = kEma ? reinterpret_cast<float*>(t.ema) : nullptr;
  const bool ea = kEma && is_aligned<float>(e);
#pragma unroll
  for (int it = 0; it < kOptIters; ++it) {
    const int64_t i = base + ((int64_t)it * kOptThreads + threadIdx.x) * kOptVec;
    if (i >= n) break;
    float pv[kOptVec], gv[kOptVec], vv[kOptVec];
    load4<P>(p, i, n, pa, pv);
    load4<G>(g, i, n, ga, gv);
    load4<float>(v, i, n, sa, vv);
    if constexpr (kMaster) {
      float wv[kOptVec];
      load4<float>(w, i, n, sa, wv);
      reconcile4<P>(pv, wv);  // the same value stage 1 started from: nothing wrote p or the master in between
    }
#pragma unroll
    for (int k = 0; k < kOptVec; ++k) {
      const float d = fmaf(wd, pv[k], gv[k] * grad_scale);
      vv[k] = fmaf(momentum, vv[k], step * d);
      pv[k] -= vv[k];
    }
    if constexpr (kMaster) store4<float>(w, i, n, sa, pv);
    store4<P>(p, i, n, pa, pv);
    store4<float>(v, i, n, sa, vv);
    if constexpr (kEma) ema4<P, kMaster>(e, i, n, ea, pv, ema_w, ema_start);
  }
}

// Adafactor (Shazeer & Stern 2018) as torch.optim.Adafactor computes it, for g the scaled gradient at step t:
//   beta_w = t^beta2_decay, rho = min(lr, 1 / sqrt(t)), alpha = max(eps2, ||w|| / sqrt(n)) * rho (w before decay)
//   factored [.., R, C]: row_var = lerp(row_var, mean_c g^2, beta_w), col_var = lerp(col_var, mean_r g^2, beta_w),
//                        v = row_var * col_var / max(mean_r row_var, eps1)
//   dim <= 1:            variance = lerp(variance, g^2, beta_w), v = variance
//   u = g * rsqrt(max(v, eps1^2)), denom = max(1, ||u|| / (sqrt(n) * d)), w = w * (1 - lr * wd) - (alpha / denom) * u
// The two clamps of v keep a NaN, as torch's clamp does; alpha's and denom's max drop one, as Python's max(eps2, nan) and
// max(1, nan) do.
// Five launches and no state between them: adafactor_stats_kernel (z = 0: one warp per row sums g^2 over the row and
// lerps row_var; z = 1: one thread per (column, chunk of kAfRowChunk rows) writes a column partial),
// adafactor_factors_kernel (z = 0: one thread per column adds its partials in fp64 in chunk order and lerps col_var;
// z = 1: one CTA per matrix of the batch takes the mean of row_var in fp64), adafactor_norms_kernel (per-CTA
// (sum w^2, sum u^2) partials in LAMB's layout; lerps and stores the variance of dim <= 1 entries), lamb_finalize_kernel,
// and adafactor_apply_kernel, which recomputes u with the same code.  Every sum has a fixed order: deterministic.
constexpr int kAfRowChunk = 64;

__device__ __forceinline__ float af_lerp(float a, float b, float w) {  // at::native::lerp's two-sided formula
  return fabsf(w) < 0.5f ? a + w * (b - a) : b - (b - a) * (1.f - w);
}

__device__ __forceinline__ unsigned af_batch(const AdafactorGeom& gm) { return (unsigned)gm.size[0] * gm.size[1] * gm.size[2]; }

// storage offset of matrix b of the batch (row-major over the leading dims)
__device__ __forceinline__ unsigned af_batch_offset(const AdafactorGeom& gm, unsigned b) {
  unsigned off = 0;
#pragma unroll
  for (int d = 2; d >= 0; --d) {
    off += (b % (unsigned)gm.size[d]) * (unsigned)gm.stride[d];
    b /= (unsigned)gm.size[d];
  }
  return off;
}

// v of the factored element at storage offset o: a dense layout's strides are a mixed radix, so coordinate
// d = (o / stride[d]) % size[d]
__device__ __forceinline__ float af_vhat(const AdafactorGeom& gm, const float* __restrict__ rmean, unsigned o, float eps1) {
  const unsigned c = (o / (unsigned)gm.stride[4]) % (unsigned)gm.size[4], r = (o / (unsigned)gm.stride[3]) % (unsigned)gm.size[3];
  unsigned b = 0;
#pragma unroll
  for (int d = 0; d < 3; ++d) b = b * (unsigned)gm.size[d] + (o / (unsigned)gm.stride[d]) % (unsigned)gm.size[d];
  const float rv = gm.row_var[(size_t)b * gm.size[3] + r], cv = gm.col_var[(size_t)b * gm.size[4] + c];
  return rv * cv / nan_max(rmean[gm.batch_off + b], eps1);
}

// u for 4 elements from the scaled gradient dv and, for dim <= 1 entries, the (lerped) variance vv; 0 past the end
__device__ __forceinline__ void af_u4(const AdafactorGeom& gm, const float* __restrict__ rmean, int64_t i, int64_t n,
                                      const float* dv, const float* vv, float eps1, float eps1_sq, float* uv) {
#pragma unroll
  for (int k = 0; k < kOptVec; ++k) {
    uv[k] = 0.f;
    if (i + k < n) {
      const float v = gm.row_var ? af_vhat(gm, rmean, (unsigned)(i + k), eps1) : vv[k];
      uv[k] = dv[k] * rsqrtf(nan_max(v, eps1_sq));
    }
  }
}

template <typename G>
__global__ void __launch_bounds__(kOptThreads)
adafactor_stats_kernel(const OptTensor* __restrict__ table, const AdafactorGeom* __restrict__ geom, float beta_w,
                       float grad_scale, const float* __restrict__ grad_scale_dev, float* __restrict__ colpart) {
  const AdafactorGeom& gm = geom[blockIdx.y];
  if (gm.row_var == nullptr) return;
  const G* g = reinterpret_cast<const G*>(table[blockIdx.y].grad);
  const unsigned R = gm.size[3], C = gm.size[4], B = af_batch(gm);
  if (blockIdx.z == 0) {
    const unsigned row = blockIdx.x * (kOptThreads / 32) + threadIdx.x / 32, lane = threadIdx.x % 32;
    if (row >= B * R) return;  // uniform per warp
    grad_scale *= grad_scale_dev ? *grad_scale_dev : 1.f;
    const G* gr = g + af_batch_offset(gm, row / R) + (size_t)(row % R) * gm.stride[3];
    float s = 0.f;
    for (unsigned c = lane; c < C; c += 32) {
      const float x = to_f<G>(gr[(size_t)c * gm.stride[4]]) * grad_scale;
      s = fmaf(x, x, s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) gm.row_var[row] = af_lerp(gm.row_var[row], s / (float)C, beta_w);
  } else {
    const unsigned chunks = (R + kAfRowChunk - 1) / kAfRowChunk, j = blockIdx.x * kOptThreads + threadIdx.x;
    if (j >= B * C * chunks) return;
    grad_scale *= grad_scale_dev ? *grad_scale_dev : 1.f;
    const unsigned c = j % C, bk = j / C, b = bk % B, k = bk / B, r1 = min(R, (k + 1) * kAfRowChunk);
    const G* gc = g + af_batch_offset(gm, b) + (size_t)c * gm.stride[4];
    float s = 0.f;
    for (unsigned r = k * kAfRowChunk; r < r1; ++r) {
      const float x = to_f<G>(gc[(size_t)r * gm.stride[3]]) * grad_scale;
      s = fmaf(x, x, s);
    }
    colpart[gm.col_off + j] = s;  // [chunk][b][c]: adjacent threads, adjacent columns
  }
}

__global__ void __launch_bounds__(kOptThreads)
adafactor_factors_kernel(const AdafactorGeom* __restrict__ geom, float beta_w, const float* __restrict__ colpart,
                         float* __restrict__ rmean) {
  __shared__ double red[kOptThreads];
  const AdafactorGeom& gm = geom[blockIdx.y];
  if (gm.row_var == nullptr) return;
  const unsigned R = gm.size[3], C = gm.size[4], B = af_batch(gm);
  if (blockIdx.z == 0) {
    const unsigned j = blockIdx.x * kOptThreads + threadIdx.x;  // b * C + c
    if (j >= B * C) return;
    const unsigned chunks = (R + kAfRowChunk - 1) / kAfRowChunk;
    double s = 0.0;
    for (unsigned k = 0; k < chunks; ++k) s += (double)colpart[gm.col_off + (size_t)k * B * C + j];
    gm.col_var[j] = af_lerp(gm.col_var[j], (float)(s / R), beta_w);
  } else {
    const unsigned b = blockIdx.x;
    if (b >= B) return;  // uniform per CTA
    double s = 0.0;
    for (unsigned r = threadIdx.x; r < R; r += kOptThreads) s += (double)gm.row_var[(size_t)b * R + r];
    red[threadIdx.x] = s;
    __syncthreads();
#pragma unroll
    for (int h = kOptThreads / 2; h > 0; h >>= 1) {
      if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
      __syncthreads();
    }
    if (threadIdx.x == 0) rmean[gm.batch_off + b] = (float)(red[0] / R);
  }
}

template <typename P, typename G, bool kMaster>
__global__ void __launch_bounds__(kOptThreads)
adafactor_norms_kernel(const OptTensor* __restrict__ table, const AdafactorGeom* __restrict__ geom, float beta_w,
                       float eps1, float eps1_sq, float grad_scale, const float* __restrict__ grad_scale_dev,
                       const float* __restrict__ rmean, float2* __restrict__ partial) {
  __shared__ float2 red[kOptThreads / 32];
  const OptTensor t = table[blockIdx.y];
  const AdafactorGeom& gm = geom[blockIdx.y];
  const int64_t n = t.count;
  const int64_t base = (int64_t)blockIdx.x * kOptPerBlock;
  if (base >= n) return;
  grad_scale *= grad_scale_dev ? *grad_scale_dev : 1.f;
  const P* p = reinterpret_cast<const P*>(t.param);
  const G* g = reinterpret_cast<const G*>(t.grad);
  float* var = reinterpret_cast<float*>(t.state0);
  const float* w = kMaster ? reinterpret_cast<const float*>(t.master) : nullptr;
  const bool pa = is_aligned<P>(p), ga = is_aligned<G>(g), va = is_aligned<float>(var), wa = kMaster && is_aligned<float>(w);
  float sw = 0.f, su = 0.f;
#pragma unroll
  for (int it = 0; it < kOptIters; ++it) {
    const int64_t i = base + ((int64_t)it * kOptThreads + threadIdx.x) * kOptVec;
    if (i >= n) break;
    float pv[kOptVec], dv[kOptVec], vv[kOptVec] = {0.f, 0.f, 0.f, 0.f}, uv[kOptVec];
    load4<P>(p, i, n, pa, pv);
    load4<G>(g, i, n, ga, dv);
    if constexpr (kMaster) {
      float wv[kOptVec];
      load4<float>(w, i, n, wa, wv);
      reconcile4<P>(pv, wv);
    }
#pragma unroll
    for (int k = 0; k < kOptVec; ++k) dv[k] *= grad_scale;
    if (!gm.row_var) {
      load4<float>(var, i, n, va, vv);
#pragma unroll
      for (int k = 0; k < kOptVec; ++k) vv[k] = af_lerp(vv[k], dv[k] * dv[k], beta_w);
      store4<float>(var, i, n, va, vv);
    }
    af_u4(gm, rmean, i, n, dv, vv, eps1, eps1_sq, uv);
#pragma unroll
    for (int k = 0; k < kOptVec; ++k) {  // past the end w reads as 0 and u is 0
      sw = fmaf(pv[k], pv[k], sw);
      su = fmaf(uv[k], uv[k], su);
    }
  }
  // CTA partial: the tree of fused_lamb_norms_kernel
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sw += __shfl_xor_sync(0xffffffffu, sw, o);
    su += __shfl_xor_sync(0xffffffffu, su, o);
  }
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = make_float2(sw, su);
  __syncthreads();
  if (threadIdx.x == 0) {
    float2 a = red[0];
    for (int k = 1; k < kOptThreads / 32; ++k) { a.x += red[k].x; a.y += red[k].y; }
    partial[t.partial + blockIdx.x] = a;
  }
}

template <typename P, typename G, bool kMaster, bool kEma>
__global__ void __launch_bounds__(kOptThreads)
adafactor_apply_kernel(const OptTensor* __restrict__ table, const AdafactorGeom* __restrict__ geom, AdafactorHyper h,
                       float grad_scale, const float* __restrict__ grad_scale_dev, const float* __restrict__ rmean,
                       const float* __restrict__ norms, float ema_w, int ema_start) {
  const OptTensor t = table[blockIdx.y];
  const AdafactorGeom& gm = geom[blockIdx.y];
  const int64_t n = t.count;
  const int64_t base = (int64_t)blockIdx.x * kOptPerBlock;
  if (base >= n) return;
  grad_scale *= grad_scale_dev ? *grad_scale_dev : 1.f;
  const float rn = sqrtf((float)n);
  const float alpha = fmaxf(h.eps2, sqrtf(norms[2 * t.slot]) / rn) * h.rho;
  const float step = alpha / fmaxf(1.f, sqrtf(norms[2 * t.slot + 1]) / (rn * h.d));
  P* p = reinterpret_cast<P*>(t.param);
  const G* g = reinterpret_cast<const G*>(t.grad);
  const float* var = reinterpret_cast<const float*>(t.state0);
  float* w = kMaster ? reinterpret_cast<float*>(t.master) : nullptr;
  const bool pa = is_aligned<P>(p), ga = is_aligned<G>(g), va = is_aligned<float>(var), wa = kMaster && is_aligned<float>(w);
  float* e = kEma ? reinterpret_cast<float*>(t.ema) : nullptr;
  const bool ea = kEma && is_aligned<float>(e);
#pragma unroll
  for (int it = 0; it < kOptIters; ++it) {
    const int64_t i = base + ((int64_t)it * kOptThreads + threadIdx.x) * kOptVec;
    if (i >= n) break;
    float pv[kOptVec], dv[kOptVec], vv[kOptVec] = {0.f, 0.f, 0.f, 0.f}, uv[kOptVec];
    load4<P>(p, i, n, pa, pv);
    load4<G>(g, i, n, ga, dv);
    if constexpr (kMaster) {
      float wv[kOptVec];
      load4<float>(w, i, n, wa, wv);
      reconcile4<P>(pv, wv);  // the same value the norms launch started from: nothing wrote p or the master in between
    }
#pragma unroll
    for (int k = 0; k < kOptVec; ++k) dv[k] *= grad_scale;
    if (!gm.row_var) load4<float>(var, i, n, va, vv);  // lerped by the norms launch
    af_u4(gm, rmean, i, n, dv, vv, h.eps1, h.eps1_sq, uv);
#pragma unroll
    for (int k = 0; k < kOptVec; ++k) pv[k] = fmaf(-step, uv[k], pv[k] * h.decay);
    if constexpr (kMaster) store4<float>(w, i, n, wa, pv);
    store4<P>(p, i, n, pa, pv);
    if constexpr (kEma) ema4<P, kMaster>(e, i, n, ea, pv, ema_w, ema_start);
  }
}

// Host bytes as kernel parameters: a launch captured into a CUDA graph keeps its own copy of them.
constexpr int kUploadChunk = 4000;
struct UploadChunk { unsigned char b[kUploadChunk]; };

__global__ void __launch_bounds__(kOptThreads) upload_bytes_kernel(unsigned char* __restrict__ dst, const UploadChunk c, int bytes) {
  for (int i = threadIdx.x; i < bytes; i += kOptThreads) dst[i] = c.b[i];
}

// Gradient statistics of a table of flat gradient shards in one read pass: optional in-place scaling by *inv_scale, the
// sum of squares (norm_inf = 0) or the max |g| (norm_inf = 1) of the scaled values as stored, and a non-finite flag.
// The grid has one CTA per kOptPerBlock-element tile of each tensor (entry e owns tiles [tile_begin, next tile_begin)), so
// a list of per-parameter gradients with one large embedding costs CTAs in proportion to its total size.  Every CTA
// writes one partial; the last CTA to finish (atomic ticket, which it resets for the next launch) combines them in fp64,
// always in the same order, and folds the result into out[0] (+= or max) and out[1] (max of 0 / 1).  So the same input
// gives the same bits on every call, and one launch per gradient dtype accumulates into one output.
template <typename G>
__global__ void __launch_bounds__(kOptThreads)
grad_shard_stats_kernel(const StatTensor* __restrict__ table, int n_entries, int64_t row_tiles,
                        const float* __restrict__ inv_scale, int norm_inf, float* __restrict__ partial,
                        int* __restrict__ partial_flag, unsigned* ticket, float* out) {
  __shared__ double red[kOptThreads];
  __shared__ int red_flag[kOptThreads / 32];
  __shared__ bool last;
  const unsigned ctas = gridDim.x, cta = blockIdx.x;
  int lo = 0, hi = n_entries - 1;  // the entry whose tiles include this CTA: the last one with tile_begin <= cta
  while (lo < hi) {
    const int mid = (lo + hi + 1) / 2;
    if (table[mid].tile_begin <= (int64_t)cta) lo = mid; else hi = mid - 1;
  }
  const StatTensor t = table[lo];
  const int64_t n = t.count;
  const int64_t base = ((int64_t)cta - t.tile_begin) * kOptPerBlock;
  float acc = 0.f;
  int bad = 0;
  if (base < n) {
    G* g = reinterpret_cast<G*>(t.grad);
    const bool ga = is_aligned<G>(g);
    const float s = inv_scale ? *inv_scale : 1.f;
#pragma unroll
    for (int it = 0; it < kOptIters; ++it) {
      const int64_t i = base + ((int64_t)it * kOptThreads + threadIdx.x) * kOptVec;
      if (i >= n) break;
      float gv[kOptVec];
      load4<G>(g, i, n, ga, gv);  // elements past the end read as 0, which changes neither statistic
      if (inv_scale) {
#pragma unroll
        for (int k = 0; k < kOptVec; ++k) gv[k] = to_f<G>(from_f<G>(gv[k] * s));  // the value as stored
        store4<G>(g, i, n, ga, gv);
      }
#pragma unroll
      for (int k = 0; k < kOptVec; ++k) {
        bad |= !isfinite(gv[k]);
        acc = norm_inf ? nan_max(acc, fabsf(gv[k])) : fmaf(gv[k], gv[k], acc);
      }
    }
  }
  // CTA partial: a fixed shuffle tree per warp, then the warps in order
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float y = __shfl_xor_sync(0xffffffffu, acc, o);
    acc = norm_inf ? nan_max(acc, y) : acc + y;
  }
  bad = __any_sync(0xffffffffu, bad);
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  if (lane == 0) { red[warp] = acc; red_flag[warp] = bad; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f;
    int f = 0;
    for (int w = 0; w < kOptThreads / 32; ++w) {
      a = norm_inf ? nan_max(a, (float)red[w]) : a + (float)red[w];
      f |= red_flag[w];
    }
    partial[cta] = a;
    partial_flag[cta] = f;
    __threadfence();
    last = atomicAdd(ticket, 1u) == ctas - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  // the last CTA: every thread combines a fixed subset of the partials in a fixed order, then a fixed tree over the
  // threads.  Thread i takes tile x of entry e when e * row_tiles + x == i (mod kOptThreads), in increasing order of that
  // index: the order of a grid of row_tiles CTAs per entry (as wide as the largest tensor), whose CTAs past the end of
  // their tensor would add partials of +0, which leave an fp64 sum and a max of non-negative values unchanged.  So the
  // statistics are bit for bit those of that rectangular grid, which earlier versions launched.
  double a = 0.0;
  int f = 0;
  for (int e = 0; e < n_entries; ++e) {
    const int64_t tb = table[e].tile_begin, te = e + 1 < n_entries ? table[e + 1].tile_begin : (int64_t)ctas;
    for (int64_t j = tb + ((int64_t)threadIdx.x + kOptThreads - (int64_t)e * row_tiles % kOptThreads) % kOptThreads;
         j < te; j += kOptThreads) {
      const double x = (double)__ldcg(partial + j);
      a = norm_inf ? nan_max(a, x) : a + x;
      f |= __ldcg(partial_flag + j);
    }
  }
  red[threadIdx.x] = a;
  f = __syncthreads_or(f);
#pragma unroll
  for (int h = kOptThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] = norm_inf ? nan_max(red[threadIdx.x], red[threadIdx.x + h]) : red[threadIdx.x] + red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    out[0] = norm_inf ? (float)nan_max((double)out[0], red[0]) : (float)((double)out[0] + red[0]);
    out[1] = fmaxf(out[1], f ? 1.f : 0.f);
    *ticket = 0u;  // ready for the next launch on this stream
  }
}

// Gradient accumulation in fp32 for bf16 / fp16 gradients: every table entry pairs a 16-bit gradient g with an fp32
// accumulator of the same element order.  kAccFirst: acc = g, g = 0.  kAccAdd: acc += g, g = 0.  kAccLast: g = acc + g
// rounded to nearest-even once (acc is not written).  Each element is one fp32 add at most, so the result is that of the
// same torch ops in fp32, bit for bit; inf / NaN propagate.  The table travels as a kernel parameter, so a launch
// captured into a CUDA graph keeps its own copy.
template <typename G>
__global__ void __launch_bounds__(kOptThreads)
grad_accumulate_kernel(const AccTable table, int mode) {
  const AccTensor t = table.t[blockIdx.y];
  const int64_t n = t.count;
  const int64_t base = (int64_t)blockIdx.x * kOptPerBlock;
  if (base >= n) return;
  G* g = reinterpret_cast<G*>(t.grad);
  float* acc = t.acc;
  const bool ga = is_aligned<G>(g), aa = is_aligned<float>(acc);
#pragma unroll
  for (int it = 0; it < kOptIters; ++it) {
    const int64_t i = base + ((int64_t)it * kOptThreads + threadIdx.x) * kOptVec;
    if (i >= n) break;
    float gv[kOptVec], av[kOptVec];
    load4<G>(g, i, n, ga, gv);
    if (mode == kAccFirst) {
      store4<float>(acc, i, n, aa, gv);
    } else {
      load4<float>(acc, i, n, aa, av);
#pragma unroll
      for (int k = 0; k < kOptVec; ++k) av[k] += gv[k];
      if (mode == kAccLast) {
        store4<G>(g, i, n, ga, av);
        continue;
      }
      store4<float>(acc, i, n, aa, av);
    }
    const float zero[kOptVec] = {0.f, 0.f, 0.f, 0.f};
    store4<G>(g, i, n, ga, zero);
  }
}

// The (param, grad, master) instantiations of the optimizer kernels: launch(OptTypes<P, G, kMaster>()) for a pair that
// has one, then the launch is counted and checked; cudaErrorInvalidValue without launching for any other pair.  The
// updates that keep an EMA pick their kEma instantiation inside `launch`, so EMA off runs the kernels it always ran.
template <typename P_, typename G_, bool kMaster_> struct OptTypes {
  using P = P_;
  using G = G_;
  static constexpr bool kMaster = kMaster_;
};

template <typename F> cudaError_t DispatchOpt(int param_dtype, int grad_dtype, bool master, F&& launch) {
  if (master) {
    if (param_dtype == 10 && grad_dtype == 10) launch(OptTypes<__nv_bfloat16, __nv_bfloat16, true>());
    else if (param_dtype == 6 && grad_dtype == 6) launch(OptTypes<__half, __half, true>());
    else return cudaErrorInvalidValue;
  }
  else if (param_dtype == 7 && grad_dtype == 7) launch(OptTypes<float, float, false>());
  else if (param_dtype == 7 && grad_dtype == 10) launch(OptTypes<float, __nv_bfloat16, false>());
  else if (param_dtype == 10 && grad_dtype == 10) launch(OptTypes<__nv_bfloat16, __nv_bfloat16, false>());
  else if (param_dtype == 6 && grad_dtype == 6) launch(OptTypes<__half, __half, false>());
  else return cudaErrorInvalidValue;
  CountKernelLaunch();
  return cudaGetLastError();
}

// blockIdx.x covers the longest entry, blockIdx.y selects the entry
dim3 OptGrid(int n, int64_t max_count) { return dim3((unsigned)NormPartials(max_count), (unsigned)n); }

// After a stage-1 launch: add each entry's partials into its norm slot.
cudaError_t FinalizeNorms(cudaError_t stage1, const OptTensor* table, int n, const float2* part, float* norms,
                          cudaStream_t stream) {
  if (stage1 != cudaSuccess) return stage1;
  lamb_finalize_kernel<<<(unsigned)n, kOptThreads, 0, stream>>>(table, part, norms);
  CountKernelLaunch();
  return cudaGetLastError();
}

}  // namespace

int64_t NormPartials(int64_t count) { return (count + kOptPerBlock - 1) / kOptPerBlock; }

cudaError_t LaunchFusedSgd(const OptTensor* table, int n, int64_t max_count, float lr, float momentum, float dampening,
                           float weight_decay, int nesterov, float grad_scale, int first_step, int param_dtype,
                           int grad_dtype, cudaStream_t stream, const float* grad_scale_dev, bool master, const OptEma& ema) {
  if (n <= 0 || max_count <= 0) return cudaSuccess;
  return DispatchOpt(param_dtype, grad_dtype, master, [&](auto t) {
    using T = decltype(t);
    if (ema.on)
      fused_sgd_kernel<typename T::P, typename T::G, T::kMaster, true><<<OptGrid(n, max_count), kOptThreads, 0, stream>>>(
          table, lr, momentum, dampening, weight_decay, nesterov, grad_scale, grad_scale_dev, first_step, ema.weight, ema.start);
    else
      fused_sgd_kernel<typename T::P, typename T::G, T::kMaster, false><<<OptGrid(n, max_count), kOptThreads, 0, stream>>>(
          table, lr, momentum, dampening, weight_decay, nesterov, grad_scale, grad_scale_dev, first_step, 0.f, 0);
  });
}

cudaError_t LaunchFusedAdamW(const OptTensor* table, int n, int64_t max_count, float lr, float beta1, float beta2,
                             float eps, float weight_decay, float bias_c1, float bias_c2, float grad_scale, int adamw,
                             int param_dtype, int grad_dtype, cudaStream_t stream, const float* grad_scale_dev,
                             bool master, const OptEma& ema) {
  if (n <= 0 || max_count <= 0) return cudaSuccess;
  return DispatchOpt(param_dtype, grad_dtype, master, [&](auto t) {
    using T = decltype(t);
    if (ema.on)
      fused_adam_kernel<typename T::P, typename T::G, T::kMaster, true><<<OptGrid(n, max_count), kOptThreads, 0, stream>>>(
          table, lr, beta1, beta2, eps, weight_decay, bias_c1, bias_c2, grad_scale, grad_scale_dev, adamw, ema.weight,
          ema.start);
    else
      fused_adam_kernel<typename T::P, typename T::G, T::kMaster, false><<<OptGrid(n, max_count), kOptThreads, 0, stream>>>(
          table, lr, beta1, beta2, eps, weight_decay, bias_c1, bias_c2, grad_scale, grad_scale_dev, adamw, 0.f, 0);
  });
}

cudaError_t LaunchLambNorms(const OptTensor* table, int n, int64_t max_count, float beta1, float beta2, float eps,
                            float weight_decay, float bias_c1, float bias_c2, float grad_scale, const float* grad_scale_dev,
                            float* partial, float* norms, int param_dtype, int grad_dtype, bool master, cudaStream_t stream) {
  if (n <= 0 || max_count <= 0) return cudaSuccess;
  float2* part = reinterpret_cast<float2*>(partial);
  return FinalizeNorms(DispatchOpt(param_dtype, grad_dtype, master, [&](auto t) {
    using T = decltype(t);
    fused_lamb_norms_kernel<typename T::P, typename T::G, T::kMaster><<<OptGrid(n, max_count), kOptThreads, 0, stream>>>(
        table, beta1, beta2, eps, weight_decay, bias_c1, bias_c2, grad_scale, grad_scale_dev, part);
  }), table, n, part, norms, stream);
}

cudaError_t LaunchLambApply(const OptTensor* table, int n, int64_t max_count, float lr, float eps, float weight_decay,
                            float bias_c1, float bias_c2, int adapt, const float* norms, int param_dtype, bool master,
                            cudaStream_t stream, const OptEma& ema) {
  if (n <= 0 || max_count <= 0) return cudaSuccess;
  // the gradient is not read: dispatch on the parameter dtype alone
  return DispatchOpt(param_dtype, param_dtype, master, [&](auto t) {
    using T = decltype(t);
    if (ema.on)
      fused_lamb_apply_kernel<typename T::P, T::kMaster, true><<<OptGrid(n, max_count), kOptThreads, 0, stream>>>(
          table, lr, eps, weight_decay, bias_c1, bias_c2, adapt, norms, ema.weight, ema.start);
    else
      fused_lamb_apply_kernel<typename T::P, T::kMaster, false><<<OptGrid(n, max_count), kOptThreads, 0, stream>>>(
          table, lr, eps, weight_decay, bias_c1, bias_c2, adapt, norms, 0.f, 0);
  });
}

cudaError_t LaunchLarsNorms(const OptTensor* table, int n, int64_t max_count, float grad_scale, const float* grad_scale_dev,
                            float* partial, float* norms, int param_dtype, int grad_dtype, bool master, cudaStream_t stream) {
  if (n <= 0 || max_count <= 0) return cudaSuccess;
  float2* part = reinterpret_cast<float2*>(partial);
  return FinalizeNorms(DispatchOpt(param_dtype, grad_dtype, master, [&](auto t) {
    using T = decltype(t);
    fused_lars_norms_kernel<typename T::P, typename T::G, T::kMaster><<<OptGrid(n, max_count), kOptThreads, 0, stream>>>(
        table, grad_scale, grad_scale_dev, part);
  }), table, n, part, norms, stream);
}

cudaError_t LaunchLarsApply(const OptTensor* table, int n, int64_t max_count, float lr, float momentum, float weight_decay,
                            float trust_coefficient, float eps, int adapt, float grad_scale, const float* grad_scale_dev,
                            const float* norms, int param_dtype, int grad_dtype, bool master, cudaStream_t stream,
                            const OptEma& ema) {
  if (n <= 0 || max_count <= 0) return cudaSuccess;
  return DispatchOpt(param_dtype, grad_dtype, master, [&](auto t) {
    using T = decltype(t);
    if (ema.on)
      fused_lars_apply_kernel<typename T::P, typename T::G, T::kMaster, true><<<OptGrid(n, max_count), kOptThreads, 0, stream>>>(
          table, lr, momentum, weight_decay, trust_coefficient, eps, adapt, grad_scale, grad_scale_dev, norms, ema.weight,
          ema.start);
    else
      fused_lars_apply_kernel<typename T::P, typename T::G, T::kMaster, false><<<OptGrid(n, max_count), kOptThreads, 0, stream>>>(
          table, lr, momentum, weight_decay, trust_coefficient, eps, adapt, grad_scale, grad_scale_dev, norms, 0.f, 0);
  });
}

int64_t AdafactorRowChunks(int64_t rows) { return (rows + kAfRowChunk - 1) / kAfRowChunk; }

int64_t AdafactorStatsCtas(int64_t batch, int64_t rows, int64_t cols) {
  const int64_t row_ctas = (batch * rows + kOptThreads / 32 - 1) / (kOptThreads / 32);
  const int64_t col_ctas = (batch * cols * AdafactorRowChunks(rows) + kOptThreads - 1) / kOptThreads;
  return std::max(row_ctas, col_ctas);
}

int64_t AdafactorFactorCtas(int64_t batch, int64_t cols) {
  return std::max(batch, (batch * cols + kOptThreads - 1) / kOptThreads);
}

cudaError_t LaunchAdafactor(const OptTensor* table, const AdafactorGeom* geom, int n, int64_t max_count, int64_t stats_ctas,
                            int64_t factor_ctas, const AdafactorHyper& h, float grad_scale, const float* grad_scale_dev,
                            float* colpart, float* rmean, float* partial, float* norms, int param_dtype, int grad_dtype,
                            bool master, cudaStream_t stream, const OptEma& ema) {
  if (n <= 0 || max_count <= 0) return cudaSuccess;
  if (stats_ctas < 1 || factor_ctas < 1 || stats_ctas > 0x7fffffff || factor_ctas > 0x7fffffff) return cudaErrorInvalidValue;
  cudaError_t e = DispatchOpt(param_dtype, grad_dtype, master, [&](auto t) {
    using T = decltype(t);
    adafactor_stats_kernel<typename T::G><<<dim3((unsigned)stats_ctas, (unsigned)n, 2), kOptThreads, 0, stream>>>(
        table, geom, h.beta_w, grad_scale, grad_scale_dev, colpart);
  });
  if (e != cudaSuccess) return e;
  adafactor_factors_kernel<<<dim3((unsigned)factor_ctas, (unsigned)n, 2), kOptThreads, 0, stream>>>(geom, h.beta_w, colpart, rmean);
  CountKernelLaunch();
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  float2* part = reinterpret_cast<float2*>(partial);
  e = FinalizeNorms(DispatchOpt(param_dtype, grad_dtype, master, [&](auto t) {
    using T = decltype(t);
    adafactor_norms_kernel<typename T::P, typename T::G, T::kMaster><<<OptGrid(n, max_count), kOptThreads, 0, stream>>>(
        table, geom, h.beta_w, h.eps1, h.eps1_sq, grad_scale, grad_scale_dev, rmean, part);
  }), table, n, part, norms, stream);
  if (e != cudaSuccess) return e;
  return DispatchOpt(param_dtype, grad_dtype, master, [&](auto t) {
    using T = decltype(t);
    if (ema.on)
      adafactor_apply_kernel<typename T::P, typename T::G, T::kMaster, true><<<OptGrid(n, max_count), kOptThreads, 0, stream>>>(
          table, geom, h, grad_scale, grad_scale_dev, rmean, norms, ema.weight, ema.start);
    else
      adafactor_apply_kernel<typename T::P, typename T::G, T::kMaster, false><<<OptGrid(n, max_count), kOptThreads, 0, stream>>>(
          table, geom, h, grad_scale, grad_scale_dev, rmean, norms, 0.f, 0);
  });
}

cudaError_t LaunchUploadBytes(void* dst, const void* host, size_t bytes, cudaStream_t stream) {
  for (size_t off = 0; off < bytes; off += kUploadChunk) {
    UploadChunk c;
    const int len = (int)std::min<size_t>(kUploadChunk, bytes - off);
    memcpy(c.b, static_cast<const unsigned char*>(host) + off, (size_t)len);
    upload_bytes_kernel<<<1, kOptThreads, 0, stream>>>(static_cast<unsigned char*>(dst) + off, c, len);
    CountKernelLaunch();
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

int64_t GradShardStatsTiles(int64_t count) { return (count + kOptPerBlock - 1) / kOptPerBlock; }

cudaError_t LaunchGradShardStats(const StatTensor* table, int n, int64_t tiles, int64_t row_tiles, const float* inv_scale,
                                 int norm_inf, float* partial, int* partial_flag, unsigned* ticket, float* out,
                                 int grad_dtype, cudaStream_t stream) {
  if (n <= 0 || tiles <= 0) return cudaSuccess;
  if (tiles > 0x7fffffff) return cudaErrorInvalidValue;
  const unsigned grid = (unsigned)tiles;
  if (grad_dtype == 7) grad_shard_stats_kernel<float><<<grid, kOptThreads, 0, stream>>>(table, n, row_tiles, inv_scale, norm_inf, partial, partial_flag, ticket, out);
  else if (grad_dtype == 10) grad_shard_stats_kernel<__nv_bfloat16><<<grid, kOptThreads, 0, stream>>>(table, n, row_tiles, inv_scale, norm_inf, partial, partial_flag, ticket, out);
  else if (grad_dtype == 6) grad_shard_stats_kernel<__half><<<grid, kOptThreads, 0, stream>>>(table, n, row_tiles, inv_scale, norm_inf, partial, partial_flag, ticket, out);
  else return cudaErrorInvalidValue;
  CountKernelLaunch();
  return cudaGetLastError();
}

cudaError_t LaunchGradAccumulate(const AccTable& table, int64_t max_count, int mode, int grad_dtype, cudaStream_t stream) {
  if (table.n <= 0 || max_count <= 0) return cudaSuccess;
  if (table.n > kAccMaxTensors || mode < kAccFirst || mode > kAccLast) return cudaErrorInvalidValue;
  dim3 grid((unsigned)((max_count + kOptPerBlock - 1) / kOptPerBlock), (unsigned)table.n);
  if (grad_dtype == 10) grad_accumulate_kernel<__nv_bfloat16><<<grid, kOptThreads, 0, stream>>>(table, mode);
  else if (grad_dtype == 6) grad_accumulate_kernel<__half><<<grid, kOptThreads, 0, stream>>>(table, mode);
  else return cudaErrorInvalidValue;
  CountKernelLaunch();
  return cudaGetLastError();
}

}  // namespace kern
}  // namespace hvd
