// Adasum (adaptive summation) on GPUs over peer-mapped symmetric buffers, sm_90a.
//
// The reference only has a CPU implementation of the pairwise Adasum reduction
// (ops/adasum/adasum.h:195-435, vector-halving distance-doubling over MPI); its
// "GPU Adasum" inside one node is an NCCL sum divided by local_size
// (ops/adasum_gpu_operations.cc).  Here all log2(N) VHDD levels run on the GPUs:
//   pack      tensors -> fp32 fused vector in my symmetric buffer (prescale)
//   level l   partner = rank ^ 2^l; I keep one half K of my current segment.
//     dots    for K: a = lower group's copy, b = upper group's copy, where the
//             partner's copy is read DIRECTLY from its buffer over NVLink;
//             per-tensor partial <a,b>, |a|^2, |b|^2 accumulate in fp64 into a
//             scratch table that lives in symmetric memory
//     combine every rank sums the partials of the 2^(l+1) ranks that jointly hold
//             the vector pair (peer loads of their scratch tables), derives
//             acoeff = 1 - <a,b>/(2|a|^2), bcoeff = 1 - <a,b>/(2|b|^2) per tensor
//             and overwrites K with acoeff*a + bcoeff*b (again pulling b / a
//             from the partner's buffer)
//   gather    every rank pulls every other rank's final 1/N slice, applies
//             postscale, casts and scatters into the output tensors.
// Every kernel begins with the CTA-index flag barrier; together with stream
// order on each GPU this orders all cross-GPU reads after the writes they need.
#include "p2p_common.cuh"

namespace hvd {
namespace kern {
namespace {

constexpr int kRow = kThreads * 16;
constexpr int kAChunk = 16384;

template <typename F>
__device__ __forceinline__ void for_my_chunks(int64_t lo_b, int64_t hi_b, int cta, int grid, F f) {
  // first chunk >= lo_b / kAChunk owned by this CTA, then every grid-th one (a 64-bit modulo per chunk per thread made
  // this walk cost more than the copies: measured 10x on the exchange kernel, which shared the pattern)
  const int64_t c0 = lo_b / kAChunk;
  for (int64_t c = c0 + ((cta - (int)(c0 % grid) + grid) % grid); c * kAChunk < hi_b; c += grid) {
    int64_t lo = c * kAChunk, hi = lo + kAChunk;
    if (lo < lo_b) lo = lo_b;
    if (hi > hi_b) hi = hi_b;
    if (lo < hi) f(lo, hi);
  }
}

__device__ __forceinline__ float4 ld_f4(const void* p) {
  uint4 v = ld_stream(p);
  return make_float4(__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z), __uint_as_float(v.w));
}
__device__ __forceinline__ void st_f4(void* p, float4 f) {
  st_stream(p, make_uint4(__float_as_uint(f.x), __float_as_uint(f.y), __float_as_uint(f.z), __float_as_uint(f.w)));
}

// ---- pack: T -> fp32 fused vector -------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads, 2)
adasum_pack_kernel(const __grid_constant__ CommParams cp, const TensorDesc* __restrict__ descs, int nd, int64_t total, float prescale) {
  const int cta = blockIdx.x, grid = gridDim.x;
  char* buf = reinterpret_cast<char*>(cp.buf[cp.rank]);
  DescCursor cur;
  cur.init(descs, nd, total);
  for_my_chunks(0, total, cta, grid, [&](int64_t lo, int64_t hi) {
    for (int64_t o = lo + (int64_t)threadIdx.x * 16; o < hi; o += kRow) {
      cur.seek(o);
      const TensorDesc& d = cur.d[cur.i];
      const int64_t e = (o - cur.lo) / 4;
      float a[4];
      load_elems<T, 4, float>(reinterpret_cast<const T*>(d.in) + e, d.count - e, a);
      st_f4(buf + o, make_float4(a[0] * prescale, a[1] * prescale, a[2] * prescale, a[3] * prescale));
    }
  });
}

// ---- level phase 1: partial dot products ---------------------------------------------
__global__ void __launch_bounds__(kThreads, 2)
adasum_dots_kernel(const __grid_constant__ CommParams cp, const TensorDesc* __restrict__ descs, int nd, int64_t total,
                   int64_t keep_lo, int64_t keep_hi, int partner, int lower, double* __restrict__ scratch) {
  extern __shared__ double s_acc[];  // [3 * nd]
  const int cta = blockIdx.x, grid = gridDim.x;
  uint32_t epoch = cp.epochs[cta];
  for (int i = threadIdx.x; i < 3 * nd; i += kThreads) s_acc[i] = 0.0;
  const bool alive = peer_barrier(cp, epoch, cta);  // also orders the smem zeroing (it ends with __syncthreads)
  const char* mine = reinterpret_cast<const char*>(cp.buf[cp.rank]);
  const char* theirs = reinterpret_cast<const char*>(cp.buf[partner]);
  DescCursor cur;
  cur.init(descs, nd, total);
  int t_cur = -1;
  double dab = 0, daa = 0, dbb = 0;
  auto flush = [&]() {
    if (t_cur >= 0 && (dab != 0 || daa != 0 || dbb != 0)) {
      atomicAdd(&s_acc[3 * t_cur], dab); atomicAdd(&s_acc[3 * t_cur + 1], daa); atomicAdd(&s_acc[3 * t_cur + 2], dbb);
    }
    dab = daa = dbb = 0;
  };
  if (alive) {
    for_my_chunks(keep_lo, keep_hi, cta, grid, [&](int64_t lo, int64_t hi) {
      for (int64_t o = lo + (int64_t)threadIdx.x * 16; o < hi; o += kRow) {
        const float4 m = ld_f4(mine + o), p = ld_f4(theirs + o);
        cur.seek(o);
        if (cur.i != t_cur) { flush(); t_cur = cur.i; }
        const float4 a = lower ? m : p, b = lower ? p : m;
        dab += (double)a.x * b.x + (double)a.y * b.y + (double)a.z * b.z + (double)a.w * b.w;
        daa += (double)a.x * a.x + (double)a.y * a.y + (double)a.z * a.z + (double)a.w * a.w;
        dbb += (double)b.x * b.x + (double)b.y * b.y + (double)b.z * b.z + (double)b.w * b.w;
      }
    });
  }
  flush();
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * nd; i += kThreads) if (s_acc[i] != 0.0) atomicAdd(&scratch[i], s_acc[i]);
  if (threadIdx.x == 0) cp.epochs[cta] = epoch;
}

// ---- level phase 2: coefficients + in-place combine of my half ----------------------------
__global__ void __launch_bounds__(kThreads, 2)
adasum_combine_kernel(const __grid_constant__ CommParams cp, const TensorDesc* __restrict__ descs, int nd, int64_t total,
                      int64_t keep_lo, int64_t keep_hi, int partner, int lower, int group_base, int group_size,
                      int64_t scratch_byte_off) {
  extern __shared__ float s_coef[];  // [2 * nd]: acoeff, bcoeff
  const int cta = blockIdx.x, grid = gridDim.x;
  uint32_t epoch = cp.epochs[cta];
  const bool alive = peer_barrier(cp, epoch, cta);
  if (alive) {
    for (int t = threadIdx.x; t < nd; t += kThreads) {
      double dab = 0, daa = 0, dbb = 0;
      for (int g = 0; g < group_size; ++g) {
        const double* s = reinterpret_cast<const double*>(reinterpret_cast<const char*>(cp.flags[group_base + g]) + scratch_byte_off);
        dab += s[3 * t]; daa += s[3 * t + 1]; dbb += s[3 * t + 2];
      }
      const double tiny = 1.4916681462400413e-154;  // sqrt(DBL_MIN), as in the reference (adasum.h:397-404)
      s_coef[2 * t] = daa >= tiny ? (float)(1.0 - dab / (2.0 * daa)) : 1.f;
      s_coef[2 * t + 1] = dbb >= tiny ? (float)(1.0 - dab / (2.0 * dbb)) : 1.f;
    }
  }
  __syncthreads();
  char* mine = reinterpret_cast<char*>(cp.buf[cp.rank]);
  const char* theirs = reinterpret_cast<const char*>(cp.buf[partner]);
  DescCursor cur;
  cur.init(descs, nd, total);
  if (alive) {
    for_my_chunks(keep_lo, keep_hi, cta, grid, [&](int64_t lo, int64_t hi) {
      for (int64_t o = lo + (int64_t)threadIdx.x * 16; o < hi; o += kRow) {
        const float4 m = ld_f4(mine + o), p = ld_f4(theirs + o);
        cur.seek(o);
        const float ac = s_coef[2 * cur.i], bc = s_coef[2 * cur.i + 1];
        const float4 a = lower ? m : p, b = lower ? p : m;
        st_f4(mine + o, make_float4(ac * a.x + bc * b.x, ac * a.y + bc * b.y, ac * a.z + bc * b.z, ac * a.w + bc * b.w));
      }
    });
  }
  if (threadIdx.x == 0) cp.epochs[cta] = epoch;
}

// ---- final: pull every rank's slice, postscale, cast, scatter --------------------------------
struct GatherRanges { int64_t lo[kMaxPeers]; int64_t hi[kMaxPeers]; };

template <typename T>
__global__ void __launch_bounds__(kThreads, 2)
adasum_gather_kernel(const __grid_constant__ CommParams cp, const TensorDesc* __restrict__ descs, int nd, int64_t total,
                     const __grid_constant__ GatherRanges rg, float postscale) {
  const int cta = blockIdx.x, grid = gridDim.x;
  uint32_t epoch = cp.epochs[cta];
  const bool alive = peer_barrier(cp, epoch, cta);
  DescCursor cur;
  cur.init(descs, nd, total);
  for (int k = 0; k < cp.nranks && alive; ++k) {
    int p = cp.rank + k; if (p >= cp.nranks) p -= cp.nranks;
    const char* src = reinterpret_cast<const char*>(cp.buf[p]);
    cur.i = -1;
    for_my_chunks(rg.lo[p], rg.hi[p], cta, grid, [&](int64_t lo, int64_t hi) {
      for (int64_t o = lo + (int64_t)threadIdx.x * 16; o < hi; o += kRow) {
        const float4 v = ld_f4(src + o);
        cur.seek(o);
        const TensorDesc& d = cur.d[cur.i];
        const int64_t e = (o - cur.lo) / 4;
        if (e >= d.count) continue;
        float a[4] = {v.x * postscale, v.y * postscale, v.z * postscale, v.w * postscale};
        store_elems<T, 4, float>(reinterpret_cast<T*>(d.out) + e, d.count - e, a);
      }
    });
  }
  if (threadIdx.x == 0) cp.epochs[cta] = epoch;
}

// =====================================================================================================================
// Persistent variant: the WHOLE Adasum (pack, log2(N) x {dots, reduce, combine}, gather) is ONE kernel.
//
// The multi-launch sequence above costs 2 + 2 log2(N) launches and log2(N) memsets per response, each launch starting
// with a cross-GPU barrier, and sums its partial dot products with fp64 atomicAdd (run-to-run differences in the last
// bits).  Here the grid stays resident and synchronises itself: a grid-wide barrier (arrival counter + generation word in
// local memory) whose LAST arriving CTA also performs the cross-GPU flag barrier on behalf of the whole grid.  Work is
// split into CONTIGUOUS per-CTA byte ranges (phases are separated by grid barriers, so the chunk -> CTA mapping no longer
// has to agree between phases), which makes a CTA touch only the few tensors its range overlaps:
//   * per-CTA partial dots are reduced inside the CTA in a fixed order (warp shuffles, then warp 0 .. 7 in order) at every
//     tensor boundary and written to a local table [cta][tensor];
//   * after a grid barrier, tensor t is summed over the CTAs in ascending CTA order and published to this rank's scratch
//     table in symmetric memory (every entry is written: no memset);
//   * after a grid + peer barrier every CTA derives the coefficients of the tensors its combine range touches by summing
//     the group's ranks in ascending rank order.
// Fixed orders everywhere: the result is bit-reproducible.  All CTAs must be co-resident (grid <= 2 x SM count).
struct GridSync { uint32_t count; uint32_t gen; uint32_t abort; uint32_t pad; };

__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t atom_add_acqrel_gpu(uint32_t* p, uint32_t v) {
  uint32_t old;
  asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}

// Grid-wide barrier; with `with_peers` the last arriving CTA runs the cross-GPU flag barrier (flag slot 0) before it
// releases the grid.  Returns false once any barrier was abandoned (peer failure / timeout): every CTA then leaves.
__device__ __forceinline__ bool grid_barrier(const CommParams& cp, GridSync* gs, bool with_peers) {
  __shared__ uint32_t s_gen;
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    s_gen = ld_acquire_gpu(&gs->gen);
    __threadfence_system();  // this CTA's writes (ordered before by the __syncthreads) are visible to peers before it arrives
    s_last = atom_add_acqrel_gpu(&gs->count, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (s_last) {
    bool alive = true;
    if (with_peers && cp.nranks > 1) {
      uint32_t epoch = cp.epochs[0];
      alive = peer_barrier(cp, epoch, 0);
      if (threadIdx.x == 0) cp.epochs[0] = epoch;
    }
    if (threadIdx.x == 0) {
      if (!alive) *reinterpret_cast<volatile uint32_t*>(&gs->abort) = 1u;
      *reinterpret_cast<volatile uint32_t*>(&gs->count) = 0u;
      __threadfence();
      st_release_gpu(&gs->gen, s_gen + 1u);
    }
  } else if (threadIdx.x == 0) {
    while (ld_acquire_gpu(&gs->gen) == s_gen) {}
  }
  __syncthreads();
  return *reinterpret_cast<volatile uint32_t*>(&gs->abort) == 0u;
}

// Deterministic CTA-wide sum of three doubles; the total lands in thread 0 (other threads get garbage).
__device__ __forceinline__ void block_sum3(double& a, double& b, double& c, double (*s_red)[3]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
  }
  const int w = threadIdx.x >> 5;
  __syncthreads();  // s_red may still be read by thread 0 from the previous call
  if ((threadIdx.x & 31) == 0) { s_red[w][0] = a; s_red[w][1] = b; s_red[w][2] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    a = b = c = 0;
    for (int k = 0; k < kThreads / 32; ++k) { a += s_red[k][0]; b += s_red[k][1]; c += s_red[k][2]; }
  }
}

struct PersistArgs {
  const TensorDesc* descs; int nd;
  int64_t total;
  float prescale, postscale;
  double* partials;      // [grid][3 * nd]   per-CTA partial dots of the current level (local)
  int2* ranges;          // [grid]           tensors a CTA's partials cover: [x, y], x > y = none
  GridSync* gs;
  int64_t scratch_stride;
  GatherRanges rg;
};

// contiguous slice of [lo, hi) owned by this CTA (row = 4 KiB granularity)
__device__ __forceinline__ void cta_slice(int64_t lo, int64_t hi, int64_t& slo, int64_t& shi) {
  const int64_t rows = (hi - lo + kRow - 1) / kRow;
  const int64_t per = (rows + gridDim.x - 1) / gridDim.x;
  slo = lo + (int64_t)blockIdx.x * per * kRow;
  shi = slo + per * kRow;
  if (slo > hi) slo = hi;
  if (shi > hi) shi = hi;
}

template <typename T>
__global__ void __launch_bounds__(kThreads, 2)
adasum_persistent_kernel(const __grid_constant__ CommParams cp, const __grid_constant__ PersistArgs a) {
  extern __shared__ double s_dyn[];         // dots: [3 * nd] doubles; combine: reused as [2 * nd] floats
  __shared__ double s_red[kThreads / 32][3];
  const int n = cp.nranks, rank = cp.rank, nd = a.nd;
  const int64_t total = a.total;
  char* mine = reinterpret_cast<char*>(cp.buf[rank]);
  DescCursor cur;
  int64_t slo, shi;

  // ---- pack: tensors -> fp32 fused vector in my symmetric buffer ----
  constexpr int UP = 4;  // rows per trip: UP independent 16 B loads per thread in flight (HBM ~0.7 us, NVLink ~2 us round trips)
  cta_slice(0, total, slo, shi);
  cur.init(a.descs, nd, total);
  for (int64_t o0 = slo + (int64_t)threadIdx.x * 16; o0 < shi; o0 += (int64_t)UP * kRow) {
    float v[UP][4];
#pragma unroll
    for (int j = 0; j < UP; ++j) {
      const int64_t o = o0 + (int64_t)j * kRow;
      if (o < shi) {
        cur.seek(o);
        const int64_t e = (o - cur.lo) / 4;
        load_elems<T, 4, float>(reinterpret_cast<const T*>(cur.in) + e, cur.count - e, v[j]);
      }
    }
#pragma unroll
    for (int j = 0; j < UP; ++j) {
      const int64_t o = o0 + (int64_t)j * kRow;
      if (o < shi) st_f4(mine + o, make_float4(v[j][0] * a.prescale, v[j][1] * a.prescale, v[j][2] * a.prescale, v[j][3] * a.prescale));
    }
  }

  int64_t lo = 0, hi = total;
  int level = 0;
  for (int d = 1; d < n; d <<= 1, ++level) {
    if (!grid_barrier(cp, a.gs, true)) return;  // every rank's vector (packed, or combined at the previous level) is final
    const int partner = rank ^ d;
    const bool lower = (rank & d) == 0;
    const int64_t mid = lo + (((hi - lo) / 2) & ~(int64_t)15);
    const int64_t klo = lower ? lo : mid, khi = lower ? mid : hi;
    const char* theirs = reinterpret_cast<const char*>(cp.buf[partner]);
    cta_slice(klo, khi, slo, shi);

    // ---- dots over my slice, reduced per tensor in a fixed order ----
    cur.init(a.descs, nd, total);
    int t_cur = -1, t_min = 0x7fffffff, t_max = -1;
    double dab = 0, daa = 0, dbb = 0;
    auto flush = [&](int t) {  // CTA-uniform call: folds the running partials into tensor t
      block_sum3(dab, daa, dbb, s_red);
      if (threadIdx.x == 0) {
        if (t > t_max) { for (int q = (t_max < 0 ? t : t_max + 1); q <= t; ++q) { s_dyn[3 * q] = 0; s_dyn[3 * q + 1] = 0; s_dyn[3 * q + 2] = 0; } }
        s_dyn[3 * t] += dab; s_dyn[3 * t + 1] += daa; s_dyn[3 * t + 2] += dbb;
      }
      if (t < t_min) t_min = t;
      if (t > t_max) t_max = t;
      dab = daa = dbb = 0;
    };
    for (int64_t row = slo; row < shi; row += kRow) {
      // fast path: the next UP rows lie inside ONE tensor -> UP x 2 loads per thread in flight, no boundary handling
      cur.seek(row);
      {
        const int64_t span_end = row + (int64_t)UP * kRow <= shi ? row + (int64_t)UP * kRow : shi;
        if (span_end - row > kRow && span_end - 16 < cur.hi) {
          const int t_span = cur.i;
          if (t_cur != t_span) { if (t_cur >= 0) flush(t_cur); t_cur = t_span; }
          float4 m[UP], p[UP];
#pragma unroll
          for (int j = 0; j < UP; ++j) {
            const int64_t o = row + (int64_t)j * kRow + (int64_t)threadIdx.x * 16;
            if (o < span_end) { m[j] = ld_f4(mine + o); p[j] = ld_f4(theirs + o); }
          }
#pragma unroll
          for (int j = 0; j < UP; ++j) {
            const int64_t o = row + (int64_t)j * kRow + (int64_t)threadIdx.x * 16;
            if (o < span_end) {
              const float4 x = lower ? m[j] : p[j], y = lower ? p[j] : m[j];
              dab += (double)x.x * y.x + (double)x.y * y.y + (double)x.z * y.z + (double)x.w * y.w;
              daa += (double)x.x * x.x + (double)x.y * x.y + (double)x.z * x.z + (double)x.w * x.w;
              dbb += (double)y.x * y.x + (double)y.y * y.y + (double)y.z * y.z + (double)y.w * y.w;
            }
          }
          row += span_end - row - kRow;  // (the loop header adds the last kRow)
          continue;
        }
      }
      // tensors at the first and last vector of this row (identical on every thread)
      const int t_first = cur.i;
      const int64_t last = (row + kRow <= shi ? row + kRow : shi) - 16;
      int t_last = t_first;
      if (last >= cur.hi) { DescCursor c2 = cur; c2.seek(last); t_last = c2.i; }
      const int64_t o = row + (int64_t)threadIdx.x * 16;
      double pab = 0, paa = 0, pbb = 0;
      int t_mine = t_first;
      if (o < shi) {
        const float4 m = ld_f4(mine + o), p = ld_f4(theirs + o);
        const float4 x = lower ? m : p, y = lower ? p : m;
        pab = (double)x.x * y.x + (double)x.y * y.y + (double)x.z * y.z + (double)x.w * y.w;
        paa = (double)x.x * x.x + (double)x.y * x.y + (double)x.z * x.z + (double)x.w * x.w;
        pbb = (double)y.x * y.x + (double)y.y * y.y + (double)y.z * y.z + (double)y.w * y.w;
        if (t_last != t_first) { DescCursor c3 = cur; c3.seek(o); t_mine = c3.i; }
      }
      if (t_first == t_last) {
        if (t_cur != t_first) { if (t_cur >= 0) flush(t_cur); t_cur = t_first; }
        dab += pab; daa += paa; dbb += pbb;
      } else {
        // a tensor boundary inside the row: close the running tensor, then one reduction per tensor of the row
        if (t_cur >= 0) flush(t_cur);
        for (int t = t_first; t <= t_last; ++t) {
          const bool sel = o < shi && t_mine == t;
          dab = sel ? pab : 0; daa = sel ? paa : 0; dbb = sel ? pbb : 0;
          flush(t);
        }
        t_cur = -1;
      }
    }
    if (t_cur >= 0) flush(t_cur);
    __syncthreads();
    if (threadIdx.x == 0) a.ranges[blockIdx.x] = make_int2(t_max >= 0 ? t_min : 1, t_max >= 0 ? t_max : 0);
    if (t_max >= 0) {
      double* out = a.partials + (size_t)blockIdx.x * 3 * nd;
      for (int i = 3 * t_min + threadIdx.x; i < 3 * (t_max + 1); i += kThreads) out[i] = s_dyn[i];
    }
    if (!grid_barrier(cp, a.gs, false)) return;

    // ---- this rank's totals: tensor t summed over the CTAs in ascending order, published to symmetric scratch ----
    const int64_t soff = kFlagWords * 4 + (int64_t)(level & 1) * a.scratch_stride;
    double* scratch = reinterpret_cast<double*>(reinterpret_cast<char*>(cp.flags[rank]) + soff);
    for (int t = blockIdx.x * kThreads + threadIdx.x; t < nd; t += gridDim.x * kThreads) {
      double sab = 0, saa = 0, sbb = 0;
      for (int b = 0; b < (int)gridDim.x; ++b) {
        const int2 rg = a.ranges[b];
        if (t >= rg.x && t <= rg.y) {
          const double* pp = a.partials + (size_t)b * 3 * nd + 3 * t;
          sab += pp[0]; saa += pp[1]; sbb += pp[2];
        }
      }
      scratch[3 * t] = sab; scratch[3 * t + 1] = saa; scratch[3 * t + 2] = sbb;
    }
    if (!grid_barrier(cp, a.gs, true)) return;  // every rank of the group published its totals

    // ---- coefficients of the tensors my combine slice touches, then the combine itself ----
    float* s_coef = reinterpret_cast<float*>(s_dyn);
    int c_first = 0, c_last = -1;
    if (slo < shi) {
      DescCursor c4; c4.init(a.descs, nd, total);
      c4.seek(slo); c_first = c4.i;
      c4.seek(shi - 16); c_last = c4.i;
    }
    const int group_base = rank & ~(2 * d - 1), group_size = 2 * d;
    for (int t = c_first + threadIdx.x; t <= c_last; t += kThreads) {
      double sab = 0, saa = 0, sbb = 0;
      for (int g = 0; g < group_size; ++g) {
        const double* sp = reinterpret_cast<const double*>(reinterpret_cast<const char*>(cp.flags[group_base + g]) + soff);
        sab += sp[3 * t]; saa += sp[3 * t + 1]; sbb += sp[3 * t + 2];
      }
      const double tiny = 1.4916681462400413e-154;  // sqrt(DBL_MIN), as in the reference (adasum.h:397-404)
      s_coef[2 * t] = saa >= tiny ? (float)(1.0 - sab / (2.0 * saa)) : 1.f;
      s_coef[2 * t + 1] = sbb >= tiny ? (float)(1.0 - sab / (2.0 * sbb)) : 1.f;
    }
    __syncthreads();
    cur.init(a.descs, nd, total);
    for (int64_t o0 = slo + (int64_t)threadIdx.x * 16; o0 < shi; o0 += (int64_t)UP * kRow) {
      float4 m[UP], p[UP];
#pragma unroll
      for (int j = 0; j < UP; ++j) {
        const int64_t o = o0 + (int64_t)j * kRow;
        if (o < shi) { m[j] = ld_f4(mine + o); p[j] = ld_f4(theirs + o); }
      }
#pragma unroll
      for (int j = 0; j < UP; ++j) {
        const int64_t o = o0 + (int64_t)j * kRow;
        if (o < shi) {
          cur.seek(o);
          const float ac = s_coef[2 * cur.i], bc = s_coef[2 * cur.i + 1];
          const float4 x = lower ? m[j] : p[j], y = lower ? p[j] : m[j];
          st_f4(mine + o, make_float4(ac * x.x + bc * y.x, ac * x.y + bc * y.y, ac * x.z + bc * y.z, ac * x.w + bc * y.w));
        }
      }
    }
    lo = klo; hi = khi;
  }

  // ---- gather: pull every rank's final slice, postscale, cast, scatter into the output tensors ----
  if (!grid_barrier(cp, a.gs, true)) return;
  for (int k = 0; k < n; ++k) {
    int p = rank + k; if (p >= n) p -= n;
    const char* src = reinterpret_cast<const char*>(cp.buf[p]);
    cta_slice(a.rg.lo[p], a.rg.hi[p], slo, shi);
    cur.init(a.descs, nd, total);
    for (int64_t o0 = slo + (int64_t)threadIdx.x * 16; o0 < shi; o0 += (int64_t)UP * kRow) {
      float4 v[UP];
#pragma unroll
      for (int j = 0; j < UP; ++j) {
        const int64_t o = o0 + (int64_t)j * kRow;
        if (o < shi) v[j] = ld_f4(src + o);
      }
#pragma unroll
      for (int j = 0; j < UP; ++j) {
        const int64_t o = o0 + (int64_t)j * kRow;
        if (o < shi) {
          cur.seek(o);
          const int64_t e = (o - cur.lo) / 4;
          if (e < cur.count) {
            float w[4] = {v[j].x * a.postscale, v[j].y * a.postscale, v[j].z * a.postscale, v[j].w * a.postscale};
            store_elems<T, 4, float>(reinterpret_cast<T*>(cur.out) + e, cur.count - e, w);
          }
        }
      }
    }
  }
  // a rank may only reuse this buffer slot after every peer finished pulling from it
  grid_barrier(cp, a.gs, true);
}

template <typename T>
cudaError_t run_adasum_persistent(const CommParams& cp, const AdasumArgs& a, double prescale, double postscale, cudaStream_t s) {
  const int n = cp.nranks;
  PersistArgs pa {};
  pa.descs = a.descs; pa.nd = a.ndesc; pa.total = a.total_bytes;
  pa.prescale = (float)prescale; pa.postscale = (float)postscale;
  pa.partials = reinterpret_cast<double*>(a.persist_scratch);
  pa.ranges = reinterpret_cast<int2*>(reinterpret_cast<char*>(a.persist_scratch) + (size_t)a.ctas * 3 * a.ndesc * sizeof(double));
  pa.gs = reinterpret_cast<GridSync*>(a.persist_sync);
  pa.scratch_stride = a.scratch_stride_bytes;
  for (int p = 0; p < n; ++p) {
    int64_t lo = 0, hi = a.total_bytes;
    for (int d = 1; d < n; d <<= 1) {
      int64_t mid = lo + (((hi - lo) / 2) & ~(int64_t)15);
      if ((p & d) == 0) hi = mid; else lo = mid;
    }
    pa.rg.lo[p] = lo; pa.rg.hi[p] = hi;
  }
  const size_t smem = (size_t)3 * a.ndesc * sizeof(double);
  cudaError_t e = cudaMemsetAsync(a.persist_sync, 0, sizeof(GridSync), s);
  if (e != cudaSuccess) return e;
  adasum_persistent_kernel<T><<<a.ctas, kThreads, smem, s>>>(cp, pa);
  CountKernelLaunch();
  return cudaGetLastError();
}

// `only` < 0: the whole sequence (production: one GPU per process).  `only` = k: just the k-th launch of the sequence
// (pack = 0, dots/combine of level l = 1 + 2l / 2 + 2l, gather last) — the single-GPU simulation issues launch k of
// EVERY rank before launch k+1 of any rank, otherwise streams that share a hardware queue deadlock (a kernel spinning in
// its barrier sits in front of the peer kernel it is waiting for).
template <typename T>
cudaError_t run_adasum(const CommParams& cp, const AdasumArgs& a, double prescale, double postscale, cudaStream_t s, int only) {
  const int n = cp.nranks, rank = cp.rank;
  const int64_t total = a.total_bytes;
  int step = 0;
  if (only < 0 || only == step) {
    adasum_pack_kernel<T><<<a.ctas, kThreads, 0, s>>>(cp, a.descs, a.ndesc, total, (float)prescale);
    CountKernelLaunch();
  }
  ++step;
  // replay the halving for every rank (element granularity: 4 floats = one 16 B vector)
  GatherRanges rg;
  for (int p = 0; p < n; ++p) {
    int64_t lo = 0, hi = total;
    for (int d = 1; d < n; d <<= 1) {
      int64_t mid = lo + (((hi - lo) / 2) & ~(int64_t)15);
      if ((p & d) == 0) hi = mid; else lo = mid;
    }
    rg.lo[p] = lo; rg.hi[p] = hi;
  }
  int64_t lo = 0, hi = total;
  int level = 0;
  const size_t dots_smem = (size_t)3 * a.ndesc * sizeof(double), coef_smem = (size_t)2 * a.ndesc * sizeof(float);
  for (int d = 1; d < n; d <<= 1, ++level) {
    const int partner = rank ^ d, lower = (rank & d) == 0;
    const int64_t mid = lo + (((hi - lo) / 2) & ~(int64_t)15);
    const int64_t klo = lower ? lo : mid, khi = lower ? mid : hi;
    const int64_t off = kFlagWords * 4 + (int64_t)(level & 1) * a.scratch_stride_bytes;
    double* scratch = reinterpret_cast<double*>(reinterpret_cast<char*>(cp.flags[rank]) + off);
    if (only < 0 || only == step) {
      cudaError_t e = cudaMemsetAsync(scratch, 0, (size_t)3 * a.ndesc * sizeof(double), s);
      if (e != cudaSuccess) return e;
      adasum_dots_kernel<<<a.ctas, kThreads, dots_smem, s>>>(cp, a.descs, a.ndesc, total, klo, khi, partner, lower, scratch);
      CountKernelLaunch();
    }
    ++step;
    if (only < 0 || only == step) {
      adasum_combine_kernel<<<a.ctas, kThreads, coef_smem, s>>>(cp, a.descs, a.ndesc, total, klo, khi, partner, lower,
                                                                 rank & ~(2 * d - 1), 2 * d, off);
      CountKernelLaunch();
    }
    ++step;
    lo = klo; hi = khi;
  }
  if (only < 0 || only == step) {
    adasum_gather_kernel<T><<<a.ctas, kThreads, 0, s>>>(cp, a.descs, a.ndesc, total, rg, (float)postscale);
    CountKernelLaunch();
  }
  return cudaGetLastError();
}

}  // namespace

int AdasumNumLaunches(int nranks) {
  int levels = 0;
  for (int d = 1; d < nranks; d <<= 1) ++levels;
  return 2 + 2 * levels;
}

cudaError_t LaunchAdasum(const CommParams& cp, const AdasumArgs& args, double prescale, double postscale, cudaStream_t stream) {
  return LaunchAdasumStep(cp, args, prescale, postscale, stream, -1);
}

size_t AdasumPersistentScratchBytes(int ctas, int ndesc) { return (size_t)ctas * 3 * ndesc * sizeof(double) + (size_t)ctas * sizeof(int2); }
size_t AdasumPersistentSyncBytes() { return sizeof(GridSync); }

cudaError_t LaunchAdasumStep(const CommParams& cp, const AdasumArgs& args, double prescale, double postscale, cudaStream_t stream,
                             int only) {
  if (args.ctas < 1 || args.ctas > kMaxCtas || (cp.nranks & (cp.nranks - 1))) return cudaErrorInvalidValue;
  if (args.ndesc > kAdasumMaxTensors) return cudaErrorInvalidValue;  // smem / scratch table bound
  if (args.persist_scratch && args.persist_sync) {
    if (only > 0) return cudaSuccess;  // (simulation driver: the single launch is step 0)
    switch (args.dtype) {
      case 7: return run_adasum_persistent<float>(cp, args, prescale, postscale, stream);
      case 6: return run_adasum_persistent<__half>(cp, args, prescale, postscale, stream);
      case 10: return run_adasum_persistent<__nv_bfloat16>(cp, args, prescale, postscale, stream);
      default: return cudaErrorInvalidValue;
    }
  }
  switch (args.dtype) {
    case 7: return run_adasum<float>(cp, args, prescale, postscale, stream, only);
    case 6: return run_adasum<__half>(cp, args, prescale, postscale, stream, only);
    case 10: return run_adasum<__nv_bfloat16>(cp, args, prescale, postscale, stream, only);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace kern
}  // namespace hvd
