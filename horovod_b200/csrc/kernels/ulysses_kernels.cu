// Ulysses sequence-parallel exchange (hvd.UlyssesExchange): sequence shards <-> head shards in one launch on a
// peer-mapped team (sm_90a), with the layout change folded into the copy.
//
// In the view [A, D1, M, D2, R] of the input (p2p_kernels.h), the block that rank p sends to rank q is a 3-D grid of
// contiguous runs of L bytes, with linear strides both in p's input and in q's output, and every (q, p) block has the
// same grid.  So one copy routine over (run j, piece k) items serves both directions and both dim orders.  Per CTA b of
// every rank:
//
//   1. stage: the items of CTA b of every block q != me of the input into block q of this rank's registered staging
//      buffer (runs packed), and block me straight into the output;
//   2. publish {direction, head_first, A, D1, M, D2, R, elem_bytes, staging_offset} into row b of the count region, and
//      barrier A with CTA b of every peer;
//   3. verdict: every rank published the same shape (integer compares in a fixed order: every rank agrees);
//   4. pull: the items of CTA b of block me from every peer's staging buffer into the output (or, on a mismatch, zero
//      the items of CTA b of every output block);
//   5. barrier B: no rank returns, and so overwrites its staging buffer or its count row, while a peer still reads them.
//
// Item t of a block belongs to CTA t % grid in every block, on every rank, and in both phases: the pull of CTA b reads
// exactly the bytes that CTA b of the sender staged, which is all that peer_barrier orders.
#include "p2p_common.cuh"

namespace hvd {
namespace kern {
namespace {

constexpr int64_t kUlyPieceBytes = 8192;  // the longest piece of a run that one lane group copies as one item
constexpr int kUlyUnroll = 4;             // units in flight per lane

__device__ __forceinline__ int64_t ld_volatile_s64(const int64_t* p) { return *reinterpret_cast<const volatile int64_t*>(p); }

template <int U> struct UnitOf;
template <> struct UnitOf<16> { using T = uint4; };
template <> struct UnitOf<8> { using T = uint2; };
template <> struct UnitOf<4> { using T = uint32_t; };
template <> struct UnitOf<2> { using T = uint16_t; };
template <> struct UnitOf<1> { using T = uint8_t; };

template <int U> __device__ __forceinline__ typename UnitOf<U>::T ld_unit(const char* p) {
  if constexpr (U == 16) return ld_stream(p);
  else return *reinterpret_cast<const typename UnitOf<U>::T*>(p);
}
template <int U> __device__ __forceinline__ void st_unit(char* p, const typename UnitOf<U>::T& v) {
  if constexpr (U == 16) st_stream(p, v);
  else *reinterpret_cast<typename UnitOf<U>::T*>(p) = v;
}
template <int U> __device__ __forceinline__ typename UnitOf<U>::T zero_unit() {
  if constexpr (U == 16) return make_uint4(0, 0, 0, 0);
  else if constexpr (U == 8) return make_uint2(0, 0);
  else return 0;
}

// The items of one block that this CTA owns, copied in units of U bytes (U divides the run length and both bases) by
// groups of G lanes, one item per group at a time.  src == nullptr stores zeros.
template <int U>
__device__ __forceinline__ void copy_items(const char* src, const int64_t* ss, char* dst, const int64_t* ds,
                                           const UlyssesGeometry& g, int cta, int grid) {
  using T = typename UnitOf<U>::T;
  const int64_t L = g.run_bytes;
  const int64_t pieces = (L + kUlyPieceBytes - 1) / kUlyPieceBytes;
  const int64_t items = g.nruns * pieces;
  const int64_t units = (L < kUlyPieceBytes ? L : kUlyPieceBytes) / U;  // units of the longest item
  int G = 1;
  while (G < 32 && G < units) G <<= 1;
  const int groups = kThreads / G, group = threadIdx.x / G, lane = threadIdx.x % G;
  for (int64_t t = cta + (int64_t)grid * group; t < items; t += (int64_t)grid * groups) {
    const int64_t j = t / pieces, piece = t - j * pieces;
    const int64_t m = j % g.nm, ai = j / g.nm, i = ai % g.ni, a = ai / g.ni;
    const int64_t off = piece * kUlyPieceBytes;
    const int64_t nu = ((L - off) < kUlyPieceBytes ? (L - off) : kUlyPieceBytes) / U;
    char* d = dst + a * ds[0] + i * ds[1] + m * ds[2] + off;
    const char* s = src ? src + a * ss[0] + i * ss[1] + m * ss[2] + off : nullptr;
    for (int64_t u0 = lane; u0 < nu; u0 += (int64_t)kUlyUnroll * G) {
      T v[kUlyUnroll];
#pragma unroll
      for (int k = 0; k < kUlyUnroll; ++k) {
        const int64_t u = u0 + (int64_t)k * G;
        if (u < nu) v[k] = s ? ld_unit<U>(s + u * U) : zero_unit<U>();
      }
#pragma unroll
      for (int k = 0; k < kUlyUnroll; ++k) {
        const int64_t u = u0 + (int64_t)k * G;
        if (u < nu) st_unit<U>(d + u * U, v[k]);
      }
    }
  }
}

// One block with the widest unit that the run length and both bases allow.
__device__ __noinline__ void copy_block(const char* src, const int64_t* ss, char* dst, const int64_t* ds,
                                        const UlyssesGeometry& g, int cta, int grid) {
  if (g.nruns == 0 || g.run_bytes == 0) return;
  const uintptr_t bits = (uintptr_t)g.run_bytes | (uintptr_t)dst | (uintptr_t)src;
  if ((bits & 15) == 0) copy_items<16>(src, ss, dst, ds, g, cta, grid);
  else if ((bits & 7) == 0) copy_items<8>(src, ss, dst, ds, g, cta, grid);
  else if ((bits & 3) == 0) copy_items<4>(src, ss, dst, ds, g, cta, grid);
  else if ((bits & 1) == 0) copy_items<2>(src, ss, dst, ds, g, cta, grid);
  else copy_items<1>(src, ss, dst, ds, g, cta, grid);
}

__global__ void __launch_bounds__(kThreads, 2)
ulysses_exchange_kernel(const __grid_constant__ CommParams cp, const __grid_constant__ UlyssesArgs a) {
  const int cta = blockIdx.x, grid = gridDim.x, n = cp.nranks, me = cp.rank, tid = threadIdx.x;
  __shared__ int64_t s_row[kMaxPeers][kUlyShapeWords + 1];
  __shared__ int s_status;
  const UlyssesGeometry& g = a.geo;
  const char* in = static_cast<const char*>(a.in);
  char* out = static_cast<char*>(a.out);
  uint32_t epoch = cp.epochs[cta];

  // ---- 1. stage ----
  char* staging = (char*)a.staging[me] + a.staging_offset;
  for (int q = 0; q < n; ++q) {
    if (q == me) copy_block(in + q * g.split_off, g.in_stride, out + me * g.cat_off, g.out_stride, g, cta, grid);
    else copy_block(in + q * g.split_off, g.in_stride, staging + q * g.block_bytes, g.packed_stride, g, cta, grid);
  }

  // ---- 2. publish, barrier A ----
  int64_t* row = a.counts[me] + (size_t)cta * kA2aRowWords;
  if (tid == 0) row[0] = a.direction;
  else if (tid == 1) row[1] = a.head_first;
  else if (tid < 7) row[tid] = a.dims[tid - 2];
  else if (tid == 7) row[7] = a.elem_bytes;
  else if (tid == kUlyStagingOffset) row[kUlyStagingOffset] = a.staging_offset;
  bool alive = true;
  if (n > 1) alive = peer_barrier(cp, epoch, cta); else __syncthreads();
  if (!alive) {
    if (cta == 0 && tid == 0 && *a.status == 0) *a.status = kA2aAborted;
    if (tid == 0) cp.epochs[cta] = epoch;
    return;
  }

  // ---- 3. verdict ----
  for (int i = tid; i < n * (kUlyShapeWords + 1); i += kThreads)
    s_row[i / (kUlyShapeWords + 1)][i % (kUlyShapeWords + 1)] =
        ld_volatile_s64(a.counts[i / (kUlyShapeWords + 1)] + (size_t)cta * kA2aRowWords + i % (kUlyShapeWords + 1));
  __syncthreads();
  if (tid == 0) {
    int st = kA2aOk;
    for (int p = 1; p < n; ++p)
      for (int w = 0; w < kUlyShapeWords; ++w) if (s_row[p][w] != s_row[0][w]) st = kA2aRowBytesMismatch;
    s_status = st;
  }
  __syncthreads();
  const int st = s_status;
  if (cta == 0 && tid == 0 && st != kA2aOk && *a.status == 0) *a.status = st;

  // ---- 4. pull, or zero the output ----
  if (st == kA2aOk) {
    for (int p = 0; p < n; ++p) {
      if (p == me) continue;
      const char* src = (const char*)a.staging[p] + s_row[p][kUlyStagingOffset] + me * g.block_bytes;
      copy_block(src, g.packed_stride, out + p * g.cat_off, g.out_stride, g, cta, grid);
    }
  } else {
    // this CTA's items of every block, own block included: exactly the bytes it wrote or would have written
    for (int p = 0; p < n; ++p) copy_block(nullptr, g.packed_stride, out + p * g.cat_off, g.out_stride, g, cta, grid);
  }

  // ---- 5. barrier B ----
  if (n > 1) peer_barrier(cp, epoch, cta);
  if (tid == 0) cp.epochs[cta] = epoch;
}

bool MulOk(int64_t a, int64_t b, int64_t* out) { return !__builtin_mul_overflow(a, b, out); }

}  // namespace

cudaError_t PlanUlyssesExchange(int n, UlyssesArgs* args) {
  if (args->ctas < 1 || args->ctas > kMaxCtas || n < 1 || n > kMaxPeers || !args->status ||
      (args->direction != kUlySeqToHeads && args->direction != kUlyHeadsToSeq) || args->elem_bytes < 1 || args->staging_offset < 0)
    return cudaErrorInvalidValue;
  for (int p = 0; p < n; ++p) if (!args->staging[p] || !args->counts[p]) return cudaErrorInvalidValue;
  for (int k = 0; k < 5; ++k) if (args->dims[k] < 0) return cudaErrorInvalidValue;
  const int64_t A = args->dims[0], d1 = args->dims[1], M = args->dims[2], d2 = args->dims[3], R = args->dims[4];
  const int64_t esz = args->elem_bytes;
  // the split dim: heads for seq -> heads, the sequence for heads -> seq
  const bool split_d1 = (args->direction == kUlySeqToHeads) == (args->head_first != 0);
  if ((split_d1 ? d1 : d2) % n != 0) return cudaErrorInvalidValue;
  int64_t total = 1;
  for (int64_t v : {A, d1, M, d2, R, esz}) if (!MulOk(total, v, &total)) return cudaErrorInvalidValue;
  if (total > args->staging_bytes) return cudaErrorInvalidValue;  // block q of the input to block q of the staging buffer
  UlyssesGeometry& g = args->geo;
  const int64_t d1b = split_d1 ? d1 / n : d1, d2b = split_d1 ? d2 : d2 / n;         // one block's extent
  const int64_t d1o = split_d1 ? d1 / n : d1 * n, d2o = split_d1 ? d2 * n : d2 / n;  // the output's
  g.ni = d1b; g.nm = M; g.nruns = A * d1b * M;
  g.run_bytes = d2b * R * esz;
  g.block_bytes = g.nruns * g.run_bytes;
  g.in_stride[2] = d2 * R * esz; g.in_stride[1] = M * g.in_stride[2]; g.in_stride[0] = d1 * g.in_stride[1];
  g.out_stride[2] = d2o * R * esz; g.out_stride[1] = M * g.out_stride[2]; g.out_stride[0] = d1o * g.out_stride[1];
  g.packed_stride[2] = g.run_bytes; g.packed_stride[1] = M * g.run_bytes; g.packed_stride[0] = d1b * g.packed_stride[1];
  g.split_off = split_d1 ? d1b * g.in_stride[1] : g.run_bytes;
  g.cat_off = split_d1 ? d2 * R * esz : d1 * g.out_stride[1];
  return cudaSuccess;
}

cudaError_t LaunchUlyssesExchange(const CommParams& cp, const UlyssesArgs& args, cudaStream_t stream) {
  if (cp.rank < 0 || cp.rank >= cp.nranks) return cudaErrorInvalidValue;
  UlyssesArgs a = args;
  const cudaError_t e = PlanUlyssesExchange(cp.nranks, &a);
  if (e != cudaSuccess) return e;
  ulysses_exchange_kernel<<<a.ctas, kThreads, 0, stream>>>(cp, a);
  CountKernelLaunch();
  return cudaGetLastError();
}

}  // namespace kern
}  // namespace hvd
