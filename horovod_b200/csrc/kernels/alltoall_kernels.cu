// Alltoall with device-resident split vectors (hvd.captured_alltoall), one launch on a peer-mapped team (sm_90a).
//
// The planned alltoall (exchange_kernels.cu) needs every rank's splits on the host to size its copies; here they are only
// ever read by the kernel, so a mixture-of-experts dispatch whose per-expert row counts come out of the router costs no
// .cpu() sync and no control-plane round, and can be captured into a CUDA graph.  Per CTA b of every rank:
//
//   1. publish: this rank's row {splits[0 .. n), rows, capacity, row_bytes, in_offset} into row b of its count region;
//   2. barrier A with CTA b of every peer: every row is visible, and every sender's input is final (each rank launched
//      after its producer);
//   3. read the n x n matrix from the peers' count regions and derive, in a fixed order with integer arithmetic only, the
//      status, this rank's output offsets (prefix sum down its column) and each sender's source offset (prefix sum along
//      that sender's row): every CTA of every rank reaches the same verdict;
//   4. pull: the received bytes [0, total) of the output, in kChunkBytes chunks, chunk c by CTA c % grid, each straight
//      from the senders' registered inputs (16 B vectors where both sides are aligned, bytes otherwise);
//   5. barrier B: no rank returns, and so overwrites its input or its count row in a later launch, while a peer still
//      reads them.
#include "p2p_common.cuh"

namespace hvd {
namespace kern {
namespace {

__device__ __forceinline__ int64_t ld_volatile_s64(const int64_t* p) { return *reinterpret_cast<const volatile int64_t*>(p); }

__global__ void __launch_bounds__(kThreads, 2)
captured_alltoall_kernel(const __grid_constant__ CommParams cp, const __grid_constant__ CapturedAlltoallArgs a) {
  const int cta = blockIdx.x, grid = gridDim.x, n = cp.nranks, me = cp.rank, tid = threadIdx.x;
  __shared__ int64_t s_row[kMaxPeers][kA2aRowWords];  // every rank's published row
  __shared__ int64_t s_out[kMaxPeers + 1];            // output byte offset of sender p's rows; s_out[n] = bytes received
  __shared__ const char* s_src[kMaxPeers];            // where those rows start in sender p's input
  __shared__ int s_status;
  uint32_t epoch = cp.epochs[cta];

  // ---- 1. publish ----
  int64_t* row = a.counts[me] + (size_t)cta * kA2aRowWords;
  if (tid < n) row[tid] = a.splits_int64 ? static_cast<const int64_t*>(a.splits)[tid] : (int64_t)static_cast<const int32_t*>(a.splits)[tid];
  else if (tid == kA2aRows) row[tid] = a.rows;
  else if (tid == kA2aCapacity) row[tid] = a.capacity;
  else if (tid == kA2aRowBytes) row[tid] = a.row_bytes;
  else if (tid == kA2aInOffset) row[tid] = a.in_offset;

  // ---- 2. barrier A ----
  bool alive = true;
  if (n > 1) alive = peer_barrier(cp, epoch, cta); else __syncthreads();
  if (!alive) {
    if (cta == 0 && tid == 0) *a.status = kA2aAborted;
    if (tid == 0) cp.epochs[cta] = epoch;
    return;
  }

  // ---- 3. the split matrix, the verdict and the offsets ----
  for (int i = tid; i < n * kA2aRowWords; i += kThreads)
    s_row[i / kA2aRowWords][i % kA2aRowWords] = ld_volatile_s64(a.counts[i / kA2aRowWords] + (size_t)cta * kA2aRowWords + i % kA2aRowWords);
  __syncthreads();
  if (tid == 0) {
    // each check over the whole matrix, in this order; the first that fails decides.  Every split is bounded by its
    // sender's rows before any sum is taken, so no sum below can overflow.
    int st = kA2aOk;
    for (int p = 0; p < n; ++p)
      for (int q = 0; q < n; ++q) if (s_row[p][q] < 0) st = kA2aNegativeSplit;
    for (int p = 0; p < n && st == kA2aOk; ++p) {
      int64_t sent = 0;
      for (int q = 0; q < n; ++q) {
        if (s_row[p][q] > s_row[p][kA2aRows]) { sent = -1; break; }
        sent += s_row[p][q];
      }
      if (sent < 0 || sent > s_row[p][kA2aRows]) st = kA2aSendOverflow;
    }
    for (int q = 0; q < n && st == kA2aOk; ++q) {
      int64_t recv = 0;
      for (int p = 0; p < n; ++p) recv += s_row[p][q];
      if (recv > s_row[q][kA2aCapacity]) st = kA2aRecvOverflow;
    }
    for (int p = 1; p < n && st == kA2aOk; ++p)
      if (s_row[p][kA2aRowBytes] != s_row[0][kA2aRowBytes]) st = kA2aRowBytesMismatch;
    s_status = st;
    if (st == kA2aOk) {
      const int64_t rb = a.row_bytes;
      int64_t out = 0;
      for (int p = 0; p < n; ++p) {
        int64_t before = 0;  // rows sender p sends to the ranks before this one
        for (int q = 0; q < me; ++q) before += s_row[p][q];
        s_out[p] = out;
        s_src[p] = static_cast<const char*>(a.in[p]) + s_row[p][kA2aInOffset] + before * rb;
        out += s_row[p][me] * rb;
      }
      s_out[n] = out;
    }
  }
  __syncthreads();
  const int st = s_status;
  if (cta == 0) {
    if (tid < n) a.recv_splits[tid] = s_row[tid][me];
    if (tid == 0) *a.status = st;
  }

  // ---- 4. pull ----
  if (st == kA2aOk) {
    char* out = static_cast<char*>(a.out);
    const int64_t total = s_out[n];
    for (int64_t lo = (int64_t)cta * kChunkBytes; lo < total; lo += (int64_t)grid * kChunkBytes) {
      const int64_t hi = lo + kChunkBytes < total ? lo + kChunkBytes : total;
      for (int p = 0; p < n; ++p) {
        const int64_t b = lo > s_out[p] ? lo : s_out[p];
        const int64_t e = hi < s_out[p + 1] ? hi : s_out[p + 1];
        if (b < e) copy_bytes_vec(s_src[p] + (b - s_out[p]), out + b, e - b);
      }
    }
  }

  // ---- 5. barrier B ----
  if (n > 1) peer_barrier(cp, epoch, cta);
  if (tid == 0) cp.epochs[cta] = epoch;
}

}  // namespace

cudaError_t LaunchCapturedAlltoall(const CommParams& cp, const CapturedAlltoallArgs& args, cudaStream_t stream) {
  if (args.ctas < 1 || args.ctas > kMaxCtas || cp.nranks < 1 || cp.nranks > kMaxPeers || cp.rank < 0 || cp.rank >= cp.nranks ||
      args.rows < 0 || args.capacity < 0 || args.row_bytes < 0 || !args.splits || !args.recv_splits || !args.status)
    return cudaErrorInvalidValue;
  captured_alltoall_kernel<<<args.ctas, kThreads, 0, stream>>>(cp, args);
  CountKernelLaunch();
  return cudaGetLastError();
}

}  // namespace kern
}  // namespace hvd
