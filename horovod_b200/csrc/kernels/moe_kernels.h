// Host-side interface of the expert-parallel dispatch and combine kernels.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace hvd {
namespace kern {

// Expert-parallel dispatch and combine (see moe_kernels.cu): the local data movement around the captured alltoall.
// Row data: fp32, bf16 or fp16 (`dtype`, hvd::DataType codes); gates fp32 or the row dtype (`gate_dtype`).
constexpr int kMoeMaxExperts = 1024, kMoeMaxTopK = 16;
// Scratch ints of LaunchMoeRoute: MoeRouteTiles(assignments) * (num_experts + 1).
int64_t MoeRouteTiles(int64_t assignments);
// The stable order by expert of `assignments` expert ids (int32 / int64; ids outside [0, num_experts) are errors):
// counts[e] (int64), splits[q] (int32: the rows for rank q's experts [q * el, q * el + el), el = num_experts / nranks),
// pos[a] (int32: send-buffer row of assignment a, -1 for a bad id).  Any bad id makes every split -1 and every count 0.
// `ticket`: a zeroed counter that the launch leaves zeroed, not shared with a launch that may run at the same time.
cudaError_t LaunchMoeRoute(const void* idx, bool idx_int64, int64_t assignments, int num_experts, int nranks, int* hist,
                           unsigned* ticket, int64_t* counts, int* splits, int* pos, cudaStream_t stream);
// Per-token row movement over [ntok, k] positions `pos` into / out of buffers of rows of h elements.
//   scatter: dst[pos[t, j]] = src[t] (no gates: the bytes) or round(gates[t, j] * src[t]); with dot_rows also
//            grad_gates[t, j] = <src[t], dot_rows[pos[t, j]]> in fp32.  Positions outside [0, dst_rows) are skipped.
//   gather:  dst[t] = round(sum_j gates[t, j] * src[pos[t, j]]), fp32, j ascending (no gates: unit gates); positions
//            outside [0, src_rows) add nothing.
// A non-zero *status (when given) writes zeros to dst (gather) or to grad_gates only (scatter).  `ctas`: 0 for the
// default grid; the results do not depend on it.
struct MoeRows {
  const void* src; void* dst; int64_t src_rows, dst_rows;
  const int* pos; int64_t ntok; int k; int64_t h; int dtype;
  const void* gates; int gate_dtype; const void* dot_rows; void* grad_gates;
  const int* status; int ctas;
};
cudaError_t LaunchMoeScatter(const MoeRows& args, cudaStream_t stream);
cudaError_t LaunchMoeGather(const MoeRows& args, cudaStream_t stream);
// Rows grouped by source rank <-> rows grouped by local expert, with counts[p * experts_per_rank + e] the rows of rank p
// for local expert e (all zero when *status is non-zero).  Forward (source-major src -> expert-major dst, `rows` rows
// each): zero past the total, offsets[e] = end row of group e.  Reverse (expert-major src -> source-major dst): the rows
// below the total, ret_splits[p] = rows of rank p.  src == dst only with experts_per_rank == 1 (nothing to move).
cudaError_t LaunchMoeRegroup(const void* src, void* dst, int64_t row_bytes, int64_t rows, const int64_t* counts, int nranks,
                             int experts_per_rank, const int* status, bool reverse, int* offsets, int* ret_splits, int ctas,
                             cudaStream_t stream);

}  // namespace kern
}  // namespace hvd
