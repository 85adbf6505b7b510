// Host-side interface of the hvd.SyncBatchNorm kernels.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace hvd {
namespace kern {

// Batch normalization over the ranks of a process set (see sync_bn_kernels.cu).  An input with channels at dim 1 is
// viewed as rows [M, C] with C innermost (channels_last, [N, C], spatial size 1) or planes [M, C, L] (contiguous NCHW).
// x / y / dy / dx: fp32, bf16 or fp16 (dtype codes of hvd::DataType), all with the same layout; weight, bias, running
// statistics and parameter gradients: fp32 or the input dtype (`wdtype` / `stat_dtype`).
enum BnLayout : int { kBnRows = 0, kBnPlanes = 1 };
struct BnGeom { int layout; int64_t M, C, L; };   // rows: L = 1
// The stats / backward-reduce grid: `tiles` channel tiles (one ticket each) x `splits` CTAs per tile (one partial per
// channel each: 16 B for the stats, 8 B for the backward reduce), `cols` threads across a rows tile.
struct BnPlan { int64_t tiles, splits; int cols; };
BnPlan BnReducePlan(const BnGeom& g, int dtype);
// This rank's {count, mean, M2} of every channel as fp64 triples into slot[0 .. 3C).  `tickets` (plan.tiles zeroed
// counters, left zeroed) must not be shared with a launch that may run at the same time.
cudaError_t LaunchBnStats(const void* x, const BnGeom& g, int dtype, void* partial, unsigned* tickets, double* slot,
                          cudaStream_t stream);
// Merges the nranks slots (slot r at slots + r * slot_stride) in rank order into mean / invstd (fp32, C) and the global
// count (1 float); updates running_mean / running_var (nullptr: not tracked) with factor 1 / *num_batches_tracked if
// that is given, else `momentum`.
cudaError_t LaunchBnCombine(const double* slots, int nranks, int64_t slot_stride, int64_t C, double eps, double momentum,
                            const int64_t* num_batches_tracked, float* mean, float* invstd, float* count, void* running_mean,
                            void* running_var, int stat_dtype, cudaStream_t stream);
// y = (x - mean) * invstd * weight + bias (weight / bias may be nullptr)
cudaError_t LaunchBnElemt(const void* x, void* y, const BnGeom& g, int dtype, const float* mean, const float* invstd,
                          const void* weight, const void* bias, int wdtype, cudaStream_t stream);
// sums[2c] = sum dy, sums[2c+1] = sum dy * (x - mean) (fp64) over this rank's batch; grad_bias = sum dy and
// grad_weight = sum dy * (x - mean) * invstd where non-null.  Partials and tickets as LaunchBnStats.
cudaError_t LaunchBnBackwardReduce(const void* dy, const void* x, const BnGeom& g, int dtype, const float* mean,
                                   const float* invstd, void* partial, unsigned* tickets, double* sums, void* grad_weight,
                                   void* grad_bias, int wdtype, cudaStream_t stream);
// dx = (dy - sums[2c] / n - (x - mean) * invstd^2 * sums[2c+1] / n) * invstd * weight, n = *count
cudaError_t LaunchBnBackwardElemt(const void* dy, const void* x, void* dx, const BnGeom& g, int dtype, const float* mean,
                                  const float* invstd, const void* weight, int wdtype, const double* sums,
                                  const float* count, cudaStream_t stream);

}  // namespace kern
}  // namespace hvd
