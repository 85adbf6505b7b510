// Host-side interface of the fused optimizer, gradient statistics and gradient accumulation kernels.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace hvd {
namespace kern {

// Fused multi-tensor optimizer updates (see optim_kernels.cu).  One table entry type serves SGD, Adam(W), LAMB and LARS:
//   param, grad    the parameter and its gradient, `count` elements each
//   master         with `master` set: the fp32 copy of the parameter that the update runs on; otherwise not read
//   state0         SGD and LARS: the momentum buffer (SGD: nullptr without momentum); Adam and LAMB: exp_avg
//   state1         Adam and LAMB: exp_avg_sq; SGD and LARS do not read it
//   partial, slot  LAMB and LARS only: the entry's first stage-1 partial and its norm slot (see LaunchLambNorms)
//   ema            with `ema.on`: the fp32 exponential moving average of the parameter (see OptEma); otherwise not read
// Every state is fp32, except SGD momentum without `master`, which has the parameter dtype.  The (param, grad) dtypes are
// fp32 / fp32, fp32 / bf16, bf16 / bf16 and fp16 / fp16; with `master` bf16 / bf16 and fp16 / fp16 only.  Any other
// combination returns cudaErrorInvalidValue before anything is launched.  The gradient factor is
// grad_scale * *grad_scale_dev (nullptr: grad_scale alone, bit for bit).
struct OptTensor { void* param; const void* grad; void* master; void* state0; void* state1; int64_t count;
                   int64_t partial; int64_t slot; void* ema; };
// The EMA epilogue of the SGD, Adam, LAMB-apply and LARS-apply launches: with `on`, every entry's `ema` becomes
// fmaf(weight, x - ema, ema) after the update (weight = 1 - decay), x being the fp32 master with `master`, else the value
// stored into the parameter; with `start` as well, ema = x (the EMA begins with this update).  Off: the kernels without
// the epilogue run, and `ema` is not read.
struct OptEma { bool on = false; float weight = 0.f; int start = 0; };
cudaError_t LaunchFusedSgd(const OptTensor* table, int n, int64_t max_count, float lr, float momentum, float dampening,
                           float weight_decay, int nesterov, float grad_scale, int first_step, int param_dtype,
                           int grad_dtype, cudaStream_t stream, const float* grad_scale_dev = nullptr, bool master = false,
                           const OptEma& ema = OptEma());
cudaError_t LaunchFusedAdamW(const OptTensor* table, int n, int64_t max_count, float lr, float beta1, float beta2,
                             float eps, float weight_decay, float bias_c1, float bias_c2, float grad_scale,
                             int adamw, int param_dtype, int grad_dtype, cudaStream_t stream,
                             const float* grad_scale_dev = nullptr, bool master = false, const OptEma& ema = OptEma());
// Fused LAMB in two phases (see optim_kernels.cu), so that the norms can be allreduced in between.  Entry i covers
// `count` elements of a parameter whose whole-tensor norms live in norms[2 * slot] (sum w^2) and norms[2 * slot + 1]
// (sum u^2); its stage-1 CTA partials start at `partial`, the running sum of NormPartials(count) over the entries before
// it.  No two entries of one launch may share a slot.
// LaunchLambNorms: moments updated, then the entries' squared norms ADDED into `norms` (two launches; `partial` holds
// 2 * sum NormPartials floats).  LaunchLambApply: w -= lr * r * u (one launch; the gradient is not read, so only the
// parameter dtype is checked).
int64_t NormPartials(int64_t count);
cudaError_t LaunchLambNorms(const OptTensor* table, int n, int64_t max_count, float beta1, float beta2, float eps,
                            float weight_decay, float bias_c1, float bias_c2, float grad_scale, const float* grad_scale_dev,
                            float* partial, float* norms, int param_dtype, int grad_dtype, bool master, cudaStream_t stream);
cudaError_t LaunchLambApply(const OptTensor* table, int n, int64_t max_count, float lr, float eps, float weight_decay,
                            float bias_c1, float bias_c2, int adapt, const float* norms, int param_dtype, bool master,
                            cudaStream_t stream, const OptEma& ema = OptEma());
// Fused LARS on LAMB's table and norms layout: norms[2 * slot] = sum w^2, norms[2 * slot + 1] = sum g^2 of the scaled
// gradient.  LaunchLarsNorms: two launches, nothing but `partial` and `norms` written.  LaunchLarsApply:
// v = momentum * v + lr * r * (g + wd * w), w -= v (one launch; reads the gradient again, scaled by
// grad_scale * *grad_scale_dev as in the first phase).
cudaError_t LaunchLarsNorms(const OptTensor* table, int n, int64_t max_count, float grad_scale, const float* grad_scale_dev,
                            float* partial, float* norms, int param_dtype, int grad_dtype, bool master, cudaStream_t stream);
cudaError_t LaunchLarsApply(const OptTensor* table, int n, int64_t max_count, float lr, float momentum, float weight_decay,
                            float trust_coefficient, float eps, int adapt, float grad_scale, const float* grad_scale_dev,
                            const float* norms, int param_dtype, int grad_dtype, bool master, cudaStream_t stream,
                            const OptEma& ema = OptEma());
// Fused Adafactor (torch.optim.Adafactor's update, see optim_kernels.cu) on the OptTensor table plus a parallel geometry
// table: entry i of both describes one whole parameter.  A parameter of dim <= 1 keeps its fp32 `variance` (its sizes and
// strides) in OptTensor::state0 and has row_var == nullptr here.  A parameter of dim 2..kAdafactorMaxDims is factored over
// its last two dims [R, C], the leading dims (up to three, padded with 1 in front) forming a batch of B matrices:
//   size, stride   the logical sizes [b0, b1, b2, R, C] and the parameter's element strides for them (any dense layout;
//                  a dim of size 1 carries stride 1), each below 2^31.  The parameter has fewer than 2^32
//                  elements: the kernels compute its element offsets in 32-bit unsigned arithmetic.
//   row_var        fp32 [B, R], col_var fp32 [B, C], both contiguous (torch's [..., R, 1] and [..., 1, C])
//   col_off        the entry's first column partial (B * C * AdafactorRowChunks(R) of them)
//   batch_off      the entry's first per-batch mean of row_var (B of them)
constexpr int kAdafactorMaxDims = 5;
struct AdafactorGeom { int32_t size[kAdafactorMaxDims]; int32_t stride[kAdafactorMaxDims]; float* row_var; float* col_var;
                       int64_t col_off; int64_t batch_off; };
// Per-launch hyper-parameters as the kernels use them: beta_w = 1 - beta2_t = step^beta2_decay, rho = min(lr, step^-0.5),
// eps1_sq = eps1 * eps1 and decay = 1 - lr * weight_decay, each rounded from double once.
struct AdafactorHyper { float beta_w, rho, eps1, eps1_sq, eps2, d, decay; };
int64_t AdafactorRowChunks(int64_t rows);
// CTAs along x that the stats and factor launches need for a factored entry of B matrices [R, C].
int64_t AdafactorStatsCtas(int64_t batch, int64_t rows, int64_t cols);
int64_t AdafactorFactorCtas(int64_t batch, int64_t cols);
// The whole step in five launches: row sums (row_var lerped) and column partials of g^2; column sums (col_var lerped) and
// the per-batch means of row_var; per-CTA (sum w^2, sum u^2) partials, which also lerp the variance of dim <= 1 entries;
// the finalize of those into `norms` (2 floats per entry, zeroed by the caller); the update.  colpart / rmean / partial
// are scratch of sum B * C * AdafactorRowChunks(R), sum B and 2 * sum NormPartials(count) floats.  `stats_ctas` /
// `factor_ctas`: the largest AdafactorStatsCtas / AdafactorFactorCtas over the entries (at least 1).
cudaError_t LaunchAdafactor(const OptTensor* table, const AdafactorGeom* geom, int n, int64_t max_count, int64_t stats_ctas,
                            int64_t factor_ctas, const AdafactorHyper& h, float grad_scale, const float* grad_scale_dev,
                            float* colpart, float* rmean, float* partial, float* norms, int param_dtype, int grad_dtype,
                            bool master, cudaStream_t stream, const OptEma& ema);
// Copies `bytes` of host memory to device memory `dst` on `stream` through kernel parameters, so that the copy of a
// launch captured into a CUDA graph is part of the graph (one launch per 4000 bytes).
cudaError_t LaunchUploadBytes(void* dst, const void* host, size_t bytes, cudaStream_t stream);
// Gradient statistics of flat gradient shards in one pass (see optim_kernels.cu): optional in-place scaling by
// *inv_scale, then out[0] += sum of squares (norm_inf: out[0] = max(out[0], max |g|)) and out[1] = max(out[1], non-finite).
// Entries are non-empty and in order; tile_begin is the sum of GradShardStatsTiles(count) of the entries before, `tiles`
// that sum over all of them and `row_tiles` its largest term.  `partial` / `partial_flag` hold `tiles` entries; `ticket`
// is a zeroed counter that the kernel leaves zeroed, which launches running at the same time must not share.
struct StatTensor { void* grad; int64_t count; int64_t tile_begin; };
int64_t GradShardStatsTiles(int64_t count);
cudaError_t LaunchGradShardStats(const StatTensor* table, int n, int64_t tiles, int64_t row_tiles, const float* inv_scale,
                                 int norm_inf, float* partial, int* partial_flag, unsigned* ticket, float* out,
                                 int grad_dtype, cudaStream_t stream);
// Gradient accumulation in fp32 (see optim_kernels.cu): `grad` is bf16 / fp16 (grad_dtype, one per launch), `acc` fp32
// with the same element order.  kAccFirst: acc = g, g = 0; kAccAdd: acc += g, g = 0; kAccLast: g = round(acc + g).  The
// table is passed by value (under the 4 KB kernel-parameter limit), so one launch covers at most kAccMaxTensors entries
// and the launch can be captured into a CUDA graph.  No atomics, no state between launches.
enum AccMode : int { kAccFirst = 0, kAccAdd = 1, kAccLast = 2 };
constexpr int kAccMaxTensors = 160;
struct AccTensor { void* grad; float* acc; int64_t count; };
struct AccTable { AccTensor t[kAccMaxTensors]; int n; };
cudaError_t LaunchGradAccumulate(const AccTable& table, int64_t max_count, int mode, int grad_dtype, cudaStream_t stream);

}  // namespace kern
}  // namespace hvd
