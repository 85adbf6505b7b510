// Host-side interface of the sm_90a peer-to-peer collective kernels.
//
// These kernels replace the reference's three-launch GPU data path
// (batched_scaled_memcpy_k -> ncclAllReduce -> batched_scaled_memcpy_k,
// horovod/common/ops/cuda/cuda_kernels.cu:259-324 + ops/nccl_operations.cc:185-287)
// with ONE launch that packs (prescale + cast) gradients into a symmetric
// buffer, synchronises with peer GPUs through release/acquire flags in peer
// memory, reduces by loading/storing peer buffers directly over NVLink (or
// through the NVSwitch with multimem.ld_reduce / multimem.st), applies
// postscale/average + cast and scatters the result to the output tensors.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace hvd {
namespace kern {

// number of kernels of this library launched by this process (bench.py reports it as gpu_launches)
unsigned long long KernelLaunchCount();
void CountKernelLaunch();

constexpr int kMaxPeers = 8;          // one NVSwitch domain of an HGX H100 box
constexpr int kMaxCtas = 256;         // flag slots per team
// 256-thread CTAs capped at 128 registers: two fit on an SM and one fits NEXT TO resident compute CTAs of an
// overlapping backward pass, so a communication kernel does not have to wait for whole SMs to drain
// (512-thread x 128-register CTAs needed an empty SM each; measured 2x step-time inflation at 2 GPUs).
constexpr int kThreads = 256;
constexpr int kChunkBytes = 32768;    // kThreads * 16 B * 8
constexpr int kInlineDescs = 6;
constexpr int kFlagWords = kMaxCtas * kMaxPeers;
// Independent barrier channels (flag words + epochs) of one team: see SymmTeam::Params
constexpr int kNumChannels = 8;
constexpr int kGraphChannel = 1;              // collectives captured into CUDA graphs (framework streams)
constexpr int kLatencyChannel = 3;            // the latency lane of small allreduce responses (channel 2 is unused)
// hvd.SyncBatchNorm's captured collectives on the compute stream: inside hvd.GraphedStep they run while the gradient
// buckets' allreduces (kGraphChannel, forked stream) may be resident, so they need flag words and epochs of their own
constexpr int kSyncBnChannel = 4;
// hvd.captured_alltoall on the compute stream: like kSyncBnChannel, it may run while the gradient buckets' allreduces are
// resident on kGraphChannel, so it has flag words and epochs of its own
constexpr int kAlltoallChannel = 5;
constexpr int kChannelFlagsOffset = 128 * 1024;  // bytes from the start of the flag region; channel c >= 1 at + (c-1) * kFlagWords * 4
// The count region of hvd.captured_alltoall, after the last channel's flag words: one row of kA2aRowWords int64 per CTA
// (see CapturedAlltoallArgs).  Reserved with the flag region when the team is created, so a first call may be captured.
constexpr int kA2aRowWords = 16;
constexpr int kCountRegionOffset = kChannelFlagsOffset + (kNumChannels - 1) * kFlagWords * 4;
constexpr int kCountRegionBytes = kMaxCtas * kA2aRowWords * 8;

// Everything a kernel needs to talk to its peers. Passed by value
// (__grid_constant__).
struct CommParams {
  int nranks;
  int rank;
  void* buf[kMaxPeers];         // op data buffer of every rank, mapped into this process
  uint32_t* flags[kMaxPeers];   // flag words of every rank: [cta][src_rank]
  void* mc_buf;                 // multicast (NVLS) mapping of the same buffer, or nullptr
  uint32_t* epochs;             // local: per-CTA barrier epoch, persists across launches
  int* abort_flag;              // host-mapped; non-zero => stop spinning (peer failure / shutdown / timeout)
  unsigned long long timeout_ns; // a barrier that waits longer sets *abort_flag = 2 and bails out (0 = wait forever)
};

// One tensor of a fused response. `offset` is the tensor's byte offset inside
// the fused buffer in WIRE dtype (128 B aligned); `count` in elements.
struct TensorDesc {
  const void* in;
  void* out;
  int64_t offset;
  int64_t count;
};

enum Variant : int { kOneShot = 0, kTwoShot = 1, kNvls = 2 };

// reduce op codes follow hvd::ReduceOp: 1 SUM (AVERAGE arrives as SUM + postscale), 3 MIN, 4 MAX, 5 PRODUCT
// dtype codes follow hvd::DataType.

struct AllreduceArgs {
  const TensorDesc* descs;      // device table (nullptr => use inline_descs)
  TensorDesc inline_descs[kInlineDescs];
  int ndesc;
  int64_t total_bytes;          // wire bytes of the fused buffer region, multiple of 128
  int64_t reduce_lo, reduce_hi; // byte range this rank must produce output for (allreduce: [0,total))
  double prescale, postscale;
  int op;
  int dtype, wire_dtype;
  int variant;
  int ctas;
  // reducescatter: outputs use their own table (offsets relative to the fused buffer)
  const TensorDesc* out_descs;  // nullptr => same as descs
  int nout;
  int oneshot_nvls;             // kOneShot only: reduce with multimem.ld_reduce on the multicast mapping instead of N peer loads
};

// Fused allreduce / reducescatter.  Returns cudaErrorInvalidValue for
// unsupported dtype combinations and for a variant other than kOneShot, kTwoShot or kNvls.
cudaError_t LaunchAllreduce(const CommParams& cp, const AllreduceArgs& args, cudaStream_t stream);

// Zero-copy allreduce on a registered (peer-mapped) tensor: ptr[r] = the tensor's address in rank r's region as
// mapped into THIS process, mc = its multicast alias (or nullptr). In place on every rank. SUM-like ops only for
// multicast; bytes must be a multiple of 16.
struct InplaceArgs {
  void* ptr[kMaxPeers];
  void* mc;
  int64_t bytes;
  double scale;       // prescale * postscale (valid for SUM / AVERAGE)
  int op;
  int dtype;
  int use_multicast;
  int ctas;
  int chunk_bytes;    // filled in by the launcher
  int nvls_unroll;    // filled in by the launcher (4 | 8 multimem.ld_reduce in flight per thread)
};
cudaError_t LaunchInplaceAllreduce(const CommParams& cp, const InplaceArgs& args, cudaStream_t stream);
// The two halves of a sharded optimizer step on a registered range, with contiguous shards: rank r owns
// [r*S, (r+1)*S), S = bytes / nranks; bytes must be a multiple of 16 * nranks (cudaErrorInvalidValue otherwise).
// Reduce-scatter: rank r's shard of its own tensor receives the reduction (scaled by `scale`); nothing else is written.
// Multicast for SUM-like ops on fp32 / fp16 / bf16 only.
cudaError_t LaunchInplaceReducescatter(const CommParams& cp, const InplaceArgs& args, cudaStream_t stream);
// Allgather: rank r's shard of its own tensor is copied into every peer's tensor.  Bytes only: `dtype`, `op` and `scale`
// are ignored.
cudaError_t LaunchInplaceAllgather(const CommParams& cp, const InplaceArgs& args, cudaStream_t stream);

// Generic "pack -> barrier -> pull" used by allgather / broadcast / alltoall.
// send: local src -> local symmetric buffer offset; recv: peer buffer offset -> local dst.
struct CopyDesc {
  const void* src;   // send: local source; recv: unused
  void* dst;         // recv: local destination; send: unused
  int64_t offset;    // byte offset in the (sender's) symmetric buffer
  int64_t bytes;
  int peer;          // recv: which rank's buffer to pull from
  int pad;           // send: kSendMulticast = store through the multicast mapping (lands in EVERY rank's buffer at `offset`)
};
constexpr int kSendMulticast = 1;  // requires a 16 B aligned offset and a 16 B-padded window
struct ExchangeArgs {
  const CopyDesc* sends; int nsend;
  const CopyDesc* recvs; int nrecv;
  int ctas;
};
cudaError_t LaunchExchange(const CommParams& cp, const ExchangeArgs& args, cudaStream_t stream);

// Alltoall whose split vectors exist only on the device (see alltoall_kernels.cu), one launch on barrier channel
// kAlltoallChannel.  Rank p sends the first splits_p[0] rows of its input to rank 0, the next splits_p[1] to rank 1, ...;
// rank q receives them into `out` in sender order.  Every CTA b publishes this rank's row {splits[0 .. n), rows, capacity,
// row_bytes, in_offset} into row b of its count region, meets CTA b of every peer, reads all n rows and derives the same
// verdict on every rank: kA2aOk, or the first of the codes below that applies, in which case no row is copied.
// `recv_splits` (int64, n) receives the column that was sent to this rank in either case; CTA 0 writes it and `status`.
enum AlltoallStatus : int {
  kA2aOk = 0,
  kA2aNegativeSplit = 1,     // some rank's split is negative
  kA2aSendOverflow = 2,      // some rank's splits sum to more than its input rows
  kA2aRecvOverflow = 3,      // some rank would receive more rows than its capacity
  kA2aRowBytesMismatch = 4,  // the ranks' row sizes in bytes differ
  kA2aAborted = 5,           // a peer did not reach the barrier (team aborted or timed out); nothing else is written
};
constexpr int kA2aRows = kMaxPeers, kA2aCapacity = kMaxPeers + 1, kA2aRowBytes = kMaxPeers + 2, kA2aInOffset = kMaxPeers + 3;
struct CapturedAlltoallArgs {
  const void* in[kMaxPeers];    // every rank's registered region as mapped into this process
  int64_t* counts[kMaxPeers];   // every rank's count region (kCountRegionOffset of its flag region) as mapped here
  int64_t in_offset;            // byte offset of this rank's input rows in its region
  int64_t rows, capacity, row_bytes;
  const void* splits;           // this rank's n splits, int32 or int64 (splits_int64)
  int splits_int64;
  void* out;                    // capacity * row_bytes bytes
  int64_t* recv_splits;
  int* status;
  int ctas;                     // the same on every rank
};
cudaError_t LaunchCapturedAlltoall(const CommParams& cp, const CapturedAlltoallArgs& args, cudaStream_t stream);

// Stand-alone batched pack / unpack / scale (NCCL-baseline path and odd cases).
// direction 0: tensors -> buffer (prescale), 1: buffer -> tensors (postscale)
cudaError_t LaunchPackUnpack(void* buffer, const TensorDesc* descs, int ndesc, int64_t total_bytes, int dtype,
                             int wire_dtype, double scale, int direction, int ctas, cudaStream_t stream);
cudaError_t LaunchScale(const void* in, void* out, int64_t count, int dtype, double scale, cudaStream_t stream);

// Adasum (vector-halving distance-doubling with per-tensor adaptive coefficients) entirely on the GPUs of a
// peer-mapped team; see adasum_kernels.cu.  Tensors are fp32 / fp16 / bf16; the fused vector lives in fp32.
struct AdasumArgs {
  const TensorDesc* descs; int ndesc;   // device table; offsets are byte offsets of the FP32 fused vector (128 B aligned)
  int64_t total_bytes;                  // fp32 bytes, multiple of 128
  int dtype;
  int ctas;
  int64_t scratch_stride_bytes;         // distance between the two per-level partial-dot tables in the flag region
  // Persistent single-launch variant (both non-null): local device scratch of AdasumPersistentScratchBytes(ctas, ndesc)
  // and a 16-byte grid-synchronisation block; `ctas` CTAs must be co-resident on the device.
  void* persist_scratch = nullptr;
  void* persist_sync = nullptr;
};
size_t AdasumPersistentScratchBytes(int ctas, int ndesc);
size_t AdasumPersistentSyncBytes();
constexpr int64_t kAdasumScratchStride = 30000;
constexpr int kAdasumMaxTensors = 1250;
cudaError_t LaunchAdasum(const CommParams& cp, const AdasumArgs& args, double prescale, double postscale, cudaStream_t stream);
// Single-GPU simulation support: launch only step `only` of the sequence (see adasum_kernels.cu); -1 = all.
cudaError_t LaunchAdasumStep(const CommParams& cp, const AdasumArgs& args, double prescale, double postscale, cudaStream_t stream,
                             int only);
int AdasumNumLaunches(int nranks);

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
