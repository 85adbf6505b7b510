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

// Ulysses sequence-parallel exchange (hvd.UlyssesExchange, see ulysses_kernels.cu), one launch on barrier channel
// kAlltoallChannel that shares the count region with the captured alltoall: a process set's captured alltoalls,
// ExpertDispatcher exchanges and Ulysses exchanges must be issued in one stream order.  The input of every rank is viewed
// as [A, D1, M, D2, R] elements of elem_bytes, where D1 and D2 are the sequence and head dims in tensor order
// (head_first: D1 is the head dim).  kUlySeqToHeads splits the head dim into N blocks, block q to rank q, and
// concatenates the sequence blocks of rank 0, 1, ...; kUlyHeadsToSeq splits the sequence dim and concatenates heads.
// Every CTA b stages exactly the runs that CTA b of every peer pulls from it, publishes
// {direction, head_first, A, D1, M, D2, R, elem_bytes, staging_offset} into row b of its count region and meets CTA b
// of every peer; if the shapes differ, status becomes kA2aRowBytesMismatch on every rank, nothing is pulled and the
// output is zero-filled.  `status` keeps the first non-zero code: the kernel only writes it while it holds 0.
enum UlyssesDirection : int { kUlySeqToHeads = 0, kUlyHeadsToSeq = 1 };
constexpr int kUlyShapeWords = 8;                  // the words of a row that every rank must agree on
constexpr int kUlyStagingOffset = kUlyShapeWords;  // then the staging offset
// The (receiver, sender) blocks of one exchange, all alike: runs j = (a * ni + i) * nm + m of run_bytes contiguous
// bytes, at a * stride[0] + i * stride[1] + m * stride[2] from the block's base.  Block q of the input starts at
// q * split_off, block p of the output at p * cat_off, block q of the staging buffer (packed runs) at q * block_bytes.
struct UlyssesGeometry {
  int64_t ni, nm, nruns, run_bytes, block_bytes, split_off, cat_off;
  int64_t in_stride[3], out_stride[3], packed_stride[3];
};
struct UlyssesArgs {
  const void* staging[kMaxPeers];  // every rank's registered region as mapped into this process
  int64_t* counts[kMaxPeers];      // every rank's count region as mapped here
  int64_t staging_offset;          // byte offset of this rank's staging buffer in its region
  int64_t staging_bytes;           // its size: at least the input's bytes
  const void* in;                  // this rank's contiguous input
  void* out;                       // its output, the same number of bytes
  int64_t dims[5];                 // A, D1, M, D2, R of the input
  int64_t elem_bytes;
  int direction;                   // UlyssesDirection
  int head_first;
  int* status;
  int ctas;                        // the same on every rank
  UlyssesGeometry geo;             // filled in by the launcher from the fields above and the team size
};
// Checks the arguments of an exchange on a team of `nranks` and fills in args->geo: cudaErrorInvalidValue when the split
// dim is not a multiple of nranks, the input does not fit the staging buffer, or a field is out of range.
cudaError_t PlanUlyssesExchange(int nranks, UlyssesArgs* args);
cudaError_t LaunchUlyssesExchange(const CommParams& cp, const UlyssesArgs& args, cudaStream_t stream);

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

}  // namespace kern
}  // namespace hvd
