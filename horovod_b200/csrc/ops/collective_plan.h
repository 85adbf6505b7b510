// Launch plans of the fused allreduce and of the exchange-style collectives (reducescatter, allgather(v), broadcast,
// alltoall(v)): plain host functions that turn per-rank sizes, a split matrix or a root into the descriptor tables and
// launch arguments of the P2P kernels, and a check that the N ranks' plans can run together.
//
// A plan is everything a rank launches for one response except the CommParams and the staged device copy of the
// tables.  The plans hold the cross-rank contract: every rank issues the same number of launches, each with the same grid,
// because CTA b of a launch rendezvouses with CTA b of every peer (a mismatch spins until the barrier timeout), and a
// receive reads the bytes that the peer's matching send packed.  GpuOps plans and launches on one rank; the single-GPU
// simulation (common/sim_api.cc) plans all N ranks, runs CheckPlans and only then launches.
#pragma once
#include <cstdint>
#include <string>
#include <vector>
#include "../common/common.h"
#include "../kernels/p2p_kernels.h"

namespace hvd {

// One kernel launch.  Exchange (`reduce` false): `sends` / `recvs` of exchange_kernel.  Reduce (`reduce` true): `table`
// holds args.ndesc in-descriptors (the packed layout) followed by args.nout out-descriptors (nout 0: the outputs are the
// in-descriptors' `out`, as in allreduce); `args` is complete except descs / out_descs / inline_descs and ctas.
struct PlanLaunch {
  bool reduce = false;
  int ctas = 1;
  std::vector<kern::CopyDesc> sends, recvs;
  std::vector<kern::TensorDesc> table;
  kern::AllreduceArgs args {};
};
using Plan = std::vector<PlanLaunch>;

// One tensor of a response.  `row`: elements per first-dim row.  `dims`:
//   allreduce      {elements} (row is not used)
//   reducescatter  {dim0}
//   allgather      the first dim of every rank, [n]
//   alltoall       the split matrix, [n][n]: dims[p * n + q] = rows rank p sends to rank q
//   broadcast      {bytes} (row and the element size are not used)
struct PlanTensor {
  const void* in = nullptr;
  void* out = nullptr;
  int64_t row = 1;
  std::vector<int64_t> dims;
};

struct ReduceParams {
  DataType dtype = DataType::FLOAT32;
  ReduceOp op = ReduceOp::SUM;
  double prescale = 1.0, postscale = 1.0;
  // reducescatter: the team may reduce through multimem, and launches of at least nvls_min_bytes then do (allreduce
  // takes both from its AllreducePolicy)
  bool nvls = false;
  int64_t nvls_min_bytes = 0;
};

// Whether multimem.ld_reduce can reduce `op` on a `dtype` wire: sums (AVERAGE included) of fp32, fp16 or bf16.
inline bool MultimemReduces(DataType dtype, ReduceOp op) {
  return (op == ReduceOp::SUM || op == ReduceOp::AVERAGE) &&
         (dtype == DataType::FLOAT32 || dtype == DataType::FLOAT16 || dtype == DataType::BFLOAT16);
}

// How the fused allreduce picks a kernel for each launch.  `variant` (HVD_ALLREDUCE_VARIANT) "oneshot" or "twoshot"
// forces that kernel, and "nvls" forces NVLS when the team has a multicast object and MultimemReduces the wire.
// Otherwise by the launch's bytes: one-shot up to oneshot_max_bytes, NVLS from nvls_min_bytes on teams of 4 or more
// GPUs that could force it, two-shot in between.
struct AllreducePolicy {
  std::string variant = "auto";
  int64_t oneshot_max_bytes = 0;
  bool multicast = false;
  int64_t nvls_min_bytes = 0;
  int64_t large_msg_ctas = 256;  // CtasFor
};

// CTAs of a fused allreduce launch of `seg_bytes` wire bytes on n ranks: at most comm_ctas, fewer for small messages,
// and at least large_msg_ctas from 64 MiB.
int CtasFor(int variant, int64_t seg_bytes, int n, int comm_ctas, int64_t large_msg_ctas);

// Whether a launch passes its descriptors by value in AllreduceArgs::inline_descs instead of a staged table.
inline bool InlineDescs(const kern::AllreduceArgs& a) { return a.nout == 0 && a.ndesc <= kern::kInlineDescs; }

// `cap`: bytes of the team's symmetric buffer available to one launch (SymmTeam::buffer_bytes()); `comm_ctas`: the
// most CTAs one launch may use.  Each returns InvalidArgument, and no plan, where `cap` leaves no room to make progress.
// Plans are appended to *plan.
// Allreduce: the pieces packed back to back (128 B aligned, in `wire` dtype), one launch per segment that fits `cap`.
Status PlanAllreduce(int n, const std::vector<PlanTensor>& ts, const ReduceParams& rp, DataType wire, const AllreducePolicy& pol,
                     int64_t cap, int comm_ctas, Plan* plan);
Status PlanReducescatter(int me, int n, const std::vector<PlanTensor>& ts, const ReduceParams& rp, int64_t cap, int comm_ctas,
                         Plan* plan);
Status PlanAllgather(int me, int n, const std::vector<PlanTensor>& ts, int64_t esz, int64_t cap, int comm_ctas, Plan* plan);
// `multicast`: the root stores through the team's multicast mapping and every rank copies out of its own buffer.
// A tensor whose `out` is nullptr or equal to `in` is not copied on the root.
Status PlanBroadcast(int me, int n, int root, const std::vector<PlanTensor>& ts, bool multicast, int64_t cap, int comm_ctas,
                     Plan* plan);
Status PlanAlltoall(int me, int n, const std::vector<PlanTensor>& ts, int64_t esz, int64_t cap, int comm_ctas, Plan* plan);

// Byte range of one output tensor.
struct OutSpan { const void* p; int64_t bytes; };

// Verifies that plans[r] (rank r's plan, r < n) can run together and write exactly outputs[r]:
//  - every rank issues the same launches: kind, ctas, and for reduce launches the arguments and the packed layout;
//  - every send and every packed region lies in [0, cap); exchange offsets are 16 B aligned and one rank's sends do not
//    overlap;
//  - every receive lies inside a send of its peer in the same launch (`root` >= 0: the peer is the root);
//  - reduce launches: N destination regions of width W (a multiple of 128) with non-decreasing, 128 B aligned in-desc
//    offsets, region q's descriptors inside [qW, (q+1)W), rank r's out-descriptors at the offsets and counts of region
//    r's in-descriptors, and [reduce_lo, reduce_hi) inside region r covering them;
//  - receive destinations and out-descriptor ranges cover every byte of every output span exactly once.
// Returns the first violation as InvalidArgument.
Status CheckPlans(const std::vector<Plan>& plans, const std::vector<std::vector<OutSpan>>& outputs, int64_t cap, int root);

}  // namespace hvd
