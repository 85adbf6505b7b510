// PyTorch entry points of the hvd.ExpertDispatcher kernels (see kernels/moe_kernels.cu).  Every argument is checked here,
// before anything is launched.  Rows are the dim-1 slices of contiguous 2-D tensors of fp32 / bf16 / fp16; positions and
// row indices are int32, byte offsets int64.
#include "../kernels/moe_kernels.h"
#include "binding_util.h"

namespace hvd {
namespace {

// a contiguous [rows, h] tensor of `dtype` on `dev`
void CheckMoeRows(const char* op, const char* what, const at::Tensor& t, int64_t h, at::ScalarType dtype, const at::Device& dev) {
  TORCH_CHECK(t.dim() == 2 && t.size(1) == h, op, ": ", what, " must be [rows, ", h, "], got sizes ", t.sizes());
  CheckVector(op, what, t, dev, {dtype}, t.numel());
  TORCH_CHECK(t.size(0) <= 0x7fffffff, op, ": ", what, " has ", t.size(0), " rows, more than int32 row indices reach");
}

at::ScalarType MoeDtype(const char* op, const at::Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.size(1) >= 1, op, ": rows must be a 2-D CUDA tensor [rows, hidden] with "
              "hidden >= 1, got sizes ", x.sizes());
  const auto st = x.scalar_type();
  TORCH_CHECK(st == at::kFloat || st == at::kBFloat16 || st == at::kHalf, op, ": rows must be float32, bfloat16 or float16, "
              "got ", st);
  return st;
}

void CheckMoePos(const char* op, const at::Tensor& pos, int64_t ntok, const at::Device& dev) {
  TORCH_CHECK(pos.dim() == 2 && pos.size(0) == ntok && pos.size(1) >= 1 && pos.size(1) <= kern::kMoeMaxTopK, op,
              ": pos must be [", ntok, ", k] with 1 <= k <= ", kern::kMoeMaxTopK, ", got sizes ", pos.sizes());
  CheckVector(op, "pos", pos, dev, {at::kInt}, pos.numel());
}

// gates: [tokens, k] contiguous, fp32 or the rows' dtype
const void* MoeGates(const char* op, const c10::optional<at::Tensor>& gates, const at::Tensor& pos, at::ScalarType dtype,
                     int* gate_dtype) {
  *gate_dtype = (int)MapDtype(at::kFloat);
  if (!gates) return nullptr;
  const at::Tensor& g = *gates;
  TORCH_CHECK(g.sizes() == pos.sizes(), op, ": gates must be ", pos.sizes(), ", got sizes ", g.sizes());
  CheckVector(op, "gates", g, pos.device(), {at::kFloat, dtype}, g.numel());
  *gate_dtype = (int)MapDtype(g.scalar_type());
  return g.data_ptr();
}

// The stable order by expert of expert_idx [T, k] (int32 / int64), and the copy of every token's row x[t] to its k
// send-buffer rows.  counts: this rank's num_experts per-expert counts (int64, contiguous), written by the kernel.
// Returns (pos int32 [T, k], splits int32 [nranks]).
std::tuple<at::Tensor, at::Tensor> MoePermute(at::Tensor x, at::Tensor expert_idx, at::Tensor send, at::Tensor counts,
                                              int64_t num_experts, int64_t nranks, int64_t ctas) {
  const char* op = "moe_permute";
  const auto dt = MoeDtype(op, x);
  const at::Device dev = x.device();
  const int64_t T = x.size(0), h = x.size(1);
  CheckMoeRows(op, "x", x, h, dt, dev);
  CheckMoeRows(op, "send", send, h, dt, dev);
  TORCH_CHECK(num_experts >= 1 && num_experts <= kern::kMoeMaxExperts, op, ": num_experts must be in [1, ",
              kern::kMoeMaxExperts, "], got ", num_experts);
  TORCH_CHECK(nranks >= 1 && num_experts % nranks == 0, op, ": num_experts (", num_experts, ") must be a multiple of nranks (",
              nranks, ")");
  TORCH_CHECK(expert_idx.dim() == 2 && expert_idx.size(0) == T && expert_idx.size(1) >= 1 &&
              expert_idx.size(1) <= kern::kMoeMaxTopK, op, ": expert_idx must be [", T, ", k] with 1 <= k <= ",
              kern::kMoeMaxTopK, ", got sizes ", expert_idx.sizes());
  CheckVector(op, "expert_idx", expert_idx, dev, {at::kInt, at::kLong}, expert_idx.numel());
  const int64_t k = expert_idx.size(1);
  TORCH_CHECK(send.size(0) >= T * k, op, ": send holds ", send.size(0), " rows, fewer than the ", T * k, " assignments");
  CheckVector(op, "counts", counts, dev, {at::kLong}, num_experts);
  TORCH_CHECK(ctas >= 0, op, ": ctas must be >= 0");
  const OnDevice on(x);
  auto iopt = x.options().dtype(at::kInt);
  at::Tensor pos = at::empty({T, k}, iopt);
  at::Tensor splits = at::empty({nranks}, iopt);
  const int64_t tiles = kern::MoeRouteTiles(T * k);
  at::Tensor hist = at::empty({tiles * (num_experts + 1)}, iopt);
  cudaError_t e = kern::LaunchMoeRoute(expert_idx.data_ptr(), expert_idx.scalar_type() == at::kLong, T * k, (int)num_experts,
                                       (int)nranks, hist.data_ptr<int>(), StreamTickets(x.get_device(), on.stream, 1),
                                       counts.data_ptr<int64_t>(), splits.data_ptr<int>(), pos.data_ptr<int>(), on.stream);
  if (e == cudaSuccess) {
    kern::MoeRows a {};
    a.src = x.data_ptr(); a.dst = send.data_ptr(); a.src_rows = T; a.dst_rows = send.size(0);
    a.pos = pos.data_ptr<int>(); a.ntok = T; a.k = (int)k; a.h = h; a.dtype = (int)MapDtype(dt);
    a.gate_dtype = (int)MapDtype(at::kFloat); a.ctas = (int)ctas;
    e = kern::LaunchMoeScatter(a, on.stream);
  }
  CheckLaunch(op, e);
  return {pos, splits};
}

// dst[pos[t, j]] = src[t] (no gates) or round(gates[t, j] * src[t]); with dot_rows also returns grad_gates [T, k] in the
// gates' dtype, grad_gates[t, j] = <src[t], dot_rows[pos[t, j]]>.
c10::optional<at::Tensor> MoeScatter(at::Tensor src, at::Tensor pos, at::Tensor dst, c10::optional<at::Tensor> gates,
                                     c10::optional<at::Tensor> dot_rows, c10::optional<at::Tensor> status, int64_t ctas) {
  const char* op = "moe_scatter";
  const auto dt = MoeDtype(op, src);
  const at::Device dev = src.device();
  const int64_t T = src.size(0), h = src.size(1);
  CheckMoeRows(op, "src", src, h, dt, dev);
  CheckMoeRows(op, "dst", dst, h, dt, dev);
  CheckMoePos(op, pos, T, dev);
  int gdt = 0;
  const void* g = MoeGates(op, gates, pos, dt, &gdt);
  TORCH_CHECK(!dot_rows || gates, op, ": dot_rows needs gates (the gate gradient has the gates' dtype)");
  if (dot_rows) CheckMoeRows(op, "dot_rows", *dot_rows, h, dt, dev);
  TORCH_CHECK(!dot_rows || dot_rows->size(0) >= dst.size(0), op, ": dot_rows must have at least dst's ", dst.size(0), " rows");
  const int* st = DeviceScalar<int>(op, "status", status, dev);
  TORCH_CHECK(ctas >= 0, op, ": ctas must be >= 0");
  const OnDevice on(src);
  c10::optional<at::Tensor> grad_gates;
  if (dot_rows) grad_gates = at::empty(pos.sizes(), gates->options());
  kern::MoeRows a {};
  a.src = src.data_ptr(); a.dst = dst.data_ptr(); a.src_rows = T; a.dst_rows = dst.size(0);
  a.pos = pos.data_ptr<int>(); a.ntok = T; a.k = (int)pos.size(1); a.h = h; a.dtype = (int)MapDtype(dt);
  a.gates = g; a.gate_dtype = gdt; a.dot_rows = dot_rows ? dot_rows->data_ptr() : nullptr;
  a.grad_gates = grad_gates ? grad_gates->data_ptr() : nullptr; a.status = st; a.ctas = (int)ctas;
  CheckLaunch(op, kern::LaunchMoeScatter(a, on.stream));
  return grad_gates;
}

// y[t] = round(sum_j gates[t, j] * src[pos[t, j]]) in fp32, j ascending (no gates: unit gates); zeros under a non-zero
// status.  Returns y [T, hidden] in src's dtype.
at::Tensor MoeGather(at::Tensor src, at::Tensor pos, c10::optional<at::Tensor> gates, c10::optional<at::Tensor> status,
                     int64_t ctas) {
  const char* op = "moe_gather";
  const auto dt = MoeDtype(op, src);
  const at::Device dev = src.device();
  const int64_t h = src.size(1);
  CheckMoeRows(op, "src", src, h, dt, dev);
  TORCH_CHECK(pos.dim() == 2, op, ": pos must be [tokens, k], got sizes ", pos.sizes());
  const int64_t T = pos.size(0);
  CheckMoePos(op, pos, T, dev);
  int gdt = 0;
  const void* g = MoeGates(op, gates, pos, dt, &gdt);
  const int* st = DeviceScalar<int>(op, "status", status, dev);
  TORCH_CHECK(ctas >= 0, op, ": ctas must be >= 0");
  const OnDevice on(src);
  at::Tensor y = at::empty({T, h}, src.options());
  kern::MoeRows a {};
  a.src = src.data_ptr(); a.dst = y.data_ptr(); a.src_rows = src.size(0); a.dst_rows = T;
  a.pos = pos.data_ptr<int>(); a.ntok = T; a.k = (int)pos.size(1); a.h = h; a.dtype = (int)MapDtype(dt);
  a.gates = g; a.gate_dtype = gdt; a.status = st; a.ctas = (int)ctas;
  CheckLaunch(op, kern::LaunchMoeGather(a, on.stream));
  return y;
}

// Source-major <-> expert-major rows (kern::LaunchMoeRegroup) with counts [nranks, experts_per_rank] int64.  Returns the
// group ends (int32 [experts_per_rank]) forward, the return splits (int32 [nranks]) in reverse.
at::Tensor MoeRegroup(at::Tensor src, at::Tensor counts, c10::optional<at::Tensor> status, at::Tensor dst, bool reverse,
                      int64_t ctas) {
  const char* op = reverse ? "moe_regroup_reverse" : "moe_regroup";
  const auto dt = MoeDtype(op, src);
  const at::Device dev = src.device();
  const int64_t rows = src.size(0), h = src.size(1);
  CheckMoeRows(op, "src", src, h, dt, dev);
  CheckMoeRows(op, "dst", dst, h, dt, dev);
  TORCH_CHECK(dst.size(0) == rows, op, ": dst must have src's ", rows, " rows, got ", dst.size(0));
  TORCH_CHECK(counts.dim() == 2 && counts.size(0) >= 1 && counts.size(1) >= 1 && counts.numel() <= kern::kMoeMaxExperts, op,
              ": counts must be [nranks, experts_per_rank] with at most ", kern::kMoeMaxExperts, " elements, got sizes ",
              counts.sizes());
  CheckVector(op, "counts", counts, dev, {at::kLong}, counts.numel());
  const int n = (int)counts.size(0), el = (int)counts.size(1);
  TORCH_CHECK(src.data_ptr() != dst.data_ptr() || el == 1, op, ": src and dst may only be the same tensor with one expert per rank");
  const int* st = DeviceScalar<int>(op, "status", status, dev);
  TORCH_CHECK(ctas >= 0, op, ": ctas must be >= 0");
  const OnDevice on(src);
  at::Tensor out = at::empty({reverse ? n : el}, src.options().dtype(at::kInt));
  CheckLaunch(op, kern::LaunchMoeRegroup(src.data_ptr(), dst.data_ptr(), h * (int64_t)src.element_size(), rows,
                                         counts.data_ptr<int64_t>(), n, el, st, reverse,
                                         reverse ? nullptr : out.data_ptr<int>(), reverse ? out.data_ptr<int>() : nullptr,
                                         (int)ctas, on.stream));
  return out;
}

}  // namespace

void DefMoe(py::module_& m) {
  m.def("moe_permute", &MoePermute, py::arg("x"), py::arg("expert_idx"), py::arg("send"), py::arg("counts"),
        py::arg("num_experts"), py::arg("nranks"), py::arg("ctas") = 0);
  m.def("moe_scatter", &MoeScatter, py::arg("src"), py::arg("pos"), py::arg("dst"), py::arg("gates") = py::none(),
        py::arg("dot_rows") = py::none(), py::arg("status") = py::none(), py::arg("ctas") = 0);
  m.def("moe_gather", &MoeGather, py::arg("src"), py::arg("pos"), py::arg("gates") = py::none(),
        py::arg("status") = py::none(), py::arg("ctas") = 0);
  m.def("moe_regroup", &MoeRegroup, py::arg("src"), py::arg("counts"), py::arg("status"), py::arg("dst"),
        py::arg("reverse"), py::arg("ctas") = 0);
}

}  // namespace hvd
