// PyTorch entry points of the hvd.SyncBatchNorm kernels (see kernels/sync_bn_kernels.cu).  Every argument is checked
// here, before anything is launched.
#include "../kernels/p2p_kernels.h"
#include "../kernels/sync_bn_kernels.h"
#include "binding_util.h"

namespace hvd {
namespace {

// The view of an input with channels at dim 1: rows [M, C] when, walking dims 1, d-1, ..., 2, 0, the strides are those of
// a packed array (channels_last, [N, C], spatial size 1; dims of size 1 do not matter), else planes [N, C, L] when it is
// contiguous.  Other layouts are the caller's to make contiguous.
kern::BnGeom BnView(const char* op, const at::Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.dim() >= 2 && x.size(1) > 0, op, ": x must be a CUDA tensor with at least 2 dimensions "
              "and at least one channel");
  const auto st = x.scalar_type();
  TORCH_CHECK(st == at::kFloat || st == at::kBFloat16 || st == at::kHalf, op, ": x must be float32, bfloat16 or float16, got ", st);
  const int64_t d = x.dim(), C = x.size(1);
  std::vector<int64_t> order {1};
  for (int64_t k = d - 1; k >= 2; --k) order.push_back(k);
  order.push_back(0);
  bool rows = true;
  int64_t expect = 1;
  for (int64_t k : order) {
    if (x.size(k) != 1 && x.stride(k) != expect) { rows = false; break; }
    expect *= x.size(k);
  }
  if (rows) return kern::BnGeom {kern::kBnRows, x.numel() / C, C, 1};
  TORCH_CHECK(x.is_contiguous(), op, ": x must be contiguous or channels-last (channels innermost), got strides ", x.strides());
  const int64_t N = x.size(0);
  return kern::BnGeom {kern::kBnPlanes, N, C, N > 0 ? x.numel() / (N * C) : 0};
}

// weight / bias: fp32 or x's dtype, both the same
int BnAffineDtype(const char* op, const c10::optional<at::Tensor>& w, const c10::optional<at::Tensor>& b, int64_t C,
                  const at::Tensor& x) {
  const at::Tensor* first = w ? &*w : (b ? &*b : nullptr);
  if (!first) return (int)MapDtype(at::kFloat);
  if (w) CheckVector(op, "weight", *w, x.device(), {at::kFloat, x.scalar_type()}, C);
  if (b) CheckVector(op, "bias", *b, x.device(), {at::kFloat, x.scalar_type()}, C);
  TORCH_CHECK(!(w && b) || w->scalar_type() == b->scalar_type(), op, ": weight and bias must have the same dtype");
  return (int)MapDtype(first->scalar_type());
}

// This rank's {count, mean, M2} of every channel of x, as fp64 triples, into slot[0 : 3C].
void SyncBnStats(at::Tensor x, at::Tensor slot) {
  const kern::BnGeom g = BnView("sync_bn_stats", x);
  CheckVector("sync_bn_stats", "slot", slot, x.device(), {at::kDouble}, 3 * g.C, true);
  const OnDevice on(x);
  const int dt = (int)MapDtype(x.scalar_type());
  const kern::BnPlan plan = kern::BnReducePlan(g, dt);
  at::Tensor part = at::empty({plan.splits * g.C * 2}, x.options().dtype(at::kDouble));  // 16 B per partial
  CheckLaunch("sync_bn_stats", kern::LaunchBnStats(x.data_ptr(), g, dt, part.data_ptr(),
                                                   StreamTickets(x.get_device(), on.stream, plan.tiles),
                                                   slot.data_ptr<double>(), on.stream));
}

// Merges the slots (rows of `slots`, in rank order) of C channels: returns (mean, invstd, count) as float32 and updates
// the running statistics where given.
std::tuple<at::Tensor, at::Tensor, at::Tensor> SyncBnCombine(at::Tensor slots, int64_t C, double eps, double momentum,
                                                             c10::optional<at::Tensor> running_mean,
                                                             c10::optional<at::Tensor> running_var,
                                                             c10::optional<at::Tensor> num_batches_tracked) {
  const char* op = "sync_bn_combine";
  TORCH_CHECK(C > 0, op, ": C must be positive");
  TORCH_CHECK(slots.is_cuda() && slots.scalar_type() == at::kDouble && slots.is_contiguous() && slots.dim() == 2 &&
              slots.size(0) >= 1 && slots.size(0) <= kern::kMaxPeers && slots.size(1) >= 3 * C, op,
              ": slots must be a contiguous float64 CUDA tensor [nranks <= ", kern::kMaxPeers, ", >= 3 * C], got ",
              slots.scalar_type(), " ", slots.sizes());
  TORCH_CHECK(running_mean.has_value() == running_var.has_value(), op, ": running_mean and running_var go together");
  int sdt = (int)MapDtype(at::kFloat);
  if (running_mean) {
    CheckVector(op, "running_mean", *running_mean, slots.device(), {at::kFloat, at::kBFloat16, at::kHalf}, C);
    CheckVector(op, "running_var", *running_var, slots.device(), {at::kFloat, at::kBFloat16, at::kHalf}, C);
    TORCH_CHECK(running_mean->scalar_type() == running_var->scalar_type(), op, ": running stats must have one dtype");
    sdt = (int)MapDtype(running_mean->scalar_type());
  }
  TORCH_CHECK(!num_batches_tracked || running_mean, op, ": num_batches_tracked goes with running stats");
  const int64_t* nbt = DeviceScalar<int64_t>(op, "num_batches_tracked", num_batches_tracked, slots.device());
  const OnDevice on(slots);
  at::Tensor mean = at::empty({C}, slots.options().dtype(at::kFloat)), invstd = at::empty_like(mean);
  at::Tensor count = at::empty({1}, mean.options());
  CheckLaunch(op, kern::LaunchBnCombine(slots.data_ptr<double>(), (int)slots.size(0), slots.size(1), C, eps, momentum, nbt,
                                        mean.data_ptr<float>(), invstd.data_ptr<float>(), count.data_ptr<float>(),
                                        running_mean ? running_mean->data_ptr() : nullptr,
                                        running_var ? running_var->data_ptr() : nullptr, sdt, on.stream));
  return {mean, invstd, count};
}

at::Tensor SyncBnElemt(at::Tensor x, at::Tensor mean, at::Tensor invstd, c10::optional<at::Tensor> weight,
                       c10::optional<at::Tensor> bias) {
  const char* op = "sync_bn_elemt";
  const kern::BnGeom g = BnView(op, x);
  CheckVector(op, "mean", mean, x.device(), {at::kFloat}, g.C);
  CheckVector(op, "invstd", invstd, x.device(), {at::kFloat}, g.C);
  const int wdt = BnAffineDtype(op, weight, bias, g.C, x);
  const OnDevice on(x);
  at::Tensor y = at::empty_like(x);  // x is dense, so y gets its strides
  CheckLaunch(op, kern::LaunchBnElemt(x.data_ptr(), y.data_ptr(), g, (int)MapDtype(x.scalar_type()), mean.data_ptr<float>(),
                                      invstd.data_ptr<float>(), weight ? weight->data_ptr() : nullptr,
                                      bias ? bias->data_ptr() : nullptr, wdt, on.stream));
  return y;
}

void CheckBnGrad(const char* op, const at::Tensor& dy, const at::Tensor& x) {
  TORCH_CHECK(dy.device() == x.device() && dy.scalar_type() == x.scalar_type() && dy.sizes() == x.sizes() &&
              dy.strides() == x.strides(), op, ": grad_output must have x's device, dtype, sizes and strides");
}

// sums[2c] = sum dy, sums[2c+1] = sum dy * (x - mean) over this rank's batch; returns the local (grad_weight, grad_bias)
// in the weight's dtype where asked for (None otherwise).
std::tuple<at::Tensor, at::Tensor> SyncBnBackwardReduce(at::Tensor dy, at::Tensor x, at::Tensor mean, at::Tensor invstd,
                                                        c10::optional<at::Tensor> weight, at::Tensor sums,
                                                        bool need_weight_grad, bool need_bias_grad) {
  const char* op = "sync_bn_backward_reduce";
  const kern::BnGeom g = BnView(op, x);
  CheckBnGrad(op, dy, x);
  CheckVector(op, "mean", mean, x.device(), {at::kFloat}, g.C);
  CheckVector(op, "invstd", invstd, x.device(), {at::kFloat}, g.C);
  CheckVector(op, "sums", sums, x.device(), {at::kDouble}, 2 * g.C, true);
  const int wdt = BnAffineDtype(op, weight, c10::nullopt, g.C, x);
  const auto wopt = x.options().dtype(weight ? weight->scalar_type() : at::kFloat);
  at::Tensor gw = need_weight_grad ? at::empty({g.C}, wopt) : at::Tensor();
  at::Tensor gb = need_bias_grad ? at::empty({g.C}, wopt) : at::Tensor();
  const OnDevice on(x);
  const int dt = (int)MapDtype(x.scalar_type());
  const kern::BnPlan plan = kern::BnReducePlan(g, dt);
  at::Tensor part = at::empty({plan.splits * g.C * 2}, x.options().dtype(at::kFloat));  // 8 B per partial
  CheckLaunch(op, kern::LaunchBnBackwardReduce(dy.data_ptr(), x.data_ptr(), g, dt, mean.data_ptr<float>(),
                                               invstd.data_ptr<float>(), part.data_ptr(),
                                               StreamTickets(x.get_device(), on.stream, plan.tiles), sums.data_ptr<double>(),
                                               gw.defined() ? gw.data_ptr() : nullptr, gb.defined() ? gb.data_ptr() : nullptr,
                                               wdt, on.stream));
  return {gw, gb};
}

at::Tensor SyncBnBackwardElemt(at::Tensor dy, at::Tensor x, at::Tensor mean, at::Tensor invstd,
                               c10::optional<at::Tensor> weight, at::Tensor sums, at::Tensor count) {
  const char* op = "sync_bn_backward_elemt";
  const kern::BnGeom g = BnView(op, x);
  CheckBnGrad(op, dy, x);
  CheckVector(op, "mean", mean, x.device(), {at::kFloat}, g.C);
  CheckVector(op, "invstd", invstd, x.device(), {at::kFloat}, g.C);
  CheckVector(op, "sums", sums, x.device(), {at::kDouble}, 2 * g.C, true);
  CheckVector(op, "count", count, x.device(), {at::kFloat}, 1);
  const int wdt = BnAffineDtype(op, weight, c10::nullopt, g.C, x);
  const OnDevice on(x);
  at::Tensor dx = at::empty_like(x);
  CheckLaunch(op, kern::LaunchBnBackwardElemt(dy.data_ptr(), x.data_ptr(), dx.data_ptr(), g, (int)MapDtype(x.scalar_type()),
                                              mean.data_ptr<float>(), invstd.data_ptr<float>(),
                                              weight ? weight->data_ptr() : nullptr, wdt, sums.data_ptr<double>(),
                                              count.data_ptr<float>(), on.stream));
  return dx;
}

}  // namespace

void DefSyncBn(py::module_& m) {
  m.def("sync_bn_stats", &SyncBnStats, py::arg("x"), py::arg("slot"));
  m.def("sync_bn_combine", &SyncBnCombine, py::arg("slots"), py::arg("num_features"), py::arg("eps"), py::arg("momentum"),
        py::arg("running_mean") = py::none(), py::arg("running_var") = py::none(),
        py::arg("num_batches_tracked") = py::none());
  m.def("sync_bn_elemt", &SyncBnElemt, py::arg("x"), py::arg("mean"), py::arg("invstd"), py::arg("weight") = py::none(),
        py::arg("bias") = py::none());
  m.def("sync_bn_backward_reduce", &SyncBnBackwardReduce, py::arg("grad_output"), py::arg("x"), py::arg("mean"),
        py::arg("invstd"), py::arg("weight"), py::arg("sums"), py::arg("need_weight_grad"), py::arg("need_bias_grad"));
  m.def("sync_bn_backward_elemt", &SyncBnBackwardElemt, py::arg("grad_output"), py::arg("x"), py::arg("mean"),
        py::arg("invstd"), py::arg("weight"), py::arg("sums"), py::arg("count"));
}

}  // namespace hvd
