// PyTorch entry points of the fused optimizer, gradient statistics and gradient accumulation kernels (an extra of this
// library; see kernels/optim_kernels.cu).  The kernels address every tensor of entry i with the element index of
// params[i] and take one element type per list, so each companion tensor must have the param's sizes and strides, one
// dtype per list, and live on the param's device (CheckLike).  Checked here, before anything is staged.
#include <set>
#include "../kernels/optim_kernels.h"
#include "../ops/gpu_ops.h"
#include "binding_util.h"

namespace hvd {
namespace {

// fp32 master weights (optional, empty: none): one fp32 tensor per param with its sizes, strides and device.  Only for
// bf16 / fp16 params with gradients of the same dtype, the pairs the master kernels are instantiated for.  Call after
// the params themselves are checked.  Returns whether masters are in use.
bool CheckMasters(const char* op, const std::vector<at::Tensor>& params, const std::vector<at::Tensor>& grads,
                  const std::vector<at::Tensor>& masters) {
  if (masters.empty()) return false;
  const auto pt = params[0].scalar_type();
  TORCH_CHECK(pt == at::kBFloat16 || pt == at::kHalf, op, ": master_params are for bfloat16 / float16 params, params are ", pt);
  TORCH_CHECK(grads[0].scalar_type() == pt, op, ": with master_params the grads must be ", pt, ", got ", grads[0].scalar_type());
  for (size_t i = 0; i < params.size(); ++i) CheckLike(op, "master_params", i, masters[i], at::kFloat, "params", params[i]);
  return true;
}

// One state list of an optimizer call and the table field it fills.  States are fp32, except a list marked
// `param_dtype` (SGD momentum), which has the param's dtype without masters.
struct OptState {
  const char* name;
  const std::vector<at::Tensor>& list;
  void* kern::OptTensor::*field;
  bool param_dtype = false;
};

// A checked call of the kern::Launch* optimizer launchers: the table, its dtypes and what the launchers take besides.
struct OptPlan {
  std::vector<kern::OptTensor> table;
  int64_t max_count = 0, partials = 0;
  int param_dtype = 0, grad_dtype = 0;
  bool master = false;
  const float* grad_scale_dev = nullptr;
  kern::OptEma ema;
};

// The EMA of one optimizer call (optional, empty list: none): one fp32 tensor per param with its sizes, strides and
// device, updated after the parameter with weight = 1 - decay; `start` begins every one of them at the updated value.
struct EmaArgs {
  const std::vector<at::Tensor>& list;
  double weight;
  bool start;
};
const std::vector<at::Tensor> kNoTensors;
const EmaArgs kNoEma{kNoTensors, 0.0, false};

// Checks every argument of one optimizer call and builds its table; nothing is staged or launched here.  Entry i is
// params[i] with grads[i], masters[i] and each state list's element in its field.  `norms` (LAMB and LARS; nullptr:
// none) is a contiguous fp32 tensor on the params' device with 2 floats per slot: entry i gets norm slot slots[i]
// (empty: i) and the offset of its stage-1 partials.  Zero-size params get no entry.
OptPlan PlanOpt(const char* op, const std::vector<at::Tensor>& params, const std::vector<at::Tensor>& grads,
                const std::vector<OptState>& states, const std::vector<at::Tensor>& masters,
                const c10::optional<at::Tensor>& grad_scale_dev, const at::Tensor* norms = nullptr,
                const std::vector<int64_t>& slots = {}, const EmaArgs& ema = kNoEma) {
  bool sizes = params.size() == grads.size();
  for (const auto& st : states) sizes = sizes && st.list.size() == params.size();
  TORCH_CHECK(sizes, op, ": list sizes differ");
  TORCH_CHECK(masters.empty() || masters.size() == params.size(), op, ": ", masters.size(), " master params for ",
              params.size(), " params");
  TORCH_CHECK(slots.empty() || slots.size() == params.size(), op, ": ", slots.size(), " slots for ", params.size(), " params");
  TORCH_CHECK(ema.list.empty() || ema.list.size() == params.size(), op, ": ", ema.list.size(), " ema params for ",
              params.size(), " params");
  OptPlan plan;
  if (params.empty()) return plan;
  for (size_t i = 0; i < params.size(); ++i) {
    CheckEntry(op, "params", i, params[i], params[0]);
    CheckLike(op, "grads", i, grads[i], grads[0].scalar_type(), "params", params[i]);
  }
  plan.master = CheckMasters(op, params, grads, masters);
  for (size_t i = 0; i < ema.list.size(); ++i) CheckLike(op, "ema_params", i, ema.list[i], at::kFloat, "params", params[i]);
  plan.ema = kern::OptEma{!ema.list.empty(), (float)ema.weight, ema.start ? 1 : 0};
  for (const auto& st : states)
    for (size_t i = 0; i < params.size(); ++i)
      CheckLike(op, st.name, i, st.list[i], st.param_dtype && !plan.master ? params[i].scalar_type() : at::kFloat,
                "params", params[i]);
  if (norms != nullptr) {
    TORCH_CHECK(norms->is_cuda() && norms->device() == params[0].device() && norms->scalar_type() == at::kFloat &&
                norms->is_contiguous(), op, ": norms must be a contiguous float32 tensor on ", params[0].device());
    const int64_t nslots = norms->numel() / 2;
    std::set<int64_t> seen;
    for (size_t i = 0; i < params.size(); ++i) {
      const int64_t s = slots.empty() ? (int64_t)i : slots[i];
      TORCH_CHECK(s >= 0 && s < nslots, op, ": slot ", s, " of params[", i, "] is out of range for norms with room for ",
                  nslots, " slots");
      TORCH_CHECK(seen.insert(s).second, op, ": slot ", s, " appears twice in one call");
    }
  }
  plan.grad_scale_dev = DeviceScalar<float>(op, "grad_scale_dev", grad_scale_dev, params[0].device());
  plan.param_dtype = (int)MapDtype(params[0].scalar_type());
  plan.grad_dtype = (int)MapDtype(grads[0].scalar_type());
  for (size_t i = 0; i < params.size(); ++i) {
    if (params[i].numel() == 0) continue;
    kern::OptTensor t{};
    t.param = params[i].data_ptr(); t.grad = grads[i].data_ptr();
    t.master = plan.master ? masters[i].data_ptr() : nullptr;
    t.ema = plan.ema.on ? ema.list[i].data_ptr() : nullptr;
    for (const auto& st : states) t.*st.field = st.list[i].data_ptr();
    t.count = params[i].numel();
    if (norms != nullptr) {
      t.partial = plan.partials;
      t.slot = slots.empty() ? (int64_t)i : slots[i];
      plan.partials += kern::NormPartials(t.count);
    }
    plan.max_count = std::max(plan.max_count, t.count);
    plan.table.push_back(t);
  }
  return plan;
}

// The optimizer kernels select the table entry with blockIdx.y, which CUDA caps at 65535.  A piece of that many entries
// (72 B each) also fits the 8 MiB staging ring of GpuContext::Stage.
constexpr size_t kOptMaxEntries = 65535;

// One launch's share of a plan's table: `n` entries staged on the device and the longest of their counts.
struct OptPiece {
  const kern::OptTensor* table;
  int n;
  int64_t max_count;
};

// Stages the plan's table on the params' device in pieces of at most kOptMaxEntries entries (one piece, so one launch
// per phase, when the table fits) and runs launch(piece, current stream) for each, which makes one or more kern::Launch*
// calls and returns the first error.  Every entry keeps its norm slot and partial offset, so the LAMB / LARS phases run
// piece by piece unchanged.
template <typename F>
void RunPlan(const char* op, const OptPlan& plan, const std::vector<at::Tensor>& params, F&& launch) {
  if (plan.table.empty()) return;
  const int device = (int)params[0].get_device();
  const OnDevice on(params[0]);
  for (size_t lo = 0; lo < plan.table.size(); lo += kOptMaxEntries) {
    const size_t n = std::min(kOptMaxEntries, plan.table.size() - lo);
    int64_t max_count = 0;
    for (size_t i = lo; i < lo + n; ++i) max_count = std::max(max_count, plan.table[i].count);
    const auto* dt = (const kern::OptTensor*)GpuContext::Get().Stage(device, plan.table.data() + lo,
                                                                      n * sizeof(kern::OptTensor), on.stream);
    TORCH_CHECK(dt != nullptr, op, ": table too large");
    CheckLaunch(op, launch(OptPiece{dt, (int)n, max_count}, on.stream));
  }
}

std::vector<OptState> MomentStates(const std::vector<at::Tensor>& exp_avg, const std::vector<at::Tensor>& exp_avg_sq) {
  return {{"exp_avgs", exp_avg, &kern::OptTensor::state0}, {"exp_avg_sqs", exp_avg_sq, &kern::OptTensor::state1}};
}

// Adam's and LAMB's bias correction 1 - beta^step; step is 1-based: step 0 would make it 0 and every parameter inf / NaN
float BiasCorrection(const char* op, double beta, int64_t step) {
  TORCH_CHECK(step >= 1, op, ": step must be >= 1, got ", step);
  return 1.0f - (float)std::pow(beta, (double)step);
}

void FusedSgdStep(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> momenta, double lr,
                  double momentum, double dampening, double weight_decay, bool nesterov, double grad_scale, bool first_step,
                  c10::optional<at::Tensor> grad_scale_dev, std::vector<at::Tensor> masters, std::vector<at::Tensor> emas,
                  double ema_weight, bool ema_start) {
  const bool has_mom = momentum != 0.0;
  // without momentum the buffers are not read: none, or a list of the params' length
  TORCH_CHECK(has_mom || momenta.empty() || momenta.size() == params.size(),
              "fused_sgd: ", momenta.size(), " momentum buffers for ", params.size(), " params");
  std::vector<OptState> states;
  if (has_mom) states.push_back({"momentum_buffers", momenta, &kern::OptTensor::state0, true});
  const OptPlan plan = PlanOpt("fused_sgd", params, grads, states, masters, grad_scale_dev, nullptr, {},
                               EmaArgs{emas, ema_weight, ema_start});
  RunPlan("fused_sgd", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    return kern::LaunchFusedSgd(pc.table, pc.n, pc.max_count, (float)lr, (float)momentum, (float)dampening,
                                (float)weight_decay, nesterov ? 1 : 0, (float)grad_scale, first_step ? 1 : 0,
                                plan.param_dtype, plan.grad_dtype, s, plan.grad_scale_dev, plan.master, plan.ema);
  });
}

void FusedAdamStep(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> exp_avg,
                   std::vector<at::Tensor> exp_avg_sq, double lr, double beta1, double beta2, double eps, double weight_decay,
                   int64_t step, double grad_scale, bool adamw, c10::optional<at::Tensor> grad_scale_dev,
                   std::vector<at::Tensor> masters, std::vector<at::Tensor> emas, double ema_weight, bool ema_start) {
  const float c1 = BiasCorrection("fused_adam", beta1, step), c2 = BiasCorrection("fused_adam", beta2, step);
  const OptPlan plan = PlanOpt("fused_adam", params, grads, MomentStates(exp_avg, exp_avg_sq), masters, grad_scale_dev,
                               nullptr, {}, EmaArgs{emas, ema_weight, ema_start});
  RunPlan("fused_adam", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    return kern::LaunchFusedAdamW(pc.table, pc.n, pc.max_count, (float)lr, (float)beta1, (float)beta2,
                                  (float)eps, (float)weight_decay, c1, c2, (float)grad_scale, adamw ? 1 : 0,
                                  plan.param_dtype, plan.grad_dtype, s, plan.grad_scale_dev, plan.master, plan.ema);
  });
}

// ---- fused LAMB and LARS: a norms phase (two launches) and an apply phase (one launch) on one table with a norm slot
// per entry, so that the norms can be allreduced in between.

// stream-ordered scratch from torch's caching allocator: one pair of sums of squares per stage-1 CTA
at::Tensor NormsScratch(const OptPlan& plan, const at::Tensor& norms) { return at::empty({2 * plan.partials}, norms.options()); }

struct LambArgs { double beta1, beta2, eps, weight_decay; float c1, c2; };

LambArgs LambHyper(const char* op, double beta1, double beta2, double eps, double weight_decay, int64_t step,
                   bool bias_correction) {
  const float c1 = BiasCorrection(op, beta1, step), c2 = BiasCorrection(op, beta2, step);  // checks step in any case
  return bias_correction ? LambArgs{beta1, beta2, eps, weight_decay, c1, c2} : LambArgs{beta1, beta2, eps, weight_decay, 1.f, 1.f};
}

cudaError_t LambNormsPhase(const OptPlan& plan, const OptPiece& pc, const LambArgs& a, double grad_scale,
                           at::Tensor& norms, cudaStream_t s) {
  at::Tensor work = NormsScratch(plan, norms);
  return kern::LaunchLambNorms(pc.table, pc.n, pc.max_count, (float)a.beta1, (float)a.beta2, (float)a.eps,
                               (float)a.weight_decay, a.c1, a.c2, (float)grad_scale, plan.grad_scale_dev,
                               work.data_ptr<float>(), norms.data_ptr<float>(), plan.param_dtype, plan.grad_dtype,
                               plan.master, s);
}

cudaError_t LambApplyPhase(const OptPlan& plan, const OptPiece& pc, const LambArgs& a, double lr, bool adapt,
                           const at::Tensor& norms, cudaStream_t s) {
  return kern::LaunchLambApply(pc.table, pc.n, pc.max_count, (float)lr, (float)a.eps, (float)a.weight_decay,
                               a.c1, a.c2, adapt ? 1 : 0, norms.data_ptr<float>(), plan.param_dtype, plan.master, s,
                               plan.ema);
}

// Phase 1: moments, then the squared norms of every entry ADDED into norms[2 * slot], norms[2 * slot + 1].
void LambNorms(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> exp_avg,
               std::vector<at::Tensor> exp_avg_sq, double beta1, double beta2, double eps, double weight_decay, int64_t step,
               bool bias_correction, double grad_scale, c10::optional<at::Tensor> grad_scale_dev,
               std::vector<at::Tensor> masters, at::Tensor out, std::vector<int64_t> slots) {
  const LambArgs a = LambHyper("lamb_norms", beta1, beta2, eps, weight_decay, step, bias_correction);
  const OptPlan plan = PlanOpt("lamb_norms", params, grads, MomentStates(exp_avg, exp_avg_sq), masters, grad_scale_dev,
                               &out, slots);
  RunPlan("lamb_norms", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    return LambNormsPhase(plan, pc, a, grad_scale, out, s);
  });
}

// Phase 2: w -= lr * r * u with r from the (allreduced) norms.  `grads` are checked like phase 1's, not read.
void LambApply(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> exp_avg,
               std::vector<at::Tensor> exp_avg_sq, double lr, double beta1, double beta2, double eps, double weight_decay,
               int64_t step, bool bias_correction, bool adapt, std::vector<at::Tensor> masters, at::Tensor norms,
               std::vector<int64_t> slots, std::vector<at::Tensor> emas, double ema_weight, bool ema_start) {
  const LambArgs a = LambHyper("lamb_apply", beta1, beta2, eps, weight_decay, step, bias_correction);
  const OptPlan plan = PlanOpt("lamb_apply", params, grads, MomentStates(exp_avg, exp_avg_sq), masters, c10::nullopt,
                               &norms, slots, EmaArgs{emas, ema_weight, ema_start});
  RunPlan("lamb_apply", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    return LambApplyPhase(plan, pc, a, lr, adapt, norms, s);
  });
}

// A fresh norms buffer for both phases on one device (slot i = params[i]).
at::Tensor FreshNorms(const char* op, const std::vector<at::Tensor>& params) {
  TORCH_CHECK(params.empty() || params[0].is_cuda(), op, ": params[0] must be a dense CUDA tensor");
  return params.empty() ? at::Tensor() : at::zeros({2 * (int64_t)params.size()}, params[0].options().dtype(at::kFloat));
}

// Both phases: three launches per staged piece of the table (one piece up to 65535 entries).
void FusedLambStep(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> exp_avg,
                   std::vector<at::Tensor> exp_avg_sq, double lr, double beta1, double beta2, double eps, double weight_decay,
                   int64_t step, bool bias_correction, bool adapt, double grad_scale,
                   c10::optional<at::Tensor> grad_scale_dev, std::vector<at::Tensor> masters, std::vector<at::Tensor> emas,
                   double ema_weight, bool ema_start) {
  at::Tensor norms = FreshNorms("fused_lamb", params);
  const LambArgs a = LambHyper("fused_lamb", beta1, beta2, eps, weight_decay, step, bias_correction);
  const OptPlan plan = PlanOpt("fused_lamb", params, grads, MomentStates(exp_avg, exp_avg_sq), masters, grad_scale_dev,
                               &norms, {}, EmaArgs{emas, ema_weight, ema_start});
  RunPlan("fused_lamb", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    const cudaError_t e = LambNormsPhase(plan, pc, a, grad_scale, norms, s);
    return e != cudaSuccess ? e : LambApplyPhase(plan, pc, a, lr, adapt, norms, s);
  });
}

// LARS keeps one fp32 state, the momentum buffer.
std::vector<OptState> LarsStates(const std::vector<at::Tensor>& momentum_buffers) {
  return {{"momentum_buffers", momentum_buffers, &kern::OptTensor::state0}};
}

cudaError_t LarsNormsPhase(const OptPlan& plan, const OptPiece& pc, double grad_scale, at::Tensor& norms,
                           cudaStream_t s) {
  at::Tensor work = NormsScratch(plan, norms);
  return kern::LaunchLarsNorms(pc.table, pc.n, pc.max_count, (float)grad_scale, plan.grad_scale_dev,
                               work.data_ptr<float>(), norms.data_ptr<float>(), plan.param_dtype, plan.grad_dtype,
                               plan.master, s);
}

cudaError_t LarsApplyPhase(const OptPlan& plan, const OptPiece& pc, double lr, double momentum, double weight_decay,
                           double trust_coefficient, double eps, bool adapt, double grad_scale, const at::Tensor& norms,
                           cudaStream_t s) {
  return kern::LaunchLarsApply(pc.table, pc.n, pc.max_count, (float)lr, (float)momentum, (float)weight_decay,
                               (float)trust_coefficient, (float)eps, adapt ? 1 : 0, (float)grad_scale, plan.grad_scale_dev,
                               norms.data_ptr<float>(), plan.param_dtype, plan.grad_dtype, plan.master, s, plan.ema);
}

// LARS phase 1: the squared norms of every entry's parameter and scaled gradient ADDED into norms[2 * slot],
// norms[2 * slot + 1].  The momentum buffers are checked like phase 2's, not read.
void LarsNorms(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> momentum_buffers,
               double grad_scale, c10::optional<at::Tensor> grad_scale_dev, std::vector<at::Tensor> masters, at::Tensor out,
               std::vector<int64_t> slots) {
  const OptPlan plan = PlanOpt("lars_norms", params, grads, LarsStates(momentum_buffers), masters, grad_scale_dev, &out,
                               slots);
  RunPlan("lars_norms", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    return LarsNormsPhase(plan, pc, grad_scale, out, s);
  });
}

// LARS phase 2: momentum and parameter update with r from the (allreduced) norms; reads the gradient again, scaled the
// same way as in phase 1.
void LarsApply(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> momentum_buffers,
               double lr, double momentum, double weight_decay, double trust_coefficient, double eps, bool adapt,
               double grad_scale, c10::optional<at::Tensor> grad_scale_dev, std::vector<at::Tensor> masters,
               at::Tensor norms, std::vector<int64_t> slots, std::vector<at::Tensor> emas, double ema_weight,
               bool ema_start) {
  const OptPlan plan = PlanOpt("lars_apply", params, grads, LarsStates(momentum_buffers), masters, grad_scale_dev, &norms,
                               slots, EmaArgs{emas, ema_weight, ema_start});
  RunPlan("lars_apply", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    return LarsApplyPhase(plan, pc, lr, momentum, weight_decay, trust_coefficient, eps, adapt, grad_scale, norms, s);
  });
}

// Both LARS phases: three launches per staged piece of the table (one piece up to 65535 entries).
void FusedLarsStep(std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> momentum_buffers,
                   double lr, double momentum, double weight_decay, double trust_coefficient, double eps, bool adapt,
                   double grad_scale, c10::optional<at::Tensor> grad_scale_dev, std::vector<at::Tensor> masters,
                   std::vector<at::Tensor> emas, double ema_weight, bool ema_start) {
  at::Tensor norms = FreshNorms("fused_lars", params);
  const OptPlan plan = PlanOpt("fused_lars", params, grads, LarsStates(momentum_buffers), masters, grad_scale_dev, &norms,
                               {}, EmaArgs{emas, ema_weight, ema_start});
  RunPlan("fused_lars", plan, params, [&](const OptPiece& pc, cudaStream_t s) {
    const cudaError_t e = LarsNormsPhase(plan, pc, grad_scale, norms, s);
    return e != cudaSuccess ? e : LarsApplyPhase(plan, pc, lr, momentum, weight_decay, trust_coefficient, eps, adapt,
                                                 grad_scale, norms, s);
  });
}

// ---- fused Adafactor: the OptTensor table of PlanOpt (variance of dim <= 1 params in state0, one norm slot per param)
// plus a geometry table parallel to it for the factored params.  Both tables and all scratch live in tensors of torch's
// caching allocator on the current stream, and the tables reach the device through kernel parameters, so the call can
// be captured into a CUDA graph.

// Checks that `f` is params[i]'s row (`dim` = -1) or column (`dim` = -2) factor: fp32, contiguous, on its device, with
// its sizes except 1 at `dim`.
void CheckAdafactorFactor(const char* op, const char* what, size_t i, const at::Tensor& param,
                          const c10::optional<at::Tensor>& f, int64_t dim) {
  TORCH_CHECK(f.has_value() && f->defined(), op, ": ", what, "[", i, "] is missing for params[", i, "] of dim ", param.dim());
  TORCH_CHECK(f->device() == param.device(), op, ": ", what, "[", i, "] is on ", f->device(), ", params[", i, "] on ",
              param.device());
  TORCH_CHECK(f->scalar_type() == at::kFloat, op, ": ", what, "[", i, "] is ", f->scalar_type(), ", expected Float");
  std::vector<int64_t> want = param.sizes().vec();
  want[want.size() + dim] = 1;
  TORCH_CHECK(f->sizes() == at::IntArrayRef(want), op, ": ", what, "[", i, "] has size ", f->sizes(), ", expected ",
              at::IntArrayRef(want));
  TORCH_CHECK(f->is_contiguous(), op, ": ", what, "[", i, "] must be contiguous");
}

void FusedAdafactorStep(std::vector<at::Tensor> params, std::vector<at::Tensor> grads,
                        std::vector<c10::optional<at::Tensor>> row_vars, std::vector<c10::optional<at::Tensor>> col_vars,
                        std::vector<c10::optional<at::Tensor>> variances, double lr, double beta2_decay, double eps1,
                        double eps2, double d, double weight_decay, int64_t step, double grad_scale,
                        c10::optional<at::Tensor> grad_scale_dev, std::vector<at::Tensor> masters,
                        std::vector<at::Tensor> emas, double ema_weight, bool ema_start) {
  const char* op = "fused_adafactor";
  TORCH_CHECK(row_vars.size() == params.size() && col_vars.size() == params.size() && variances.size() == params.size(),
              op, ": list sizes differ");
  TORCH_CHECK(step >= 1, op, ": step must be >= 1, got ", step);
  TORCH_CHECK(eps1 >= 0.0 && d > 0.0, op, ": eps1 must be >= 0 and d > 0, got eps1 = ", eps1, ", d = ", d);
  if (params.empty()) return;
  // the kernels address a parameter's elements with 32-bit unsigned offsets, and the geometry of a factored parameter
  // holds its sizes and strides as int32
  for (size_t i = 0; i < params.size(); ++i) {
    const at::Tensor& p = params[i];
    TORCH_CHECK(p.numel() < ((int64_t)1 << 32), op, ": params[", i, "] has ", p.numel(),
                " elements, at most 2^32 - 1 are supported");
    if (p.dim() < 2) continue;
    for (int64_t k = 0; k < p.dim(); ++k)
      TORCH_CHECK(p.size(k) < ((int64_t)1 << 31) && (p.size(k) == 1 || p.stride(k) < ((int64_t)1 << 31)), op,
                  ": params[", i, "] has size ", p.size(k), " and stride ", p.stride(k), " in dim ", k,
                  ", at most 2^31 - 1 are supported in each dim of a factored parameter");
  }
  // not zeroed yet: nothing is launched before every argument is checked
  at::Tensor norms = at::empty({2 * (int64_t)params.size()}, params[0].options().dtype(at::kFloat));
  OptPlan plan = PlanOpt(op, params, grads, {}, masters, grad_scale_dev, &norms, {}, EmaArgs{emas, ema_weight, ema_start});
  for (size_t i = 0; i < params.size(); ++i) {
    const at::Tensor& p = params[i];
    TORCH_CHECK(p.dim() <= kern::kAdafactorMaxDims, op, ": params[", i, "] has ", p.dim(), " dims, at most ",
                kern::kAdafactorMaxDims, " are supported");
    if (p.dim() >= 2) {
      CheckAdafactorFactor(op, "row_vars", i, p, row_vars[i], -1);
      CheckAdafactorFactor(op, "col_vars", i, p, col_vars[i], -2);
      TORCH_CHECK(!(variances[i].has_value() && variances[i]->defined()), op, ": variances[", i,
                  "] is given for params[", i, "] of dim ", p.dim(), ", which keeps row / column factors");
    } else {
      TORCH_CHECK(!(row_vars[i].has_value() && row_vars[i]->defined()) && !(col_vars[i].has_value() && col_vars[i]->defined()),
                  op, ": row_vars[", i, "] / col_vars[", i, "] are given for params[", i, "] of dim ", p.dim(),
                  ", which keeps a variance");
      TORCH_CHECK(variances[i].has_value() && variances[i]->defined(), op, ": variances[", i, "] is missing for params[",
                  i, "] of dim ", p.dim());
      CheckLike(op, "variances", i, *variances[i], at::kFloat, "params", params[i]);
    }
  }
  // the geometry of every table entry (PlanOpt gives zero-size params no entry) and the scratch offsets
  std::vector<kern::AdafactorGeom> geom;
  int64_t colparts = 0, batches = 0, stats_ctas = 1, factor_ctas = 1;
  for (size_t i = 0, e = 0; i < params.size(); ++i) {
    const at::Tensor& p = params[i];
    if (p.numel() == 0) continue;
    kern::AdafactorGeom g{};
    for (int k = 0; k < kern::kAdafactorMaxDims; ++k) { g.size[k] = 1; g.stride[k] = 1; }
    if (p.dim() >= 2) {
      for (int64_t k = 0; k < p.dim(); ++k) {
        const int slot = kern::kAdafactorMaxDims - (int)p.dim() + (int)k;
        g.size[slot] = (int32_t)p.size(k);
        g.stride[slot] = p.size(k) == 1 ? 1 : (int32_t)p.stride(k);
      }
      g.row_var = row_vars[i]->data_ptr<float>();
      g.col_var = col_vars[i]->data_ptr<float>();
      const int64_t B = (int64_t)g.size[0] * g.size[1] * g.size[2], R = g.size[3], C = g.size[4];
      g.col_off = colparts;
      g.batch_off = batches;
      colparts += B * C * kern::AdafactorRowChunks(R);
      batches += B;
      stats_ctas = std::max(stats_ctas, kern::AdafactorStatsCtas(B, R, C));
      factor_ctas = std::max(factor_ctas, kern::AdafactorFactorCtas(B, C));
    } else {
      plan.table[e].state0 = variances[i]->data_ptr();
    }
    geom.push_back(g);
    ++e;
  }
  if (plan.table.empty()) return;
  TORCH_CHECK(plan.table.size() <= 65535, op, ": at most 65535 non-empty params per call, got ", plan.table.size());
  kern::AdafactorHyper h;
  const double t = (double)step;
  h.beta_w = (float)std::pow(t, beta2_decay);
  h.rho = (float)std::min(lr, 1.0 / std::sqrt(t));
  h.eps1 = (float)eps1;
  h.eps1_sq = (float)(eps1 * eps1);
  h.eps2 = (float)eps2;
  h.d = (float)d;
  h.decay = (float)(1.0 - lr * weight_decay);
  const size_t tab_bytes = plan.table.size() * sizeof(kern::OptTensor);
  const size_t geom_at = (tab_bytes + 255) / 256 * 256, bytes = geom_at + geom.size() * sizeof(kern::AdafactorGeom);
  std::vector<unsigned char> host(bytes);
  memcpy(host.data(), plan.table.data(), tab_bytes);
  memcpy(host.data() + geom_at, geom.data(), geom.size() * sizeof(kern::AdafactorGeom));
  const OnDevice on(params[0]);
  at::Tensor tables = at::empty({(int64_t)bytes}, params[0].options().dtype(at::kByte));
  at::Tensor work = at::empty({colparts + batches + 2 * plan.partials}, norms.options());
  norms.zero_();
  float* w = work.data_ptr<float>();
  cudaError_t e = kern::LaunchUploadBytes(tables.data_ptr(), host.data(), bytes, on.stream);
  if (e == cudaSuccess) {
    const auto* dt = reinterpret_cast<const kern::OptTensor*>(tables.data_ptr<uint8_t>());
    const auto* dg = reinterpret_cast<const kern::AdafactorGeom*>(tables.data_ptr<uint8_t>() + geom_at);
    // the float2 CTA partials first, where the allocator's alignment holds; then the column partials and batch means
    float* part = w;
    float* cols = part + 2 * plan.partials;
    e = kern::LaunchAdafactor(dt, dg, (int)plan.table.size(), plan.max_count, stats_ctas, factor_ctas, h,
                              (float)grad_scale, plan.grad_scale_dev, cols, cols + colparts, part,
                              norms.data_ptr<float>(), plan.param_dtype, plan.grad_dtype, plan.master, on.stream,
                              plan.ema);
  }
  CheckLaunch(op, e);
}

// One launch of the gradient statistics kernel over `grads` (one dtype: fp32 / bf16 / fp16), folded into out[0:2].
void GradShardStats(std::vector<at::Tensor> grads, at::Tensor out, c10::optional<at::Tensor> inv_scale, bool norm_inf) {
  TORCH_CHECK(out.is_cuda() && out.scalar_type() == at::kFloat && out.is_contiguous() && out.numel() >= 2,
              "grad_shard_stats: out must be a contiguous float32 CUDA tensor with at least 2 elements");
  for (size_t i = 0; i < grads.size(); ++i) CheckEntry("grad_shard_stats", "tensors", i, grads[i], grads[0]);
  if (!grads.empty()) {
    TORCH_CHECK(grads[0].device() == out.device(), "grad_shard_stats: tensors are on ", grads[0].device(), ", out on ",
                out.device());
    const auto st = grads[0].scalar_type();
    TORCH_CHECK(st == at::kFloat || st == at::kBFloat16 || st == at::kHalf,
                "grad_shard_stats: gradients must be float32, bfloat16 or float16, got ", st);
  }
  const float* isc = DeviceScalar<float>("grad_shard_stats", "inv_scale", inv_scale, out.device());
  std::vector<kern::StatTensor> table;
  int64_t tiles = 0, row_tiles = 0;  // one CTA per tile of every tensor
  for (auto& g : grads) {
    if (g.numel() == 0) continue;
    table.push_back({g.data_ptr(), g.numel(), tiles});
    const int64_t t = kern::GradShardStatsTiles(g.numel());
    tiles += t;
    row_tiles = std::max(row_tiles, t);
  }
  if (table.empty()) return;
  TORCH_CHECK(tiles <= 0x7fffffff, "grad_shard_stats: ", tiles, " tiles exceed one launch's grid");
  int device = (int)out.get_device();
  const OnDevice on(out);
  // stream-ordered scratch from torch's caching allocator: fp32 partials followed by int flags
  at::Tensor work = at::empty({2 * tiles}, out.options());
  const auto* dt = (const kern::StatTensor*)GpuContext::Get().Stage(device, table.data(), table.size() * sizeof(kern::StatTensor),
                                                                    on.stream);
  TORCH_CHECK(dt != nullptr, "grad_shard_stats: table too large");
  CheckLaunch("grad_shard_stats",
              kern::LaunchGradShardStats(dt, (int)table.size(), tiles, row_tiles, isc, norm_inf ? 1 : 0,
                                         work.data_ptr<float>(), reinterpret_cast<int*>(work.data_ptr<float>() + tiles),
                                         StreamTickets(device, on.stream, 1), out.data_ptr<float>(),
                                         (int)MapDtype(grads[0].scalar_type()), on.stream));
}

// Fold bf16 / fp16 gradients into fp32 accumulators (kern::LaunchGradAccumulate): mode 0 first, 1 add, 2 last.  Every
// argument is checked before anything is launched; one launch per kAccMaxTensors non-empty entries, on the current stream,
// with the table as a kernel parameter, so the call can be captured into a CUDA graph.
void GradAccumulate(std::vector<at::Tensor> grads, std::vector<at::Tensor> accs, int64_t mode) {
  TORCH_CHECK(mode >= kern::kAccFirst && mode <= kern::kAccLast, "grad_accumulate: mode must be 0 (first), 1 (add) or 2 "
              "(last), got ", mode);
  TORCH_CHECK(grads.size() == accs.size(), "grad_accumulate: ", grads.size(), " gradients but ", accs.size(), " accumulators");
  if (grads.empty()) return;
  const auto st = grads[0].scalar_type();
  TORCH_CHECK(st == at::kBFloat16 || st == at::kHalf, "grad_accumulate: gradients must be bfloat16 or float16, got ", st);
  for (size_t i = 0; i < grads.size(); ++i) {
    CheckEntry("grad_accumulate", "grads", i, grads[i], grads[0]);
    CheckLike("grad_accumulate", "accs", i, accs[i], at::kFloat, "grads", grads[i]);
  }
  std::vector<kern::AccTensor> entries;
  int64_t maxc = 0;
  for (size_t i = 0; i < grads.size(); ++i) {
    if (grads[i].numel() == 0) continue;
    entries.push_back({grads[i].data_ptr(), accs[i].data_ptr<float>(), grads[i].numel()});
  }
  if (entries.empty()) return;
  const OnDevice on(grads[0]);
  for (size_t lo = 0; lo < entries.size(); lo += kern::kAccMaxTensors) {
    kern::AccTable table;
    table.n = (int)std::min<size_t>(kern::kAccMaxTensors, entries.size() - lo);
    maxc = 0;
    for (int k = 0; k < table.n; ++k) {
      table.t[k] = entries[lo + k];
      maxc = std::max(maxc, table.t[k].count);
    }
    CheckLaunch("grad_accumulate", kern::LaunchGradAccumulate(table, maxc, (int)mode, (int)MapDtype(st), on.stream));
  }
}

}  // namespace

void DefOptim(py::module_& m) {
  m.def("fused_sgd_step", &FusedSgdStep, py::arg("params"), py::arg("grads"), py::arg("momenta"), py::arg("lr"),
        py::arg("momentum"), py::arg("dampening"), py::arg("weight_decay"), py::arg("nesterov"), py::arg("grad_scale"),
        py::arg("first_step"), py::arg("grad_scale_dev") = py::none(), py::arg("master_params") = std::vector<at::Tensor>(),
        py::arg("ema_params") = std::vector<at::Tensor>(), py::arg("ema_weight") = 0.0, py::arg("ema_start") = false);
  m.def("fused_adam_step", &FusedAdamStep, py::arg("params"), py::arg("grads"), py::arg("exp_avg"), py::arg("exp_avg_sq"),
        py::arg("lr"), py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("weight_decay"), py::arg("step"),
        py::arg("grad_scale"), py::arg("adamw"), py::arg("grad_scale_dev") = py::none(),
        py::arg("master_params") = std::vector<at::Tensor>(),
        py::arg("ema_params") = std::vector<at::Tensor>(), py::arg("ema_weight") = 0.0, py::arg("ema_start") = false);
  m.def("fused_lamb_step", &FusedLambStep, py::arg("params"), py::arg("grads"), py::arg("exp_avg"), py::arg("exp_avg_sq"),
        py::arg("lr"), py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("weight_decay"), py::arg("step"),
        py::arg("bias_correction"), py::arg("adapt"), py::arg("grad_scale"), py::arg("grad_scale_dev") = py::none(),
        py::arg("master_params") = std::vector<at::Tensor>(),
        py::arg("ema_params") = std::vector<at::Tensor>(), py::arg("ema_weight") = 0.0, py::arg("ema_start") = false);
  m.def("lamb_norms", &LambNorms, py::arg("params"), py::arg("grads"), py::arg("exp_avg"), py::arg("exp_avg_sq"),
        py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("weight_decay"), py::arg("step"),
        py::arg("bias_correction"), py::arg("grad_scale"), py::arg("grad_scale_dev"), py::arg("master_params"),
        py::arg("out"), py::arg("slots"));
  m.def("lamb_apply", &LambApply, py::arg("params"), py::arg("grads"), py::arg("exp_avg"), py::arg("exp_avg_sq"),
        py::arg("lr"), py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("weight_decay"), py::arg("step"),
        py::arg("bias_correction"), py::arg("adapt"), py::arg("master_params"), py::arg("norms"), py::arg("slots"),
        py::arg("ema_params") = std::vector<at::Tensor>(), py::arg("ema_weight") = 0.0, py::arg("ema_start") = false);
  m.def("fused_lars_step", &FusedLarsStep, py::arg("params"), py::arg("grads"), py::arg("momentum_buffers"), py::arg("lr"),
        py::arg("momentum"), py::arg("weight_decay"), py::arg("trust_coefficient"), py::arg("eps"), py::arg("adapt"),
        py::arg("grad_scale"), py::arg("grad_scale_dev") = py::none(), py::arg("master_params") = std::vector<at::Tensor>(),
        py::arg("ema_params") = std::vector<at::Tensor>(), py::arg("ema_weight") = 0.0, py::arg("ema_start") = false);
  m.def("lars_norms", &LarsNorms, py::arg("params"), py::arg("grads"), py::arg("momentum_buffers"), py::arg("grad_scale"),
        py::arg("grad_scale_dev"), py::arg("master_params"), py::arg("out"), py::arg("slots"));
  m.def("lars_apply", &LarsApply, py::arg("params"), py::arg("grads"), py::arg("momentum_buffers"), py::arg("lr"),
        py::arg("momentum"), py::arg("weight_decay"), py::arg("trust_coefficient"), py::arg("eps"), py::arg("adapt"),
        py::arg("grad_scale"), py::arg("grad_scale_dev"), py::arg("master_params"), py::arg("norms"), py::arg("slots"),
        py::arg("ema_params") = std::vector<at::Tensor>(), py::arg("ema_weight") = 0.0, py::arg("ema_start") = false);
  m.def("fused_adafactor_step", &FusedAdafactorStep, py::arg("params"), py::arg("grads"), py::arg("row_vars"),
        py::arg("col_vars"), py::arg("variances"), py::arg("lr"), py::arg("beta2_decay"), py::arg("eps1"), py::arg("eps2"),
        py::arg("d"), py::arg("weight_decay"), py::arg("step"), py::arg("grad_scale"), py::arg("grad_scale_dev"),
        py::arg("master_params"), py::arg("ema_params"), py::arg("ema_weight"), py::arg("ema_start"));
  m.def("grad_shard_stats", &GradShardStats, py::arg("grads"), py::arg("out"), py::arg("inv_scale") = py::none(),
        py::arg("norm_inf") = false);
  m.def("grad_accumulate", &GradAccumulate, py::arg("grads"), py::arg("accs"), py::arg("mode"));
}

}  // namespace hvd
