// CUDA-side bindings: GPU communicators and the sm_90a operator library.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <pybind11/stl.h>
#include <torch/extension.h>

#include <cmath>
#include <cstring>
#include <map>
#include <mutex>

#include "conv_wgmma.h"
#include "fused_convnet.h"
#include "cuda_comm.h"
#include "cuda_utils.h"
#include "ops_kernels.h"

namespace py = pybind11;

namespace pdt {

namespace {

using NoGil = py::call_guard<py::gil_scoped_release>;

cudaStream_t cur_stream(const at::Tensor& t) { return c10::cuda::getCurrentCUDAStream(t.device().index()).stream(); }

void chk(const at::Tensor& t, const char* name, at::ScalarType dt = at::kFloat) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
  TORCH_CHECK(t.scalar_type() == dt, name, " must have dtype ", c10::toString(dt), " (got ", c10::toString(t.scalar_type()), ")");
  TORCH_CHECK(t.is_contiguous(), name, " must be contiguous");
}

const float* opt_ptr(const c10::optional<at::Tensor>& t, const char* name) {
  if (!t.has_value() || !t->defined()) return nullptr;
  chk(*t, name);
  return t->data_ptr<float>();
}
float* opt_mut(c10::optional<at::Tensor>& t, const char* name) {
  if (!t.has_value() || !t->defined()) return nullptr;
  chk(*t, name);
  return t->data_ptr<float>();
}

// The hyper-parameters of sgd_multi and of the SGD rider of convnet_l1_bwd_wgrad.
SgdHyper sgd_hyper(double lr, const c10::optional<at::Tensor>& lr_tensor, double momentum, double dampening, double weight_decay, bool nesterov,
                   bool maximize, bool first_step) {
  return SgdHyper{static_cast<float>(lr), static_cast<float>(momentum), static_cast<float>(dampening), static_cast<float>(weight_decay),
                  nesterov ? 1 : 0, maximize ? 1 : 0, first_step ? 1 : 0, opt_ptr(lr_tensor, "lr_tensor")};
}
// The hyper-parameters of adam_multi and of the Adam rider of convnet_l1_bwd_wgrad.
AdamHyper adam_hyper(double lr, const c10::optional<at::Tensor>& lr_tensor, double beta1, double beta2, double eps, double weight_decay,
                     bool decoupled, bool maximize) {
  return AdamHyper{lr, beta1, beta2, static_cast<float>(eps), static_cast<float>(weight_decay), decoupled ? 1 : 0, maximize ? 1 : 0,
                   opt_ptr(lr_tensor, "lr_tensor")};
}
// The hyper-parameters of rmsprop_multi and of the RMSprop rider of convnet_l1_bwd_wgrad.
RmspropHyper rmsprop_hyper(double lr, const c10::optional<at::Tensor>& lr_tensor, double alpha, double eps, double weight_decay, double momentum,
                           bool maximize) {
  return RmspropHyper{static_cast<float>(lr), static_cast<float>(alpha), static_cast<float>(1.0 - alpha), static_cast<float>(eps),
                      static_cast<float>(weight_decay), static_cast<float>(momentum), maximize ? 1 : 0, opt_ptr(lr_tensor, "lr_tensor")};
}
// The hyper-parameters of adagrad_multi and of the Adagrad rider of convnet_l1_bwd_wgrad.
AdagradHyper adagrad_hyper(double lr, const c10::optional<at::Tensor>& lr_tensor, double lr_decay, double eps, double weight_decay, bool maximize) {
  return AdagradHyper{lr, lr_decay, static_cast<float>(eps), static_cast<float>(weight_decay), maximize ? 1 : 0, opt_ptr(lr_tensor, "lr_tensor")};
}

using TensorList = std::vector<c10::optional<at::Tensor>>;
TensorList tensors(const py::dict& d, const char* key) { return d[key].cast<TensorList>(); }

// The hyper-parameters of adadelta_multi and of the Adadelta rider of convnet_l1_bwd_wgrad.
AdadeltaHyper adadelta_hyper(double lr, const c10::optional<at::Tensor>& lr_tensor, double rho, double eps, double weight_decay, bool maximize) {
  return AdadeltaHyper{static_cast<float>(lr), static_cast<float>(rho), static_cast<float>(1.0 - rho), static_cast<float>(eps),
                       static_cast<float>(weight_decay), maximize ? 1 : 0, opt_ptr(lr_tensor, "lr_tensor")};
}
// The hyper-parameters of asgd_multi and of the ASGD rider of convnet_l1_bwd_wgrad.
AsgdHyper asgd_hyper(double lr, const c10::optional<at::Tensor>& lr_tensor, double lambd, double alpha, double t0, double weight_decay,
                     bool maximize) {
  return AsgdHyper{lr, lambd, alpha, t0, static_cast<float>(weight_decay), maximize ? 1 : 0, opt_ptr(lr_tensor, "lr_tensor")};
}
// The hyper-parameters of rprop_multi and of the Rprop rider of convnet_l1_bwd_wgrad.
RpropHyper rprop_hyper(double etaminus, double etaplus, double step_min, double step_max, bool maximize) {
  return RpropHyper{static_cast<float>(etaminus), static_cast<float>(etaplus), static_cast<float>(step_min), static_cast<float>(step_max),
                    maximize ? 1 : 0};
}

// The parameters of a rider description (dict: "params", the ten parameters in the order conv1.w, conv1.b, bn1.w, bn1.b, conv2.w,
// conv2.b, fc.w, fc.b, bn2.w, bn2.b, entries may be None; "prev_grads", the gradients of the last four) into r; state(k, param)
// fills the optimizer state of parameter k.
template <class R, class State>
void fill_rider(R& r, const py::dict& d, const char* kind, State state) {
  static const int64_t want[10] = {400, 16, 16, 16, 12800, 32, -1, -1, 32, 32};
  const TensorList params = tensors(d, "params"), prev = tensors(d, "prev_grads");
  TORCH_CHECK(params.size() == 10 && prev.size() == 4, "convnet_l1_bwd_wgrad: ", kind, " lists have the wrong length");
  for (int k = 0; k < 10; ++k) {
    if (!params[k].has_value() || !params[k]->defined()) continue;
    const at::Tensor& p = *params[k];
    chk(p, "rider param");
    TORCH_CHECK(want[k] < 0 || p.numel() == want[k], "convnet_l1_bwd_wgrad: ", kind, " parameter ", k, " has the wrong size");
    r.p[k] = p.data_ptr<float>();
    state(k, p);
    if (k >= 6) {
      TORCH_CHECK(prev[k - 6].has_value() && prev[k - 6]->numel() == p.numel(), "convnet_l1_bwd_wgrad: gradient of ", kind, " parameter ", k, " missing");
      chk(*prev[k - 6], "rider gradient");
      r.g_prev[k - 6] = prev[k - 6]->data_ptr<float>();
      r.n_prev[k - 6] = static_cast<int>(p.numel());
    }
  }
  TORCH_CHECK(r.p[0] && r.p[4], "convnet_l1_bwd_wgrad: the convolution weights must take part in the fused update");
  r.on = 1;
}

// {"kind": "sgd", "params", "prev_grads", "momentum_buffer" (ten, or empty when momentum == 0), "lr", "lr_tensor", "momentum",
// "dampening", "weight_decay", "nesterov", "maximize", "first_step"}
SgdRider sgd_rider(const py::dict& d) {
  SgdRider r;
  const double momentum = d["momentum"].cast<double>();
  const TensorList bufs = tensors(d, "momentum_buffer");
  TORCH_CHECK(bufs.empty() || bufs.size() == 10, "convnet_l1_bwd_wgrad: sgd lists have the wrong length");
  fill_rider(r, d, "sgd", [&](int k, const at::Tensor& p) {
    if (momentum == 0.0) return;
    TORCH_CHECK(!bufs.empty() && bufs[k].has_value() && bufs[k]->numel() == p.numel(), "convnet_l1_bwd_wgrad: momentum buffer ", k, " missing");
    chk(*bufs[k], "momentum buffer");
    r.m[k] = bufs[k]->data_ptr<float>();
  });
  r.h = sgd_hyper(d["lr"].cast<double>(), d["lr_tensor"].cast<c10::optional<at::Tensor>>(), momentum, d["dampening"].cast<double>(),
                  d["weight_decay"].cast<double>(), d["nesterov"].cast<bool>(), d["maximize"].cast<bool>(), d["first_step"].cast<bool>());
  return r;
}

// {"kind": "adam", "params", "prev_grads", "exp_avg", "exp_avg_sq", "step" (fp32 scalars on the device), "lr", "lr_tensor", "beta1",
// "beta2", "eps", "weight_decay", "decoupled", "maximize"}, and for AMSGrad "max_exp_avg_sq" (ten tensors; amsgrad_rider below).
// The "nadam" and "radam" descriptions have the same entries (nadam_rider, radam_rider below); kind names them in errors.
AdamRider adam_rider(const py::dict& d, const char* kind = "adam") {
  AdamRider r;
  const TensorList ms = tensors(d, "exp_avg"), vs = tensors(d, "exp_avg_sq"), steps = tensors(d, "step");
  TORCH_CHECK(ms.size() == 10 && vs.size() == 10 && steps.size() == 10, "convnet_l1_bwd_wgrad: ", kind, " lists have the wrong length");
  fill_rider(r, d, kind, [&](int k, const at::Tensor& p) {
    TORCH_CHECK(ms[k].has_value() && vs[k].has_value() && steps[k].has_value(), "convnet_l1_bwd_wgrad: ", kind, " state of parameter ", k,
                " missing");
    chk(*ms[k], "exp_avg"); chk(*vs[k], "exp_avg_sq"); chk(*steps[k], "step");
    TORCH_CHECK(ms[k]->numel() == p.numel() && vs[k]->numel() == p.numel() && steps[k]->numel() == 1, "convnet_l1_bwd_wgrad: ", kind,
                " state of parameter ", k, " has the wrong size");
    r.m[k] = ms[k]->data_ptr<float>();
    r.v[k] = vs[k]->data_ptr<float>();
    r.step[k] = steps[k]->data_ptr<float>();
  });
  r.h = adam_hyper(d["lr"].cast<double>(), d["lr_tensor"].cast<c10::optional<at::Tensor>>(), d["beta1"].cast<double>(), d["beta2"].cast<double>(),
                   d["eps"].cast<double>(), d["weight_decay"].cast<double>(), d["decoupled"].cast<bool>(), d["maximize"].cast<bool>());
  return r;
}
// the "adam" description with a "max_exp_avg_sq" entry
AmsgradRider amsgrad_rider(const py::dict& d) {
  AmsgradRider r;
  static_cast<AdamRider&>(r) = adam_rider(d);
  const TensorList vmax = tensors(d, "max_exp_avg_sq"), params = tensors(d, "params");
  TORCH_CHECK(vmax.size() == 10, "convnet_l1_bwd_wgrad: adam lists have the wrong length");
  for (int k = 0; k < 10; ++k) {
    if (!r.p[k]) continue;
    TORCH_CHECK(vmax[k].has_value() && vmax[k]->numel() == params[k]->numel(), "convnet_l1_bwd_wgrad: max_exp_avg_sq of parameter ", k,
                " missing or of the wrong size");
    chk(*vmax[k], "max_exp_avg_sq");
    r.vmax[k] = vmax[k]->data_ptr<float>();
  }
  return r;
}

// State tensor `name` of rider parameter k: present, `numel` elements, fp32 contiguous on the device.
float* rider_state(const TensorList& ts, int k, int64_t numel, const char* kind, const char* name) {
  TORCH_CHECK(ts[k].has_value() && ts[k]->defined(), "convnet_l1_bwd_wgrad: ", kind, " state ", name, " of parameter ", k, " missing");
  chk(*ts[k], name);
  TORCH_CHECK(ts[k]->numel() == numel, "convnet_l1_bwd_wgrad: ", kind, " state ", name, " of parameter ", k, " has the wrong size");
  return ts[k]->data_ptr<float>();
}

// {"kind": "nadam", the "adam" entries, "mu_product" (ten fp32 scalars on the device), "momentum_decay"}
NadamRider nadam_rider(const py::dict& d) {
  NadamRider r;
  static_cast<AdamRider&>(r) = adam_rider(d, "nadam");
  const TensorList mps = tensors(d, "mu_product");
  TORCH_CHECK(mps.size() == 10, "convnet_l1_bwd_wgrad: nadam lists have the wrong length");
  for (int k = 0; k < 10; ++k)
    if (r.p[k]) r.mu_product[k] = rider_state(mps, k, 1, "nadam", "mu_product");
  r.momentum_decay = d["momentum_decay"].cast<double>();
  return r;
}

// {"kind": "radam", the "adam" entries}
RadamRider radam_rider(const py::dict& d) {
  RadamRider r;
  static_cast<AdamRider&>(r) = adam_rider(d, "radam");
  return r;
}

// {"kind": "rmsprop", "params", "prev_grads", "square_avg", "step" (fp32 scalars on the device), "momentum_buffer" (ten, or empty when
// momentum == 0), "grad_avg" (ten, or empty when not centered), "lr", "lr_tensor", "alpha", "eps", "weight_decay", "momentum",
// "maximize"}
RmspropRider rmsprop_rider(const py::dict& d) {
  RmspropRider r;
  const double momentum = d["momentum"].cast<double>();
  const TensorList sqs = tensors(d, "square_avg"), steps = tensors(d, "step"), bufs = tensors(d, "momentum_buffer"), gas = tensors(d, "grad_avg");
  TORCH_CHECK(sqs.size() == 10 && steps.size() == 10 && (bufs.empty() || bufs.size() == 10) && (gas.empty() || gas.size() == 10),
              "convnet_l1_bwd_wgrad: rmsprop lists have the wrong length");
  TORCH_CHECK((momentum > 0.0) == !bufs.empty(), "convnet_l1_bwd_wgrad: rmsprop momentum buffers are given exactly when momentum > 0");
  fill_rider(r, d, "rmsprop", [&](int k, const at::Tensor& p) {
    r.sq[k] = rider_state(sqs, k, p.numel(), "rmsprop", "square_avg");
    r.step[k] = rider_state(steps, k, 1, "rmsprop", "step");
    if (!bufs.empty()) r.buf[k] = rider_state(bufs, k, p.numel(), "rmsprop", "momentum_buffer");
    if (!gas.empty()) r.ga[k] = rider_state(gas, k, p.numel(), "rmsprop", "grad_avg");
  });
  r.h = rmsprop_hyper(d["lr"].cast<double>(), d["lr_tensor"].cast<c10::optional<at::Tensor>>(), d["alpha"].cast<double>(), d["eps"].cast<double>(),
                      d["weight_decay"].cast<double>(), momentum, d["maximize"].cast<bool>());
  return r;
}

// {"kind": "adagrad", "params", "prev_grads", "sum", "step" (fp32 scalars on the device), "lr", "lr_tensor", "lr_decay", "eps",
// "weight_decay", "maximize"}
AdagradRider adagrad_rider(const py::dict& d) {
  AdagradRider r;
  const TensorList sums = tensors(d, "sum"), steps = tensors(d, "step");
  TORCH_CHECK(sums.size() == 10 && steps.size() == 10, "convnet_l1_bwd_wgrad: adagrad lists have the wrong length");
  fill_rider(r, d, "adagrad", [&](int k, const at::Tensor& p) {
    r.sum[k] = rider_state(sums, k, p.numel(), "adagrad", "sum");
    r.step[k] = rider_state(steps, k, 1, "adagrad", "step");
  });
  r.h = adagrad_hyper(d["lr"].cast<double>(), d["lr_tensor"].cast<c10::optional<at::Tensor>>(), d["lr_decay"].cast<double>(),
                      d["eps"].cast<double>(), d["weight_decay"].cast<double>(), d["maximize"].cast<bool>());
  return r;
}

// {"kind": "adamax", the "adam" entries with "exp_inf" in place of "exp_avg_sq" ("decoupled" unused)}
AdamaxRider adamax_rider(const py::dict& d) {
  AdamaxRider r;
  const TensorList ms = tensors(d, "exp_avg"), us = tensors(d, "exp_inf"), steps = tensors(d, "step");
  TORCH_CHECK(ms.size() == 10 && us.size() == 10 && steps.size() == 10, "convnet_l1_bwd_wgrad: adamax lists have the wrong length");
  fill_rider(r, d, "adamax", [&](int k, const at::Tensor& p) {
    r.m[k] = rider_state(ms, k, p.numel(), "adamax", "exp_avg");
    r.v[k] = rider_state(us, k, p.numel(), "adamax", "exp_inf");
    r.step[k] = rider_state(steps, k, 1, "adamax", "step");
  });
  r.h = adam_hyper(d["lr"].cast<double>(), d["lr_tensor"].cast<c10::optional<at::Tensor>>(), d["beta1"].cast<double>(), d["beta2"].cast<double>(),
                   d["eps"].cast<double>(), d["weight_decay"].cast<double>(), false, d["maximize"].cast<bool>());
  return r;
}

// {"kind": "adadelta", "params", "prev_grads", "square_avg", "acc_delta", "step" (fp32 scalars on the device), "lr", "lr_tensor", "rho",
// "eps", "weight_decay", "maximize"}
AdadeltaRider adadelta_rider(const py::dict& d) {
  AdadeltaRider r;
  const TensorList sqs = tensors(d, "square_avg"), accs = tensors(d, "acc_delta"), steps = tensors(d, "step");
  TORCH_CHECK(sqs.size() == 10 && accs.size() == 10 && steps.size() == 10, "convnet_l1_bwd_wgrad: adadelta lists have the wrong length");
  fill_rider(r, d, "adadelta", [&](int k, const at::Tensor& p) {
    r.sq[k] = rider_state(sqs, k, p.numel(), "adadelta", "square_avg");
    r.acc[k] = rider_state(accs, k, p.numel(), "adadelta", "acc_delta");
    r.step[k] = rider_state(steps, k, 1, "adadelta", "step");
  });
  r.h = adadelta_hyper(d["lr"].cast<double>(), d["lr_tensor"].cast<c10::optional<at::Tensor>>(), d["rho"].cast<double>(), d["eps"].cast<double>(),
                       d["weight_decay"].cast<double>(), d["maximize"].cast<bool>());
  return r;
}

// {"kind": "asgd", "params", "prev_grads", "ax", "step", "eta", "mu" (fp32 scalars on the device), "lr", "lr_tensor", "lambd", "alpha",
// "t0", "weight_decay", "maximize"}
AsgdRider asgd_rider(const py::dict& d) {
  AsgdRider r;
  const TensorList axs = tensors(d, "ax"), steps = tensors(d, "step"), etas = tensors(d, "eta"), mus = tensors(d, "mu");
  TORCH_CHECK(axs.size() == 10 && steps.size() == 10 && etas.size() == 10 && mus.size() == 10, "convnet_l1_bwd_wgrad: asgd lists have the wrong length");
  fill_rider(r, d, "asgd", [&](int k, const at::Tensor& p) {
    r.ax[k] = rider_state(axs, k, p.numel(), "asgd", "ax");
    r.step[k] = rider_state(steps, k, 1, "asgd", "step");
    r.eta[k] = rider_state(etas, k, 1, "asgd", "eta");
    r.mu[k] = rider_state(mus, k, 1, "asgd", "mu");
  });
  r.h = asgd_hyper(d["lr"].cast<double>(), d["lr_tensor"].cast<c10::optional<at::Tensor>>(), d["lambd"].cast<double>(), d["alpha"].cast<double>(),
                   d["t0"].cast<double>(), d["weight_decay"].cast<double>(), d["maximize"].cast<bool>());
  return r;
}

// {"kind": "rprop", "params", "prev_grads", "prev", "step_size", "step" (fp32 scalars on the device), "etaminus", "etaplus",
// "step_size_min", "step_size_max", "maximize"}
RpropRider rprop_rider(const py::dict& d) {
  RpropRider r;
  const TensorList prevs = tensors(d, "prev"), sizes = tensors(d, "step_size"), steps = tensors(d, "step");
  TORCH_CHECK(prevs.size() == 10 && sizes.size() == 10 && steps.size() == 10, "convnet_l1_bwd_wgrad: rprop lists have the wrong length");
  fill_rider(r, d, "rprop", [&](int k, const at::Tensor& p) {
    r.prev[k] = rider_state(prevs, k, p.numel(), "rprop", "prev");
    r.step_size[k] = rider_state(sizes, k, p.numel(), "rprop", "step_size");
    r.step[k] = rider_state(steps, k, 1, "rprop", "step");
  });
  r.h = rprop_hyper(d["etaminus"].cast<double>(), d["etaplus"].cast<double>(), d["step_size_min"].cast<double>(), d["step_size_max"].cast<double>(),
                    d["maximize"].cast<bool>());
  return r;
}

// torch's cross-entropy options for C classes of logits on `like`'s device
CeSpec ce_spec(const c10::optional<at::Tensor>& weight, int64_t ignore_index, double label_smoothing, const std::string& reduction, int64_t C,
               const at::Tensor& like, const char* who) {
  TORCH_CHECK(reduction == "mean" || reduction == "sum", who, ": reduction must be 'mean' or 'sum' (got '", reduction, "')");
  TORCH_CHECK(label_smoothing >= 0.0 && label_smoothing <= 1.0, who, ": label_smoothing must lie in [0, 1] (got ", label_smoothing, ")");
  CeSpec s;
  s.weight = opt_ptr(weight, "weight");
  if (s.weight != nullptr)
    TORCH_CHECK(weight->dim() == 1 && weight->size(0) == C && weight->device() == like.device(), who, ": weight must be [", C, "] on ", like.device());
  s.smoothing = static_cast<float>(label_smoothing);
  s.ignore_index = ignore_index;
  s.sum = reduction == "sum";
  return s;
}

// Whether `target` holds class probabilities (a floating-point tensor, which must then be fp32 and shaped like the [B, C] `logits`)
// rather than int64 class indices
bool soft_target(const at::Tensor& target, const at::Tensor& logits, int64_t ignore_index, const char* who) {
  if (!at::isFloatingType(target.scalar_type())) {
    chk(target, "target", at::kLong);
    return false;
  }
  chk(target, "target");
  TORCH_CHECK(logits.dim() == 2 && target.sizes() == logits.sizes(), who, ": a probability target must have the logits' shape ",
              logits.sizes(), " (got ", target.sizes(), ")");
  TORCH_CHECK(target.device() == logits.device(), who, ": target must be on ", logits.device());
  TORCH_CHECK(ignore_index == -100, who, ": ignore_index is not supported for floating point target");
  return true;
}

// Per-device scratch for deterministic cross-CTA reductions. Kernels that use it run on one
// stream at a time (the compute stream), which is what serialises access.
struct Scratch {
  at::Tensor partials, counter;
  // conv2's weight-gradient partials per image ([one per SM][512][32]), written by the layer-2 backward kernel and folded by the
  // layer-1 one: a buffer of their own, so that no per-op kernel launched between the two (on any stream) can overwrite them
  at::Tensor wgrad;
  int wgrad_batch = 0;   // batch whose partials wgrad holds and nobody has folded yet (0: none)
};
Scratch& scratch_entry(const at::Tensor& like) {
  static std::mutex mu;
  static auto& per_dev = *new std::map<int, Scratch>();  // leaked on purpose: CUDA tensors must not die at static teardown
  std::lock_guard<std::mutex> g(mu);
  const int dev = like.device().index();
  auto it = per_dev.find(dev);
  if (it == per_dev.end()) {
    Scratch s;
    s.partials = at::empty({kScratchFloats}, like.options().dtype(at::kFloat));
    s.counter = at::zeros({kCounterWords}, like.options().dtype(at::kInt));   // layout: ops_kernels.h
    s.wgrad = at::empty({static_cast<int64_t>(at::cuda::getDeviceProperties(dev)->multiProcessorCount) * 400 * 32}, like.options().dtype(at::kFloat));
    it = per_dev.emplace(dev, std::move(s)).first;
  }
  return it->second;
}
ReduceScratch scratch(const at::Tensor& like) {
  Scratch& s = scratch_entry(like);
  ReduceScratch r;
  r.partials = s.partials.data_ptr<float>();
  r.counter = reinterpret_cast<unsigned int*>(s.counter.data_ptr<int>());
  r.capacity_floats = static_cast<int>(s.partials.numel());
  r.fold_counters = kFoldCounterWords;
  return r;
}
// Where the layer-2 backward kernel of a batch of B leaves conv2's per-image weight-gradient partials for the layer-1 one.
float* conv2_wgrad_partials(const at::Tensor& like, int B, const char* what) {
  Scratch& s = scratch_entry(like);
  TORCH_CHECK(static_cast<int64_t>(B) * 400 * 32 <= s.wgrad.numel(), what, ": batch ", B, " exceeds one CTA per SM");
  return s.wgrad.data_ptr<float>();
}

// conv2's input frame p1 [B,18,18,16] of the layer-2 backward bindings, or nullptr when not given.
const float* conv2_input(const c10::optional<at::Tensor>& p1, int B, const char* what) {
  if (!p1.has_value() || !p1->defined()) return nullptr;
  chk(*p1, "p1");
  TORCH_CHECK(p1->numel() == static_cast<int64_t>(B) * 324 * 16, what, ": p1 must be the [B,18,18,16] frame of layer 1");
  return p1->data_ptr<float>();
}

// Test-only: rank `rank` of a world emulated on one GPU, for launching the collective kernels one at a time.  The W heaps are
// plain uint8 device tensors laid out like the symmetric heap (the flag pads of every channel first, kSymmFlagPadBytes, then
// data), and the SymmDev's peer[r] points at heap r; there is no multicast mapping.  Whoever drives it stages what the other
// ranks would have written (their data, and their barrier flags far enough ahead that no kernel waits) before each launch.
// Pointer arguments are device addresses (0 = nullptr), so that tests can pass misaligned ones; every launch goes to the current
// stream of the heaps' device.
constexpr size_t kSymmFlagPadBytes = sizeof(uint32_t) * kSymmChannels * kSymmMaxBlocks * kSymmMaxWorld;

class SymmEmu {
 public:
  SymmEmu(std::vector<at::Tensor> heaps, int rank, int channel, int64_t timeout_ns, at::Tensor epochs, at::Tensor status)
      : heaps_(std::move(heaps)), epochs_(std::move(epochs)), status_(std::move(status)) {
    const int world = static_cast<int>(heaps_.size());
    TORCH_CHECK(world >= 1 && world <= kSymmMaxWorld, "SymmEmu: 1 to ", kSymmMaxWorld, " heaps required");
    TORCH_CHECK(rank >= 0 && rank < world && channel >= 0 && channel < kSymmChannels && timeout_ns > 0, "SymmEmu: bad rank, channel or timeout");
    std::memset(&d_, 0, sizeof(d_));
    for (int r = 0; r < world; ++r) {
      chk(heaps_[r], "heap", at::kByte);
      TORCH_CHECK(heaps_[r].device() == heaps_[0].device() && heaps_[r].numel() >= static_cast<int64_t>(kSymmFlagPadBytes) &&
                      reinterpret_cast<uintptr_t>(heaps_[r].data_ptr()) % 16 == 0,
                  "SymmEmu: heaps must be 16-byte aligned, on one device, and hold at least the flag pads");
      d_.peer[r] = static_cast<char*>(heaps_[r].data_ptr());
    }
    chk(epochs_, "epochs", at::kInt);
    chk(status_, "status", at::kInt);
    TORCH_CHECK(epochs_.numel() == kSymmMaxBlocks && status_.numel() >= 1 && epochs_.device() == heaps_[0].device() &&
                    status_.device() == heaps_[0].device(),
                "SymmEmu: epochs [", kSymmMaxBlocks, "] and status [1] on the heaps' device required");
    d_.mc = nullptr;
    d_.flags = nullptr;
    d_.flags_off = static_cast<size_t>(channel) * kSymmMaxBlocks * kSymmMaxWorld * sizeof(uint32_t);
    d_.epochs = reinterpret_cast<uint32_t*>(epochs_.data_ptr<int>());
    d_.status = status_.data_ptr<int>();
    d_.timeout_ns = static_cast<unsigned long long>(timeout_ns);
    d_.rank = rank;
    d_.world = world;
    d_.channel = channel;
  }
  const SymmDev& dev() const { return d_; }
  cudaStream_t stream() const { return c10::cuda::getCurrentCUDAStream(heaps_[0].device().index()).stream(); }

 private:
  std::vector<at::Tensor> heaps_;
  at::Tensor epochs_, status_;
  SymmDev d_;
};

template <typename P = void> P* dptr(int64_t a) { return reinterpret_cast<P*>(static_cast<uintptr_t>(a)); }
SymmLaunchCfg launch_cfg(int blocks, int threads) {
  SymmLaunchCfg c;
  c.blocks = blocks;
  c.threads = threads;
  return c;
}

// The grid barrier of the cooperative kernels lives in the fixed words behind the fold region.
GridSync grid_sync(const ReduceScratch& r) { return GridSync{r.counter + kGridEpochWord, r.counter + kGridArrivalWord}; }

ConvShape conv_shape(const at::Tensor& x_nhwc, const at::Tensor& w) {
  TORCH_CHECK(x_nhwc.dim() == 4 && w.dim() == 4 && w.size(2) == 5 && w.size(3) == 5, "conv5x5: x [B,H,W,Cin] and w [Cout,Cin,5,5] expected");
  ConvShape s;
  s.B = static_cast<int>(x_nhwc.size(0));
  s.H = static_cast<int>(x_nhwc.size(1));
  s.W = static_cast<int>(x_nhwc.size(2));
  s.Cin = static_cast<int>(w.size(1));
  s.Cout = static_cast<int>(w.size(0));
  return s;
}

}  // namespace

void register_cuda_bindings(py::module_& m) {
  m.attr("ops_ready") = true;
  m.def("_mark_exiting", [] { mark_process_exiting(); });
  m.def("kernel_launch_count", [] { return kernel_launch_count(); },
        "number of kernels this library has launched (or recorded into CUDA graphs) so far");
  m.def("nccl_available", [] { return NcclComm::available(); });
  m.def("nccl_version", [] { return NcclComm::version(); });

  py::class_<SymmComm, Comm, std::shared_ptr<SymmComm>>(m, "SymmComm")
      .def(py::init([](std::shared_ptr<Store> store, int rank, int size, int device, double timeout_s, int64_t heap_bytes) {
             py::gil_scoped_release r;
             return std::make_shared<SymmComm>(std::move(store), rank, size, device, Millis(static_cast<int64_t>(timeout_s * 1000)),
                                               static_cast<size_t>(heap_bytes));
           }),
           py::arg("store"), py::arg("rank"), py::arg("size"), py::arg("device"), py::arg("timeout") = 600.0,
           py::arg("heap_bytes") = int64_t(1) << 30)
      .def("allreduce_inline", &SymmComm::allreduce_inline, py::arg("tensor"), py::arg("op") = ReduceOp::SUM, py::arg("postscale") = 1.0)
      .def("broadcast_inline", &SymmComm::broadcast_inline, py::arg("tensor"), py::arg("root") = 0)
      .def("allreduce_sgd_inline", &SymmComm::allreduce_sgd_inline, py::arg("grad"), py::arg("param"), py::arg("momentum_buf") = py::none(),
           py::arg("lr") = 0.0, py::arg("lr_tensor") = py::none(), py::arg("momentum") = 0.0, py::arg("dampening") = 0.0,
           py::arg("weight_decay") = 0.0, py::arg("nesterov") = false, py::arg("first_step") = false)
      .def_property_readonly("has_multicast", &SymmComm::has_multicast)
      .def_property_readonly("fused_step_max_bytes",
                             [](SymmComm& c) { return static_cast<int64_t>(c.heap().staging_half_bytes(kChanInline) / std::max(1, c.size())); })
      .def_property("algo", &SymmComm::algo, &SymmComm::set_algo)
      .def("set_oneshot_max_bytes", &SymmComm::set_oneshot_max_bytes)
      .def("set_launch", &SymmComm::set_launch, py::arg("blocks") = 0, py::arg("threads") = 0)
      .def("describe", &SymmComm::describe)
      .def("status", &SymmComm::status)
      .def("status_string", &SymmComm::status_string)
      .def("parity_state", [](SymmComm& c) {
        // which half of each channel's double-buffered staging the NEXT collective will use; a CUDA graph bakes
        // these in, so a captured step with an odd number of staged collectives must alternate between two captures
        std::vector<int> v;
        for (int ch = 0; ch < kSymmChannels; ++ch) v.push_back(c.heap().peek_parity(ch));
        return v;
      })
      .def("heap_bytes_in_use", [](SymmComm& c) { return c.heap().user_bytes_in_use(); })
      .def("is_symmetric", [](SymmComm& c, const at::Tensor& t) { return c.heap().contains(t.data_ptr(), t.nbytes()); });

  // Test-only (see SymmEmu): thin wrappers over every launcher of symm_kernels.h except the multicast forms.
  m.attr("_symm_max_world") = kSymmMaxWorld;
  m.attr("_symm_max_blocks") = kSymmMaxBlocks;
  m.attr("_symm_channels") = kSymmChannels;
  m.attr("_symm_p2p_blocks") = kSymmP2PBlocks;
  m.attr("_symm_flag_pad_bytes") = kSymmFlagPadBytes;
  py::class_<SymmEmu>(m, "_SymmEmu")
      .def(py::init<std::vector<at::Tensor>, int, int, int64_t, at::Tensor, at::Tensor>(), py::arg("heaps"), py::arg("rank"),
           py::arg("channel"), py::arg("timeout_ns"), py::arg("epochs"), py::arg("status"))
      .def("oneshot", [](SymmEmu& e, int64_t in, int64_t out, int64_t stage_off, int64_t count, int dtype, int op, double scale, int blocks,
                         int threads) {
        launch_allreduce_oneshot_push(e.dev(), dptr(in), dptr(out), stage_off, count, dtype, op, scale, false, launch_cfg(blocks, threads), e.stream());
      }, py::arg("inp"), py::arg("out"), py::arg("stage_off"), py::arg("count"), py::arg("dtype"), py::arg("op"), py::arg("scale") = 1.0,
         py::arg("blocks") = 0, py::arg("threads") = 0)
      .def("twoshot", [](SymmEmu& e, int64_t buf_off, int64_t count, int dtype, int op, double scale, int blocks, int threads) {
        launch_allreduce_twoshot(e.dev(), buf_off, count, dtype, op, scale, false, launch_cfg(blocks, threads), e.stream());
      }, py::arg("buf_off"), py::arg("count"), py::arg("dtype"), py::arg("op"), py::arg("scale") = 1.0, py::arg("blocks") = 0, py::arg("threads") = 0)
      .def("reduce_pull", [](SymmEmu& e, int64_t stage_off, int64_t begin_vec, int64_t count_vec, int64_t total_vec, int64_t out, int dtype, int op,
                             double scale, int blocks, int threads) {
        launch_reduce_pull(e.dev(), stage_off, begin_vec, count_vec, total_vec, dptr(out), dtype, op, scale, launch_cfg(blocks, threads), e.stream());
      }, py::arg("stage_off"), py::arg("begin_vec"), py::arg("count_vec"), py::arg("total_vec"), py::arg("out"), py::arg("dtype"), py::arg("op"),
         py::arg("scale") = 1.0, py::arg("blocks") = 0, py::arg("threads") = 0)
      .def("broadcast", [](SymmEmu& e, int64_t src_off, int64_t dst, int64_t nbytes, int root, bool exit_barrier, int blocks, int threads) {
        launch_broadcast_pull(e.dev(), src_off, dptr(dst), nbytes, root, exit_barrier, launch_cfg(blocks, threads), e.stream());
      }, py::arg("src_off"), py::arg("dst"), py::arg("nbytes"), py::arg("root"), py::arg("exit_barrier"), py::arg("blocks") = 0, py::arg("threads") = 0)
      .def("allgather", [](SymmEmu& e, int64_t src_off, int64_t dst, int64_t nbytes, int64_t dst_stride, bool exit_barrier, int blocks, int threads) {
        launch_allgather_pull(e.dev(), src_off, dptr(dst), nbytes, dst_stride, exit_barrier, launch_cfg(blocks, threads), e.stream());
      }, py::arg("src_off"), py::arg("dst"), py::arg("nbytes"), py::arg("dst_stride"), py::arg("exit_barrier"), py::arg("blocks") = 0,
         py::arg("threads") = 0)
      .def("alltoall", [](SymmEmu& e, int64_t src_off, int64_t dst, int64_t nbytes, int64_t stride, bool exit_barrier, int blocks, int threads) {
        launch_alltoall_pull(e.dev(), src_off, dptr(dst), nbytes, stride, exit_barrier, launch_cfg(blocks, threads), e.stream());
      }, py::arg("src_off"), py::arg("dst"), py::arg("nbytes"), py::arg("stride"), py::arg("exit_barrier"), py::arg("blocks") = 0, py::arg("threads") = 0)
      .def("allreduce_sgd", [](SymmEmu& e, int64_t grad, int64_t param, int64_t mom, int64_t stage_off, int64_t count, double scale, int64_t lr_dev,
                               double lr, double momentum, double dampening, double weight_decay, bool nesterov, bool first_step, int64_t bcast,
                               int64_t bcast_bytes, int bcast_root, int blocks, int threads) {
        launch_allreduce_sgd_oneshot(e.dev(), dptr<float>(grad), dptr<float>(param), dptr<float>(mom), stage_off, count, static_cast<float>(scale),
                                     dptr<const float>(lr_dev), static_cast<float>(lr), static_cast<float>(momentum), static_cast<float>(dampening),
                                     static_cast<float>(weight_decay), nesterov, first_step, false, launch_cfg(blocks, threads), e.stream(),
                                     dptr(bcast), bcast_bytes, bcast_root);
      }, py::arg("grad"), py::arg("param"), py::arg("mom"), py::arg("stage_off"), py::arg("count"), py::arg("scale"), py::arg("lr_dev"), py::arg("lr"),
         py::arg("momentum"), py::arg("dampening"), py::arg("weight_decay"), py::arg("nesterov"), py::arg("first_step"), py::arg("bcast") = 0,
         py::arg("bcast_bytes") = 0, py::arg("bcast_root") = 0, py::arg("blocks") = 0, py::arg("threads") = 0)
      .def("p2p_send", [](SymmEmu& e, int64_t src, int64_t nbytes, int dst_rank, int64_t slot_off, uint32_t seq) {
        launch_p2p_send(e.dev(), dptr(src), nbytes, dst_rank, slot_off, seq, e.stream());
      }, py::arg("src"), py::arg("nbytes"), py::arg("dst_rank"), py::arg("slot_off"), py::arg("seq"))
      .def("p2p_recv", [](SymmEmu& e, int64_t dst, int64_t nbytes, int src_rank, int64_t slot_off, uint32_t seq) {
        launch_p2p_recv(e.dev(), dptr(dst), nbytes, src_rank, slot_off, seq, e.stream());
      }, py::arg("dst"), py::arg("nbytes"), py::arg("src_rank"), py::arg("slot_off"), py::arg("seq"))
      .def("barrier", [](SymmEmu& e) { launch_barrier(e.dev(), e.stream()); });

  py::class_<NcclComm, Comm, std::shared_ptr<NcclComm>>(m, "NcclComm")
      .def(py::init([](std::shared_ptr<Store> store, int rank, int size, int device, double timeout_s) {
             py::gil_scoped_release r;
             return std::make_shared<NcclComm>(std::move(store), rank, size, device, Millis(static_cast<int64_t>(timeout_s * 1000)));
           }),
           py::arg("store"), py::arg("rank"), py::arg("size"), py::arg("device"), py::arg("timeout") = 600.0);

  // ---- convolution ---------------------------------------------------------------------------------
  // The shape picks the kernels: conv2 (16→32) runs on the tensor cores (TMA-im2col wgmma forward and data gradient, mma.sync
  // weight gradient), every other shape on the SIMT kernels, which cover conv1 (1→16: forward, weight gradient, and the data
  // gradient an input that requires grad takes) and refuse the rest.
  // centred: stats = [mean, M2, n] (ops_kernels.h), without the cancellation of Σy² when |mean| ≫ std; fp64_sums: the fp64
  // [Σy, Σy², n, 0] formed from the same centred fold, which SyncBatchNorm all-reduces; the default is the fp32 [Σ, Σ², n]
  m.def("conv5x5_fwd", [](const at::Tensor& x, const at::Tensor& w, c10::optional<at::Tensor> bias, bool want_stats, bool zero_pad,
                          bool centred, bool fp64_sums) {
    chk(x, "x"); chk(w, "w");
    c10::cuda::CUDAGuard g(x.device());
    ConvShape s = conv_shape(x, w);
    TORCH_CHECK(x.size(3) == s.Cin, "conv5x5_fwd: x channels ", x.size(3), " != weight Cin ", s.Cin);
    TORCH_CHECK(!(centred && fp64_sums), "conv5x5_fwd: stats are either centred or fp64_sums");
    TORCH_CHECK(want_stats || !fp64_sums, "conv5x5_fwd: fp64_sums needs want_stats");
    at::Tensor y = at::empty({s.B, s.H, s.W, s.Cout}, x.options());
    at::Tensor stats;
    if (fp64_sums) {
      // [2C+2] doubles, every entry written by the kernel: already a 16-byte multiple for the allreduce
      stats = at::empty({2 * s.Cout + 2}, x.options().dtype(at::kDouble));
    } else if (want_stats) {
      // [2C+1] statistics live in a [2C+4] vector (a 16-byte multiple), the three pad entries zeroed on request
      at::Tensor stats_full = zero_pad ? at::zeros({2 * s.Cout + 4}, x.options()) : at::empty({2 * s.Cout + 4}, x.options());
      stats = stats_full.narrow(0, 0, 2 * s.Cout + 1);
    }
    const ConvStats form = fp64_sums ? kConvSums64 : centred ? kConvCentred : kConvSums;
    auto launch = conv_wgmma_supported(s) ? launch_conv5x5_fwd_im2col : launch_conv5x5_fwd;
    launch(x.data_ptr<float>(), w.data_ptr<float>(), opt_ptr(bias, "bias"), y.data_ptr<float>(), want_stats ? stats.data_ptr() : nullptr,
           form, s, scratch(x), cur_stream(x));
    return py::make_tuple(y, stats);  // fp32 stats: a view of the first 2C+1 entries of the padded vector
  }, py::arg("x"), py::arg("w"), py::arg("bias") = py::none(), py::arg("want_stats") = true, py::arg("zero_pad") = false,
     py::arg("centred") = false, py::arg("fp64_sums") = false);

  m.def("conv5x5_dgrad", [](const at::Tensor& dy, const at::Tensor& w) {
    chk(dy, "dy"); chk(w, "w");
    c10::cuda::CUDAGuard g(dy.device());
    ConvShape s = conv_shape(dy, w);
    s.Cin = static_cast<int>(w.size(1));
    TORCH_CHECK(dy.size(3) == s.Cout, "conv5x5_dgrad: dy channels must equal weight Cout");
    at::Tensor dx = at::empty({s.B, s.H, s.W, s.Cin}, dy.options());
    auto launch = conv_wgmma_supported(s) ? launch_conv5x5_dgrad_im2col : launch_conv5x5_dgrad;
    launch(dy.data_ptr<float>(), w.data_ptr<float>(), dx.data_ptr<float>(), s, cur_stream(dy));
    return dx;
  }, py::arg("dy"), py::arg("w"));

  m.def("conv5x5_wgrad", [](const at::Tensor& dy, const at::Tensor& x, at::Tensor dw, c10::optional<at::Tensor> db) {
    chk(dy, "dy"); chk(x, "x"); chk(dw, "dw");
    c10::cuda::CUDAGuard g(dy.device());
    ConvShape s = conv_shape(x, dw);
    auto launch = conv_wgmma_supported(s) ? launch_conv5x5_wgrad_mma : launch_conv5x5_wgrad;
    launch(dy.data_ptr<float>(), x.data_ptr<float>(), dw.data_ptr<float>(), opt_mut(db, "db"), s, scratch(x), cur_stream(x));
  }, py::arg("dy"), py::arg("x"), py::arg("dw"), py::arg("db") = py::none());

  // ---- cooperative fused ConvNet layers (fused_convnet.cu): one CTA per image, grid barrier for the batch statistics ----
  m.def("fused_convnet_supported", [](int64_t B) { return fused_convnet_supported(static_cast<int>(B)); });
  // A captured launch with programmatic stream serialization becomes a programmatic edge only when the node before it in the
  // captured stream is a kernel; behind anything else the capture records a full dependency.
  m.def("graph_programmatic_edges", [](uintptr_t graph) {
    auto g = reinterpret_cast<cudaGraph_t>(graph);
    size_t n = 0;
    PDT_CUDA_CHECK(cudaGraphGetEdges_v2(g, nullptr, nullptr, nullptr, &n));
    std::vector<cudaGraphNode_t> from(n), to(n);
    std::vector<cudaGraphEdgeData> data(n);
    PDT_CUDA_CHECK(cudaGraphGetEdges_v2(g, from.data(), to.data(), data.data(), &n));
    int64_t programmatic = 0;
    for (size_t i = 0; i < n; ++i) programmatic += data[i].type == cudaGraphDependencyTypeProgrammatic ? 1 : 0;
    return programmatic;
  }, py::arg("graph"), "number of programmatic-dependency edges of a cudaGraph_t (torch.cuda.CUDAGraph(keep_graph=True).raw_cuda_graph())");
  m.def("fused_convnet_trace_enable", [](bool on) { fused_convnet_trace_enable(on); });
  m.def("fused_convnet_trace_read", [] {
    at::Tensor t = at::zeros({4, 160, 12}, at::kLong);
    fused_convnet_trace_read(reinterpret_cast<unsigned long long*>(t.data_ptr<int64_t>()));
    return t;
  });
  m.def("convnet_l1_bwd_wgrad", [](const at::Tensor& dp, c10::optional<at::Tensor> y, const at::Tensor& x, const at::Tensor& saved,
                                   c10::optional<at::Tensor> gamma, c10::optional<at::Tensor> beta, at::Tensor dgamma, at::Tensor dbeta, at::Tensor dw,
                                   c10::optional<at::Tensor> db, c10::optional<at::Tensor> dy2_pad, c10::optional<at::Tensor> x2_pad,
                                   const at::Tensor& dysum2, at::Tensor dw2, c10::optional<at::Tensor> db2, py::object rider, py::object clip,
                                   bool accumulate, c10::optional<at::Tensor> w1, c10::optional<at::Tensor> b1) {
    chk(dp, "dp"); chk(x, "x"); chk(saved, "saved"); chk(dgamma, "dgamma"); chk(dbeta, "dbeta"); chk(dw, "dw");
    chk(dysum2, "dysum2"); chk(dw2, "dw2");
    c10::cuda::CUDAGuard g(x.device());
    TORCH_CHECK(x.numel() % 784 == 0, "convnet_l1_bwd_wgrad: x [B,1,28,28] expected");
    const int B = static_cast<int>(x.numel() / 784);
    TORCH_CHECK(dp.numel() == static_cast<int64_t>(B) * 5184 && dw.numel() == 400 && dgamma.numel() == 16 && dbeta.numel() == 16,
                "convnet_l1_bwd_wgrad: layer-1 shape mismatch");
    // y: conv1's output as convnet_fwd(…, keep_y1=True) returns it, or None: the kernel recomputes it from x and w1 / b1 (bit for bit)
    const float* y_ptr = opt_ptr(y, "y");
    const float* w1_ptr = opt_ptr(w1, "w1");
    const float* b1_ptr = opt_ptr(b1, "b1");
    TORCH_CHECK(y_ptr != nullptr || w1_ptr != nullptr, "convnet_l1_bwd_wgrad: without y, conv1's weights w1 are needed to recompute it");
    TORCH_CHECK(y_ptr == nullptr || y->numel() == static_cast<int64_t>(B) * 12544, "convnet_l1_bwd_wgrad: y [B,28,28,16] expected");
    TORCH_CHECK(w1_ptr == nullptr || w1->numel() == 400, "convnet_l1_bwd_wgrad: w1 [16,1,5,5] expected");
    TORCH_CHECK(b1_ptr == nullptr || b1->numel() == 16, "convnet_l1_bwd_wgrad: b1 [16] expected");
    TORCH_CHECK(dysum2.numel() == static_cast<int64_t>(B) * 32 && dw2.numel() == 12800, "convnet_l1_bwd_wgrad: layer-2 shape mismatch");
    // conv2's per-image weight-gradient partials: from the given frames (the tests' reference), or (both None) left by
    // convnet_l2_bwd_fc(…, p1) of this batch
    const bool frames = dy2_pad.has_value() && dy2_pad->defined();
    TORCH_CHECK(frames == (x2_pad.has_value() && x2_pad->defined()), "convnet_l1_bwd_wgrad: dy2_pad and x2_pad are given together or not at all");
    float* wpart = conv2_wgrad_partials(x, B, "convnet_l1_bwd_wgrad");
    Scratch& entry = scratch_entry(x);
    if (frames) {
      chk(*dy2_pad, "dy2_pad"); chk(*x2_pad, "x2_pad");
      TORCH_CHECK(dy2_pad->numel() == static_cast<int64_t>(B) * 324 * 32 && x2_pad->numel() == static_cast<int64_t>(B) * 324 * 16,
                  "convnet_l1_bwd_wgrad: layer-2 frame shape mismatch");
    } else {
      TORCH_CHECK(entry.wgrad_batch == B, "convnet_l1_bwd_wgrad: without dy2_pad / x2_pad it folds the partials of convnet_l2_bwd_fc(…, p1) "
                  "of the same batch, and none are pending");
    }
    // rider: the optimizer update riding on the kernel, a description with named entries (sgd_rider / adam_rider above), or None.
    // clip = (max_norm, norm_type 2 or inf, norm_out): gradient-norm clipping in front of the update (ClipRider); norm_out receives the
    // norm.  accumulate: gradient accumulation — dgamma, dbeta, dw, db, dw2, db2 are added to (they hold the earlier micro-batches' sum),
    // and the rider updates with the accumulated gradients.
    ReduceScratch scr = scratch(x);
    const size_t l1_floats = static_cast<size_t>(B) * (64 + 512);
    TORCH_CHECK(static_cast<long long>(l1_floats) + B <= scr.capacity_floats, "convnet_l1_bwd_wgrad: scratch too small");
    auto launch = [&](auto rider) {
      if (frames) launch_conv2_wgrad_partials(dy2_pad->data_ptr<float>(), x2_pad->data_ptr<float>(), B, wpart, cur_stream(x));
      launch_convnet_l1_bwd_wgrad(dp.data_ptr<float>(), y_ptr, w1_ptr, b1_ptr, x.data_ptr<float>(), saved.data_ptr<float>(), opt_ptr(gamma, "gamma"),
                                  opt_ptr(beta, "beta"), dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), dw.data_ptr<float>(), opt_mut(db, "db"),
                                  wpart, dysum2.data_ptr<float>(), dw2.data_ptr<float>(), opt_mut(db2, "db2"), B, scr.partials,
                                  scr.partials + static_cast<size_t>(B) * 64, grid_sync(scr), cur_stream(x), rider, accumulate);
      entry.wgrad_batch = 0;
    };
    // the rider with clipping → its clipping variant
    auto launch_rider = [&](auto base) {
      if (clip.is_none()) return launch(base);
      auto c = clip.cast<py::tuple>();
      TORCH_CHECK(c.size() == 3, "convnet_l1_bwd_wgrad: clip entry (max_norm, norm_type, norm_out) expected");
      const double norm_type = c[1].cast<double>();
      TORCH_CHECK(norm_type == 2.0 || (std::isinf(norm_type) && norm_type > 0), "convnet_l1_bwd_wgrad: clip norm_type must be 2 or inf");
      at::Tensor out = c[2].cast<at::Tensor>();
      chk(out, "norm_out");
      TORCH_CHECK(out.numel() == 1, "convnet_l1_bwd_wgrad: norm_out must have one element");
      ClipRider<decltype(base)> r;
      static_cast<decltype(base)&>(r) = base;
      r.max_norm = static_cast<float>(c[0].cast<double>());
      r.norm_inf = std::isinf(norm_type) ? 1 : 0;
      r.norm_out = out.data_ptr<float>();
      r.part = scr.partials + l1_floats;
      launch(r);
    };
    if (rider.is_none()) {
      TORCH_CHECK(clip.is_none(), "convnet_l1_bwd_wgrad: clip needs a rider");
      return launch(SgdRider{});
    }
    const auto d = rider.cast<py::dict>();
    const auto kind = d["kind"].cast<std::string>();
    TORCH_CHECK(kind == "sgd" || kind == "adam" || kind == "nadam" || kind == "radam" || kind == "rmsprop" || kind == "adagrad" ||
                    kind == "adamax" || kind == "adadelta" || kind == "asgd" || kind == "rprop",
                "convnet_l1_bwd_wgrad: rider kind must be 'sgd', 'adam', 'nadam', 'radam', 'rmsprop', 'adagrad', 'adamax', 'adadelta', 'asgd' "
                "or 'rprop' (got '", kind, "')");
    if (kind == "sgd") launch_rider(sgd_rider(d));
    else if (kind == "adamax") launch_rider(adamax_rider(d));
    else if (kind == "adadelta") launch_rider(adadelta_rider(d));
    else if (kind == "asgd") launch_rider(asgd_rider(d));
    else if (kind == "rprop") launch_rider(rprop_rider(d));
    else if (kind == "nadam") launch_rider(nadam_rider(d));
    else if (kind == "radam") launch_rider(radam_rider(d));
    else if (kind == "rmsprop") launch_rider(rmsprop_rider(d));
    else if (kind == "adagrad") launch_rider(adagrad_rider(d));
    else if (d.contains("max_exp_avg_sq")) launch_rider(amsgrad_rider(d));
    else launch_rider(adam_rider(d));
  }, py::arg("dp"), py::arg("y"), py::arg("x"), py::arg("saved"), py::arg("gamma"), py::arg("beta"), py::arg("dgamma"), py::arg("dbeta"),
     py::arg("dw"), py::arg("db"), py::arg("dy2_pad"), py::arg("x2_pad"), py::arg("dysum2"), py::arg("dw2"), py::arg("db2"),
     py::arg("rider") = py::none(), py::kw_only(), py::arg("clip") = py::none(), py::arg("accumulate") = false, py::arg("w1") = py::none(),
     py::arg("b1") = py::none());
  m.def("convnet_fwd", [](const at::Tensor& x, const at::Tensor& w1, c10::optional<at::Tensor> b1, c10::optional<at::Tensor> g1,
                          c10::optional<at::Tensor> be1, c10::optional<at::Tensor> rm1, c10::optional<at::Tensor> rv1, c10::optional<at::Tensor> nbt1,
                          double mom1, double eps1, const at::Tensor& w2, c10::optional<at::Tensor> b2, c10::optional<at::Tensor> g2,
                          c10::optional<at::Tensor> be2, c10::optional<at::Tensor> rm2, c10::optional<at::Tensor> rv2, c10::optional<at::Tensor> nbt2,
                          double mom2, double eps2, const at::Tensor& fcw, c10::optional<at::Tensor> fcb, c10::optional<at::Tensor> target,
                          bool defer_loss_mean, double grad_scale, c10::optional<at::Tensor> ce_weight, int64_t ignore_index,
                          double label_smoothing, const std::string& reduction, bool keep_y1) {
    chk(x, "x"); chk(w1, "w1"); chk(w2, "w2"); chk(fcw, "fc weight");
    c10::cuda::CUDAGuard g(x.device());
    TORCH_CHECK(x.numel() % 784 == 0 && w1.numel() == 400 && w2.numel() == 12800 && fcw.dim() == 2 && fcw.size(1) == 1568 && fcw.size(0) <= 16,
                "convnet_fwd: x [B,1,28,28], w1 [16,1,5,5], w2 [32,16,5,5], fc weight [<=16, 1568] expected");
    const int B = static_cast<int>(x.numel() / 784), ncls = static_cast<int>(fcw.size(0));
    TORCH_CHECK(fused_convnet_supported(B), "convnet_fwd: batch ", B, " exceeds one CTA per SM");
    // keep_y1=False: conv1's output is not stored (None in its place); convnet_l1_bwd_wgrad(y=None, w1=…, b1=…) recomputes it
    at::Tensor y1 = keep_y1 ? at::empty({B, 28, 28, 16}, x.options()) : at::Tensor();
    at::Tensor p1 = at::empty({B, 18, 18, 16}, x.options()), saved1 = at::empty({32}, x.options());
    at::Tensor y2 = at::empty({B, 14, 14, 32}, x.options()), out = at::empty({B, 32, 7, 7}, x.options()), saved2 = at::empty({64}, x.options());
    at::Tensor logits = at::empty({B, ncls}, x.options());
    auto nbt_ptr = [](c10::optional<at::Tensor>& t) -> long long* {
      if (!t.has_value() || !t->defined()) return nullptr;
      chk(*t, "num_batches_tracked", at::kLong);
      return reinterpret_cast<long long*>(t->data_ptr<int64_t>());
    };
    ReduceScratch scr = scratch(x);
    TORCH_CHECK(grad_scale > 0.0, "convnet_fwd: grad_scale must be positive");
    // grad_scale (gradient accumulation over k micro-batches: 1/k): the loss is grad_scale · mean cross-entropy, dlogits its gradient
    SoftCe ce;
    ce.scale = static_cast<float>(grad_scale);
    at::Tensor loss, dlogits, loss_parts;
    if (target.has_value() && target->defined()) {
      // int64 class indices [B], or fp32 class probabilities [B, ncls] (SoftCe)
      const bool soft = soft_target(*target, logits, ignore_index, "convnet_fwd");
      TORCH_CHECK(soft || target->numel() == B, "convnet_fwd: one target per image expected");
      // ce_weight / ignore_index / label_smoothing / reduction: torch's cross-entropy options (a non-default spec runs SmoothCe)
      const CeSpec spec = ce_spec(ce_weight, ignore_index, label_smoothing, reduction, ncls, x, "convnet_fwd");
      ce.weight = spec.weight;
      ce.smoothing = spec.smoothing;
      ce.ignore_index = spec.ignore_index;
      ce.sum = spec.sum;
      loss = at::empty({}, x.options());
      dlogits = at::empty({B, ncls}, x.options());
      loss_parts = at::empty({B + 1}, x.options());   // one term per image, then the number of counted images
      if (soft) ce.target_probs = target->data_ptr<float>();
      else ce.target = reinterpret_cast<const long long*>(target->data_ptr<int64_t>());
      ce.loss_parts = loss_parts.data_ptr<float>();
      ce.loss = defer_loss_mean ? nullptr : loss.data_ptr<float>();   // deferred: convnet_l2_bwd_fc(…, loss_parts, loss) writes it
      ce.dlogits = dlogits.data_ptr<float>();
      ce.counter = scr.counter + kCeCounterWord;
    }
    launch_convnet_fwd(x.data_ptr<float>(), w1.data_ptr<float>(), opt_ptr(b1, "b1"), opt_ptr(g1, "g1"), opt_ptr(be1, "be1"), keep_y1 ? y1.data_ptr<float>() : nullptr,
                       p1.data_ptr<float>(), saved1.data_ptr<float>(), opt_mut(rm1, "rm1"), opt_mut(rv1, "rv1"), nbt_ptr(nbt1), static_cast<float>(mom1),
                       static_cast<float>(eps1), w2.data_ptr<float>(), opt_ptr(b2, "b2"), opt_ptr(g2, "g2"), opt_ptr(be2, "be2"), y2.data_ptr<float>(),
                       out.data_ptr<float>(), saved2.data_ptr<float>(), opt_mut(rm2, "rm2"), opt_mut(rv2, "rv2"), nbt_ptr(nbt2), static_cast<float>(mom2),
                       static_cast<float>(eps2), fcw.data_ptr<float>(), opt_ptr(fcb, "fc bias"), logits.data_ptr<float>(), ncls, B, scr.partials,
                       grid_sync(scr), cur_stream(x), ce);
    return py::make_tuple(p1, y1, saved1, out, y2, saved2, logits, loss, dlogits, loss_parts);
  }, py::arg("x"), py::arg("w1"), py::arg("b1"), py::arg("g1"), py::arg("be1"), py::arg("rm1"), py::arg("rv1"), py::arg("nbt1"), py::arg("mom1"),
     py::arg("eps1"), py::arg("w2"), py::arg("b2"), py::arg("g2"), py::arg("be2"), py::arg("rm2"), py::arg("rv2"), py::arg("nbt2"), py::arg("mom2"),
     py::arg("eps2"), py::arg("fcw"), py::arg("fcb"), py::arg("target") = py::none(), py::arg("defer_loss_mean") = false,
     py::arg("grad_scale") = 1.0, py::arg("ce_weight") = py::none(), py::arg("ignore_index") = -100, py::arg("label_smoothing") = 0.0,
     py::arg("reduction") = "mean", py::arg("keep_y1") = true);
  // p1 (conv2's input frame [B,18,18,16], optional): conv2's per-image weight-gradient partials are computed inside the kernel for
  // convnet_l1_bwd_wgrad(…, None, None, …) to fold, and the dy frame is not written (None in its place).  The training step always
  // passes p1; the dy frame of the form without it, fed to convnet_l1_bwd_wgrad, is the tests' reference for those partials.
  m.def("convnet_l2_bwd_fc", [](const at::Tensor& dlogits, const at::Tensor& fcw, const at::Tensor& pooled, at::Tensor dfcw, c10::optional<at::Tensor> dfcb,
                                const at::Tensor& y, const at::Tensor& saved, c10::optional<at::Tensor> gamma, c10::optional<at::Tensor> beta,
                                const at::Tensor& w, at::Tensor dgamma, at::Tensor dbeta, c10::optional<at::Tensor> loss_parts,
                                c10::optional<at::Tensor> loss_out, c10::optional<at::Tensor> p1, bool accumulate) {
    chk(dlogits, "dlogits"); chk(fcw, "fc weight"); chk(pooled, "pooled"); chk(dfcw, "dfcw");
    chk(y, "y"); chk(saved, "saved"); chk(w, "w"); chk(dgamma, "dgamma"); chk(dbeta, "dbeta");
    c10::cuda::CUDAGuard g(y.device());
    const int B = static_cast<int>(y.size(0));
    const int ncls = static_cast<int>(fcw.size(0));
    TORCH_CHECK(fcw.dim() == 2 && fcw.size(1) == 1568 && ncls <= 16 && dlogits.numel() == static_cast<int64_t>(B) * ncls &&
                    pooled.numel() == static_cast<int64_t>(B) * 1568 && dfcw.numel() == fcw.numel() && y.numel() == static_cast<int64_t>(B) * 6272 &&
                    w.numel() == 12800 && dgamma.numel() == 32 && dbeta.numel() == 32, "convnet_l2_bwd_fc: shape mismatch");
    TORCH_CHECK(reinterpret_cast<uintptr_t>(fcw.data_ptr()) % 16 == 0, "convnet_l2_bwd_fc: fc weight must be 16-byte aligned");
    TORCH_CHECK(!loss_parts.has_value() || !loss_parts->defined() || (loss_parts->numel() == B + 1 && loss_out.has_value() && loss_out->defined()),
                "convnet_l2_bwd_fc: loss_parts must be the [B + 1] tensor of convnet_fwd, and loss_out given with it");
    const float* x2 = conv2_input(p1, B, "convnet_l2_bwd_fc");
    // accumulate: dfcw, dfcb, dgamma, dbeta (and loss_out) hold the earlier micro-batches' sum and are added to
    TORCH_CHECK(!accumulate || x2 != nullptr, "convnet_l2_bwd_fc: accumulate mode is the variant with conv2's weight-gradient partials (p1)");
    at::Tensor dy = x2 ? at::Tensor() : at::empty({B, 18, 18, 32}, y.options());
    at::Tensor dx = at::empty({B, 18, 18, 16}, y.options());
    at::Tensor dysum = at::empty({B, 32}, y.options());
    ReduceScratch scr = scratch(y);
    float* wpart = x2 ? conv2_wgrad_partials(y, B, "convnet_l2_bwd_fc") : nullptr;
    launch_convnet_l2_bwd_fc(dlogits.data_ptr<float>(), fcw.data_ptr<float>(), pooled.data_ptr<float>(), dfcw.data_ptr<float>(), opt_mut(dfcb, "dfcb"),
                             ncls, y.data_ptr<float>(), saved.data_ptr<float>(), opt_ptr(gamma, "gamma"), opt_ptr(beta, "beta"), w.data_ptr<float>(),
                             dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), x2 ? nullptr : dy.data_ptr<float>(), dx.data_ptr<float>(),
                             dysum.data_ptr<float>(), B, scr.partials, grid_sync(scr), cur_stream(y), opt_ptr(loss_parts, "loss_parts"),
                             opt_mut(loss_out, "loss_out"), x2, wpart, accumulate);
    if (x2) scratch_entry(y).wgrad_batch = B;
    return py::make_tuple(x2 ? py::none() : py::cast(dy), dx, dysum);
  }, py::arg("dlogits"), py::arg("fcw"), py::arg("pooled"), py::arg("dfcw"), py::arg("dfcb"), py::arg("y"), py::arg("saved"), py::arg("gamma"),
     py::arg("beta"), py::arg("w"), py::arg("dgamma"), py::arg("dbeta"), py::arg("loss_parts") = py::none(), py::arg("loss_out") = py::none(),
     py::arg("p1") = py::none(), py::arg("accumulate") = false);
  // ---- BN + ReLU + pool ------------------------------------------------------------------------------
  // fp64_sums: stats are conv5x5_fwd's fp64 [Σy, Σy², n, 0] (all-reduced by SyncBatchNorm); saved then has 2C+1 entries, the count
  // last, for bn_relu_pool_bwd_apply
  m.def("bn_relu_pool_fwd", [](const at::Tensor& y, const at::Tensor& stats, c10::optional<at::Tensor> gamma, c10::optional<at::Tensor> beta,
                               c10::optional<at::Tensor> running_mean, c10::optional<at::Tensor> running_var,
                               c10::optional<at::Tensor> nbt, double momentum, double eps, bool out_nchw, bool mean_var, bool centred,
                               bool fp64_sums) {
    chk(y, "y"); chk(stats, "stats", fp64_sums ? at::kDouble : at::kFloat);
    c10::cuda::CUDAGuard g(y.device());
    TORCH_CHECK(y.dim() == 4, "bn_relu_pool_fwd: y [B,H,W,C] expected");
    const int B = y.size(0), H = y.size(1), W = y.size(2), C = y.size(3);
    TORCH_CHECK(int(mean_var) + int(centred) + int(fp64_sums) <= 1, "bn_relu_pool_fwd: stats are one of mean_var, centred or fp64_sums");
    if (mean_var) {
      TORCH_CHECK(stats.numel() == 2 * C, "bn_relu_pool_fwd: mean_var stats must have 2C entries (mean, var)");
      TORCH_CHECK(!(running_mean.has_value() && running_mean->defined()) && !(running_var.has_value() && running_var->defined()) &&
                      !(nbt.has_value() && nbt->defined()), "bn_relu_pool_fwd: mean_var statistics update no running statistics");
    } else if (fp64_sums) {
      TORCH_CHECK(stats.numel() == 2 * C + 2, "bn_relu_pool_fwd: fp64_sums stats must have 2C+2 entries");
    } else {
      TORCH_CHECK(stats.numel() == 2 * C + 1, "bn_relu_pool_fwd: stats must have 2C+1 entries");
    }
    at::Tensor out = out_nchw ? at::empty({B, C, H / 2, W / 2}, y.options()) : at::empty({B, H / 2, W / 2, C}, y.options());
    at::Tensor saved = at::empty({fp64_sums ? 2 * C + 1 : 2 * C}, y.options());
    long long* nbt_p = nullptr;
    if (nbt.has_value() && nbt->defined()) { chk(*nbt, "num_batches_tracked", at::kLong); nbt_p = reinterpret_cast<long long*>(nbt->data_ptr<int64_t>()); }
    launch_bn_relu_pool_fwd(y.data_ptr<float>(), stats.data_ptr(), opt_ptr(gamma, "gamma"), opt_ptr(beta, "beta"), out.data_ptr<float>(),
                            saved.data_ptr<float>(), opt_mut(running_mean, "running_mean"), opt_mut(running_var, "running_var"), nbt_p,
                            static_cast<float>(momentum), static_cast<float>(eps), B, H, W, C, out_nchw,
                            mean_var ? kBnMeanVar : centred ? kBnCentred : fp64_sums ? kBnSums64 : kBnSums, cur_stream(y));
    return py::make_tuple(out, saved);
  }, py::arg("y"), py::arg("stats"), py::arg("gamma"), py::arg("beta"), py::arg("running_mean"), py::arg("running_var"), py::arg("nbt"),
     py::arg("momentum"), py::arg("eps"), py::arg("out_nchw"), py::arg("mean_var") = false, py::arg("centred") = false,
     py::arg("fp64_sums") = false);
  m.def("bn_relu_pool_bwd_reduce", [](const at::Tensor& dout, const at::Tensor& y, const at::Tensor& saved, c10::optional<at::Tensor> gamma,
                                      c10::optional<at::Tensor> beta, bool dout_nchw, c10::optional<at::Tensor> dgamma_out,
                                      c10::optional<at::Tensor> dbeta_out) {
    chk(dout, "dout"); chk(y, "y"); chk(saved, "saved");
    c10::cuda::CUDAGuard g(y.device());
    const int B = y.size(0), H = y.size(1), W = y.size(2), C = y.size(3);
    at::Tensor sums = at::empty({2 * C}, y.options());
    at::Tensor dgamma = dgamma_out.has_value() && dgamma_out->defined() ? *dgamma_out : at::empty({C}, y.options());
    at::Tensor dbeta = dbeta_out.has_value() && dbeta_out->defined() ? *dbeta_out : at::empty({C}, y.options());
    chk(dgamma, "dgamma"); chk(dbeta, "dbeta");
    TORCH_CHECK(dgamma.numel() == C && dbeta.numel() == C, "bn_relu_pool_bwd_reduce: dgamma/dbeta must have C elements");
    launch_bn_relu_pool_bwd_reduce(dout.data_ptr<float>(), y.data_ptr<float>(), saved.data_ptr<float>(), opt_ptr(gamma, "gamma"),
                                   opt_ptr(beta, "beta"), sums.data_ptr<float>(), dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), B, H, W, C,
                                   dout_nchw, scratch(y), cur_stream(y));
    return py::make_tuple(sums, dgamma, dbeta);
  }, py::arg("dout"), py::arg("y"), py::arg("saved"), py::arg("gamma"), py::arg("beta"), py::arg("dout_nchw"),
     py::arg("dgamma_out") = py::none(), py::arg("dbeta_out") = py::none());
  // Batch statistics take bn_relu_pool_bwd_reduce's (possibly all-reduced) sums and the element count.  mean_var=True: the forward
  // ran with mean_var=True (eval: the running statistics, constants of the graph), so dy has no batch-mean terms and takes neither.
  m.def("bn_relu_pool_bwd_apply", [](const at::Tensor& dout, const at::Tensor& y, const at::Tensor& saved, c10::optional<at::Tensor> gamma,
                                     c10::optional<at::Tensor> beta, c10::optional<at::Tensor> sums, c10::optional<at::Tensor> count,
                                     bool dout_nchw, bool mean_var) {
    chk(dout, "dout"); chk(y, "y"); chk(saved, "saved");
    const bool has_sums = sums.has_value() && sums->defined(), has_count = count.has_value() && count->defined();
    TORCH_CHECK(has_sums != mean_var && has_count != mean_var,
                "bn_relu_pool_bwd_apply: batch statistics take sums and count, mean_var=True takes neither");
    c10::cuda::CUDAGuard g(y.device());
    const int B = y.size(0), H = y.size(1), W = y.size(2), C = y.size(3);
    at::Tensor dy = at::empty_like(y);
    launch_bn_relu_pool_bwd_apply(dout.data_ptr<float>(), y.data_ptr<float>(), saved.data_ptr<float>(), opt_ptr(gamma, "gamma"),
                                  opt_ptr(beta, "beta"), opt_ptr(sums, "sums"), opt_ptr(count, "count"), dy.data_ptr<float>(), B, H, W, C,
                                  dout_nchw, mean_var, cur_stream(y));
    return dy;
  }, py::arg("dout"), py::arg("y"), py::arg("saved"), py::arg("gamma"), py::arg("beta"), py::arg("sums"), py::arg("count"),
     py::arg("dout_nchw"), py::arg("mean_var") = false);

  // ---- generic NCHW BatchNorm (SyncBatchNorm) ----------------------------------------------------------
  m.def("bn_stats_nchw_f64", [](const at::Tensor& x) {
    chk(x, "x");
    TORCH_CHECK(x.dim() >= 2, "bn_stats: at least 2-D input");
    c10::cuda::CUDAGuard g(x.device());
    const int N = x.size(0), C = x.size(1);
    const int HW = static_cast<int>(x.numel() / std::max<int64_t>(1, static_cast<int64_t>(N) * C));
    at::Tensor stats = at::zeros({2 * C + 2}, x.options().dtype(at::kDouble));  // [2C+1] + one pad: 16-byte multiple for the allreduce
    if (x.numel() > 0) launch_bn_stats_nchw_f64(x.data_ptr<float>(), stats.data_ptr<double>(), N, C, HW, scratch(x), cur_stream(x));
    return stats;
  });
  m.def("bn_finalize", [](const at::Tensor& stats, int64_t C, double eps, double momentum, c10::optional<at::Tensor> running_mean,
                          c10::optional<at::Tensor> running_var) {
    chk(stats, "stats", at::kDouble);
    TORCH_CHECK(stats.numel() >= 2 * C + 1, "bn_finalize: stats must hold 2C+1 entries");
    TORCH_CHECK(running_mean.has_value() == running_var.has_value(), "bn_finalize: running_mean and running_var go together");
    c10::cuda::CUDAGuard g(stats.device());
    auto opt = stats.options().dtype(at::kFloat);
    at::Tensor mean = at::empty({C}, opt), invstd = at::empty({C}, opt), count = at::empty({1}, opt);
    launch_bn_finalize(stats.data_ptr<double>(), static_cast<int>(C), eps, static_cast<float>(momentum), mean.data_ptr<float>(),
                       invstd.data_ptr<float>(), count.data_ptr<float>(), opt_mut(running_mean, "running_mean"),
                       opt_mut(running_var, "running_var"), cur_stream(stats));
    return py::make_tuple(mean, invstd, count);
  });
  m.def("bn_apply_nchw", [](const at::Tensor& x, const at::Tensor& mean, const at::Tensor& invstd, c10::optional<at::Tensor> gamma,
                            c10::optional<at::Tensor> beta) {
    chk(x, "x"); chk(mean, "mean"); chk(invstd, "invstd");
    c10::cuda::CUDAGuard g(x.device());
    const int N = x.size(0), C = x.size(1);
    const int HW = static_cast<int>(x.numel() / std::max<int64_t>(1, static_cast<int64_t>(N) * C));
    at::Tensor out = at::empty_like(x);
    if (x.numel() > 0) launch_bn_apply_nchw(x.data_ptr<float>(), mean.data_ptr<float>(), invstd.data_ptr<float>(), opt_ptr(gamma, "gamma"),
                                            opt_ptr(beta, "beta"), out.data_ptr<float>(), N, C, HW, cur_stream(x));
    return out;
  });
  m.def("bn_bwd_reduce_nchw", [](const at::Tensor& dy, const at::Tensor& x, const at::Tensor& mean, const at::Tensor& invstd) {
    chk(dy, "dy"); chk(x, "x"); chk(mean, "mean"); chk(invstd, "invstd");
    c10::cuda::CUDAGuard g(x.device());
    const int N = x.size(0), C = x.size(1);
    const int HW = static_cast<int>(x.numel() / std::max<int64_t>(1, static_cast<int64_t>(N) * C));
    at::Tensor red = at::zeros({4 * C}, x.options());
    if (x.numel() > 0) launch_bn_bwd_reduce_nchw(dy.data_ptr<float>(), x.data_ptr<float>(), mean.data_ptr<float>(), invstd.data_ptr<float>(),
                                                 red.data_ptr<float>(), N, C, HW, scratch(x), cur_stream(x));
    return red;
  });
  m.def("bn_bwd_apply_nchw", [](const at::Tensor& dy, const at::Tensor& x, const at::Tensor& mean, const at::Tensor& invstd,
                                c10::optional<at::Tensor> gamma, const at::Tensor& mean_dy, const at::Tensor& mean_dy_xmu) {
    chk(dy, "dy"); chk(x, "x"); chk(mean_dy, "mean_dy"); chk(mean_dy_xmu, "mean_dy_xmu");
    c10::cuda::CUDAGuard g(x.device());
    const int N = x.size(0), C = x.size(1);
    const int HW = static_cast<int>(x.numel() / std::max<int64_t>(1, static_cast<int64_t>(N) * C));
    at::Tensor dx = at::empty_like(x);
    if (x.numel() > 0) launch_bn_bwd_apply_nchw(dy.data_ptr<float>(), x.data_ptr<float>(), mean.data_ptr<float>(), invstd.data_ptr<float>(),
                                                opt_ptr(gamma, "gamma"), mean_dy.data_ptr<float>(), mean_dy_xmu.data_ptr<float>(),
                                                dx.data_ptr<float>(), N, C, HW, cur_stream(x));
    return dx;
  });

  // ---- head ---------------------------------------------------------------------------------------------
  m.def("linear_fwd", [](const at::Tensor& x, const at::Tensor& w, c10::optional<at::Tensor> b) {
    chk(x, "x"); chk(w, "w");
    c10::cuda::CUDAGuard g(x.device());
    TORCH_CHECK(x.dim() == 2 && w.dim() == 2 && x.size(1) == w.size(1), "linear_fwd: x [B,K], w [N,K]");
    at::Tensor out = at::empty({x.size(0), w.size(0)}, x.options());
    launch_linear_fwd(x.data_ptr<float>(), w.data_ptr<float>(), opt_ptr(b, "bias"), out.data_ptr<float>(), x.size(0), x.size(1), w.size(0), cur_stream(x));
    return out;
  });
  m.def("linear_bwd", [](const at::Tensor& dout, const at::Tensor& x, const at::Tensor& w, bool need_dx, at::Tensor dw, c10::optional<at::Tensor> db) {
    chk(dout, "dout"); chk(x, "x"); chk(w, "w"); chk(dw, "dw");
    c10::cuda::CUDAGuard g(x.device());
    at::Tensor dx = need_dx ? at::empty_like(x) : at::Tensor();
    launch_linear_bwd(dout.data_ptr<float>(), x.data_ptr<float>(), w.data_ptr<float>(), need_dx ? dx.data_ptr<float>() : nullptr,
                      dw.data_ptr<float>(), opt_mut(db, "db"), x.size(0), x.size(1), w.size(0), cur_stream(x));
    return dx;
  });
  // weight / ignore_index / label_smoothing / reduction: torch's options (ops_kernels.h: CeSpec); the defaults run the plain mean kernels.
  // target: int64 class indices [B], or fp32 class probabilities shaped like the logits (soft_target)
  m.def("cross_entropy_fwd", [](const at::Tensor& logits, const at::Tensor& target, bool emit_grad, c10::optional<at::Tensor> weight,
                                int64_t ignore_index, double label_smoothing, const std::string& reduction) {
    chk(logits, "logits");
    const bool soft = soft_target(target, logits, ignore_index, "cross_entropy_fwd");
    c10::cuda::CUDAGuard g(logits.device());
    const CeSpec spec = ce_spec(weight, ignore_index, label_smoothing, reduction, logits.size(1), logits, "cross_entropy_fwd");
    at::Tensor loss = at::empty({}, logits.options()), probs = at::empty_like(logits);
    if (soft)
      launch_cross_entropy_fwd_soft(logits.data_ptr<float>(), target.data_ptr<float>(), loss.data_ptr<float>(), probs.data_ptr<float>(),
                                    logits.size(0), logits.size(1), cur_stream(logits), emit_grad, spec);
    else
      launch_cross_entropy_fwd(logits.data_ptr<float>(), reinterpret_cast<const long long*>(target.data_ptr<int64_t>()), loss.data_ptr<float>(),
                               probs.data_ptr<float>(), logits.size(0), logits.size(1), cur_stream(logits), emit_grad, spec);
    return py::make_tuple(loss, probs);  // emit_grad: the second tensor is d(loss)/d(logits) for a unit incoming gradient
  }, py::arg("logits"), py::arg("target"), py::arg("emit_grad") = false, py::arg("weight") = py::none(), py::arg("ignore_index") = -100,
     py::arg("label_smoothing") = 0.0, py::arg("reduction") = "mean");
  m.def("cross_entropy_bwd", [](const at::Tensor& probs, const at::Tensor& target, const at::Tensor& dloss, c10::optional<at::Tensor> weight,
                                int64_t ignore_index, double label_smoothing, const std::string& reduction) {
    chk(probs, "probs"); chk(dloss, "dloss");
    const bool soft = soft_target(target, probs, ignore_index, "cross_entropy_bwd");
    c10::cuda::CUDAGuard g(probs.device());
    const CeSpec spec = ce_spec(weight, ignore_index, label_smoothing, reduction, probs.size(1), probs, "cross_entropy_bwd");
    at::Tensor d = at::empty_like(probs);
    if (soft)
      launch_cross_entropy_bwd_soft(probs.data_ptr<float>(), target.data_ptr<float>(), dloss.data_ptr<float>(), d.data_ptr<float>(),
                                    probs.size(0), probs.size(1), cur_stream(probs), spec);
    else
      launch_cross_entropy_bwd(probs.data_ptr<float>(), reinterpret_cast<const long long*>(target.data_ptr<int64_t>()), dloss.data_ptr<float>(),
                               d.data_ptr<float>(), probs.size(0), probs.size(1), cur_stream(probs), spec);
    return d;
  }, py::arg("probs"), py::arg("target"), py::arg("dloss"), py::arg("weight") = py::none(), py::arg("ignore_index") = -100,
     py::arg("label_smoothing") = 0.0, py::arg("reduction") = "mean");
  // acc[0..3] += Σ loss terms, Σ counted target weights, top-1 hits, counted rows of logits[:rows] (ops_kernels.h); no sync
  m.def("cross_entropy_eval", [](const at::Tensor& logits, const at::Tensor& target, at::Tensor acc, int64_t rows,
                                 c10::optional<at::Tensor> weight, int64_t ignore_index, double label_smoothing) {
    chk(logits, "logits"); chk(target, "target", at::kLong); chk(acc, "acc", at::kDouble);
    TORCH_CHECK(logits.dim() == 2 && logits.size(1) >= 1 && logits.size(1) <= 1024, "cross_entropy_eval: logits must be [B, C <= 1024]");
    TORCH_CHECK(target.dim() == 1 && target.size(0) == logits.size(0), "cross_entropy_eval: target must be [", logits.size(0), "]");
    TORCH_CHECK(acc.numel() == 4 && acc.device() == logits.device(), "cross_entropy_eval: acc must be 4 doubles on ", logits.device());
    TORCH_CHECK(rows >= 0 && rows <= logits.size(0), "cross_entropy_eval: rows must lie in [0, ", logits.size(0), "] (got ", rows, ")");
    c10::cuda::CUDAGuard g(logits.device());
    const CeSpec spec = ce_spec(weight, ignore_index, label_smoothing, "mean", logits.size(1), logits, "cross_entropy_eval");
    launch_cross_entropy_eval(logits.data_ptr<float>(), reinterpret_cast<const long long*>(target.data_ptr<int64_t>()), acc.data_ptr<double>(),
                              static_cast<int>(rows), logits.size(1), cur_stream(logits), spec);
  }, py::arg("logits"), py::arg("target"), py::arg("acc"), py::arg("rows"), py::arg("weight") = py::none(), py::arg("ignore_index") = -100,
     py::arg("label_smoothing") = 0.0);

  // ---- optimizer ------------------------------------------------------------------------------------------
  m.def("sgd_multi", [](std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> bufs, double lr,
                        c10::optional<at::Tensor> lr_tensor, double momentum, double dampening, double weight_decay, bool nesterov,
                        bool maximize, bool first_step) {
    TORCH_CHECK(params.size() == grads.size(), "sgd_multi: params/grads length mismatch");
    TORCH_CHECK(momentum == 0.0 || bufs.size() == params.size(), "sgd_multi: momentum buffers required");
    if (params.empty()) return;
    c10::cuda::CUDAGuard g(params[0].device());
    const SgdHyper h = sgd_hyper(lr, lr_tensor, momentum, dampening, weight_decay, nesterov, maximize, first_step);
    cudaStream_t st = cur_stream(params[0]);
    for (size_t base = 0; base < params.size(); base += SgdTensorList::kMax) {
      SgdTensorList tl;
      tl.count = static_cast<int>(std::min<size_t>(SgdTensorList::kMax, params.size() - base));
      for (int i = 0; i < tl.count; ++i) {
        at::Tensor& p = params[base + i];
        at::Tensor& gr = grads[base + i];
        chk(p, "param"); chk(gr, "grad");
        TORCH_CHECK(p.numel() == gr.numel() && p.numel() < (int64_t(1) << 31), "sgd_multi: bad tensor sizes");
        tl.p[i] = p.data_ptr<float>();
        tl.g[i] = gr.data_ptr<float>();
        tl.m[i] = momentum != 0.0 ? bufs[base + i].data_ptr<float>() : nullptr;
        tl.n[i] = static_cast<int>(p.numel());
      }
      launch_sgd_multi(tl, h, st);
    }
  });
  m.def("adam_multi", [](std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> exp_avgs,
                         std::vector<at::Tensor> exp_avg_sqs, std::vector<at::Tensor> steps, double lr, c10::optional<at::Tensor> lr_tensor,
                         double beta1, double beta2, double eps, double weight_decay, bool decoupled, bool maximize,
                         c10::optional<std::vector<at::Tensor>> max_exp_avg_sqs) {
    const size_t n = params.size();
    TORCH_CHECK(grads.size() == n && exp_avgs.size() == n && exp_avg_sqs.size() == n && steps.size() == n, "adam_multi: list lengths differ");
    // max_exp_avg_sqs: AMSGrad (amsgrad_multi_kernel)
    const bool ams = max_exp_avg_sqs.has_value();
    TORCH_CHECK(!ams || max_exp_avg_sqs->size() == n, "adam_multi: list lengths differ");
    if (n == 0) return;
    c10::cuda::CUDAGuard g(params[0].device());
    const AdamHyper h = adam_hyper(lr, lr_tensor, beta1, beta2, eps, weight_decay, decoupled, maximize);
    cudaStream_t st = cur_stream(params[0]);
    // the ticket word of the step hand-over (adam_multi_kernel); launches on one device are ordered by the compute stream, and
    // every launch leaves the word at zero
    unsigned int* ticket = scratch(params[0]).counter + kAdamTicketWord;
    for (size_t base = 0; base < n; base += AdamTensorList::kMax) {
      AmsgradTensorList tl;
      tl.count = static_cast<int>(std::min<size_t>(AdamTensorList::kMax, n - base));
      for (int i = 0; i < tl.count; ++i) {
        const size_t j = base + i;
        chk(params[j], "param"); chk(grads[j], "grad"); chk(exp_avgs[j], "exp_avg"); chk(exp_avg_sqs[j], "exp_avg_sq"); chk(steps[j], "step");
        const int64_t numel = params[j].numel();
        TORCH_CHECK(grads[j].numel() == numel && exp_avgs[j].numel() == numel && exp_avg_sqs[j].numel() == numel && steps[j].numel() == 1 &&
                        numel < (int64_t(1) << 31), "adam_multi: bad tensor sizes");
        TORCH_CHECK(params[j].device() == params[0].device() && steps[j].device() == params[0].device(), "adam_multi: all tensors on one device");
        tl.p[i] = params[j].data_ptr<float>();
        tl.g[i] = grads[j].data_ptr<float>();
        tl.m[i] = exp_avgs[j].data_ptr<float>();
        tl.v[i] = exp_avg_sqs[j].data_ptr<float>();
        tl.step[i] = steps[j].data_ptr<float>();
        tl.n[i] = static_cast<int>(numel);
        if (ams) {
          const at::Tensor& vm = (*max_exp_avg_sqs)[j];
          chk(vm, "max_exp_avg_sq");
          TORCH_CHECK(vm.numel() == numel, "adam_multi: bad tensor sizes");
          TORCH_CHECK(vm.device() == params[0].device(), "adam_multi: all tensors on one device");
          tl.vmax[i] = vm.data_ptr<float>();
        }
      }
      if (ams) launch_adam_multi(tl, h, ticket, st);
      else launch_adam_multi(static_cast<const AdamTensorList&>(tl), h, ticket, st);
    }
  });
  // NAdam (mu_products given) and RAdam (mu_products empty, momentum_decay unused): adam_multi's tables and checks; the step counts
  // and mu_products take adam_multi's ticket word.
  auto nadam_radam = [](bool nadam, std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> exp_avgs,
                        std::vector<at::Tensor> exp_avg_sqs, std::vector<at::Tensor> steps, std::vector<at::Tensor> mu_products, double lr,
                        c10::optional<at::Tensor> lr_tensor, double beta1, double beta2, double eps, double weight_decay, bool decoupled,
                        bool maximize, double momentum_decay) {
    const size_t n = params.size();
    const char* who = nadam ? "nadam_multi" : "radam_multi";
    TORCH_CHECK(grads.size() == n && exp_avgs.size() == n && exp_avg_sqs.size() == n && steps.size() == n &&
                    mu_products.size() == (nadam ? n : 0), who, ": list lengths differ");
    if (n == 0) return;
    c10::cuda::CUDAGuard g(params[0].device());
    NadamHyper h;
    static_cast<AdamHyper&>(h) = adam_hyper(lr, lr_tensor, beta1, beta2, eps, weight_decay, decoupled, maximize);
    h.momentum_decay = momentum_decay;
    cudaStream_t st = cur_stream(params[0]);
    unsigned int* ticket = scratch(params[0]).counter + kAdamTicketWord;
    for (size_t base = 0; base < n; base += AdamTensorList::kMax) {
      NadamTensorList tl;
      tl.count = static_cast<int>(std::min<size_t>(AdamTensorList::kMax, n - base));
      for (int i = 0; i < tl.count; ++i) {
        const size_t j = base + i;
        chk(params[j], "param"); chk(grads[j], "grad"); chk(exp_avgs[j], "exp_avg"); chk(exp_avg_sqs[j], "exp_avg_sq"); chk(steps[j], "step");
        const int64_t numel = params[j].numel();
        TORCH_CHECK(grads[j].numel() == numel && exp_avgs[j].numel() == numel && exp_avg_sqs[j].numel() == numel && steps[j].numel() == 1 &&
                        numel < (int64_t(1) << 31), who, ": bad tensor sizes");
        TORCH_CHECK(params[j].device() == params[0].device() && steps[j].device() == params[0].device(), who, ": all tensors on one device");
        tl.p[i] = params[j].data_ptr<float>();
        tl.g[i] = grads[j].data_ptr<float>();
        tl.m[i] = exp_avgs[j].data_ptr<float>();
        tl.v[i] = exp_avg_sqs[j].data_ptr<float>();
        tl.step[i] = steps[j].data_ptr<float>();
        tl.n[i] = static_cast<int>(numel);
        if (nadam) {
          chk(mu_products[j], "mu_product");
          TORCH_CHECK(mu_products[j].numel() == 1, who, ": bad tensor sizes");
          TORCH_CHECK(mu_products[j].device() == params[0].device(), who, ": all tensors on one device");
          tl.mu_product[i] = mu_products[j].data_ptr<float>();
        }
      }
      if (nadam) launch_nadam_multi(tl, h, ticket, st);
      else launch_radam_multi(static_cast<const AdamTensorList&>(tl), static_cast<const AdamHyper&>(h), ticket, st);
    }
  };
  m.def("nadam_multi", [nadam_radam](std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> exp_avgs,
                                     std::vector<at::Tensor> exp_avg_sqs, std::vector<at::Tensor> steps, std::vector<at::Tensor> mu_products,
                                     double lr, c10::optional<at::Tensor> lr_tensor, double beta1, double beta2, double eps, double weight_decay,
                                     bool decoupled, bool maximize, double momentum_decay) {
    nadam_radam(true, params, grads, exp_avgs, exp_avg_sqs, steps, mu_products, lr, lr_tensor, beta1, beta2, eps, weight_decay,
                decoupled, maximize, momentum_decay);
  });
  m.def("radam_multi", [nadam_radam](std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> exp_avgs,
                                     std::vector<at::Tensor> exp_avg_sqs, std::vector<at::Tensor> steps, double lr,
                                     c10::optional<at::Tensor> lr_tensor, double beta1, double beta2, double eps, double weight_decay,
                                     bool decoupled, bool maximize) {
    nadam_radam(false, params, grads, exp_avgs, exp_avg_sqs, steps, {}, lr, lr_tensor, beta1, beta2, eps, weight_decay, decoupled,
                maximize, 0.0);
  });
  // RMSprop: momentum_buffers given exactly when momentum > 0, grad_avgs exactly when centered (empty lists otherwise).  The step
  // counts take adam_multi's ticket word: launches on one device are ordered by the compute stream.
  m.def("rmsprop_multi", [](std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> square_avgs,
                            std::vector<at::Tensor> momentum_buffers, std::vector<at::Tensor> grad_avgs, std::vector<at::Tensor> steps,
                            double lr, c10::optional<at::Tensor> lr_tensor, double alpha, double eps, double weight_decay, double momentum,
                            bool maximize) {
    const size_t n = params.size();
    TORCH_CHECK(grads.size() == n && square_avgs.size() == n && steps.size() == n, "rmsprop_multi: list lengths differ");
    TORCH_CHECK(momentum > 0.0 ? momentum_buffers.size() == n : momentum_buffers.empty(),
                "rmsprop_multi: momentum buffers are given exactly when momentum > 0");
    TORCH_CHECK(grad_avgs.empty() || grad_avgs.size() == n, "rmsprop_multi: list lengths differ");
    if (n == 0) return;
    c10::cuda::CUDAGuard g(params[0].device());
    const RmspropHyper h = rmsprop_hyper(lr, lr_tensor, alpha, eps, weight_decay, momentum, maximize);
    cudaStream_t st = cur_stream(params[0]);
    unsigned int* ticket = scratch(params[0]).counter + kAdamTicketWord;
    const bool centered = !grad_avgs.empty(), mom = !momentum_buffers.empty();
    for (size_t base = 0; base < n; base += RmspropTensorList::kMax) {
      RmspropTensorList tl;
      tl.count = static_cast<int>(std::min<size_t>(RmspropTensorList::kMax, n - base));
      for (int i = 0; i < tl.count; ++i) {
        const size_t j = base + i;
        chk(params[j], "param"); chk(grads[j], "grad"); chk(square_avgs[j], "square_avg"); chk(steps[j], "step");
        const int64_t numel = params[j].numel();
        TORCH_CHECK(grads[j].numel() == numel && square_avgs[j].numel() == numel && steps[j].numel() == 1 && numel < (int64_t(1) << 31),
                    "rmsprop_multi: bad tensor sizes");
        TORCH_CHECK(params[j].device() == params[0].device() && steps[j].device() == params[0].device(), "rmsprop_multi: all tensors on one device");
        tl.p[i] = params[j].data_ptr<float>();
        tl.g[i] = grads[j].data_ptr<float>();
        tl.sq[i] = square_avgs[j].data_ptr<float>();
        tl.step[i] = steps[j].data_ptr<float>();
        tl.n[i] = static_cast<int>(numel);
        tl.buf[i] = tl.ga[i] = nullptr;
        if (mom) {
          chk(momentum_buffers[j], "momentum_buffer");
          TORCH_CHECK(momentum_buffers[j].numel() == numel, "rmsprop_multi: bad tensor sizes");
          TORCH_CHECK(momentum_buffers[j].device() == params[0].device(), "rmsprop_multi: all tensors on one device");
          tl.buf[i] = momentum_buffers[j].data_ptr<float>();
        }
        if (centered) {
          chk(grad_avgs[j], "grad_avg");
          TORCH_CHECK(grad_avgs[j].numel() == numel, "rmsprop_multi: bad tensor sizes");
          TORCH_CHECK(grad_avgs[j].device() == params[0].device(), "rmsprop_multi: all tensors on one device");
          tl.ga[i] = grad_avgs[j].data_ptr<float>();
        }
      }
      launch_rmsprop_multi(tl, h, ticket, st);
    }
  });
  m.def("adagrad_multi", [](std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> sums,
                            std::vector<at::Tensor> steps, double lr, c10::optional<at::Tensor> lr_tensor, double lr_decay, double eps,
                            double weight_decay, bool maximize) {
    const size_t n = params.size();
    TORCH_CHECK(grads.size() == n && sums.size() == n && steps.size() == n, "adagrad_multi: list lengths differ");
    if (n == 0) return;
    c10::cuda::CUDAGuard g(params[0].device());
    const AdagradHyper h = adagrad_hyper(lr, lr_tensor, lr_decay, eps, weight_decay, maximize);
    cudaStream_t st = cur_stream(params[0]);
    unsigned int* ticket = scratch(params[0]).counter + kAdamTicketWord;
    for (size_t base = 0; base < n; base += AdagradTensorList::kMax) {
      AdagradTensorList tl;
      tl.count = static_cast<int>(std::min<size_t>(AdagradTensorList::kMax, n - base));
      for (int i = 0; i < tl.count; ++i) {
        const size_t j = base + i;
        chk(params[j], "param"); chk(grads[j], "grad"); chk(sums[j], "sum"); chk(steps[j], "step");
        const int64_t numel = params[j].numel();
        TORCH_CHECK(grads[j].numel() == numel && sums[j].numel() == numel && steps[j].numel() == 1 && numel < (int64_t(1) << 31),
                    "adagrad_multi: bad tensor sizes");
        TORCH_CHECK(params[j].device() == params[0].device() && steps[j].device() == params[0].device(), "adagrad_multi: all tensors on one device");
        tl.p[i] = params[j].data_ptr<float>();
        tl.g[i] = grads[j].data_ptr<float>();
        tl.sum[i] = sums[j].data_ptr<float>();
        tl.step[i] = steps[j].data_ptr<float>();
        tl.n[i] = static_cast<int>(numel);
      }
      launch_adagrad_multi(tl, h, ticket, st);
    }
  });
  // Adamax: adam_multi's tables (exp_infs in place of exp_avg_sqs), checks and ticket word.
  m.def("adamax_multi", [](std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> exp_avgs,
                           std::vector<at::Tensor> exp_infs, std::vector<at::Tensor> steps, double lr, c10::optional<at::Tensor> lr_tensor,
                           double beta1, double beta2, double eps, double weight_decay, bool maximize) {
    const size_t n = params.size();
    TORCH_CHECK(grads.size() == n && exp_avgs.size() == n && exp_infs.size() == n && steps.size() == n, "adamax_multi: list lengths differ");
    if (n == 0) return;
    c10::cuda::CUDAGuard g(params[0].device());
    const AdamHyper h = adam_hyper(lr, lr_tensor, beta1, beta2, eps, weight_decay, false, maximize);
    cudaStream_t st = cur_stream(params[0]);
    unsigned int* ticket = scratch(params[0]).counter + kAdamTicketWord;
    for (size_t base = 0; base < n; base += AdamTensorList::kMax) {
      AdamTensorList tl;
      tl.count = static_cast<int>(std::min<size_t>(AdamTensorList::kMax, n - base));
      for (int i = 0; i < tl.count; ++i) {
        const size_t j = base + i;
        chk(params[j], "param"); chk(grads[j], "grad"); chk(exp_avgs[j], "exp_avg"); chk(exp_infs[j], "exp_inf"); chk(steps[j], "step");
        const int64_t numel = params[j].numel();
        TORCH_CHECK(grads[j].numel() == numel && exp_avgs[j].numel() == numel && exp_infs[j].numel() == numel && steps[j].numel() == 1 &&
                        numel < (int64_t(1) << 31), "adamax_multi: bad tensor sizes");
        TORCH_CHECK(params[j].device() == params[0].device() && steps[j].device() == params[0].device(), "adamax_multi: all tensors on one device");
        tl.p[i] = params[j].data_ptr<float>();
        tl.g[i] = grads[j].data_ptr<float>();
        tl.m[i] = exp_avgs[j].data_ptr<float>();
        tl.v[i] = exp_infs[j].data_ptr<float>();
        tl.step[i] = steps[j].data_ptr<float>();
        tl.n[i] = static_cast<int>(numel);
      }
      launch_adamax_multi(tl, h, ticket, st);
    }
  });
  m.def("adadelta_multi", [](std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> square_avgs,
                             std::vector<at::Tensor> acc_deltas, std::vector<at::Tensor> steps, double lr, c10::optional<at::Tensor> lr_tensor,
                             double rho, double eps, double weight_decay, bool maximize) {
    const size_t n = params.size();
    TORCH_CHECK(grads.size() == n && square_avgs.size() == n && acc_deltas.size() == n && steps.size() == n, "adadelta_multi: list lengths differ");
    if (n == 0) return;
    c10::cuda::CUDAGuard g(params[0].device());
    const AdadeltaHyper h = adadelta_hyper(lr, lr_tensor, rho, eps, weight_decay, maximize);
    cudaStream_t st = cur_stream(params[0]);
    unsigned int* ticket = scratch(params[0]).counter + kAdamTicketWord;
    for (size_t base = 0; base < n; base += AdadeltaTensorList::kMax) {
      AdadeltaTensorList tl;
      tl.count = static_cast<int>(std::min<size_t>(AdadeltaTensorList::kMax, n - base));
      for (int i = 0; i < tl.count; ++i) {
        const size_t j = base + i;
        chk(params[j], "param"); chk(grads[j], "grad"); chk(square_avgs[j], "square_avg"); chk(acc_deltas[j], "acc_delta"); chk(steps[j], "step");
        const int64_t numel = params[j].numel();
        TORCH_CHECK(grads[j].numel() == numel && square_avgs[j].numel() == numel && acc_deltas[j].numel() == numel && steps[j].numel() == 1 &&
                        numel < (int64_t(1) << 31), "adadelta_multi: bad tensor sizes");
        TORCH_CHECK(params[j].device() == params[0].device() && steps[j].device() == params[0].device(), "adadelta_multi: all tensors on one device");
        tl.p[i] = params[j].data_ptr<float>();
        tl.g[i] = grads[j].data_ptr<float>();
        tl.sq[i] = square_avgs[j].data_ptr<float>();
        tl.acc[i] = acc_deltas[j].data_ptr<float>();
        tl.step[i] = steps[j].data_ptr<float>();
        tl.n[i] = static_cast<int>(numel);
      }
      launch_adadelta_multi(tl, h, ticket, st);
    }
  });
  m.def("asgd_multi", [](std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> axs, std::vector<at::Tensor> steps,
                         std::vector<at::Tensor> etas, std::vector<at::Tensor> mus, double lr, c10::optional<at::Tensor> lr_tensor, double lambd,
                         double alpha, double t0, double weight_decay, bool maximize) {
    const size_t n = params.size();
    TORCH_CHECK(grads.size() == n && axs.size() == n && steps.size() == n && etas.size() == n && mus.size() == n, "asgd_multi: list lengths differ");
    if (n == 0) return;
    c10::cuda::CUDAGuard g(params[0].device());
    const AsgdHyper h = asgd_hyper(lr, lr_tensor, lambd, alpha, t0, weight_decay, maximize);
    cudaStream_t st = cur_stream(params[0]);
    unsigned int* ticket = scratch(params[0]).counter + kAdamTicketWord;
    for (size_t base = 0; base < n; base += AsgdTensorList::kMax) {
      AsgdTensorList tl;
      tl.count = static_cast<int>(std::min<size_t>(AsgdTensorList::kMax, n - base));
      for (int i = 0; i < tl.count; ++i) {
        const size_t j = base + i;
        chk(params[j], "param"); chk(grads[j], "grad"); chk(axs[j], "ax"); chk(steps[j], "step"); chk(etas[j], "eta"); chk(mus[j], "mu");
        const int64_t numel = params[j].numel();
        TORCH_CHECK(grads[j].numel() == numel && axs[j].numel() == numel && steps[j].numel() == 1 && etas[j].numel() == 1 && mus[j].numel() == 1 &&
                        numel < (int64_t(1) << 31), "asgd_multi: bad tensor sizes");
        TORCH_CHECK(params[j].device() == params[0].device() && steps[j].device() == params[0].device() && etas[j].device() == params[0].device() &&
                        mus[j].device() == params[0].device(), "asgd_multi: all tensors on one device");
        tl.p[i] = params[j].data_ptr<float>();
        tl.g[i] = grads[j].data_ptr<float>();
        tl.ax[i] = axs[j].data_ptr<float>();
        tl.step[i] = steps[j].data_ptr<float>();
        tl.eta[i] = etas[j].data_ptr<float>();
        tl.mu[i] = mus[j].data_ptr<float>();
        tl.n[i] = static_cast<int>(numel);
      }
      launch_asgd_multi(tl, h, ticket, st);
    }
  });
  m.def("rprop_multi", [](std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> prevs,
                          std::vector<at::Tensor> step_sizes, std::vector<at::Tensor> steps, double etaminus, double etaplus, double step_min,
                          double step_max, bool maximize) {
    const size_t n = params.size();
    TORCH_CHECK(grads.size() == n && prevs.size() == n && step_sizes.size() == n && steps.size() == n, "rprop_multi: list lengths differ");
    if (n == 0) return;
    c10::cuda::CUDAGuard g(params[0].device());
    const RpropHyper h = rprop_hyper(etaminus, etaplus, step_min, step_max, maximize);
    cudaStream_t st = cur_stream(params[0]);
    unsigned int* ticket = scratch(params[0]).counter + kAdamTicketWord;
    for (size_t base = 0; base < n; base += RpropTensorList::kMax) {
      RpropTensorList tl;
      tl.count = static_cast<int>(std::min<size_t>(RpropTensorList::kMax, n - base));
      for (int i = 0; i < tl.count; ++i) {
        const size_t j = base + i;
        chk(params[j], "param"); chk(grads[j], "grad"); chk(prevs[j], "prev"); chk(step_sizes[j], "step_size"); chk(steps[j], "step");
        const int64_t numel = params[j].numel();
        TORCH_CHECK(grads[j].numel() == numel && prevs[j].numel() == numel && step_sizes[j].numel() == numel && steps[j].numel() == 1 &&
                        numel < (int64_t(1) << 31), "rprop_multi: bad tensor sizes");
        TORCH_CHECK(params[j].device() == params[0].device() && steps[j].device() == params[0].device(), "rprop_multi: all tensors on one device");
        tl.p[i] = params[j].data_ptr<float>();
        tl.g[i] = grads[j].data_ptr<float>();
        tl.prev[i] = prevs[j].data_ptr<float>();
        tl.step_size[i] = step_sizes[j].data_ptr<float>();
        tl.step[i] = steps[j].data_ptr<float>();
        tl.n[i] = static_cast<int>(numel);
      }
      launch_rprop_multi(tl, h, ticket, st);
    }
  });
  // Gradient-norm clipping: returns the total norm (a 0-d view of a [2] buffer whose second element is the clip coefficient);
  // scale=False stops after the norm kernel (grad_scale then applies the coefficient).
  m.def("grad_norm_clip", [](std::vector<at::Tensor> grads, double max_norm, double norm_type, bool scale) {
    TORCH_CHECK(!grads.empty(), "grad_norm_clip: no gradients");
    TORCH_CHECK(norm_type == 2.0 || (std::isinf(norm_type) && norm_type > 0), "grad_norm_clip: norm_type must be 2 or inf");
    c10::cuda::CUDAGuard g(grads[0].device());
    std::vector<GradTensorList> tables;
    for (size_t base = 0; base < grads.size(); base += GradTensorList::kMax) {
      GradTensorList tl;
      tl.count = static_cast<int>(std::min<size_t>(GradTensorList::kMax, grads.size() - base));
      for (int i = 0; i < tl.count; ++i) {
        at::Tensor& gr = grads[base + i];
        chk(gr, "grad");
        TORCH_CHECK(gr.device() == grads[0].device(), "grad_norm_clip: all gradients on one device");
        TORCH_CHECK(gr.numel() < (int64_t(1) << 31), "grad_norm_clip: gradient too large");
        tl.g[i] = gr.data_ptr<float>();
        tl.n[i] = static_cast<int>(gr.numel());
      }
      tables.push_back(tl);
    }
    int total = 0;
    for (const auto& tl : tables) total += grad_multi_blocks_x(tl) * tl.count;
    ReduceScratch scr = scratch(grads[0]);
    TORCH_CHECK(total <= scr.capacity_floats, "grad_norm_clip: too many gradients for the reduction scratch");
    at::Tensor out = at::empty({2}, grads[0].options());
    cudaStream_t st = cur_stream(grads[0]);
    // the ticket word of the fold (grad_norm_multi_kernel): launches on one device are ordered by the compute stream, and every
    // set leaves the word at zero
    GradNormArgs a{scr.partials, 0, total, 0, std::isinf(norm_type) ? 1 : 0, static_cast<float>(max_norm), out.data_ptr<float>(),
                   scr.counter + kClipTicketWord};
    for (size_t k = 0; k < tables.size(); ++k) {
      a.last = k + 1 == tables.size() ? 1 : 0;
      launch_grad_norm_multi(tables[k], a, st);
      a.part_base += grad_multi_blocks_x(tables[k]) * tables[k].count;
    }
    if (scale)
      for (const auto& tl : tables) launch_grad_scale_multi(tl, out.data_ptr<float>() + 1, st);
    return out.select(0, 0);
  }, py::arg("grads"), py::arg("max_norm"), py::arg("norm_type") = 2.0, py::arg("scale") = true);
  // g *= the clip coefficient stored behind `norm` (a tensor returned by grad_norm_clip)
  m.def("grad_scale", [](std::vector<at::Tensor> grads, const at::Tensor& norm) {
    TORCH_CHECK(norm.is_cuda() && norm.scalar_type() == at::kFloat && norm.dim() == 0 &&
                    norm.storage().nbytes() >= (static_cast<size_t>(norm.storage_offset()) + 2) * sizeof(float),
                "grad_scale: norm must be a tensor returned by grad_norm_clip");
    if (grads.empty()) return;
    c10::cuda::CUDAGuard g(norm.device());
    cudaStream_t st = cur_stream(norm);
    for (size_t base = 0; base < grads.size(); base += GradTensorList::kMax) {
      GradTensorList tl;
      tl.count = static_cast<int>(std::min<size_t>(GradTensorList::kMax, grads.size() - base));
      for (int i = 0; i < tl.count; ++i) {
        at::Tensor& gr = grads[base + i];
        chk(gr, "grad");
        TORCH_CHECK(gr.device() == norm.device() && gr.numel() < (int64_t(1) << 31), "grad_scale: bad gradient");
        tl.g[i] = gr.data_ptr<float>();
        tl.n[i] = static_cast<int>(gr.numel());
      }
      launch_grad_scale_multi(tl, norm.data_ptr<float>() + 1, st);
    }
  });
  // Weight averaging (AveragedModel.update_parameters with the EMA or SWA multi_avg_fn): averaged[i] follows current[i] (fp32, or
  // int64 under EMA), copied[i] takes copied_from[i]; n_averaged (int64 scalar on the device) advances by one.  decay < 0: SWA.
  // One launch per 48 pairs, no host synchronisation.
  m.def("avg_multi", [](std::vector<at::Tensor> averaged, std::vector<at::Tensor> current, at::Tensor n_averaged, double decay,
                        std::vector<at::Tensor> copied, std::vector<at::Tensor> copied_from) {
    TORCH_CHECK(averaged.size() == current.size() && copied.size() == copied_from.size(), "avg_multi: list lengths differ");
    TORCH_CHECK(!averaged.empty() || !copied.empty(), "avg_multi: no tensors");
    chk(n_averaged, "n_averaged", at::kLong);
    TORCH_CHECK(n_averaged.numel() == 1, "avg_multi: n_averaged must be one element");
    const bool swa = decay < 0.0;
    TORCH_CHECK(swa || decay <= 1.0, "avg_multi: decay must lie in [0, 1]");
    c10::cuda::CUDAGuard g(n_averaged.device());
    std::vector<AvgTensorList> tables;
    auto add = [&](at::Tensor& d, at::Tensor& s, bool copy) {
      TORCH_CHECK(d.scalar_type() == at::kFloat || d.scalar_type() == at::kLong, "avg_multi: tensors must be float32 or int64");
      chk(d, "averaged tensor", d.scalar_type());
      chk(s, "model tensor", d.scalar_type());
      TORCH_CHECK(d.device() == n_averaged.device() && s.device() == n_averaged.device(), "avg_multi: all tensors on one device");
      TORCH_CHECK(d.numel() == s.numel() && d.numel() < (int64_t(1) << 31), "avg_multi: bad tensor sizes");
      const bool f32 = d.scalar_type() == at::kFloat;
      TORCH_CHECK(copy || f32 || !swa, "avg_multi: SWA does not average int64 tensors (torch's swa_update raises)");
      if (tables.empty() || tables.back().count == AvgTensorList::kMax) {
        tables.emplace_back();
        tables.back().count = 0;
      }
      AvgTensorList& tl = tables.back();
      tl.avg[tl.count] = d.data_ptr();
      tl.src[tl.count] = s.data_ptr();
      tl.n[tl.count] = static_cast<int>(d.numel());
      tl.mode[tl.count] = f32 ? (copy ? AvgTensorList::kCopyF32 : AvgTensorList::kAvgF32) : (copy ? AvgTensorList::kCopyI64 : AvgTensorList::kAvgI64);
      ++tl.count;
    };
    for (size_t i = 0; i < averaged.size(); ++i) add(averaged[i], current[i], false);
    for (size_t i = 0; i < copied.size(); ++i) add(copied[i], copied_from[i], true);
    // the ticket word of the n_averaged hand-over (avg_multi_kernel): launches on one device are ordered by the compute stream,
    // and every set leaves the word at zero
    AvgArgs a{reinterpret_cast<long long*>(n_averaged.data_ptr<int64_t>()), swa ? 1 : 0, static_cast<float>(swa ? 0.0 : decay), static_cast<float>(swa ? 0.0 : 1.0 - decay), 0,
              scratch(n_averaged).counter + kAvgTicketWord};
    cudaStream_t st = cur_stream(n_averaged);
    for (size_t k = 0; k < tables.size(); ++k) {
      a.last = k + 1 == tables.size() ? 1 : 0;
      launch_avg_multi(tables[k], a, st);
    }
  }, py::arg("averaged"), py::arg("current"), py::arg("n_averaged"), py::arg("decay"), py::arg("copied") = std::vector<at::Tensor>{},
     py::arg("copied_from") = std::vector<at::Tensor>{});
}

}  // namespace pdt
