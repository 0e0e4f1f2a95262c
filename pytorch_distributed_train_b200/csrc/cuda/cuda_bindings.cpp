// CUDA-side bindings: GPU communicators and the sm_90a operator library.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <pybind11/stl.h>
#include <torch/extension.h>

#include <cmath>
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

// Per-device scratch for deterministic cross-CTA reductions. Kernels that use it run on one
// stream at a time (the compute stream), which is what serialises access.
struct Scratch {
  at::Tensor partials, counter;
};
ReduceScratch scratch(const at::Tensor& like) {
  static std::mutex mu;
  static auto& per_dev = *new std::map<int, Scratch>();  // leaked on purpose: CUDA tensors must not die at static teardown
  std::lock_guard<std::mutex> g(mu);
  const int dev = like.device().index();
  auto it = per_dev.find(dev);
  if (it == per_dev.end()) {
    Scratch s;
    const int64_t cap = 4 << 20;  // 4 Mi floats = 16 MiB
    s.partials = at::empty({cap}, like.options().dtype(at::kFloat));
    s.counter = at::zeros({1024}, like.options().dtype(at::kInt));
    it = per_dev.emplace(dev, std::move(s)).first;
  }
  ReduceScratch r;
  r.partials = it->second.partials.data_ptr<float>();
  r.counter = reinterpret_cast<unsigned int*>(it->second.counter.data_ptr<int>());
  r.capacity_floats = static_cast<int>(it->second.partials.numel());
  r.counters = static_cast<int>(it->second.counter.numel());
  return r;
}

// Kernel family of the per-op conv2, selected by the `impl` argument of the conv5x5_* bindings:
//   auto, tma → TMA-im2col wgmma forward / data gradient;
//   tcgen05   → the cp.async-gather wgmma kernel for forward / data gradient;
//   simt      → the CUDA-core kernels for all three.
// Both tensor-core choices compute the weight gradient with the mma.sync split-K kernel.  Shapes the tensor-core kernels
// do not cover (conv1: K = 25) always take SIMT.
enum class ConvImpl { kIm2col, kGather, kSimt };

ConvImpl conv_impl(const std::string& impl) {
  if (impl == "auto" || impl == "tma") return ConvImpl::kIm2col;
  if (impl == "tcgen05") return ConvImpl::kGather;
  TORCH_CHECK(impl == "simt", "conv5x5: impl must be one of auto, tma, tcgen05, simt (got '", impl, "')");
  return ConvImpl::kSimt;
}

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

  py::class_<NcclComm, Comm, std::shared_ptr<NcclComm>>(m, "NcclComm")
      .def(py::init([](std::shared_ptr<Store> store, int rank, int size, int device, double timeout_s) {
             py::gil_scoped_release r;
             return std::make_shared<NcclComm>(std::move(store), rank, size, device, Millis(static_cast<int64_t>(timeout_s * 1000)));
           }),
           py::arg("store"), py::arg("rank"), py::arg("size"), py::arg("device"), py::arg("timeout") = 600.0);

  // ---- convolution ---------------------------------------------------------------------------------
  m.def("conv5x5_fwd", [](const at::Tensor& x, const at::Tensor& w, c10::optional<at::Tensor> bias, bool want_stats, const std::string& impl,
                          bool zero_pad) {
    const ConvImpl family = conv_impl(impl);
    chk(x, "x"); chk(w, "w");
    c10::cuda::CUDAGuard g(x.device());
    ConvShape s = conv_shape(x, w);
    TORCH_CHECK(x.size(3) == s.Cin, "conv5x5_fwd: x channels ", x.size(3), " != weight Cin ", s.Cin);
    at::Tensor y = at::empty({s.B, s.H, s.W, s.Cout}, x.options());
    // [2C+1] statistics live in a [2C+4] vector: a 16-byte multiple goes through the vectorised one-shot allreduce
    // directly (SyncBatchNorm asks for the three pad entries to be zeroed), an odd length would bounce through a
    // padded temporary (3 extra kernels)
    at::Tensor stats_full = !want_stats ? at::Tensor() : (zero_pad ? at::zeros({2 * s.Cout + 4}, x.options()) : at::empty({2 * s.Cout + 4}, x.options()));
    at::Tensor stats = want_stats ? stats_full.narrow(0, 0, 2 * s.Cout + 1) : at::Tensor();
    const ConvImpl k = conv_wgmma_supported(s) ? family : ConvImpl::kSimt;
    auto launch = k == ConvImpl::kIm2col ? launch_conv5x5_fwd_im2col : k == ConvImpl::kGather ? launch_conv5x5_fwd_gather : launch_conv5x5_fwd;
    launch(x.data_ptr<float>(), w.data_ptr<float>(), opt_ptr(bias, "bias"), y.data_ptr<float>(), want_stats ? stats.data_ptr<float>() : nullptr, s,
           scratch(x), cur_stream(x));
    return py::make_tuple(y, stats);  // stats is a view of the first 2C+1 entries of the zero-padded vector
  }, py::arg("x"), py::arg("w"), py::arg("bias") = py::none(), py::arg("want_stats") = true, py::arg("impl") = "auto",
     py::arg("zero_pad") = false);

  m.def("conv5x5_dgrad", [](const at::Tensor& dy, const at::Tensor& w, const std::string& impl) {
    const ConvImpl family = conv_impl(impl);
    chk(dy, "dy"); chk(w, "w");
    c10::cuda::CUDAGuard g(dy.device());
    ConvShape s = conv_shape(dy, w);
    s.Cin = static_cast<int>(w.size(1));
    TORCH_CHECK(dy.size(3) == s.Cout, "conv5x5_dgrad: dy channels must equal weight Cout");
    at::Tensor dx = at::empty({s.B, s.H, s.W, s.Cin}, dy.options());
    const ConvImpl k = conv_wgmma_supported(s) ? family : ConvImpl::kSimt;
    auto launch = k == ConvImpl::kIm2col ? launch_conv5x5_dgrad_im2col : k == ConvImpl::kGather ? launch_conv5x5_dgrad_gather : launch_conv5x5_dgrad;
    launch(dy.data_ptr<float>(), w.data_ptr<float>(), dx.data_ptr<float>(), s, cur_stream(dy));
    return dx;
  }, py::arg("dy"), py::arg("w"), py::arg("impl") = "auto");

  m.def("conv5x5_wgrad", [](const at::Tensor& dy, const at::Tensor& x, at::Tensor dw, c10::optional<at::Tensor> db, const std::string& impl) {
    const ConvImpl family = conv_impl(impl);
    chk(dy, "dy"); chk(x, "x"); chk(dw, "dw");
    c10::cuda::CUDAGuard g(dy.device());
    ConvShape s = conv_shape(x, dw);
    auto launch = conv_wgmma_supported(s) && family != ConvImpl::kSimt ? launch_conv5x5_wgrad_mma : launch_conv5x5_wgrad;
    launch(dy.data_ptr<float>(), x.data_ptr<float>(), dw.data_ptr<float>(), opt_mut(db, "db"), s, scratch(x), cur_stream(x));
  }, py::arg("dy"), py::arg("x"), py::arg("dw"), py::arg("db") = py::none(), py::arg("impl") = "auto");

  // ---- cooperative fused ConvNet layers (fused_convnet.cu): one CTA per image, grid barrier for the batch statistics ----
  m.def("fused_convnet_supported", [](int64_t B) { return fused_convnet_supported(static_cast<int>(B)); });
  m.def("fused_convnet_trace_enable", [](bool on) { fused_convnet_trace_enable(on); });
  m.def("fused_convnet_trace_read", [] {
    at::Tensor t = at::zeros({4, 160, 12}, at::kLong);
    fused_convnet_trace_read(reinterpret_cast<unsigned long long*>(t.data_ptr<int64_t>()));
    return t;
  });
  m.def("convnet_l1_fwd", [](const at::Tensor& x, const at::Tensor& w, c10::optional<at::Tensor> bias, c10::optional<at::Tensor> gamma,
                             c10::optional<at::Tensor> beta, c10::optional<at::Tensor> running_mean, c10::optional<at::Tensor> running_var,
                             c10::optional<at::Tensor> nbt, double momentum, double eps) {
    chk(x, "x"); chk(w, "w");
    c10::cuda::CUDAGuard g(x.device());
    TORCH_CHECK(x.numel() % 784 == 0 && w.numel() == 400, "convnet_l1_fwd: x [B,1,28,28] and w [16,1,5,5] expected");
    const int B = static_cast<int>(x.numel() / 784);
    TORCH_CHECK(fused_convnet_supported(B), "convnet_l1_fwd: batch ", B, " exceeds one CTA per SM");
    at::Tensor y = at::empty({B, 28, 28, 16}, x.options());
    at::Tensor out = at::empty({B, 18, 18, 16}, x.options());   // zero-haloed frame
    at::Tensor saved = at::empty({32}, x.options());
    long long* nbt_p = nullptr;
    if (nbt.has_value() && nbt->defined()) { chk(*nbt, "num_batches_tracked", at::kLong); nbt_p = reinterpret_cast<long long*>(nbt->data_ptr<int64_t>()); }
    ReduceScratch scr = scratch(x);
    TORCH_CHECK(static_cast<long long>(B) * 512 <= scr.capacity_floats, "fused convnet: reduction scratch too small");
    launch_convnet_l1_fwd(x.data_ptr<float>(), w.data_ptr<float>(), opt_ptr(bias, "bias"), opt_ptr(gamma, "gamma"), opt_ptr(beta, "beta"),
                          y.data_ptr<float>(), out.data_ptr<float>(), saved.data_ptr<float>(), opt_mut(running_mean, "running_mean"),
                          opt_mut(running_var, "running_var"), nbt_p, static_cast<float>(momentum), static_cast<float>(eps), B, scr.partials,
                          GridSync{scr.counter + 512, scr.counter + 520}, cur_stream(x));
    return py::make_tuple(out, y, saved);
  });
  m.def("convnet_l1_bwd", [](const at::Tensor& dp, const at::Tensor& y, const at::Tensor& x, const at::Tensor& saved,
                             c10::optional<at::Tensor> gamma, c10::optional<at::Tensor> beta, at::Tensor dgamma, at::Tensor dbeta, at::Tensor dw,
                             c10::optional<at::Tensor> db) {
    chk(dp, "dp"); chk(y, "y"); chk(x, "x"); chk(saved, "saved"); chk(dgamma, "dgamma"); chk(dbeta, "dbeta"); chk(dw, "dw");
    c10::cuda::CUDAGuard g(x.device());
    const int B = static_cast<int>(y.size(0));
    TORCH_CHECK(dp.numel() == static_cast<int64_t>(B) * 5184 && x.numel() == static_cast<int64_t>(B) * 784 && dw.numel() == 400 &&
                    dgamma.numel() == 16 && dbeta.numel() == 16, "convnet_l1_bwd: shape mismatch");
    ReduceScratch scr = scratch(x);
    launch_convnet_l1_bwd(dp.data_ptr<float>(), y.data_ptr<float>(), x.data_ptr<float>(), saved.data_ptr<float>(), opt_ptr(gamma, "gamma"),
                          opt_ptr(beta, "beta"), dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), dw.data_ptr<float>(), opt_mut(db, "db"), B,
                          scr.partials, scr.partials + static_cast<size_t>(B) * 64,
                          GridSync{scr.counter + 512, scr.counter + 520}, cur_stream(x));
  });
  m.def("convnet_l1_bwd_wgrad", [](const at::Tensor& dp, const at::Tensor& y, const at::Tensor& x, const at::Tensor& saved,
                                   c10::optional<at::Tensor> gamma, c10::optional<at::Tensor> beta, at::Tensor dgamma, at::Tensor dbeta, at::Tensor dw,
                                   c10::optional<at::Tensor> db, const at::Tensor& dy2_pad, const at::Tensor& x2_pad, const at::Tensor& dysum2,
                                   at::Tensor dw2, c10::optional<at::Tensor> db2, py::object sgd) {
    chk(dp, "dp"); chk(y, "y"); chk(x, "x"); chk(saved, "saved"); chk(dgamma, "dgamma"); chk(dbeta, "dbeta"); chk(dw, "dw");
    chk(dy2_pad, "dy2_pad"); chk(x2_pad, "x2_pad"); chk(dysum2, "dysum2"); chk(dw2, "dw2");
    c10::cuda::CUDAGuard g(x.device());
    const int B = static_cast<int>(y.size(0));
    TORCH_CHECK(dp.numel() == static_cast<int64_t>(B) * 5184 && x.numel() == static_cast<int64_t>(B) * 784 && dw.numel() == 400 &&
                    dgamma.numel() == 16 && dbeta.numel() == 16, "convnet_l1_bwd_wgrad: layer-1 shape mismatch");
    TORCH_CHECK(dy2_pad.numel() == static_cast<int64_t>(B) * 324 * 32 && x2_pad.numel() == static_cast<int64_t>(B) * 324 * 16 &&
                    dysum2.numel() == static_cast<int64_t>(B) * 32 && dw2.numel() == 12800, "convnet_l1_bwd_wgrad: layer-2 shape mismatch");
    // sgd = (params[10], prev_grads[4], momentum_bufs[10] or [], lr, lr_tensor, momentum, dampening, weight_decay, nesterov, maximize, first_step):
    // parameters in the order conv1.w, conv1.b, bn1.w, bn1.b, conv2.w, conv2.b, fc.w, fc.b, bn2.w, bn2.b (entries may be None)
    // or the Adam rider: ("adam", params[10], prev_grads[4], exp_avgs[10], exp_avg_sqs[10], steps[10], lr, lr_tensor, beta1, beta2,
    // eps, weight_decay, decoupled, maximize), steps being fp32 scalars on the device.  Either tuple may end in a clip entry
    // (max_norm, norm_type 2 or inf, norm_out): gradient-norm clipping in front of the update (ClipRider); norm_out receives the norm.
    static const int64_t want[10] = {400, 16, 16, 16, 12800, 32, -1, -1, 32, 32};
    ReduceScratch scr = scratch(x);
    const size_t l1_floats = static_cast<size_t>(B) * (64 + 512);
    TORCH_CHECK(static_cast<long long>(l1_floats) + static_cast<long long>(B) * 512 * 32 + B <= scr.capacity_floats, "convnet_l1_bwd_wgrad: scratch too small");
    auto launch = [&](auto rider) {
      launch_convnet_l1_bwd_wgrad(dp.data_ptr<float>(), y.data_ptr<float>(), x.data_ptr<float>(), saved.data_ptr<float>(), opt_ptr(gamma, "gamma"),
                                  opt_ptr(beta, "beta"), dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), dw.data_ptr<float>(), opt_mut(db, "db"),
                                  dy2_pad.data_ptr<float>(), x2_pad.data_ptr<float>(), dysum2.data_ptr<float>(), dw2.data_ptr<float>(),
                                  opt_mut(db2, "db2"), B, scr.partials, scr.partials + static_cast<size_t>(B) * 64, scr.partials + l1_floats,
                                  GridSync{scr.counter + 512, scr.counter + 520}, cur_stream(x), rider);
    };
    // the clip entry of a rider tuple → the clipping variant of the rider
    auto clipped = [&](auto base, const py::handle& entry) {
      auto c = entry.cast<py::tuple>();
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
      r.part = scr.partials + l1_floats + static_cast<size_t>(B) * 512 * 32;
      return r;
    };
    if (!sgd.is_none() && py::isinstance<py::tuple>(sgd) && py::len(sgd) > 0 && py::isinstance<py::str>(sgd.cast<py::tuple>()[0])) {
      auto t = sgd.cast<py::tuple>();
      TORCH_CHECK((t.size() == 14 || t.size() == 15) && t[0].cast<std::string>() == "adam", "convnet_l1_bwd_wgrad: adam tuple of 14 or 15 entries expected");
      auto params = t[1].cast<std::vector<c10::optional<at::Tensor>>>();
      auto prev = t[2].cast<std::vector<c10::optional<at::Tensor>>>();
      auto ms = t[3].cast<std::vector<c10::optional<at::Tensor>>>();
      auto vs = t[4].cast<std::vector<c10::optional<at::Tensor>>>();
      auto steps = t[5].cast<std::vector<c10::optional<at::Tensor>>>();
      TORCH_CHECK(params.size() == 10 && prev.size() == 4 && ms.size() == 10 && vs.size() == 10 && steps.size() == 10,
                  "convnet_l1_bwd_wgrad: adam lists have the wrong length");
      AdamRider rider;
      for (int k = 0; k < 10; ++k) {
        if (!params[k].has_value() || !params[k]->defined()) continue;
        chk(*params[k], "adam param");
        const int64_t numel = params[k]->numel();
        TORCH_CHECK(want[k] < 0 || numel == want[k], "convnet_l1_bwd_wgrad: adam parameter ", k, " has the wrong size");
        TORCH_CHECK(ms[k].has_value() && vs[k].has_value() && steps[k].has_value(), "convnet_l1_bwd_wgrad: adam state of parameter ", k, " missing");
        chk(*ms[k], "exp_avg"); chk(*vs[k], "exp_avg_sq"); chk(*steps[k], "step");
        TORCH_CHECK(ms[k]->numel() == numel && vs[k]->numel() == numel && steps[k]->numel() == 1, "convnet_l1_bwd_wgrad: adam state of parameter ", k,
                    " has the wrong size");
        rider.p[k] = params[k]->data_ptr<float>();
        rider.m[k] = ms[k]->data_ptr<float>();
        rider.v[k] = vs[k]->data_ptr<float>();
        rider.step[k] = steps[k]->data_ptr<float>();
        if (k >= 6) {
          TORCH_CHECK(prev[k - 6].has_value() && prev[k - 6]->numel() == numel, "convnet_l1_bwd_wgrad: gradient of adam parameter ", k, " missing");
          chk(*prev[k - 6], "adam gradient");
          rider.g_prev[k - 6] = prev[k - 6]->data_ptr<float>();
          rider.n_prev[k - 6] = static_cast<int>(numel);
        }
      }
      TORCH_CHECK(rider.p[0] && rider.p[4], "convnet_l1_bwd_wgrad: the convolution weights must take part in the fused update");
      rider.h = AdamHyper{t[6].cast<double>(), t[8].cast<double>(), t[9].cast<double>(), static_cast<float>(t[10].cast<double>()),
                          static_cast<float>(t[11].cast<double>()), t[12].cast<bool>() ? 1 : 0, t[13].cast<bool>() ? 1 : 0, nullptr};
      if (!t[7].is_none()) {
        at::Tensor lrt = t[7].cast<at::Tensor>();
        chk(lrt, "lr_tensor");
        rider.h.lr_dev = lrt.data_ptr<float>();
      }
      rider.on = 1;
      if (t.size() == 15) launch(clipped(rider, t[14]));
      else launch(rider);
      return;
    }
    SgdRider rider;
    if (!sgd.is_none()) {
      auto t = sgd.cast<py::tuple>();
      TORCH_CHECK(t.size() == 11 || t.size() == 12, "convnet_l1_bwd_wgrad: sgd tuple of 11 or 12 entries expected");
      auto params = t[0].cast<std::vector<c10::optional<at::Tensor>>>();
      auto prev = t[1].cast<std::vector<c10::optional<at::Tensor>>>();
      auto bufs = t[2].cast<std::vector<c10::optional<at::Tensor>>>();
      TORCH_CHECK(params.size() == 10 && prev.size() == 4 && (bufs.empty() || bufs.size() == 10), "convnet_l1_bwd_wgrad: sgd lists have the wrong length");
      const double momentum = t[5].cast<double>();
      for (int k = 0; k < 10; ++k) {
        if (!params[k].has_value() || !params[k]->defined()) continue;
        chk(*params[k], "sgd param");
        TORCH_CHECK(want[k] < 0 || params[k]->numel() == want[k], "convnet_l1_bwd_wgrad: sgd parameter ", k, " has the wrong size");
        rider.p[k] = params[k]->data_ptr<float>();
        if (momentum != 0.0) {
          TORCH_CHECK(!bufs.empty() && bufs[k].has_value() && bufs[k]->numel() == params[k]->numel(), "convnet_l1_bwd_wgrad: momentum buffer ", k, " missing");
          chk(*bufs[k], "momentum buffer");
          rider.m[k] = bufs[k]->data_ptr<float>();
        }
        if (k >= 6) {
          TORCH_CHECK(prev[k - 6].has_value() && prev[k - 6]->numel() == params[k]->numel(), "convnet_l1_bwd_wgrad: gradient of sgd parameter ", k, " missing");
          chk(*prev[k - 6], "sgd gradient");
          rider.g_prev[k - 6] = prev[k - 6]->data_ptr<float>();
          rider.n_prev[k - 6] = static_cast<int>(params[k]->numel());
        }
      }
      TORCH_CHECK(rider.p[0] && rider.p[4], "convnet_l1_bwd_wgrad: the convolution weights must take part in the fused update");
      rider.h = SgdHyper{static_cast<float>(t[3].cast<double>()), static_cast<float>(momentum), static_cast<float>(t[6].cast<double>()),
                         static_cast<float>(t[7].cast<double>()), t[8].cast<bool>() ? 1 : 0, t[9].cast<bool>() ? 1 : 0, t[10].cast<bool>() ? 1 : 0, nullptr};
      if (!t[4].is_none()) {
        at::Tensor lrt = t[4].cast<at::Tensor>();
        chk(lrt, "lr_tensor");
        rider.h.lr_dev = lrt.data_ptr<float>();
      }
      rider.on = 1;
      if (t.size() == 12) {
        launch(clipped(rider, t[11]));
        return;
      }
    }
    launch(rider);
  }, py::arg("dp"), py::arg("y"), py::arg("x"), py::arg("saved"), py::arg("gamma"), py::arg("beta"), py::arg("dgamma"), py::arg("dbeta"),
     py::arg("dw"), py::arg("db"), py::arg("dy2_pad"), py::arg("x2_pad"), py::arg("dysum2"), py::arg("dw2"), py::arg("db2"),
     py::arg("sgd") = py::none());
  m.def("convnet_l2_fwd", [](const at::Tensor& x, const at::Tensor& w, c10::optional<at::Tensor> bias, c10::optional<at::Tensor> gamma,
                             c10::optional<at::Tensor> beta, c10::optional<at::Tensor> running_mean, c10::optional<at::Tensor> running_var,
                             c10::optional<at::Tensor> nbt, double momentum, double eps, c10::optional<at::Tensor> fcw,
                             c10::optional<at::Tensor> fcb) {
    chk(x, "x"); chk(w, "w");
    c10::cuda::CUDAGuard g(x.device());
    TORCH_CHECK(x.dim() == 4 && x.size(1) == 18 && x.size(2) == 18 && x.size(3) == 16 && w.numel() == 12800,
                "convnet_l2_fwd: x [B,18,18,16] (zero-haloed NHWC frame) and w [32,16,5,5] expected");
    const int B = static_cast<int>(x.size(0));
    TORCH_CHECK(fused_convnet_supported(B), "convnet_l2_fwd: batch ", B, " exceeds one CTA per SM");
    at::Tensor y = at::empty({B, 14, 14, 32}, x.options());
    at::Tensor out = at::empty({B, 32, 7, 7}, x.options());
    at::Tensor saved = at::empty({64}, x.options());
    at::Tensor logits;
    int ncls = 0;
    if (fcw.has_value() && fcw->defined()) {
      chk(*fcw, "fc weight");
      TORCH_CHECK(fcw->dim() == 2 && fcw->size(1) == 1568, "convnet_l2_fwd: fc weight [classes, 1568] expected");
      ncls = static_cast<int>(fcw->size(0));
      logits = at::empty({B, ncls}, x.options());
    }
    long long* nbt_p = nullptr;
    if (nbt.has_value() && nbt->defined()) { chk(*nbt, "num_batches_tracked", at::kLong); nbt_p = reinterpret_cast<long long*>(nbt->data_ptr<int64_t>()); }
    ReduceScratch scr = scratch(x);
    launch_convnet_l2_fwd(x.data_ptr<float>(), w.data_ptr<float>(), opt_ptr(bias, "bias"), opt_ptr(gamma, "gamma"), opt_ptr(beta, "beta"),
                          y.data_ptr<float>(), out.data_ptr<float>(), saved.data_ptr<float>(), opt_mut(running_mean, "running_mean"),
                          opt_mut(running_var, "running_var"), nbt_p, static_cast<float>(momentum), static_cast<float>(eps),
                          ncls ? fcw->data_ptr<float>() : nullptr, ncls ? opt_ptr(fcb, "fc bias") : nullptr,
                          ncls ? logits.data_ptr<float>() : nullptr, ncls, B, scr.partials,
                          GridSync{scr.counter + 512, scr.counter + 520}, cur_stream(x));
    return py::make_tuple(out, y, saved, logits);
  });
  m.def("convnet_fwd", [](const at::Tensor& x, const at::Tensor& w1, c10::optional<at::Tensor> b1, c10::optional<at::Tensor> g1,
                          c10::optional<at::Tensor> be1, c10::optional<at::Tensor> rm1, c10::optional<at::Tensor> rv1, c10::optional<at::Tensor> nbt1,
                          double mom1, double eps1, const at::Tensor& w2, c10::optional<at::Tensor> b2, c10::optional<at::Tensor> g2,
                          c10::optional<at::Tensor> be2, c10::optional<at::Tensor> rm2, c10::optional<at::Tensor> rv2, c10::optional<at::Tensor> nbt2,
                          double mom2, double eps2, const at::Tensor& fcw, c10::optional<at::Tensor> fcb, c10::optional<at::Tensor> target,
                          bool defer_loss_mean) {
    chk(x, "x"); chk(w1, "w1"); chk(w2, "w2"); chk(fcw, "fc weight");
    c10::cuda::CUDAGuard g(x.device());
    TORCH_CHECK(x.numel() % 784 == 0 && w1.numel() == 400 && w2.numel() == 12800 && fcw.dim() == 2 && fcw.size(1) == 1568 && fcw.size(0) <= 16,
                "convnet_fwd: x [B,1,28,28], w1 [16,1,5,5], w2 [32,16,5,5], fc weight [<=16, 1568] expected");
    const int B = static_cast<int>(x.numel() / 784), ncls = static_cast<int>(fcw.size(0));
    TORCH_CHECK(fused_convnet_supported(B), "convnet_fwd: batch ", B, " exceeds one CTA per SM");
    at::Tensor y1 = at::empty({B, 28, 28, 16}, x.options()), p1 = at::empty({B, 18, 18, 16}, x.options()), saved1 = at::empty({32}, x.options());
    at::Tensor y2 = at::empty({B, 14, 14, 32}, x.options()), out = at::empty({B, 32, 7, 7}, x.options()), saved2 = at::empty({64}, x.options());
    at::Tensor logits = at::empty({B, ncls}, x.options());
    auto nbt_ptr = [](c10::optional<at::Tensor>& t) -> long long* {
      if (!t.has_value() || !t->defined()) return nullptr;
      chk(*t, "num_batches_tracked", at::kLong);
      return reinterpret_cast<long long*>(t->data_ptr<int64_t>());
    };
    ReduceScratch scr = scratch(x);
    FusedCe ce;
    at::Tensor loss, dlogits, loss_parts;
    if (target.has_value() && target->defined()) {
      chk(*target, "target", at::kLong);
      TORCH_CHECK(target->numel() == B, "convnet_fwd: one target per image expected");
      loss = at::empty({}, x.options());
      dlogits = at::empty({B, ncls}, x.options());
      loss_parts = at::empty({B}, x.options());
      ce.target = reinterpret_cast<const long long*>(target->data_ptr<int64_t>());
      ce.loss_parts = loss_parts.data_ptr<float>();
      ce.loss = defer_loss_mean ? nullptr : loss.data_ptr<float>();   // deferred: convnet_l2_bwd_fc(…, loss_parts, loss) writes it
      ce.dlogits = dlogits.data_ptr<float>();
      ce.counter = scr.counter + 528;
    }
    launch_convnet_fwd(x.data_ptr<float>(), w1.data_ptr<float>(), opt_ptr(b1, "b1"), opt_ptr(g1, "g1"), opt_ptr(be1, "be1"), y1.data_ptr<float>(),
                       p1.data_ptr<float>(), saved1.data_ptr<float>(), opt_mut(rm1, "rm1"), opt_mut(rv1, "rv1"), nbt_ptr(nbt1), static_cast<float>(mom1),
                       static_cast<float>(eps1), w2.data_ptr<float>(), opt_ptr(b2, "b2"), opt_ptr(g2, "g2"), opt_ptr(be2, "be2"), y2.data_ptr<float>(),
                       out.data_ptr<float>(), saved2.data_ptr<float>(), opt_mut(rm2, "rm2"), opt_mut(rv2, "rv2"), nbt_ptr(nbt2), static_cast<float>(mom2),
                       static_cast<float>(eps2), fcw.data_ptr<float>(), opt_ptr(fcb, "fc bias"), logits.data_ptr<float>(), ncls, B, scr.partials,
                       GridSync{scr.counter + 512, scr.counter + 520}, cur_stream(x), ce);
    return py::make_tuple(p1, y1, saved1, out, y2, saved2, logits, loss, dlogits, loss_parts);
  }, py::arg("x"), py::arg("w1"), py::arg("b1"), py::arg("g1"), py::arg("be1"), py::arg("rm1"), py::arg("rv1"), py::arg("nbt1"), py::arg("mom1"),
     py::arg("eps1"), py::arg("w2"), py::arg("b2"), py::arg("g2"), py::arg("be2"), py::arg("rm2"), py::arg("rv2"), py::arg("nbt2"), py::arg("mom2"),
     py::arg("eps2"), py::arg("fcw"), py::arg("fcb"), py::arg("target") = py::none(), py::arg("defer_loss_mean") = false);
  m.def("convnet_l2_bwd", [](const at::Tensor& dout, const at::Tensor& y, const at::Tensor& saved, c10::optional<at::Tensor> gamma,
                             c10::optional<at::Tensor> beta, const at::Tensor& w, at::Tensor dgamma, at::Tensor dbeta) {
    chk(dout, "dout"); chk(y, "y"); chk(saved, "saved"); chk(w, "w"); chk(dgamma, "dgamma"); chk(dbeta, "dbeta");
    c10::cuda::CUDAGuard g(y.device());
    const int B = static_cast<int>(y.size(0));
    TORCH_CHECK(dout.numel() == static_cast<int64_t>(B) * 1568 && y.numel() == static_cast<int64_t>(B) * 6272 && w.numel() == 12800 &&
                    dgamma.numel() == 32 && dbeta.numel() == 32, "convnet_l2_bwd: shape mismatch");
    at::Tensor dy = at::empty({B, 18, 18, 32}, y.options());
    at::Tensor dx = at::empty({B, 18, 18, 16}, y.options());
    at::Tensor dysum = at::empty({B, 32}, y.options());
    ReduceScratch scr = scratch(y);
    launch_convnet_l2_bwd(dout.data_ptr<float>(), y.data_ptr<float>(), saved.data_ptr<float>(), opt_ptr(gamma, "gamma"), opt_ptr(beta, "beta"),
                          w.data_ptr<float>(), dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), dy.data_ptr<float>(), dx.data_ptr<float>(),
                          dysum.data_ptr<float>(), B, scr.partials, GridSync{scr.counter + 512, scr.counter + 520},
                          cur_stream(y));
    return py::make_tuple(dy, dx, dysum);
  });
  m.def("convnet_l2_bwd_fc", [](const at::Tensor& dlogits, const at::Tensor& fcw, const at::Tensor& pooled, at::Tensor dfcw, c10::optional<at::Tensor> dfcb,
                                const at::Tensor& y, const at::Tensor& saved, c10::optional<at::Tensor> gamma, c10::optional<at::Tensor> beta,
                                const at::Tensor& w, at::Tensor dgamma, at::Tensor dbeta, c10::optional<at::Tensor> loss_parts,
                                c10::optional<at::Tensor> loss_out) {
    chk(dlogits, "dlogits"); chk(fcw, "fc weight"); chk(pooled, "pooled"); chk(dfcw, "dfcw");
    chk(y, "y"); chk(saved, "saved"); chk(w, "w"); chk(dgamma, "dgamma"); chk(dbeta, "dbeta");
    c10::cuda::CUDAGuard g(y.device());
    const int B = static_cast<int>(y.size(0));
    const int ncls = static_cast<int>(fcw.size(0));
    TORCH_CHECK(fcw.dim() == 2 && fcw.size(1) == 1568 && ncls <= 16 && dlogits.numel() == static_cast<int64_t>(B) * ncls &&
                    pooled.numel() == static_cast<int64_t>(B) * 1568 && dfcw.numel() == fcw.numel() && y.numel() == static_cast<int64_t>(B) * 6272 &&
                    w.numel() == 12800 && dgamma.numel() == 32 && dbeta.numel() == 32, "convnet_l2_bwd_fc: shape mismatch");
    TORCH_CHECK(reinterpret_cast<uintptr_t>(fcw.data_ptr()) % 16 == 0, "convnet_l2_bwd_fc: fc weight must be 16-byte aligned");
    at::Tensor dy = at::empty({B, 18, 18, 32}, y.options());
    at::Tensor dx = at::empty({B, 18, 18, 16}, y.options());
    at::Tensor dysum = at::empty({B, 32}, y.options());
    ReduceScratch scr = scratch(y);
    launch_convnet_l2_bwd_fc(dlogits.data_ptr<float>(), fcw.data_ptr<float>(), pooled.data_ptr<float>(), dfcw.data_ptr<float>(), opt_mut(dfcb, "dfcb"),
                             ncls, y.data_ptr<float>(), saved.data_ptr<float>(), opt_ptr(gamma, "gamma"), opt_ptr(beta, "beta"), w.data_ptr<float>(),
                             dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), dy.data_ptr<float>(), dx.data_ptr<float>(), dysum.data_ptr<float>(), B,
                             scr.partials, GridSync{scr.counter + 512, scr.counter + 520}, cur_stream(y), opt_ptr(loss_parts, "loss_parts"),
                             opt_mut(loss_out, "loss_out"));
    return py::make_tuple(dy, dx, dysum);
  }, py::arg("dlogits"), py::arg("fcw"), py::arg("pooled"), py::arg("dfcw"), py::arg("dfcb"), py::arg("y"), py::arg("saved"), py::arg("gamma"),
     py::arg("beta"), py::arg("w"), py::arg("dgamma"), py::arg("dbeta"), py::arg("loss_parts") = py::none(), py::arg("loss_out") = py::none());
  m.def("conv5x5_wgrad_win", [](const at::Tensor& dy_pad, const at::Tensor& x_pad, const at::Tensor& dysum, at::Tensor dw, c10::optional<at::Tensor> db) {
    chk(dy_pad, "dy_pad"); chk(x_pad, "x_pad"); chk(dysum, "dysum"); chk(dw, "dw");
    c10::cuda::CUDAGuard g(dy_pad.device());
    const int B = static_cast<int>(dy_pad.size(0));
    TORCH_CHECK(dy_pad.numel() == static_cast<int64_t>(B) * 324 * 32 && x_pad.numel() == static_cast<int64_t>(B) * 324 * 16 &&
                    dysum.numel() == static_cast<int64_t>(B) * 32 && dw.numel() == 12800, "conv5x5_wgrad_win: shape mismatch");
    ReduceScratch scr = scratch(dy_pad);
    launch_conv5x5_wgrad_win(dy_pad.data_ptr<float>(), x_pad.data_ptr<float>(), dysum.data_ptr<float>(), dw.data_ptr<float>(), opt_mut(db, "db"), B,
                             scr, cur_stream(dy_pad), GridSync{scr.counter + 512, scr.counter + 520});
  }, py::arg("dy_pad"), py::arg("x_pad"), py::arg("dysum"), py::arg("dw"), py::arg("db") = py::none());

  // ---- BN + ReLU + pool ------------------------------------------------------------------------------
  m.def("bn_relu_pool_fwd", [](const at::Tensor& y, const at::Tensor& stats, c10::optional<at::Tensor> gamma, c10::optional<at::Tensor> beta,
                               c10::optional<at::Tensor> running_mean, c10::optional<at::Tensor> running_var,
                               c10::optional<at::Tensor> nbt, double momentum, double eps, bool out_nchw) {
    chk(y, "y"); chk(stats, "stats");
    c10::cuda::CUDAGuard g(y.device());
    const int B = y.size(0), H = y.size(1), W = y.size(2), C = y.size(3);
    TORCH_CHECK(stats.numel() == 2 * C + 1, "bn_relu_pool_fwd: stats must have 2C+1 entries");
    at::Tensor out = out_nchw ? at::empty({B, C, H / 2, W / 2}, y.options()) : at::empty({B, H / 2, W / 2, C}, y.options());
    at::Tensor saved = at::empty({2 * C}, y.options());
    long long* nbt_p = nullptr;
    if (nbt.has_value() && nbt->defined()) { chk(*nbt, "num_batches_tracked", at::kLong); nbt_p = reinterpret_cast<long long*>(nbt->data_ptr<int64_t>()); }
    launch_bn_relu_pool_fwd(y.data_ptr<float>(), stats.data_ptr<float>(), opt_ptr(gamma, "gamma"), opt_ptr(beta, "beta"), out.data_ptr<float>(),
                            saved.data_ptr<float>(), opt_mut(running_mean, "running_mean"), opt_mut(running_var, "running_var"), nbt_p,
                            static_cast<float>(momentum), static_cast<float>(eps), B, H, W, C, out_nchw, cur_stream(y));
    return py::make_tuple(out, saved);
  });
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
  m.def("bn_relu_pool_bwd_apply", [](const at::Tensor& dout, const at::Tensor& y, const at::Tensor& saved, c10::optional<at::Tensor> gamma,
                                     c10::optional<at::Tensor> beta, const at::Tensor& sums, const at::Tensor& count, bool dout_nchw) {
    chk(dout, "dout"); chk(y, "y"); chk(saved, "saved"); chk(sums, "sums"); chk(count, "count");
    c10::cuda::CUDAGuard g(y.device());
    const int B = y.size(0), H = y.size(1), W = y.size(2), C = y.size(3);
    at::Tensor dy = at::empty_like(y);
    launch_bn_relu_pool_bwd_apply(dout.data_ptr<float>(), y.data_ptr<float>(), saved.data_ptr<float>(), opt_ptr(gamma, "gamma"),
                                  opt_ptr(beta, "beta"), sums.data_ptr<float>(), count.data_ptr<float>(), dy.data_ptr<float>(), B, H, W, C,
                                  dout_nchw, cur_stream(y));
    return dy;
  });

  // ---- generic NCHW BatchNorm (SyncBatchNorm) ----------------------------------------------------------
  m.def("bn_stats_nchw", [](const at::Tensor& x) {
    chk(x, "x");
    TORCH_CHECK(x.dim() >= 2, "bn_stats: at least 2-D input");
    c10::cuda::CUDAGuard g(x.device());
    const int N = x.size(0), C = x.size(1);
    const int HW = static_cast<int>(x.numel() / std::max<int64_t>(1, static_cast<int64_t>(N) * C));
    at::Tensor stats = at::zeros({2 * C + 1}, x.options());
    if (x.numel() > 0) launch_bn_stats_nchw(x.data_ptr<float>(), stats.data_ptr<float>(), N, C, HW, scratch(x), cur_stream(x));
    return stats;
  });
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
  m.def("cross_entropy_fwd", [](const at::Tensor& logits, const at::Tensor& target, bool emit_grad) {
    chk(logits, "logits"); chk(target, "target", at::kLong);
    c10::cuda::CUDAGuard g(logits.device());
    at::Tensor loss = at::empty({}, logits.options()), probs = at::empty_like(logits);
    launch_cross_entropy_fwd(logits.data_ptr<float>(), reinterpret_cast<const long long*>(target.data_ptr<int64_t>()), loss.data_ptr<float>(),
                             probs.data_ptr<float>(), logits.size(0), logits.size(1), cur_stream(logits), emit_grad);
    return py::make_tuple(loss, probs);  // emit_grad: the second tensor is d(loss)/d(logits) for a unit incoming gradient
  }, py::arg("logits"), py::arg("target"), py::arg("emit_grad") = false);
  m.def("cross_entropy_bwd", [](const at::Tensor& probs, const at::Tensor& target, const at::Tensor& dloss) {
    chk(probs, "probs"); chk(target, "target", at::kLong); chk(dloss, "dloss");
    c10::cuda::CUDAGuard g(probs.device());
    at::Tensor d = at::empty_like(probs);
    launch_cross_entropy_bwd(probs.data_ptr<float>(), reinterpret_cast<const long long*>(target.data_ptr<int64_t>()), dloss.data_ptr<float>(),
                             d.data_ptr<float>(), probs.size(0), probs.size(1), cur_stream(probs));
    return d;
  });

  // ---- optimizer ------------------------------------------------------------------------------------------
  m.def("sgd_multi", [](std::vector<at::Tensor> params, std::vector<at::Tensor> grads, std::vector<at::Tensor> bufs, double lr,
                        c10::optional<at::Tensor> lr_tensor, double momentum, double dampening, double weight_decay, bool nesterov,
                        bool maximize, bool first_step) {
    TORCH_CHECK(params.size() == grads.size(), "sgd_multi: params/grads length mismatch");
    TORCH_CHECK(momentum == 0.0 || bufs.size() == params.size(), "sgd_multi: momentum buffers required");
    if (params.empty()) return;
    c10::cuda::CUDAGuard g(params[0].device());
    SgdHyper h{static_cast<float>(lr), static_cast<float>(momentum), static_cast<float>(dampening), static_cast<float>(weight_decay),
               nesterov ? 1 : 0, maximize ? 1 : 0, first_step ? 1 : 0, nullptr};
    if (lr_tensor.has_value() && lr_tensor->defined()) { chk(*lr_tensor, "lr_tensor"); h.lr_dev = lr_tensor->data_ptr<float>(); }
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
                         double beta1, double beta2, double eps, double weight_decay, bool decoupled, bool maximize) {
    const size_t n = params.size();
    TORCH_CHECK(grads.size() == n && exp_avgs.size() == n && exp_avg_sqs.size() == n && steps.size() == n, "adam_multi: list lengths differ");
    if (n == 0) return;
    c10::cuda::CUDAGuard g(params[0].device());
    AdamHyper h{lr, beta1, beta2, static_cast<float>(eps), static_cast<float>(weight_decay), decoupled ? 1 : 0, maximize ? 1 : 0, nullptr};
    if (lr_tensor.has_value() && lr_tensor->defined()) { chk(*lr_tensor, "lr_tensor"); h.lr_dev = lr_tensor->data_ptr<float>(); }
    cudaStream_t st = cur_stream(params[0]);
    // the ticket word of the step hand-over (adam_multi_kernel); launches on one device are ordered by the compute stream, and
    // every launch leaves the word at zero
    unsigned int* ticket = scratch(params[0]).counter + 536;
    for (size_t base = 0; base < n; base += AdamTensorList::kMax) {
      AdamTensorList tl;
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
      }
      launch_adam_multi(tl, h, ticket, st);
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
                   scr.counter + 544};
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

  // ---- TF32 wgmma GEMM self-test (D[M,N] = A[M,K]·B[N,K]^T) — validates descriptors/TMA/accumulator layout ---
  m.def("gemm_tf32_wgmma", [](const at::Tensor& a, const at::Tensor& b) {
    chk(a, "a"); chk(b, "b");
    c10::cuda::CUDAGuard g(a.device());
    TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && a.size(1) == b.size(1), "gemm_tf32: A [M,K], B [N,K]");
    at::Tensor d = at::empty({a.size(0), b.size(0)}, a.options());
    launch_gemm_tf32_wgmma(a.data_ptr<float>(), b.data_ptr<float>(), d.data_ptr<float>(), a.size(0), b.size(0), a.size(1), cur_stream(a));
    return d;
  });
}

}  // namespace pdt
