// Python bindings for the native runtime (module pytorch_distributed_train_b200._C).
#include <pybind11/chrono.h>
#include <pybind11/functional.h>
#include <pybind11/stl.h>
#include <torch/extension.h>

#include "comm/comm.h"
#include "data/batch_loader.h"
#include "engine/step_pipeline.h"
#include "common/net.h"
#include "reducer/bucket_plan.h"
#include "reducer/reducer.h"
#include "store/store.h"

namespace py = pybind11;
using namespace pdt;

namespace pdt {
void register_cuda_bindings(py::module_& m);  // csrc/cuda/cuda_bindings.cpp
}

namespace {

using NoGil = py::call_guard<py::gil_scoped_release>;

Millis ms(double seconds) { return Millis(static_cast<int64_t>(seconds * 1000.0)); }

template <typename S, typename... Extra>
py::class_<S, Store, std::shared_ptr<S>> bind_store(py::module_& m, const char* name, Extra&&... extra) {
  return py::class_<S, Store, std::shared_ptr<S>>(m, name, std::forward<Extra>(extra)...);
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "pytorch_distributed_train_b200 native runtime: stores, CPU/NVLink/NCCL collectives, reducer, sm_90a ops";

  py::register_exception<TimeoutError>(m, "TimeoutError", PyExc_TimeoutError);
  py::register_exception<PeerClosedError>(m, "PeerClosedError", PyExc_ConnectionError);

  // ---- stores --------------------------------------------------------------------------
  py::class_<Store, std::shared_ptr<Store>>(m, "Store")
      .def("set", [](Store& s, const std::string& k, const py::bytes& v) { std::string val = v; py::gil_scoped_release r; s.set(k, val); })
      .def("set", [](Store& s, const std::string& k, const std::string& v) { py::gil_scoped_release r; s.set(k, v); })
      .def("get", [](Store& s, const std::string& k) { std::string v; { py::gil_scoped_release r; v = s.get(k); } return py::bytes(v); })
      .def("add", &Store::add, NoGil())
      .def("compare_set", [](Store& s, const std::string& k, const std::string& e, const std::string& d) {
        std::string v; { py::gil_scoped_release r; v = s.compare_set(k, e, d); } return py::bytes(v); })
      .def("wait", [](Store& s, const std::vector<std::string>& keys) { py::gil_scoped_release r; s.wait(keys); })
      .def("wait", [](Store& s, const std::vector<std::string>& keys, double timeout_s) { py::gil_scoped_release r; s.wait(keys, ms(timeout_s)); })
      .def("check", &Store::check, NoGil())
      .def("delete_key", &Store::delete_key, NoGil())
      .def("num_keys", &Store::num_keys, NoGil())
      .def("append", [](Store& s, const std::string& k, const std::string& v) { py::gil_scoped_release r; s.append(k, v); })
      .def("multi_get", [](Store& s, const std::vector<std::string>& keys) {
        std::vector<std::string> v; { py::gil_scoped_release r; v = s.multi_get(keys); }
        py::list out; for (auto& x : v) out.append(py::bytes(x)); return out; })
      .def("multi_set", [](Store& s, const std::vector<std::string>& keys, const std::vector<std::string>& vals) { py::gil_scoped_release r; s.multi_set(keys, vals); })
      .def("queue_push", [](Store& s, const std::string& k, const std::string& v) { py::gil_scoped_release r; s.queue_push(k, v); })
      .def("queue_pop", [](Store& s, const std::string& k, bool block) { std::string v; { py::gil_scoped_release r; v = s.queue_pop(k, block); } return py::bytes(v); },
           py::arg("key"), py::arg("block") = true)
      .def("queue_len", &Store::queue_len, NoGil())
      .def("set_timeout", [](Store& s, double seconds) { s.set_timeout(ms(seconds)); })
      .def_property_readonly("timeout", [](Store& s) { return static_cast<double>(s.timeout().count()) / 1000.0; });

  bind_store<HashStore>(m, "HashStore").def(py::init<>());
  bind_store<FileStore>(m, "FileStore")
      .def(py::init<std::string, int>(), py::arg("path"), py::arg("world_size") = -1)
      .def_property_readonly("path", &FileStore::path);
  bind_store<PrefixStore>(m, "PrefixStore")
      .def(py::init<std::string, std::shared_ptr<Store>>(), py::arg("prefix"), py::arg("store"))
      .def_property_readonly("prefix", &PrefixStore::prefix)
      .def_property_readonly("underlying_store", &PrefixStore::underlying);
  bind_store<TCPStore>(m, "TCPStore")
      .def(py::init([](const std::string& host, int port, int world_size, bool is_master, double timeout_s, bool wait_for_workers) {
             py::gil_scoped_release r;
             return std::make_shared<TCPStore>(host, port, world_size, is_master, ms(timeout_s), wait_for_workers);
           }),
           py::arg("host_name"), py::arg("port"), py::arg("world_size") = -1, py::arg("is_master") = false,
           py::arg("timeout") = 300.0, py::arg("wait_for_workers") = true)
      .def("ping", &TCPStore::ping, NoGil())
      .def_property_readonly("port", &TCPStore::port)
      .def_property_readonly("host", &TCPStore::host)
      .def_property_readonly("is_master", &TCPStore::is_master);

  m.def("store_barrier", [](std::shared_ptr<Store> s, const std::string& name, int rank, int world, double timeout_s) {
    py::gil_scoped_release r;
    store_barrier(*s, name, rank, world, ms(timeout_s));
  });

  // ---- fd passing (used to ship CUDA VMM handles between the per-GPU processes) ---------
  m.def("unix_listen", [](const std::string& name) { return unix_listen(name).release(); });
  m.def("unix_connect", [](const std::string& name, double timeout_s) { py::gil_scoped_release r; return unix_connect(name, ms(timeout_s)).release(); });
  m.def("unix_accept", [](int lfd, double timeout_s) { py::gil_scoped_release r; return tcp_accept(lfd, ms(timeout_s)).release(); });
  m.def("send_fd", [](int sock, int fd, double timeout_s) { py::gil_scoped_release r; send_fd(sock, fd, ms(timeout_s)); });
  m.def("recv_fd", [](int sock, double timeout_s) { py::gil_scoped_release r; return recv_fd(sock, ms(timeout_s)); });

  // ---- collectives ---------------------------------------------------------------------
  py::enum_<ReduceOp>(m, "ReduceOp")
      .value("SUM", ReduceOp::SUM).value("AVG", ReduceOp::AVG).value("PRODUCT", ReduceOp::PRODUCT)
      .value("MIN", ReduceOp::MIN).value("MAX", ReduceOp::MAX).value("BAND", ReduceOp::BAND)
      .value("BOR", ReduceOp::BOR).value("BXOR", ReduceOp::BXOR);

  py::class_<CommWork, std::shared_ptr<CommWork>>(m, "Work")
      .def("wait", [](CommWork& w) { py::gil_scoped_release r; w.wait(); return true; })
      .def("synchronize", &CommWork::synchronize, NoGil())
      .def("is_completed", &CommWork::is_completed);

  py::class_<Comm, std::shared_ptr<Comm>>(m, "Comm")
      .def_property_readonly("rank", &Comm::rank)
      .def_property_readonly("size", &Comm::size)
      .def_property_readonly("backend_name", &Comm::backend_name)
      .def_property_readonly("is_cuda", &Comm::is_cuda)
      .def("alloc_flat", [](Comm& c, int64_t numel, py::object dtype, py::object device) {
        return c.alloc_flat(numel, torch::python::detail::py_object_to_dtype(dtype), torch::python::detail::py_object_to_device(device));
      })
      .def("allreduce", &Comm::allreduce, py::arg("tensor"), py::arg("op") = ReduceOp::SUM, py::arg("postscale") = 1.0, NoGil())
      .def("broadcast", &Comm::broadcast, py::arg("tensor"), py::arg("root"), NoGil())
      .def("allgather", &Comm::allgather, py::arg("output"), py::arg("input"), NoGil())
      .def("reduce", &Comm::reduce, py::arg("tensor"), py::arg("op"), py::arg("root"), NoGil())
      .def("reduce_scatter", &Comm::reduce_scatter, py::arg("output"), py::arg("input"), py::arg("op") = ReduceOp::SUM, NoGil())
      .def("gather", &Comm::gather, py::arg("output"), py::arg("input"), py::arg("root"), NoGil())
      .def("scatter", &Comm::scatter, py::arg("output"), py::arg("input"), py::arg("root"), NoGil())
      .def("alltoall", &Comm::alltoall, py::arg("output"), py::arg("input"), NoGil())
      .def("send", &Comm::send, py::arg("tensor"), py::arg("dst"), NoGil())
      .def("recv", &Comm::recv, py::arg("tensor"), py::arg("src"), NoGil())
      .def("barrier", &Comm::barrier, NoGil())
      .def("shutdown", &Comm::shutdown, NoGil())
      .def("flight_records", [](Comm& c) {
        py::list out;
        for (auto& r : c.flight_records()) {
          py::dict d;
          d["seq"] = r.seq; d["op"] = r.op; d["numel"] = r.numel; d["dtype"] = r.dtype; d["t_enqueue"] = r.t_enqueue;
          out.append(d);
        }
        return out;
      });

  py::class_<CpuComm, Comm, std::shared_ptr<CpuComm>>(m, "CpuComm")
      .def(py::init([](std::shared_ptr<Store> store, int rank, int size, double timeout_s, const std::string& bind_host) {
             py::gil_scoped_release r;
             return std::make_shared<CpuComm>(std::move(store), rank, size, ms(timeout_s), bind_host);
           }),
           py::arg("store"), py::arg("rank"), py::arg("size"), py::arg("timeout") = 1800.0, py::arg("bind_host") = "127.0.0.1")
      .def("inject_delay", [](CpuComm& c, int n, int msec) { c.backend().inject_delay(n, msec); })
      .def("inject_skip", [](CpuComm& c, int n) { c.backend().inject_skip(n); })
      .def("ops_completed", [](CpuComm& c) { return c.backend().ops_completed(); });

  // ---- bucket planner + reducer ----------------------------------------------------------
  m.def("plan_buckets",
        [](const std::vector<int64_t>& nbytes, const std::vector<int64_t>& group_keys, const std::vector<int64_t>& limits,
           const std::vector<int64_t>& order) {
          TORCH_CHECK(nbytes.size() == group_keys.size(), "plan_buckets: nbytes/group_keys length mismatch");
          std::vector<PlanInput> in;
          for (size_t i = 0; i < nbytes.size(); ++i) in.push_back({nbytes[i], group_keys[i]});
          auto r = plan_buckets(in, limits, order);
          return py::make_tuple(r.buckets, r.size_limits);
        },
        py::arg("nbytes"), py::arg("group_keys"), py::arg("size_limits"), py::arg("order") = std::vector<int64_t>{});

  py::class_<GradBucket>(m, "GradBucket")
      .def("index", [](GradBucket& b) { return b.index; })
      .def("is_last", [](GradBucket& b) { return b.is_last; })
      .def("buffer", [](GradBucket& b) { return b.buffer; })
      .def("set_buffer", [](GradBucket& b, at::Tensor t) { b.buffer = std::move(t); })
      .def("gradients", [](GradBucket& b) { return b.gradients; })
      .def("parameters", [](GradBucket& b) { return b.parameters; })
      .def("offsets", [](GradBucket& b) { return b.offsets; })
      .def("lengths", [](GradBucket& b) { return b.lengths; });

  py::class_<BatchStager, std::shared_ptr<BatchStager>>(m, "BatchStager")
      .def(py::init<at::Tensor, at::Tensor, std::vector<int64_t>, int64_t, bool, double, int64_t, bool, int>(), py::arg("data"), py::arg("targets"),
           py::arg("sample_shape"), py::arg("batch_size"), py::arg("drop_last") = false, py::arg("scale") = 1.0, py::arg("depth") = 8,
           py::arg("pin_memory") = false, py::arg("device") = -1)
      .def("start", &BatchStager::start, py::arg("indices"))
      .def("num_batches", &BatchStager::num_batches)
      .def("stats", &BatchStager::stats)
      .def("next", [](BatchStager& s) -> py::object {
        at::Tensor images, targets;
        bool ok;
        {
          py::gil_scoped_release r;   // the worker thread may still be staging this batch
          ok = s.next(&images, &targets);
        }
        if (!ok) return py::none();
        return py::make_tuple(images, targets);
      });

  py::class_<StepPipeline, std::shared_ptr<StepPipeline>>(m, "StepPipeline")
      .def(py::init([](int device, int num_sets, const at::Tensor& loss_like) {
             return std::make_shared<StepPipeline>(device, num_sets, loss_like.scalar_type());
           }), py::arg("device"), py::arg("num_sets"), py::arg("loss_like"))
      .def("stage_inputs", &StepPipeline::stage_inputs, py::arg("set"), py::arg("dst"), py::arg("src"), py::arg("inputs_ready") = false,
           py::arg("overlap") = true)
      .def("replayed", &StepPipeline::replayed)
      .def("loss_to_host", &StepPipeline::loss_to_host)
      .def("loss_value", [](StepPipeline& p, int64_t gen) {
        py::gil_scoped_release r;
        return p.loss_value(gen);
      });

  py::class_<Reducer, std::shared_ptr<Reducer>>(m, "Reducer")
      .def(py::init<std::vector<at::Tensor>, std::vector<std::vector<int64_t>>, std::shared_ptr<Comm>, int64_t, int64_t, bool, bool, bool>(),
           py::arg("params"), py::arg("bucket_indices"), py::arg("comm"), py::arg("bucket_bytes_cap") = 25 * 1024 * 1024,
           py::arg("first_bucket_bytes_cap") = 1024 * 1024, py::arg("find_unused_parameters") = false,
           py::arg("gradient_as_bucket_view") = true, py::arg("static_graph") = false)
      .def("prepare_for_forward", &Reducer::prepare_for_forward)
      .def("prepare_for_backward", &Reducer::prepare_for_backward, py::arg("outputs") = std::vector<at::Tensor>{})
      .def("set_require_sync", &Reducer::set_require_sync)
      .def("should_rebuild", &Reducer::should_rebuild)
      .def("propose_rebuild", &Reducer::propose_rebuild)
      .def("apply_rebuild", &Reducer::apply_rebuild)
      .def("register_comm_hook", &Reducer::register_comm_hook)
      .def("bucket_buffers", &Reducer::bucket_buffers)
      .def("grad_views", &Reducer::grad_views)
      .def("grads_are_views", &Reducer::grads_are_views)
      .def("install_grad_views", &Reducer::install_grad_views, py::arg("zero") = true)
      .def("set_postscale", &Reducer::set_postscale)
      .def("set_defer_comm", &Reducer::set_defer_comm)
      .def_property_readonly("defer_comm", &Reducer::defer_comm)
      .def("set_chunking", &Reducer::set_chunking, py::arg("min_chunk_bytes"), py::arg("max_chunks"))
      .def("set_fused_sgd",
           [](Reducer& r, c10::optional<at::Tensor> param_flat, c10::optional<at::Tensor> momentum_flat, double lr,
              c10::optional<at::Tensor> lr_tensor, double momentum, double dampening, double weight_decay, bool nesterov, bool first_step,
              c10::optional<at::Tensor> bcast, int64_t bcast_root) {
             FusedSgd h;
             h.lr = lr; h.momentum = momentum; h.dampening = dampening; h.weight_decay = weight_decay;
             h.nesterov = nesterov; h.first_step = first_step;
             if (lr_tensor.has_value()) h.lr_tensor = *lr_tensor;
             r.set_fused_sgd(param_flat.value_or(at::Tensor()), momentum_flat.value_or(at::Tensor()), h, bcast.value_or(at::Tensor()), bcast_root);
           },
           py::arg("param_flat"), py::arg("momentum_flat") = py::none(), py::arg("lr") = 0.0, py::arg("lr_tensor") = py::none(),
           py::arg("momentum") = 0.0, py::arg("dampening") = 0.0, py::arg("weight_decay") = 0.0, py::arg("nesterov") = false,
           py::arg("first_step") = false, py::arg("bcast") = py::none(), py::arg("bcast_root") = 0)
      .def_property_readonly("fused_sgd", &Reducer::fused_sgd)
      .def("stats", [](Reducer& r) {
        ReducerStats s = r.stats();
        py::dict d;
        d["num_iterations"] = s.num_iterations;
        d["num_buckets_reduced"] = s.num_buckets_reduced;
        d["num_rebuilds"] = s.num_rebuilds;
        d["bucket_sizes"] = s.bucket_sizes_bytes;
        d["bucket_indices"] = s.bucket_indices;
        d["grad_ready_order"] = s.grad_ready_order;
        d["forward_us"] = s.forward_us;
        d["backward_compute_us"] = s.backward_compute_us;
        d["backward_comm_us"] = s.backward_comm_us;
        d["backward_comm_exposed_us"] = s.backward_comm_exposed_us;
        d["backward_total_us"] = s.backward_total_us;
        d["reduce_chunks"] = s.reduce_chunks;
        d["timed_iterations"] = s.timed_iterations;
        d["avg_forward_compute_time_us"] = s.avg_forward_us;
        d["avg_backward_compute_time_us"] = s.avg_backward_compute_us;
        d["avg_backward_comm_time_us"] = s.avg_backward_comm_us;
        d["avg_backward_comm_exposed_time_us"] = s.avg_backward_comm_exposed_us;
        d["has_rebuilt_buckets"] = s.has_rebuilt;
        d["gradient_as_bucket_view"] = s.gradient_as_bucket_view;
        d["find_unused_parameters"] = s.find_unused_parameters;
        d["total_parameter_size_bytes"] = s.total_param_bytes;
        d["copies_into_bucket"] = s.copies_into_bucket;
        return d;
      });

  pdt::register_cuda_bindings(m);
}
