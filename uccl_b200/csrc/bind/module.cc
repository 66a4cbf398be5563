// pybind11 bindings (nanobind, which the reference uses for uccl.p2p / uccl.ep, is not
// available offline).  Device pointers and CUDA streams cross the boundary as integers
// (tensor.data_ptr(), torch.cuda.current_stream().cuda_stream) so this module does not
// need any torch headers and builds in seconds.
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include "../coll/comm.h"
#include "../coll/multi_comm.h"
#include "../common/log.h"
#include "../common/param.h"
#include "../kernels/launch.h"

namespace py = pybind11;
using namespace ub;

void bind_ep(py::module_& m);
void bind_p2p(py::module_& m);
void bind_util(py::module_& m);
void bind_uk(py::module_& m);
void bind_net(py::module_& m);

static inline cudaStream_t S(uintptr_t s) { return reinterpret_cast<cudaStream_t>(s); }
static inline void* P(uintptr_t p) { return reinterpret_cast<void*>(p); }

PYBIND11_MODULE(_C, m) {
  m.doc() = "uccl_b200 native core: symmetric-heap fabric, sm_90a collectives, EP, P2P engine";
  m.attr("MAX_RANKS") = kMaxRanks;
  m.attr("LL_MAX_BYTES") = (uint64_t)kLLMaxData;

  m.def("create_unique_id", [] {
    UniqueId id = Bootstrap::create_id();
    return py::bytes(id.data, sizeof(id.data));
  });
  m.def("preload_kernels", [] {
    cudaError_t e = preload_all_kernels();
    UB_CHECK(e == cudaSuccess, "preload failed: %s", cudaGetErrorString(e));
  });
  m.def("set_log_level", [](int lv) { set_log_level(lv); });
  m.def("dtype_size", [](int dt) { return dtype_size(dt); });
  m.def("algo_name", [](int a) { return std::string(algo_name(a)); });
  m.def("param", [](const std::string& name, int64_t dflt) { return param_load(name.c_str(), dflt); });

  py::class_<TuneEntry>(m, "TuneEntry")
      .def(py::init([](uint64_t max_bytes, int algo, int ctas) { return TuneEntry{max_bytes, algo, ctas}; }))
      .def_readwrite("max_bytes", &TuneEntry::max_bytes)
      .def_readwrite("algo", &TuneEntry::algo)
      .def_readwrite("ctas", &TuneEntry::ctas);

  py::class_<Comm, std::shared_ptr<Comm>>(m, "Comm")
      .def_static(
          "create",
          [](py::bytes uid, int rank, int nranks, int device, size_t heap_bytes, size_t stage_bytes, bool host_fake,
             int timeout_ms, int max_ctas) {
            std::string s = uid;
            UB_CHECK(s.size() == sizeof(UniqueId), "unique id must be %zu bytes", sizeof(UniqueId));
            UniqueId id;
            memcpy(id.data, s.data(), sizeof(id.data));
            CommConfig cfg;
            cfg.heap_bytes = heap_bytes;
            cfg.stage_bytes = stage_bytes;
            cfg.host_fake = host_fake;
            cfg.timeout_ms = timeout_ms;
            cfg.max_ctas = max_ctas;
            py::gil_scoped_release rel;
            return Comm::create(id, rank, nranks, device, cfg);
          },
          py::arg("uid"), py::arg("rank"), py::arg("nranks"), py::arg("device"), py::arg("heap_bytes"),
          py::arg("stage_bytes") = (size_t)(64ull << 20), py::arg("host_fake") = false, py::arg("timeout_ms") = -1,
          py::arg("max_ctas") = -1)
      .def_static(
          "create_local",
          [](std::vector<int> devices, size_t heap_bytes, size_t stage_bytes, bool host_fake, int timeout_ms,
             int max_ctas) {
            CommConfig cfg;
            cfg.heap_bytes = heap_bytes;
            cfg.stage_bytes = stage_bytes;
            cfg.host_fake = host_fake;
            cfg.timeout_ms = timeout_ms;
            cfg.max_ctas = max_ctas;
            return Comm::create_local(devices, cfg);
          },
          py::arg("devices"), py::arg("heap_bytes"), py::arg("stage_bytes") = (size_t)(64ull << 20),
          py::arg("host_fake") = false, py::arg("timeout_ms") = -1, py::arg("max_ctas") = -1)
      .def_property_readonly("rank", &Comm::rank)
      .def_property_readonly("nranks", &Comm::nranks)
      .def_property_readonly("device", &Comm::device)
      .def_property_readonly("has_multicast", &Comm::has_multicast)
      .def_property_readonly("is_host", &Comm::is_host)
      .def_property_readonly("single_process", [](const Comm& c) { return c.fabric().single_process(); })
      .def_property_readonly("launches", &Comm::launches)
      .def_property_readonly("error_word", &Comm::error_word)
      .def_property_readonly("heap_base", [](const Comm& c) { return (uintptr_t)c.fabric().local(); })
      .def_property_readonly("heap_bytes", [](const Comm& c) { return c.fabric().heap_bytes(); })
      .def_property_readonly("heap_free_bytes", &Comm::heap_free_bytes)
      .def_property_readonly("stage_bytes", [](const Comm& c) { return (uint64_t)c.layout().stage_bytes; })
      .def("describe", &Comm::describe)
      .def("alloc", [](Comm& c, size_t bytes, size_t align) { return (uintptr_t)c.alloc(bytes, align); },
           py::arg("bytes"), py::arg("align") = 256)
      .def("free", [](Comm& c, uintptr_t p) { c.free(P(p)); })
      .def("in_heap", [](const Comm& c, uintptr_t p, size_t n) { return c.in_heap(P(p), n); })
      .def("heap_offset", [](const Comm& c, uintptr_t p) { return c.heap_offset(P(p)); })
      .def("peer_ptr", [](const Comm& c, uintptr_t p, int peer) { return (uintptr_t)c.peer_ptr(P(p), peer); })
      .def("mc_ptr", [](const Comm& c, uintptr_t p) { return (uintptr_t)c.mc_ptr(P(p)); })
      .def(
          "allreduce",
          [](Comm& c, uintptr_t in, uintptr_t out, size_t count, int dtype, int op, uintptr_t stream, int algo,
             float scale, int out_dtype, int max_ctas) {
            ArOpts o;
            o.algo = algo;
            o.scale = scale;
            o.out_dtype = out_dtype;
            o.max_ctas = max_ctas;
            py::gil_scoped_release rel;
            c.allreduce(P(in), P(out), count, dtype, op, S(stream), o);
          },
          py::arg("inp"), py::arg("out"), py::arg("count"), py::arg("dtype"), py::arg("op"), py::arg("stream"),
          py::arg("algo") = 0, py::arg("scale") = 1.0f, py::arg("out_dtype") = -1, py::arg("max_ctas") = -1)
      .def("allgather",
           [](Comm& c, uintptr_t in, uintptr_t out, size_t count, int dtype, uintptr_t stream) {
             py::gil_scoped_release rel;
             c.allgather(P(in), P(out), count, dtype, S(stream));
           })
      .def("reduce_scatter",
           [](Comm& c, uintptr_t in, uintptr_t out, size_t count, int dtype, int op, uintptr_t stream) {
             py::gil_scoped_release rel;
             c.reduce_scatter(P(in), P(out), count, dtype, op, S(stream));
           })
      .def("broadcast",
           [](Comm& c, uintptr_t in, uintptr_t out, size_t count, int dtype, int root, uintptr_t stream) {
             py::gil_scoped_release rel;
             c.broadcast(P(in), P(out), count, dtype, root, S(stream));
           })
      .def("reduce",
           [](Comm& c, uintptr_t in, uintptr_t out, size_t count, int dtype, int op, int root, uintptr_t stream) {
             py::gil_scoped_release rel;
             c.reduce(P(in), P(out), count, dtype, op, root, S(stream));
           })
      .def("alltoall",
           [](Comm& c, uintptr_t in, uintptr_t out, size_t count, int dtype, uintptr_t stream) {
             py::gil_scoped_release rel;
             c.alltoall(P(in), P(out), count, dtype, S(stream));
           })
      .def("alltoallv",
           [](Comm& c, uintptr_t in, std::vector<size_t> scounts, std::vector<size_t> sdispls, uintptr_t out,
              std::vector<size_t> rcounts, std::vector<size_t> rdispls, int dtype, uintptr_t stream) {
             const size_t n = (size_t)c.nranks();
             UB_CHECK(scounts.size() == n && sdispls.size() == n && rcounts.size() == n && rdispls.size() == n,
                      "alltoallv: count/displacement lists must have nranks entries");
             py::gil_scoped_release rel;
             c.alltoallv(P(in), scounts.data(), sdispls.data(), P(out), rcounts.data(), rdispls.data(), dtype,
                         S(stream));
           })
      .def("barrier",
           [](Comm& c, uintptr_t stream) {
             py::gil_scoped_release rel;
             c.barrier(S(stream));
           })
      .def("select_allreduce",
           [](const Comm& c, size_t bytes, bool symmetric, int dtype, int op) {
             int ctas = 0;
             int algo = c.select_allreduce(bytes, symmetric, dtype, op, &ctas);
             return py::make_tuple(algo, ctas);
           })
      // grouped point-to-point: ops = [(is_send, ptr, bytes, peer), ...] (ncclGroupStart/Send/Recv/End)
      .def("group_p2p",
           [](Comm& c, const std::vector<std::tuple<bool, uintptr_t, size_t, int>>& ops, uintptr_t stream) {
             std::vector<Comm::P2pOp> v;
             for (auto& o : ops) v.push_back(Comm::P2pOp{std::get<0>(o), P(std::get<1>(o)), std::get<2>(o), std::get<3>(o)});
             py::gil_scoped_release rel;
             c.group_p2p(v, S(stream));
           },
           py::arg("ops"), py::arg("stream") = 0)
      .def("set_tuning", &Comm::set_tuning)
      .def("set_xchg_ll_max", &Comm::set_xchg_ll_max)
      .def("set_rs_push", &Comm::set_rs_push)
      .def("rs_push", &Comm::rs_push)
      .def("xchg_ll_max", &Comm::xchg_ll_max)
      .def("enable_trace", &Comm::enable_trace)
      .def("disable_trace", &Comm::disable_trace)
      .def("dump_trace",
           [](Comm& c, bool reset) {
             py::list out;
             for (auto& e : c.dump_trace(reset)) out.append(py::make_tuple(e.t_ns, e.code, e.block, e.aux));
             return out;
           },
           py::arg("reset") = true);

  // slicing helpers of the chunked kernels (host-callable twins, for property tests)
  m.def("split_range", [](uint64_t total, int parts, int idx, uint64_t gran) {
    uint64_t lo, hi;
    split_range(total, parts, idx, lo, hi, gran);
    return py::make_tuple(lo, hi);
  }, py::arg("total"), py::arg("parts"), py::arg("idx"), py::arg("gran") = 1);
  m.def("chunk_slice", [](uint64_t msg_bytes, uint64_t chunk_bytes, uint64_t cb, int parts, int idx, uint64_t gran) {
    uint64_t lo, hi;
    chunk_slice_hd(msg_bytes, chunk_bytes, cb, parts, idx, lo, hi, gran);
    return py::make_tuple(lo, hi);
  }, py::arg("msg_bytes"), py::arg("chunk_bytes"), py::arg("cb"), py::arg("parts"), py::arg("idx"), py::arg("gran") = 1);
  m.def("pool_install", &pool_install);
  m.def("pool_set_thread_comm", &pool_set_thread_comm);
  m.def("pool_clear_thread_comm", &pool_clear_thread_comm);
  m.def("pool_stats", [] {
    uint64_t a, f, l, fb;
    pool_stats(&a, &f, &l, &fb);
    py::dict d;
    d["allocs"] = a, d["frees"] = f, d["live_bytes"] = l, d["fallback_allocs"] = fb;
    return d;
  });

  bind_util(m);
  bind_ep(m);
  bind_p2p(m);
  // hierarchical communicator across boxes in C++ (what the NCCL drop-in uses); same calling convention as Comm
  py::class_<MultiComm, std::shared_ptr<MultiComm>>(m, "MultiComm")
      .def_static(
          "create",
          [](py::bytes uid, int rank, int nranks, int local_size, int device, size_t heap_bytes, size_t stage_bytes,
             bool host_fake, int timeout_ms) {
            std::string s = uid;
            UB_CHECK(s.size() == sizeof(UniqueId), "unique id must be %zu bytes", sizeof(UniqueId));
            UniqueId id;
            memcpy(id.data, s.data(), sizeof(id.data));
            CommConfig cfg;
            cfg.heap_bytes = heap_bytes;
            cfg.stage_bytes = stage_bytes;
            cfg.host_fake = host_fake;
            cfg.timeout_ms = timeout_ms;
            py::gil_scoped_release rel;
            return MultiComm::create(id, rank, nranks, local_size, device, cfg);
          },
          py::arg("uid"), py::arg("rank"), py::arg("nranks"), py::arg("local_size"), py::arg("device"),
          py::arg("heap_bytes"), py::arg("stage_bytes") = (size_t)(64ull << 20), py::arg("host_fake") = false,
          py::arg("timeout_ms") = -1)
      .def_property_readonly("rank", &MultiComm::rank)
      .def_property_readonly("nranks", &MultiComm::nranks)
      .def_property_readonly("local_rank", &MultiComm::local_rank)
      .def_property_readonly("local_size", &MultiComm::local_size)
      .def_property_readonly("node", &MultiComm::node)
      .def_property_readonly("nnodes", &MultiComm::nnodes)
      .def_property_readonly("is_host", &MultiComm::is_host)
      .def_property_readonly("device", &MultiComm::device)
      .def_property_readonly("local", [](MultiComm& c) { return c.local(); })
      .def("describe", &MultiComm::describe)
      .def("allreduce",
           [](MultiComm& c, uintptr_t in, uintptr_t out, size_t count, int dtype, int op, uintptr_t stream, float scale) {
             py::gil_scoped_release rel;
             c.allreduce(P(in), P(out), count, dtype, op, S(stream), scale);
           },
           py::arg("inp"), py::arg("out"), py::arg("count"), py::arg("dtype"), py::arg("op"), py::arg("stream") = 0,
           py::arg("scale") = 1.0f)
      .def("allgather",
           [](MultiComm& c, uintptr_t in, uintptr_t out, size_t count, int dtype, uintptr_t stream) {
             py::gil_scoped_release rel;
             c.allgather(P(in), P(out), count, dtype, S(stream));
           })
      .def("reduce_scatter",
           [](MultiComm& c, uintptr_t in, uintptr_t out, size_t count, int dtype, int op, uintptr_t stream) {
             py::gil_scoped_release rel;
             c.reduce_scatter(P(in), P(out), count, dtype, op, S(stream));
           })
      .def("broadcast",
           [](MultiComm& c, uintptr_t in, uintptr_t out, size_t count, int dtype, int root, uintptr_t stream) {
             py::gil_scoped_release rel;
             c.broadcast(P(in), P(out), count, dtype, root, S(stream));
           })
      .def("reduce",
           [](MultiComm& c, uintptr_t in, uintptr_t out, size_t count, int dtype, int op, int root, uintptr_t stream) {
             py::gil_scoped_release rel;
             c.reduce(P(in), P(out), count, dtype, op, root, S(stream));
           })
      .def("alltoall",
           [](MultiComm& c, uintptr_t in, uintptr_t out, size_t count, int dtype, uintptr_t stream) {
             py::gil_scoped_release rel;
             c.alltoall(P(in), P(out), count, dtype, S(stream));
           })
      .def("alltoallv",
           [](MultiComm& c, uintptr_t in, std::vector<size_t> sc, std::vector<size_t> sd, uintptr_t out, std::vector<size_t> rc,
              std::vector<size_t> rd, int dtype, uintptr_t stream) {
             UB_CHECK((int)sc.size() == c.nranks() && (int)sd.size() == c.nranks() && (int)rc.size() == c.nranks() &&
                          (int)rd.size() == c.nranks(),
                      "alltoallv: count / displacement lists must have one entry per rank");
             py::gil_scoped_release rel;
             c.alltoallv(P(in), sc.data(), sd.data(), P(out), rc.data(), rd.data(), dtype, S(stream));
           })
      .def("barrier",
           [](MultiComm& c, uintptr_t stream) {
             py::gil_scoped_release rel;
             c.barrier(S(stream));
           },
           py::arg("stream") = 0)
      .def("group_p2p",
           [](MultiComm& c, std::vector<std::tuple<bool, uintptr_t, size_t, int>> ops, uintptr_t stream) {
             std::vector<Comm::P2pOp> v;
             for (auto& o : ops) v.push_back(Comm::P2pOp{std::get<0>(o), P(std::get<1>(o)), std::get<2>(o), std::get<3>(o)});
             py::gil_scoped_release rel;
             c.group_p2p(v, S(stream));
           },
           py::arg("ops"), py::arg("stream") = 0);
  bind_uk(m);
  bind_net(m);
}
