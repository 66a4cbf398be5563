// Python bindings of the EP runtime (role of the reference's NB_MODULE in ep/src/uccl_ep.cc:1641-2410).
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include "../common/log.h"
#include "ep_buffer.h"
#include "ep_logfmt.h"
#include "proxy.h"

namespace py = pybind11;
using namespace ub;

void bind_ep(py::module_& m) {
  m.attr("EP_X_BF16") = (int)EP_X_BF16;
  m.attr("EP_X_FP8_SCALED") = (int)EP_X_FP8_SCALED;
  m.attr("EP_X_FUSED_FP8") = (int)EP_X_FUSED_FP8;
  m.attr("EP_MAX_TOPK") = kEpMaxTopk;
  m.attr("EP_IMPL_AUTO") = (int)EP_IMPL_AUTO;
  m.attr("EP_IMPL_REG") = (int)EP_IMPL_REG;
  m.attr("EP_IMPL_TMA") = (int)EP_IMPL_TMA;
  m.attr("EP_LL_FULL") = (int)EP_LL_FULL;
  m.attr("EP_LL_SEND") = (int)EP_LL_SEND;
  m.attr("EP_LL_RECV") = (int)EP_LL_RECV;
  m.attr("EP_LL_SCALES_ROW_MAJOR") = (int)EP_LL_SCALES_ROW_MAJOR;
  m.attr("EP_LL_SCALES_COL_MAJOR") = (int)EP_LL_SCALES_COL_MAJOR;
  m.attr("EP_LL_SCALES_COL_UE8M0") = (int)EP_LL_SCALES_COL_UE8M0;
  py::class_<EpDispatchOut>(m, "EpDispatchOut")
      .def_readonly("recv_x", &EpDispatchOut::recv_x)
      .def_readonly("recv_scales", &EpDispatchOut::recv_scales)
      .def_readonly("recv_topk_idx", &EpDispatchOut::recv_topk_idx)
      .def_readonly("recv_topk_w", &EpDispatchOut::recv_topk_w)
      .def_readonly("recv_src_idx", &EpDispatchOut::recv_src_idx)
      .def_readonly("slot", &EpDispatchOut::slot)
      .def_readonly("capacity", &EpDispatchOut::capacity);
  py::class_<EpBuffer, std::shared_ptr<EpBuffer>>(m, "EpBuffer")
      .def(py::init<std::shared_ptr<Comm>, size_t, int>(), py::arg("comm"), py::arg("num_nvl_bytes"),
           py::arg("num_slots") = 2)
      .def_property_readonly("rank", &EpBuffer::rank)
      .def_property_readonly("nranks", &EpBuffer::nranks)
      .def_property_readonly("arena_bytes", &EpBuffer::arena_bytes)
      .def_property_readonly("num_slots", &EpBuffer::num_slots)
      .def_property_readonly("launches", &EpBuffer::launches)
      .def_property_readonly("dev_counts_ptr", &EpBuffer::dev_counts_ptr)
      .def_property("impl", &EpBuffer::impl, &EpBuffer::set_impl)
      .def("set_stages", &EpBuffer::set_stages, py::arg("dispatch_in") = 0, py::arg("dispatch_out") = 0,
           py::arg("combine") = 0)
      .def_property_readonly("last_dispatch_impl", &EpBuffer::last_dispatch_impl)
      .def_property_readonly("last_combine_impl", &EpBuffer::last_combine_impl)
      .def("capacity_for", &EpBuffer::capacity_for)
      .def("combine_capacity_for", &EpBuffer::combine_capacity_for)
      .def("layout",
           [](EpBuffer& b, uintptr_t topk_idx, int T, int K, int E, uintptr_t tpr, uintptr_t tpe, uintptr_t itir,
              uintptr_t pos, uintptr_t st) { b.layout(topk_idx, T, K, E, tpr, tpe, itir, pos, (cudaStream_t)st); })
      .def("dispatch",
           [](EpBuffer& b, uintptr_t x, uintptr_t xs, uintptr_t ti, uintptr_t tw, uintptr_t pos, uintptr_t ss,
              uintptr_t tpr, uintptr_t tpe, int T, int H, int K, int E, int mode, bool cached, int reuse_slot,
              uintptr_t rank_prefix, int expert_alignment, int num_worst_tokens, bool round_scale, int num_sms,
              uintptr_t st) {
             return b.dispatch(x, xs, ti, tw, pos, ss, tpr, tpe, T, H, K, E, mode, cached, reuse_slot, rank_prefix,
                               expert_alignment, num_worst_tokens, round_scale, num_sms, (cudaStream_t)st);
           })
      .def_property_readonly("base_offset", &EpBuffer::base_offset)
      .def_property_readonly("arena_area_ptr", &EpBuffer::arena_area_ptr)
      .def_property_readonly("arena_area_bytes", &EpBuffer::arena_area_bytes)
      .def_property_readonly("ll_ptr", &EpBuffer::ll_ptr)
      .def_property_readonly("ll_nbytes", &EpBuffer::ll_nbytes)
      .def("wait_counts",
           [](EpBuffer& b, int E_local, double timeout_s) {
             std::vector<int> pe;
             int total;
             {
               py::gil_scoped_release rel;
               total = b.wait_counts(E_local, &pe, timeout_s);
             }
             return py::make_tuple(total, pe);
           },
           py::arg("E_local"), py::arg("timeout_s") = 0.0)
      .def("ll_init", &EpBuffer::ll_init)
      .def_static("ll_size_hint", &EpBuffer::ll_size_hint)
      .def("ll_dispatch",
           [](EpBuffer& b, uintptr_t x, uintptr_t ti, int T, int H, int K, int E, int M, bool use_fp8, bool round_scale,
              uintptr_t recv_count, uintptr_t layout_range, uintptr_t send_pos, int num_sms, uintptr_t st, int phase,
              int scale_layout, uintptr_t wait_stats) {
             auto o = b.ll_dispatch(x, ti, T, H, K, E, M, use_fp8, round_scale, recv_count, layout_range, send_pos,
                                    num_sms, (cudaStream_t)st, phase, scale_layout, wait_stats);
             return py::make_tuple(o.recv_x, o.recv_scales, o.recv_src_info, o.combine_x, o.buffer_idx);
           },
           py::arg("x"), py::arg("topk_idx"), py::arg("T"), py::arg("H"), py::arg("K"), py::arg("E"), py::arg("M"),
           py::arg("use_fp8"), py::arg("round_scale"), py::arg("recv_count"), py::arg("layout_range"),
           py::arg("send_pos"), py::arg("num_sms"), py::arg("stream"), py::arg("phase") = (int)EP_LL_FULL,
           py::arg("scale_layout") = (int)EP_LL_SCALES_ROW_MAJOR, py::arg("wait_stats") = 0)
      .def("ll_dispatch_recv",
           [](EpBuffer& b, int num_sms, uintptr_t wait_stats, uintptr_t st) { b.ll_dispatch_recv(num_sms, wait_stats, (cudaStream_t)st); },
           py::arg("num_sms"), py::arg("wait_stats"), py::arg("stream"))
      .def("ll_combine_buffer", &EpBuffer::ll_combine_buffer)
      .def("ll_combine",
           [](EpBuffer& b, uintptr_t x, int idx, uintptr_t tw, uintptr_t sp, uintptr_t out, int T, int H, int K, int E,
              int M, int num_sms, uintptr_t st, int phase, uintptr_t layout_range, uintptr_t wait_stats, bool use_logfmt) {
             b.ll_combine(x, idx, tw, sp, out, T, H, K, E, M, num_sms, (cudaStream_t)st, phase, layout_range, wait_stats,
                          use_logfmt);
           },
           py::arg("x"), py::arg("buffer_idx"), py::arg("topk_weights"), py::arg("send_pos"), py::arg("out"),
           py::arg("T"), py::arg("H"), py::arg("K"), py::arg("E"), py::arg("M"), py::arg("num_sms"), py::arg("stream"),
           py::arg("phase") = (int)EP_LL_FULL, py::arg("layout_range") = 0, py::arg("wait_stats") = 0,
           py::arg("use_logfmt") = false)
      .def("ll_combine_rmsnorm",
           [](EpBuffer& b, uintptr_t x, int idx, uintptr_t tw, uintptr_t sp, uintptr_t shared, uintptr_t residual,
              uintptr_t residual_out, uintptr_t weight, uintptr_t out, uintptr_t out_scales, int T, int H, int K, int E,
              int M, float eps, int num_sms, uintptr_t st, int phase, uintptr_t layout_range, uintptr_t wait_stats,
              bool use_logfmt) {
             b.ll_combine_rmsnorm(x, idx, tw, sp, shared, residual, residual_out, weight, out, out_scales, T, H, K, E,
                                  M, eps, num_sms, (cudaStream_t)st, phase, layout_range, wait_stats, use_logfmt);
           },
           py::arg("x"), py::arg("buffer_idx"), py::arg("topk_weights"), py::arg("send_pos"), py::arg("shared"),
           py::arg("residual"), py::arg("residual_out"), py::arg("weight"), py::arg("out"), py::arg("out_scales"),
           py::arg("T"), py::arg("H"), py::arg("K"), py::arg("E"), py::arg("M"), py::arg("eps"), py::arg("num_sms"),
           py::arg("stream"), py::arg("phase") = (int)EP_LL_FULL, py::arg("layout_range") = 0,
           py::arg("wait_stats") = 0, py::arg("use_logfmt") = false)
      .def("combine_input_ptr", &EpBuffer::combine_input_ptr)
      .def("combine", [](EpBuffer& b, uintptr_t x, int num_recv, uintptr_t tw, uintptr_t ss, uintptr_t b0,
                         uintptr_t b1, uintptr_t out, uintptr_t otw, int T, int H, int K, int num_sms, uintptr_t st) {
        b.combine(x, num_recv, tw, ss, b0, b1, out, otw, T, H, K, num_sms, (cudaStream_t)st);
      })
      .def("combine_rmsnorm",
           [](EpBuffer& b, uintptr_t x, int num_recv, uintptr_t ss, uintptr_t b0, uintptr_t b1, uintptr_t residual,
              uintptr_t residual_out, uintptr_t weight, uintptr_t out, uintptr_t out_scales, int T, int H, float eps,
              int num_sms, uintptr_t st) {
             b.combine_rmsnorm(x, num_recv, ss, b0, b1, residual, residual_out, weight, out, out_scales, T, H, eps,
                               num_sms, (cudaStream_t)st);
           },
           py::arg("x"), py::arg("num_recv"), py::arg("send_slot"), py::arg("bias0"), py::arg("bias1"),
           py::arg("residual"), py::arg("residual_out"), py::arg("weight"), py::arg("out"), py::arg("out_scales"),
           py::arg("T"), py::arg("H"), py::arg("eps"), py::arg("num_sms"), py::arg("stream"));

  // host reference of the LogFMT-10 simulated cast: the same arithmetic the CUDA pass compiles (ep_logfmt.h), in place
  // on [rows, H] bf16 host memory
  m.def("ep_logfmt10_host", [](uintptr_t ptr, size_t rows, size_t H) {
    UB_CHECK(H % 128 == 0, "ep_logfmt10_host: hidden %% 128 != 0");
    py::gil_scoped_release rel;
    logfmt10_host((uint16_t*)ptr, rows, H);
  });

  // ---- GPU -> CPU command queue + proxy
  m.attr("D2H_NOP") = (int)D2H_NOP;
  m.attr("D2H_WRITE") = (int)D2H_WRITE;
  m.attr("D2H_ATOMIC") = (int)D2H_ATOMIC;
  m.attr("D2H_NOTIFY") = (int)D2H_NOTIFY;
  // network half of the proxy on its own (host heaps): what tests and CPU-only runs use
  py::class_<ProxyLink, std::shared_ptr<ProxyLink>>(m, "EpProxyLink")
      .def(py::init([](int box, int nboxes, std::shared_ptr<net::Engine> engine, std::vector<uint32_t> flows,
                       std::vector<uintptr_t> heaps, uint64_t heap_bytes) {
             std::vector<char*> hs;
             for (auto h : heaps) hs.push_back((char*)h);
             return std::shared_ptr<ProxyLink>(
                 new ProxyLink(box, nboxes, std::move(engine), std::move(flows), ProxyLink::host_write(hs, heap_bytes),
                               ProxyLink::host_add(hs, heap_bytes)),
                 [](ProxyLink* l) {
                   if (PyGILState_Check()) {
                     py::gil_scoped_release rel;
                     delete l;
                   } else {
                     delete l;
                   }
                 });
           }),
           py::arg("box"), py::arg("nboxes"), py::arg("engine"), py::arg("flows"), py::arg("heaps"), py::arg("heap_bytes"))
      .def("put", [](ProxyLink& l, int dst_box, int dst_local, uint64_t off, uintptr_t src, uint32_t bytes) {
        l.put(dst_box, dst_local, off, (const void*)src, bytes);
      })
      .def("add", &ProxyLink::add)
      .def("notify", &ProxyLink::notify)
      .def("flush", &ProxyLink::flush, py::arg("timeout_ms") = 30000, py::call_guard<py::gil_scoped_release>())
      .def("stats", [](ProxyLink& l) {
        auto s = l.stats();
        py::dict d;
        d["puts"] = s.puts, d["adds"] = s.adds, d["notifies"] = s.notifies, d["bytes_out"] = s.bytes_out;
        d["applied_writes"] = s.applied_writes, d["applied_adds"] = s.applied_adds, d["bytes_in"] = s.bytes_in;
        d["applied_notifies"] = s.applied_notifies;
        return d;
      });
  py::class_<Proxy, std::shared_ptr<Proxy>>(m, "EpProxy")
      .def("attach_link", &Proxy::attach_link, py::arg("engine"), py::arg("flows"), py::arg("box"), py::arg("nboxes"),
           py::arg("local_size"))
      .def(py::init([](std::shared_ptr<Comm> c, uint32_t cap) {
             py::gil_scoped_release rel;
             return std::make_shared<Proxy>(c, cap);
           }),
           py::arg("comm"), py::arg("capacity") = 4096)
      .def("start", &Proxy::start)
      .def("stop", &Proxy::stop, py::call_guard<py::gil_scoped_release>())
      .def_property_readonly("running", &Proxy::running)
      .def("drain", &Proxy::drain, py::arg("timeout_s") = 30.0, py::call_guard<py::gil_scoped_release>())
      .def("consumed", &Proxy::consumed)
      .def("poll_notifications", &Proxy::poll_notifications)
      // raw device handle (ring, head, tail, ack, capacity) for kernels of other extensions
      .def("queue_handle",
           [](Proxy& p) {
             D2HQueueDev q = p.queue();
             return py::make_tuple((uintptr_t)q.ring, (uintptr_t)q.head, (uintptr_t)q.tail, (uintptr_t)q.ack, q.capacity);
           })
      .def("issue_from_device",
           [](Proxy& p, int type, int dst, uint32_t aux, uint64_t so, uint64_t doff, uint32_t bytes, uint32_t value,
              uintptr_t st) { p.issue_from_device((uint32_t)type, dst, aux, so, doff, bytes, value, (cudaStream_t)st); },
           py::arg("type"), py::arg("dst_rank") = 0, py::arg("aux") = 0, py::arg("src_off") = 0, py::arg("dst_off") = 0,
           py::arg("bytes") = 0, py::arg("value") = 0, py::arg("stream") = 0)
      .def("bench_throughput",
           [](Proxy& p, int blocks, int threads, int per_thread, uintptr_t st) {
             py::gil_scoped_release rel;
             return p.bench_throughput(blocks, threads, per_thread, (cudaStream_t)st);
           },
           py::arg("blocks") = 8, py::arg("threads") = 128, py::arg("per_thread") = 64, py::arg("stream") = 0)
      .def("bench_latency",
           [](Proxy& p, int iters, uintptr_t st) {
             py::gil_scoped_release rel;
             return p.bench_latency(iters, (cudaStream_t)st);
           },
           py::arg("iters") = 1000, py::arg("stream") = 0)
      .def("stats", [](Proxy& p) {
        auto s = p.stats();
        py::dict d;
        d["cmds"] = s.cmds, d["nops"] = s.nops, d["writes"] = s.writes, d["atomics"] = s.atomics;
        d["notifies"] = s.notifies, d["bytes"] = s.bytes, d["avg_handle_us"] = s.avg_handle_us;
        return d;
      });
}
