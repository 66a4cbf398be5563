// Force-load every kernel of this library (see launch.h for why).
#include <cstring>
#include <mutex>

#include "../common/log.h"
#include "../ep/ep_buffer.h"
#include "../ep/proxy.h"
#include "../p2p/compress.h"
#include "../kernels/launch.h"

namespace ub {

bool g_preload = false;
cudaError_t preload_p2p_kernels();  // p2p/p2p_kernels.cu
}  // namespace ub
#include "../ukernel/uk_worker.h"
namespace ub {

cudaError_t preload_all_kernels() {
  static std::mutex mu;
  static uint64_t done_mask = 0;  // per device (lazy loading is per context)
  std::lock_guard<std::mutex> g(mu);
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    (void)cudaGetLastError();
    return cudaSuccess;
  }
  if (done_mask & (1ull << (dev & 63))) return cudaSuccess;
  DevComm c;
  memset(&c, 0, sizeof(c));
  CollArgs a;
  memset(&a, 0, sizeof(a));
  A2AvArgs v;
  memset(&v, 0, sizeof(v));
  g_preload = true;
  int loaded = 0;
  auto ok = [&](cudaError_t e) {
    if (e == cudaSuccess) ++loaded;
    else (void)cudaGetLastError();  // unsupported combination: nothing to load
  };
  for (int algo = 1; algo <= 7; ++algo)
    for (int op = 0; op < 4; ++op) {
      for (int dt : {(int)kF32, (int)kBF16, (int)kF16}) ok(launch_allreduce_f(algo, dt, op, dt, c, a, 1, 512, 0));
      for (int dt : {(int)kI8, (int)kU8, (int)kI32, (int)kU32, (int)kI64, (int)kU64})
        ok(launch_allreduce_i(algo, dt, op, c, a, 1, 512, 0));
      for (int dt : {(int)kF64, (int)kF8E4M3, (int)kF8E5M2}) ok(launch_allreduce_x(algo, dt, op, c, a, 1, 512, 0));
    }
  for (int algo = 3; algo <= 6; ++algo) {
    ok(launch_allreduce_f(algo, kF32, kSum, kBF16, c, a, 1, 512, 0));
    ok(launch_allreduce_f(algo, kF32, kSum, kF16, c, a, 1, 512, 0));
    ok(launch_allreduce_f(algo, kBF16, kSum, kF32, c, a, 1, 512, 0));
    ok(launch_allreduce_f(algo, kF16, kSum, kF32, c, a, 1, 512, 0));
  }
  {
    RmsNormArgs r;
    memset(&r, 0, sizeof(r));
    for (int algo : {0, 1, 2})
      for (int dt : {(int)kBF16, (int)kF16})
        for (bool fp8 : {false, true}) ok(launch_allreduce_rmsnorm(algo, dt, fp8, c, a, r, 1, 0));
    for (int dt : {(int)kBF16, (int)kF16})
      for (bool fp8 : {false, true}) ok(launch_reduce_scatter_rmsnorm(dt, fp8, c, a, r, 1, 0));
  }
  for (int m = 0; m < 5; ++m) ok(launch_allgather(m, c, a, 1, 512, 0));
  for (int m = 0; m < 4; ++m) ok(launch_broadcast(m, c, a, 1, 512, 0));
  for (int m = 0; m < 3; ++m) ok(launch_alltoall(m, c, a, 1, 512, 0));
  ok(launch_alltoallv(c, a, v, 1, 512, 0));
  ok(launch_barrier(c, 0, 0));
  {
    SendRecvArgs sr;
    memset(&sr, 0, sizeof(sr));
    ok(launch_sendrecv(c, sr, 0));
  }
  for (int which = 0; which < 2; ++which)
    for (int op = 0; op < 4; ++op) {
      for (int dt : {(int)kF32, (int)kBF16, (int)kF16, (int)kF64, (int)kF8E4M3, (int)kF8E5M2})
        for (int nv = 0; nv < 2; ++nv) ok(launch_red_f(which, dt, op, nv != 0, c, a, 1, 512, 0));
      for (int dt : {(int)kI8, (int)kU8, (int)kI32, (int)kU32, (int)kI64, (int)kU64})
        ok(launch_red_i(which, dt, op, c, a, 1, 512, 0));
    }
  for (int op = 0; op < 4; ++op) {
    for (int dt : {(int)kF32, (int)kBF16, (int)kF16, (int)kF64, (int)kF8E4M3, (int)kF8E5M2})
      ok(launch_rs_ll_f(dt, op, c, a, 1, 512, 0));
    for (int dt : {(int)kI8, (int)kU8, (int)kI32, (int)kU32, (int)kI64, (int)kU64})
      ok(launch_rs_ll_i(dt, op, c, a, 1, 512, 0));
  }
  EpLayoutArgs la;
  memset(&la, 0, sizeof(la));
  ok(launch_ep_layout(la, 0));
  {
    uint32_t dummy_scratch = 0;
    la.scratch = &dummy_scratch;  // multi-CTA variant
    ok(launch_ep_layout(la, 0));
  }
  EpDispatchArgs da;
  memset(&da, 0, sizeof(da));
  EpCombineArgs ca;
  memset(&ca, 0, sizeof(ca));
  int dummy_bias = 0;
  for (int nr : {1, 2, 4, 8}) {
    DevComm cn = c;
    cn.nranks = nr;
    for (int m = 0; m < 3; ++m) {
      da.mode = m;
      ok(launch_ep_dispatch(cn, da, 1, 0));
    }
    ca.bias0 = nullptr;
    ok(launch_ep_combine(cn, ca, 1, 0));
    ca.bias0 = &dummy_bias;
    ok(launch_ep_combine(cn, ca, 1, 0));
    RmsNormArgs r;
    memset(&r, 0, sizeof(r));
    for (bool fp8 : {false, true}) {
      ca.bias0 = nullptr;
      ok(launch_ep_combine_rmsnorm(cn, ca, r, fp8, 1, 0));
      ca.bias0 = &dummy_bias;
      ok(launch_ep_combine_rmsnorm(cn, ca, r, fp8, 1, 0));
    }
  }
  {
    DevComm cn = c;
    cn.nranks = 8;
    da.H = ca.H = 1024;
    for (int m = 0; m < 3; ++m) {
      da.mode = m;
      ok(launch_ep_dispatch_tma(cn, da, 1, 0));
    }
    ca.bias0 = nullptr;
    ok(launch_ep_combine_tma(cn, ca, 1, 0));
    ca.bias0 = &dummy_bias;
    ok(launch_ep_combine_tma(cn, ca, 1, 0));
  }
  {
    EpLLDispatchArgs ld;
    memset(&ld, 0, sizeof(ld));
    ld.H = 128;
    ld.E = 8;
    ok(launch_ep_ll_dispatch(c, ld, 1, 0));
    EpLLCombineArgs lc;
    memset(&lc, 0, sizeof(lc));
    ok(launch_ep_ll_combine(c, lc, 1, 0));
    RmsNormArgs lr;
    memset(&lr, 0, sizeof(lr));
    int dummy_shared = 0;
    for (bool fp8 : {false, true}) {
      ok(launch_ep_ll_combine_rmsnorm(c, lc, nullptr, lr, fp8, 1, 0));
      ok(launch_ep_ll_combine_rmsnorm(c, lc, &dummy_shared, lr, fp8, 1, 0));
    }
    EpLLPackArgs lp;
    memset(&lp, 0, sizeof(lp));
    ok(launch_ep_ll_pack(lp, 0));
    lp.logfmt = 1;
    lp.H = 128;
    ok(launch_ep_ll_pack(lp, 0));
  }
  ok(preload_p2p_kernels());
  ok(launch_smid_probe(nullptr, 1, 0, 0));
  ok(cmp_compress_async(nullptr, 0, kBF16, nullptr, 0));
  ok(cmp_compress_async(nullptr, 0, kF32, nullptr, 0));
  ok(cmp_decompress_async(nullptr, nullptr, 0, kBF16, 0));
  ok(cmp_decompress_async(nullptr, nullptr, 0, kF32, 0));
  {
    D2HQueueDev dq;
    memset(&dq, 0, sizeof(dq));
    ok(launch_d2h_bench(dq, 1, 32, 0, 0));
    ok(launch_d2h_latency(dq, 0, nullptr, 0));
    ok(launch_d2h_issue(dq, 0, 0, 0, 0, 0, 0, 0, 0));
    ok(launch_u64_add(nullptr, 0, 0));
  }
  {
    UkWorkerArgs uw;
    memset(&uw, 0, sizeof(uw));
    ok(launch_uk_worker(uw, 0));
  }
  g_preload = false;
  done_mask |= 1ull << (dev & 63);
  UB_INFO(SUB_INIT, "preloaded %d kernel functions", loaded);
  return cudaSuccess;
}

}  // namespace ub
