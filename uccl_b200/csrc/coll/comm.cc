#include "comm.h"

#include <algorithm>
#include <cstring>

#include "../common/log.h"
#include "../common/param.h"
#include "../fabric/cu_api.h"
#include "../kernels/launch.h"

namespace ub {

UB_PARAM(TimeoutMs, "TIMEOUT_MS", 20000)
UB_PARAM(MaxCtas, "MAX_CTAS", 128)
UB_PARAM(ArLLMaxBytes, "AR_LL_MAX_BYTES", 0)  // 0: per-world-size default
UB_PARAM(ArP2PMinBytes, "AR_P2P_MIN_BYTES", -1)  // symmetric buffers >= this use twoshot_p2p even with NVLS (-1: default)
UB_PARAM(ArForceAlgo, "AR_ALGO", 0)
// LL-packet AllGather / AllToAll / ReduceScatter for per-rank pieces up to this many bytes
// (0: per-world-size default, -1: never)
UB_PARAM(XchgLLMaxBytes, "XCHG_LL_MAX_BYTES", 0)
UB_PARAM(RsPush, "RS_PUSH", 1)  // staged ReduceScatter: 1 = push into the peers' stages (default), 0 = copy-in + pull
UB_PARAM(NvlsCtas, "NVLS_CTAS", 0)  // 0: 256 / nranks
// 1: a one-rank communicator launches the real kernels instead of a cudaMemcpy (profiling / smoke tests on one GPU)
UB_PARAM(ForceKernels, "FORCE_KERNELS", 0)
UB_PARAM(NvlsUnroll, "NVLS_UNROLL", 4)  // multimem.ld_reduce in flight per thread of twoshot_nvls (4 or 8)
// plain (non-symmetric) buffers of at least this size take the block-pipelined staged kernel (needs NVLS, > 2 ranks)
UB_PARAM(ArPipeMinBytes, "AR_PIPE_MIN_BYTES", 512 << 20)  // from 8-GPU sweeps of benchmarks/allreduce_perf.py: wins at 1 GiB, loses at 256 MiB

const char* algo_name(int algo) {
  switch (algo) {
    case ALGO_AUTO: return "auto";
    case ALGO_ONESHOT_LL: return "oneshot_ll";
    case ALGO_ONESHOT_MC: return "oneshot_mc";
    case ALGO_TWOSHOT_P2P: return "twoshot_p2p";
    case ALGO_TWOSHOT_NVLS: return "twoshot_nvls";
    case ALGO_STAGED_P2P: return "staged_p2p";
    case ALGO_STAGED_NVLS: return "staged_nvls";
    case ALGO_STAGED_PIPE: return "staged_pipe";
    default: return "?";
  }
}

namespace {
struct DeviceGuard {
  int prev = -1;
  bool active = false;
  explicit DeviceGuard(int dev) {
    if (dev < 0) return;
    if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) {
      cudaSetDevice(dev);
      active = true;
    }
  }
  ~DeviceGuard() {
    if (active) cudaSetDevice(prev);
  }
};
bool aligned16(const void* p) { return (((uintptr_t)p) & 15) == 0; }
bool is_float_dtype(int dt) { return dt == kF16 || dt == kF32 || dt == kF64 || dt == kBF16 || dt == kF8E4M3 || dt == kF8E5M2; }
}  // namespace

std::shared_ptr<Comm> Comm::create(const UniqueId& id, int rank, int nranks, int device, const CommConfig& cfg) {
  Bootstrap bs(id, rank, nranks);
  HeapLayout l = HeapLayout::make(cfg.stage_bytes);
  UB_CHECK(cfg.heap_bytes > l.user_off, "heap_bytes (%zu) must exceed the control+staging region (%lu)",
           cfg.heap_bytes, (unsigned long)l.user_off);
  auto f = Fabric::create(bs, device, cfg.heap_bytes, l.ctrl_bytes(), cfg.host_fake);
  std::shared_ptr<Comm> c(new Comm());
  c->init(f, cfg);
  bs.barrier();
  return c;
}

std::vector<std::shared_ptr<Comm>> Comm::create_local(const std::vector<int>& devices, const CommConfig& cfg) {
  HeapLayout l = HeapLayout::make(cfg.stage_bytes);
  UB_CHECK(cfg.heap_bytes > l.user_off, "heap_bytes (%zu) must exceed the control+staging region (%lu)",
           cfg.heap_bytes, (unsigned long)l.user_off);
  auto fs = Fabric::create_local(devices, cfg.heap_bytes, l.ctrl_bytes(), cfg.host_fake);
  std::vector<std::shared_ptr<Comm>> out;
  for (auto& f : fs) {
    std::shared_ptr<Comm> c(new Comm());
    c->init(f, cfg);
    out.push_back(c);
  }
  return out;
}

void Comm::init(std::shared_ptr<Fabric> f, const CommConfig& cfg) {
  fabric_ = f;
  cfg_ = cfg;
  layout_ = HeapLayout::make(cfg.stage_bytes);
  max_ctas_ = cfg.max_ctas > 0 ? cfg.max_ctas : (int)ubParamMaxCtas();
  max_ctas_ = std::min(max_ctas_, kMaxSyncBlocks);
  xchg_ll_max_ = ubParamXchgLLMaxBytes();
  rs_push_ = ubParamRsPush() != 0;
  memset(&dev_, 0, sizeof(dev_));
  dev_.rank = f->rank();
  dev_.nranks = f->nranks();
  for (int r = 0; r < f->nranks(); ++r) dev_.heap[r] = f->heap(r);
  dev_.mc = f->mc();
  dev_.sig_off = layout_.sig_off;
  dev_.epoch_off = layout_.epoch_off;
  dev_.xchg_off = layout_.xchg_off;
  int64_t tmo = cfg.timeout_ms >= 0 ? cfg.timeout_ms : ubParamTimeoutMs();
  dev_.timeout_ns = (uint64_t)tmo * 1000000ull;
  if (!f->is_host()) {
    DeviceGuard g(f->device());
    void* h = nullptr;
    if (cudaHostAlloc(&h, 64, cudaHostAllocMapped) == cudaSuccess) {
      memset(h, 0, 64);
      err_host_ = (uint32_t*)h;
      void* d = nullptr;
      if (cudaHostGetDevicePointer(&d, h, 0) == cudaSuccess) dev_.err = (uint32_t*)d;
    } else {
      (void)cudaGetLastError();
    }
  }
  if (!f->is_host()) {
    DeviceGuard g(f->device());
    preload_all_kernels();
  }
  free_[layout_.user_off] = f->heap_bytes() - layout_.user_off;
  UB_INFO(SUB_INIT, "%s", describe().c_str());
}

Comm::~Comm() {
  if (err_host_) cudaFreeHost(err_host_);
  if (trace_dev_) cudaFree(trace_dev_);
}

void Comm::enable_trace(size_t max_events) {
  UB_CHECK(!is_host(), "tracing needs a CUDA communicator");
  DeviceGuard g(device());
  disable_trace();
  UB_CUDA(cudaMalloc((void**)&trace_dev_, (2 + 2 * max_events) * sizeof(unsigned long long)));
  UB_CUDA(cudaMemset(trace_dev_, 0, (2 + 2 * max_events) * sizeof(unsigned long long)));
  trace_cap_ = max_events;
  dev_.trace = trace_dev_;
  dev_.trace_cap = (uint32_t)max_events;
}

void Comm::disable_trace() {
  if (trace_dev_) {
    DeviceGuard g(device());
    cudaDeviceSynchronize();
    cudaFree(trace_dev_);
  }
  trace_dev_ = nullptr;
  trace_cap_ = 0;
  dev_.trace = nullptr;
  dev_.trace_cap = 0;
}

std::vector<Comm::TraceEvent> Comm::dump_trace(bool reset) {
  std::vector<TraceEvent> out;
  if (!trace_dev_) return out;
  DeviceGuard g(device());
  UB_CUDA(cudaDeviceSynchronize());
  std::vector<unsigned long long> h(2 + 2 * trace_cap_);
  UB_CUDA(cudaMemcpy(h.data(), trace_dev_, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  const size_t n = std::min<size_t>((size_t)h[0], trace_cap_);
  out.reserve(n);
  for (size_t i = 0; i < n; ++i) {
    const unsigned long long tag = h[3 + 2 * i];
    out.push_back(TraceEvent{h[2 + 2 * i], (uint32_t)(tag >> 48), (uint32_t)((tag >> 32) & 0xffff), (uint32_t)(tag & 0xffffffffu)});
  }
  std::sort(out.begin(), out.end(), [](const TraceEvent& a, const TraceEvent& b) { return a.t_ns < b.t_ns; });
  if (reset) UB_CUDA(cudaMemset(trace_dev_, 0, 2 * sizeof(unsigned long long)));
  return out;
}

std::string Comm::describe() const {
  char b[320];
  snprintf(b, sizeof(b), "Comm(rank=%d/%d, dev=%d, heap=%zuMiB user_off=%luMiB stage=%luMiB, nvls=%d, max_ctas=%d)",
           rank(), nranks(), device(), fabric_->heap_bytes() >> 20, (unsigned long)(layout_.user_off >> 20),
           (unsigned long)(layout_.stage_bytes >> 20), has_multicast() ? 1 : 0, max_ctas_);
  return std::string(b);
}

// ------------------------------------------------------------- heap allocator
void* Comm::alloc(size_t bytes, size_t align) {
  std::lock_guard<std::mutex> g(mu_);
  if (align < 256) align = 256;
  bytes = (bytes + 255) / 256 * 256;
  if (bytes == 0) bytes = 256;
  for (auto it = free_.begin(); it != free_.end(); ++it) {
    uint64_t off = it->first, sz = it->second;
    uint64_t aoff = (off + align - 1) / align * align;
    if (aoff + bytes > off + sz) continue;
    free_.erase(it);
    if (aoff > off) free_[off] = aoff - off;
    if (aoff + bytes < off + sz) free_[aoff + bytes] = off + sz - (aoff + bytes);
    used_[aoff] = bytes;
    return fabric_->local() + aoff;
  }
  UB_THROW("symmetric heap exhausted: need %zu bytes (heap %zu MiB); raise heap_bytes", bytes,
           fabric_->heap_bytes() >> 20);
}

void Comm::free(void* p) {
  if (!p) return;
  std::lock_guard<std::mutex> g(mu_);
  uint64_t off = fabric_->offset_of(p);
  auto it = used_.find(off);
  UB_CHECK(it != used_.end(), "free(): pointer %p was not allocated from this heap", p);
  uint64_t sz = it->second;
  used_.erase(it);
  auto ins = free_.emplace(off, sz).first;
  // coalesce with next / previous
  auto nx = std::next(ins);
  if (nx != free_.end() && ins->first + ins->second == nx->first) {
    ins->second += nx->second;
    free_.erase(nx);
  }
  if (ins != free_.begin()) {
    auto pv = std::prev(ins);
    if (pv->first + pv->second == ins->first) {
      pv->second += ins->second;
      free_.erase(ins);
    }
  }
}

size_t Comm::heap_free_bytes() const {
  std::lock_guard<std::mutex> g(mu_);
  size_t t = 0;
  for (auto& kv : free_) t += kv.second;
  return t;
}

// ------------------------------------------------------------------ helpers
CollArgs Comm::base_args() const {
  CollArgs a;
  memset(&a, 0, sizeof(a));
  a.in_off = kNoOff;
  a.out_off = kNoOff;
  a.ep.scale = 1.0f;
  a.ep.idiv = 1;
  a.misc_off = layout_.misc_off;
  a.ll_off = layout_.ll_off;
  a.stage_in_off = layout_.stage_in_off;
  a.stage_out_off = layout_.stage_out_off;
  a.stage_bytes = layout_.stage_bytes;
  return a;
}

int Comm::nvls_ctas() const {
  // bytes in flight needed per rank ~ (algbw / nranks) x multimem latency  =>  CTAs ~ 1 / nranks
  int64_t v = ubParamNvlsCtas();
  if (v <= 0) v = 256 / std::max(1, nranks());
  return (int)std::max<int64_t>(8, std::min<int64_t>(v, max_ctas_));
}

int Comm::ctas_for(uint64_t bytes, int cap, int per_cta_bytes) const {
  uint64_t c = (bytes + per_cta_bytes - 1) / per_cta_bytes;
  if (c < 1) c = 1;
  if (c > (uint64_t)cap) c = cap;
  return (int)c;
}

void Comm::check_buf(const void* p, const char* what) const {
  UB_CHECK(p != nullptr, "%s is null", what);
}

void Comm::set_tuning(bool symmetric, const std::vector<TuneEntry>& table) {
  auto t = table;
  std::sort(t.begin(), t.end(), [](const TuneEntry& a, const TuneEntry& b) { return a.max_bytes < b.max_bytes; });
  (symmetric ? tune_sym_ : tune_unsym_) = t;
}

int Comm::select_allreduce(size_t bytes, bool symmetric, int dtype, int op, int* ctas) const {
  const int n = nranks();
  const bool mc = has_multicast();
  const bool nvls_ok = mc && nvls_reduce_supported(dtype, op);
  int algo = (int)ubParamArForceAlgo();
  int c = -1;
  if (algo == ALGO_AUTO) {
    const auto& tab = symmetric ? tune_sym_ : tune_unsym_;
    for (const auto& e : tab) {
      if (bytes <= e.max_bytes) {
        algo = e.algo;
        c = e.ctas;
        break;
      }
    }
  }
  if (algo == ALGO_AUTO) {
    // defaults from benchmarks/allreduce_perf.py sweeps on NVSwitch boxes: the packet path wins
    // until its N-fold traffic outweighs the two barriers of the two-shot kernels
    uint64_t ll_max = (uint64_t)ubParamArLLMaxBytes();
    // n = 2: the two barriers of the two-shot kernels dominate when both GPUs are driven by one host thread, so
    // packets carry up to the 1 MiB cap there; n = 4: ordinary buffers of 512 KiB - 1 MiB are slower through the
    // staged kernels than through NCCL, and the packet path has no barrier
    if (ll_max == 0) ll_max = n <= 4 ? (1u << 20) : (128u << 10);
    ll_max = std::min<uint64_t>(ll_max, kLLMaxData);
    // with 2 ranks the switch cannot reduce traffic (both paths move `size` per direction) and the
    // plain P2P kernel sustains more bytes in flight per SM than multimem.ld_reduce
    int64_t p2p_min = ubParamArP2PMinBytes();
    if (p2p_min < 0) p2p_min = n <= 2 ? (8 << 20) : INT64_MAX;
    if (bytes <= ll_max || n == 1) algo = mc ? ALGO_ONESHOT_MC : ALGO_ONESHOT_LL;
    else if (symmetric) algo = (nvls_ok && (int64_t)bytes < p2p_min) ? ALGO_TWOSHOT_NVLS : ALGO_TWOSHOT_P2P;
    else if (nvls_ok && n > 2)
      algo = ((int64_t)bytes >= ubParamArPipeMinBytes() && max_ctas_ >= 48 && layout_.stage_bytes >= (32u << 20))
                 ? ALGO_STAGED_PIPE : ALGO_STAGED_NVLS;
    else algo = ALGO_STAGED_P2P;
    if (n == 1 && bytes > kLLMaxData) algo = ALGO_STAGED_P2P;
  }
  // degrade gracefully when a tuned/forced choice is impossible here
  if ((algo == ALGO_ONESHOT_MC) && !mc) algo = ALGO_ONESHOT_LL;
  if ((algo == ALGO_TWOSHOT_NVLS) && !nvls_ok) algo = ALGO_TWOSHOT_P2P;
  if (algo == ALGO_STAGED_PIPE && (!nvls_ok || bytes % 16 != 0 || max_ctas_ < 12)) algo = ALGO_STAGED_NVLS;
  if ((algo == ALGO_STAGED_NVLS) && !nvls_ok) algo = ALGO_STAGED_P2P;
  if ((algo == ALGO_TWOSHOT_P2P || algo == ALGO_TWOSHOT_NVLS) && !symmetric)
    algo = (algo == ALGO_TWOSHOT_NVLS) ? ALGO_STAGED_NVLS : ALGO_STAGED_P2P;
  if ((algo == ALGO_ONESHOT_LL || algo == ALGO_ONESHOT_MC) && bytes > kLLMaxData)
    algo = symmetric ? (nvls_ok ? ALGO_TWOSHOT_NVLS : ALGO_TWOSHOT_P2P) : (nvls_ok ? ALGO_STAGED_NVLS : ALGO_STAGED_P2P);
  if (c <= 0) {
    switch (algo) {
      case ALGO_ONESHOT_LL:
      case ALGO_ONESHOT_MC: c = ctas_for(bytes, std::min(max_ctas_, 64), 8192); break;  // 512 thr x 16 B
      case ALGO_TWOSHOT_NVLS: c = ctas_for(bytes, nvls_ctas(), 64 << 10); break;
      case ALGO_STAGED_PIPE: c = std::min(max_ctas_, 112); break;  // split into the three groups at launch
      case ALGO_STAGED_NVLS:
      case ALGO_STAGED_P2P: c = ctas_for(bytes, max_ctas_, 64 << 10); break;
      default: c = ctas_for(bytes, max_ctas_, 128 << 10); break;
    }
  }
  c = std::max(1, std::min(c, std::min(max_ctas_, kMaxSyncBlocks)));
  if (ctas) *ctas = c;
  return algo;
}

static cudaError_t launch_ar_any(int algo, int dtype, int op, int out_dtype, const DevComm& d, const CollArgs& a,
                                 int grid, int block, cudaStream_t st) {
  switch (dtype) {
    case kF32: case kBF16: case kF16: return launch_allreduce_f(algo, dtype, op, out_dtype, d, a, grid, block, st);
    case kI8: case kU8: case kI32: case kU32: case kI64: case kU64:
      if (out_dtype != dtype) return cudaErrorInvalidValue;
      return launch_allreduce_i(algo, dtype, op, d, a, grid, block, st);
    default:
      if (out_dtype != dtype) return cudaErrorInvalidValue;
      return launch_allreduce_x(algo, dtype, op, d, a, grid, block, st);
  }
}

// per-rank piece size up to which the barrier-free LL exchange kernels are used
static uint64_t xchg_ll_limit(int64_t v, int n, bool symmetric_push) {
  if (v < 0) return 0;
  uint64_t m = v > 0 ? (uint64_t)v : (n <= 4 ? (256u << 10) : (128u << 10));  // 4 ranks: a staged 1 MiB reduce_scatter was slower than NCCL
  if (v == 0 && symmetric_push) m = 32u << 10;  // the push kernels only pay one barrier
  return std::min<uint64_t>(m, kLLMaxData);
}

// ------------------------------------------------------------------ allreduce
void Comm::allreduce(const void* in, void* out, size_t count, int dtype, int op, cudaStream_t stream,
                     const ArOpts& opts) {
  UB_CHECK(dtype >= 0 && dtype < kNumDTypes, "allreduce: bad dtype %d", dtype);
  UB_CHECK(op >= 0 && op < kNumOps, "allreduce: bad op %d", op);
  if (count == 0) return;
  check_buf(in, "sendbuff");
  check_buf(out, "recvbuff");
  const int n = nranks();
  const int out_dtype = opts.out_dtype < 0 ? dtype : opts.out_dtype;
  const size_t esize = dtype_size(dtype), osize = dtype_size(out_dtype);
  const size_t bytes = count * esize, out_bytes = count * osize;
  float scale = opts.scale;
  int idiv = 1;
  if (op == kAvg) {
    if (is_float_dtype(dtype)) scale *= 1.0f / (float)n;
    else idiv = n;
  }
  if (is_host()) {
    host_allreduce(in, out, count, dtype, op, is_float_dtype(dtype) ? scale : 1.0f, out_dtype);
    return;
  }
  DeviceGuard g(device());
  if (!ubParamForceKernels() && n == 1 && out_dtype == dtype && scale == 1.0f && idiv == 1) {
    if (in != out) UB_CUDA(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice, stream));
    return;
  }
  UB_CHECK(aligned16(in) && aligned16(out), "allreduce: buffers must be 16-byte aligned (in=%p out=%p)", in, out);
  const bool sym = in_heap(in, bytes) && in_heap(out, out_bytes);
  int ctas = 0;
  int algo = opts.algo != ALGO_AUTO ? opts.algo : ALGO_AUTO;
  if (algo == ALGO_AUTO) {
    algo = select_allreduce(bytes, sym, dtype, op, &ctas);
  } else {
    (void)select_allreduce(bytes, sym, dtype, op, &ctas);
    // validate a forced choice
    if (algo == ALGO_ONESHOT_MC || algo == ALGO_TWOSHOT_NVLS || algo == ALGO_STAGED_NVLS || algo == ALGO_STAGED_PIPE)
      UB_CHECK(has_multicast(), "allreduce: algo %s needs NVLS multicast", algo_name(algo));
    if (algo == ALGO_STAGED_PIPE)
      UB_CHECK(bytes % 16 == 0 && out_dtype == dtype && max_ctas_ >= 12,
               "allreduce: staged_pipe needs 16-byte multiples, no fused cast and >= 12 CTAs");
    if (algo == ALGO_TWOSHOT_NVLS || algo == ALGO_STAGED_NVLS || algo == ALGO_STAGED_PIPE)
      UB_CHECK(nvls_reduce_supported(dtype, op), "allreduce: NVLS cannot reduce dtype %d op %d", dtype, op);
    if (algo == ALGO_TWOSHOT_P2P || algo == ALGO_TWOSHOT_NVLS)
      UB_CHECK(sym, "allreduce: algo %s needs buffers from the symmetric heap", algo_name(algo));
    if (algo == ALGO_ONESHOT_LL || algo == ALGO_ONESHOT_MC)
      UB_CHECK(bytes <= kLLMaxData, "allreduce: one-shot limited to %lu bytes", (unsigned long)kLLMaxData);
    if (algo == ALGO_ONESHOT_LL || algo == ALGO_ONESHOT_MC) ctas = ctas_for(bytes, std::min(max_ctas_, 64), 8192);
    else if (algo == ALGO_TWOSHOT_NVLS) ctas = ctas_for(bytes, nvls_ctas(), 64 << 10);
    else if (algo == ALGO_STAGED_PIPE) ctas = std::min(max_ctas_, 112);
    else if (algo == ALGO_STAGED_NVLS || algo == ALGO_STAGED_P2P) ctas = ctas_for(bytes, max_ctas_, 64 << 10);
    else ctas = ctas_for(bytes, max_ctas_, 128 << 10);
  }
  if (opts.max_ctas > 0) ctas = std::min(ctas, opts.max_ctas);
  if (algo == ALGO_STAGED_PIPE && (out_dtype != dtype || ctas < 12)) algo = ALGO_STAGED_NVLS;
  if (out_dtype != dtype) {
    if (algo == ALGO_ONESHOT_LL || algo == ALGO_ONESHOT_MC)
      algo = sym ? ALGO_TWOSHOT_P2P : ALGO_STAGED_P2P;  // cast is fused only in the two-shot/staged kernels
    UB_CHECK(bytes % 16 == 0 && out_bytes % 16 == 0,
             "allreduce with fused cast needs 16-byte multiples on both sides (count=%zu)", count);
  }

  CollArgs a = base_args();
  a.ep.scale = scale;
  a.ep.idiv = idiv;
  const bool oneshot = (algo == ALGO_ONESHOT_LL || algo == ALGO_ONESHOT_MC);
  const size_t main_bytes = oneshot ? bytes : (bytes / 16 * 16);
  const int block = 512;
  if (main_bytes) {
    a.in = in;
    a.out = out;
    a.bytes = main_bytes;
    a.count = main_bytes / esize;
    if (sym) {
      a.in_off = heap_offset(in);
      a.out_off = heap_offset(out);
    }
    if (algo == ALGO_TWOSHOT_NVLS) a.variant = ubParamNvlsUnroll() >= 8 ? 8 : 4;
    if (algo == ALGO_STAGED_PIPE) {
      // the in-switch reduce saturates with ~32 CTAs; the copy groups get the rest (they bound the fill / drain time)
      const int nB = std::max(4, std::min(32, ctas * 2 / 5)), nA = std::max(4, (ctas - nB) / 2), nC = std::max(4, ctas - nB - nA);
      a.variant = nB | (nA << 8) | (nC << 16);
      ctas = nA + nB + nC;
    }
    cudaError_t e = launch_ar_any(algo, dtype, op, out_dtype, dev_, a, ctas, block, stream);
    if (e != cudaSuccess) {
      int cur = -1;
      cudaGetDevice(&cur);
      CUcontext cctx = nullptr, sctx = nullptr;
      CUdevice cdev = -1;
      if (cu().CtxGetCurrent) cu().CtxGetCurrent(&cctx);
      if (cu().CtxGetDevice) cu().CtxGetDevice(&cdev);
      if (cu().StreamGetCtx) cu().StreamGetCtx((CUstream)stream, &sctx);
      UB_THROW("allreduce launch failed (rank %d algo=%s dtype=%d op=%d ctas=%d, comm device %d, current device %d, "
               "driver ctx %p on device %d, stream %p in ctx %p): %s",
               rank(), algo_name(algo), dtype, op, ctas, device(), cur, (void*)cctx, (int)cdev, (void*)stream,
               (void*)sctx, cudaGetErrorString(e));
    }
    ++launches_;
  }
  if (main_bytes < bytes) {  // < 16-byte tail through the packet path
    CollArgs t = base_args();
    t.ep = a.ep;
    t.in = (const char*)in + main_bytes;
    t.out = (char*)out + main_bytes;
    t.bytes = bytes - main_bytes;
    t.count = t.bytes / esize;
    cudaError_t e = launch_ar_any(has_multicast() ? ALGO_ONESHOT_MC : ALGO_ONESHOT_LL, dtype, op, dtype, dev_, t, 1,
                                  block, stream);
    UB_CHECK(e == cudaSuccess, "allreduce tail launch failed: %s", cudaGetErrorString(e));
    ++launches_;
  }
  UB_TRACE(SUB_COLL, "allreduce bytes=%zu algo=%s ctas=%d sym=%d", bytes, algo_name(algo), ctas, sym ? 1 : 0);
}

// ------------------------------------------------------------------ allgather
void Comm::allgather(const void* in, void* out, size_t count_per_rank, int dtype, cudaStream_t stream) {
  UB_CHECK(dtype >= 0 && dtype < kNumDTypes, "allgather: bad dtype %d", dtype);
  if (count_per_rank == 0) return;
  check_buf(in, "sendbuff");
  check_buf(out, "recvbuff");
  const int n = nranks();
  const size_t bytes = count_per_rank * dtype_size(dtype);
  if (is_host()) {
    host_allgather(in, out, bytes);
    return;
  }
  DeviceGuard g(device());
  if (!ubParamForceKernels() && n == 1) {
    if (in != out) UB_CUDA(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice, stream));
    return;
  }
  UB_CHECK(aligned16(in) && aligned16(out), "allgather: buffers must be 16-byte aligned");
  CollArgs a = base_args();
  a.in = in;
  a.out = out;
  a.bytes = bytes;
  a.count = count_per_rank;
  const bool out_sym = in_heap(out, bytes * n);
  const bool in_sym = in_heap(in, bytes);
  int mode;
  int ctas;
  const bool ll_mc = has_multicast() && n > 2;
  // with multicast one multimem.st publishes a packet to every peer, which keeps the LL path ahead
  // of the barrier-based kernels up to 512 KiB pieces (8-GPU all-gather sweeps)
  uint64_t ag_ll_max = xchg_ll_limit(xchg_ll_max_, n, out_sym && !ll_mc);
  if (xchg_ll_max_ == 0 && ll_mc) ag_ll_max = std::min<uint64_t>(512u << 10, kLLMaxData);
  if (bytes % 16 == 0 && bytes <= ag_ll_max) {
    mode = ll_mc ? 4 : 3;
    ctas = ctas_for(bytes * (uint64_t)(n - 1), std::min(max_ctas_, 64), 16 << 10);
  } else if (out_sym && bytes % 16 == 0) {
    a.out_off = heap_offset(out);
    mode = (has_multicast() && n > 2) ? 1 : 0;  // with 2 ranks multicast saves nothing and issues slower
    ctas = ctas_for(bytes, max_ctas_, 64 << 10);
  } else {
    mode = 2;
    if (in_sym) a.in_off = heap_offset(in);
    ctas = ctas_for(bytes * (uint64_t)n, max_ctas_, 64 << 10);  // every CTA moves a slice of all n pieces
  }
  cudaError_t e = launch_allgather(mode, dev_, a, ctas, 512, stream);
  UB_CHECK(e == cudaSuccess, "allgather launch failed: %s", cudaGetErrorString(e));
  ++launches_;
}

// ------------------------------------------------------------- reduce_scatter
void Comm::reduce_scatter(const void* in, void* out, size_t recv_count, int dtype, int op, cudaStream_t stream,
                          float scale) {
  UB_CHECK(dtype >= 0 && dtype < kNumDTypes, "reduce_scatter: bad dtype %d", dtype);
  UB_CHECK(op >= 0 && op < kNumOps, "reduce_scatter: bad op %d", op);
  if (recv_count == 0) return;
  check_buf(in, "sendbuff");
  check_buf(out, "recvbuff");
  const int n = nranks();
  const size_t bytes = recv_count * dtype_size(dtype);
  UB_CHECK(scale == 1.0f || is_float_dtype(dtype), "reduce_scatter: scale needs a floating-point dtype");
  if (is_host()) {
    UB_CHECK(scale == 1.0f, "host backend: fused scale unsupported");
    host_reduce_scatter(in, out, recv_count, dtype, op);
    return;
  }
  DeviceGuard g(device());
  CollArgs a = base_args();
  a.ep.scale = scale;
  if (op == kAvg) {
    if (is_float_dtype(dtype)) a.ep.scale *= 1.0f / (float)n;
    else a.ep.idiv = n;
  }
  if (!ubParamForceKernels() && n == 1 && op != kAvg && scale == 1.0f) {
    if (in != out) UB_CUDA(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice, stream));
    return;
  }
  UB_CHECK(aligned16(in) && aligned16(out), "reduce_scatter: buffers must be 16-byte aligned");
  a.in = in;
  a.out = out;
  a.bytes = bytes;
  a.count = recv_count;
  const bool in_sym = in_heap(in, bytes * n) && (bytes % 16 == 0);
  if (in_sym) a.in_off = heap_offset(in);
  // staged input: pushing pieces into the peers' stages wins except for very large messages on
  // NVLS systems, where copy-in + multimem.ld_reduce is ahead (8-GPU reduce-scatter sweeps, from 256 MiB)
  const bool nvls_possible = has_multicast() && nvls_reduce_supported(dtype, op) && n > 2;
  a.variant = (rs_push_ && !(nvls_possible && bytes * (uint64_t)n >= (256ull << 20))) ? 1 : 0;
  const bool nvls = has_multicast() && nvls_reduce_supported(dtype, op) && n > 2;
  const bool fdt =
      dtype == kF32 || dtype == kBF16 || dtype == kF16 || dtype == kF64 || dtype == kF8E4M3 || dtype == kF8E5M2;
  cudaError_t e;
  if (n > 1 && bytes % 16 == 0 && bytes <= xchg_ll_limit(xchg_ll_max_, n, false)) {
    const int ctas = ctas_for(bytes * (uint64_t)(n - 1), std::min(max_ctas_, 64), 16 << 10);
    e = fdt ? launch_rs_ll_f(dtype, op, dev_, a, ctas, 512, stream) : launch_rs_ll_i(dtype, op, dev_, a, ctas, 512, stream);
    UB_CHECK(e == cudaSuccess, "reduce_scatter (LL) launch failed: %s", cudaGetErrorString(e));
    ++launches_;
    return;
  }
  int ctas = ctas_for(in_sym ? bytes : bytes * (uint64_t)n, nvls && in_sym ? nvls_ctas() : max_ctas_, 64 << 10);
  if (fdt) e = launch_red_f(0, dtype, op, nvls, dev_, a, ctas, 512, stream);
  else e = launch_red_i(0, dtype, op, dev_, a, ctas, 512, stream);
  UB_CHECK(e == cudaSuccess, "reduce_scatter launch failed: %s", cudaGetErrorString(e));
  ++launches_;
}

// ------------------------------------------------------------------ broadcast
void Comm::broadcast(const void* in, void* out, size_t count, int dtype, int root, cudaStream_t stream) {
  UB_CHECK(dtype >= 0 && dtype < kNumDTypes, "broadcast: bad dtype %d", dtype);
  UB_CHECK(root >= 0 && root < nranks(), "broadcast: bad root %d", root);
  if (count == 0) return;
  check_buf(out, "recvbuff");
  const size_t bytes = count * dtype_size(dtype);
  if (rank() == root) check_buf(in, "sendbuff");
  if (is_host()) {
    host_broadcast(in, out, bytes, root);
    return;
  }
  DeviceGuard g(device());
  if (!ubParamForceKernels() && nranks() == 1) {
    if (in != out) UB_CUDA(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice, stream));
    return;
  }
  UB_CHECK(aligned16(out) && (rank() != root || aligned16(in)), "broadcast: buffers must be 16-byte aligned");
  CollArgs a = base_args();
  a.in = rank() == root ? in : out;
  a.out = out;
  a.bytes = bytes;
  a.count = count;
  a.root = root;
  int mode = 0;
  if (in_heap(out, bytes)) {
    a.out_off = heap_offset(out);
    mode = (has_multicast() && nranks() > 2) ? 1 : 2;
  } else if (has_multicast() && nranks() > 2 && bytes >= (256u << 10) && layout_.stage_bytes >= (2u << 20)) {
    mode = 3;  // ordinary output: multicast into the staging area, local copy-out (a pull is bound by the root's egress)
  }
  int ctas = ctas_for(bytes, max_ctas_, 64 << 10);
  cudaError_t e = launch_broadcast(mode, dev_, a, ctas, 512, stream);
  UB_CHECK(e == cudaSuccess, "broadcast launch failed: %s", cudaGetErrorString(e));
  ++launches_;
}

// --------------------------------------------------------------------- reduce
void Comm::reduce(const void* in, void* out, size_t count, int dtype, int op, int root, cudaStream_t stream,
                  float scale) {
  UB_CHECK(dtype >= 0 && dtype < kNumDTypes, "reduce: bad dtype %d", dtype);
  UB_CHECK(op >= 0 && op < kNumOps, "reduce: bad op %d", op);
  UB_CHECK(root >= 0 && root < nranks(), "reduce: bad root %d", root);
  if (count == 0) return;
  check_buf(in, "sendbuff");
  if (rank() == root) check_buf(out, "recvbuff");
  const int n = nranks();
  const size_t bytes = count * dtype_size(dtype);
  UB_CHECK(scale == 1.0f || is_float_dtype(dtype), "reduce: scale needs a floating-point dtype");
  if (is_host()) {
    UB_CHECK(scale == 1.0f, "host backend: fused scale unsupported");
    host_reduce(in, out, count, dtype, op, root);
    return;
  }
  DeviceGuard g(device());
  CollArgs a = base_args();
  a.ep.scale = scale;
  if (op == kAvg) {
    if (is_float_dtype(dtype)) a.ep.scale *= 1.0f / (float)n;
    else a.ep.idiv = n;
  }
  if (!ubParamForceKernels() && n == 1 && op != kAvg && scale == 1.0f) {
    if (in != out) UB_CUDA(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice, stream));
    return;
  }
  UB_CHECK(aligned16(in) && (rank() != root || aligned16(out)), "reduce: buffers must be 16-byte aligned");
  a.in = in;
  a.out = rank() == root ? out : const_cast<void*>(in);
  a.bytes = bytes;
  a.count = count;
  a.root = root;
  if (in_heap(in, bytes)) a.in_off = heap_offset(in);
  const bool nvls = has_multicast() && nvls_reduce_supported(dtype, op) && n > 2;
  int ctas = ctas_for(bytes, max_ctas_, 64 << 10);
  cudaError_t e;
  if (is_float_dtype(dtype)) e = launch_red_f(1, dtype, op, nvls, dev_, a, ctas, 512, stream);
  else e = launch_red_i(1, dtype, op, dev_, a, ctas, 512, stream);
  UB_CHECK(e == cudaSuccess, "reduce launch failed: %s", cudaGetErrorString(e));
  ++launches_;
}

// ------------------------------------------------------------------- alltoall
void Comm::alltoall(const void* in, void* out, size_t count_per_peer, int dtype, cudaStream_t stream) {
  UB_CHECK(dtype >= 0 && dtype < kNumDTypes, "alltoall: bad dtype %d", dtype);
  if (count_per_peer == 0) return;
  check_buf(in, "sendbuff");
  check_buf(out, "recvbuff");
  const int n = nranks();
  const size_t bytes = count_per_peer * dtype_size(dtype);
  if (is_host()) {
    host_alltoall(in, out, bytes);
    return;
  }
  DeviceGuard g(device());
  if (!ubParamForceKernels() && n == 1) {
    if (in != out) UB_CUDA(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice, stream));
    return;
  }
  UB_CHECK(in != out, "alltoall: in-place operation is not supported");
  UB_CHECK(aligned16(in) && aligned16(out), "alltoall: buffers must be 16-byte aligned");
  CollArgs a = base_args();
  a.in = in;
  a.out = out;
  a.bytes = bytes;
  a.count = count_per_peer;
  int mode = 0;
  int ctas = ctas_for(bytes * (uint64_t)n, max_ctas_, 64 << 10);
  const bool out_sym = in_heap(out, bytes * n);
  if (bytes % 16 == 0 && bytes <= xchg_ll_limit(xchg_ll_max_, n, out_sym)) {
    mode = 2;
    ctas = ctas_for(bytes * (uint64_t)(n - 1), std::min(max_ctas_, 64), 16 << 10);
  } else if (out_sym) {
    a.out_off = heap_offset(out);
    mode = 1;
  } else if (in_heap(in, bytes * n)) {
    a.in_off = heap_offset(in);
  }
  cudaError_t e = launch_alltoall(mode, dev_, a, ctas, 512, stream);
  UB_CHECK(e == cudaSuccess, "alltoall launch failed: %s", cudaGetErrorString(e));
  ++launches_;
}

void Comm::alltoallv(const void* in, const size_t* send_counts, const size_t* send_displs, void* out,
                     const size_t* recv_counts, const size_t* recv_displs, int dtype, cudaStream_t stream) {
  UB_CHECK(dtype >= 0 && dtype < kNumDTypes, "alltoallv: bad dtype %d", dtype);
  const int n = nranks();
  const size_t es = dtype_size(dtype);
  if (is_host()) {
    std::vector<size_t> sb(n), so(n), rb(n), ro(n);
    for (int p = 0; p < n; ++p) {
      sb[p] = send_counts[p] * es, so[p] = send_displs[p] * es;
      rb[p] = recv_counts[p] * es, ro[p] = recv_displs[p] * es;
    }
    host_alltoallv(in, sb.data(), so.data(), out, rb.data(), ro.data());
    return;
  }
  DeviceGuard g(device());
  size_t in_total = 0;
  for (int p = 0; p < n; ++p) in_total = std::max(in_total, (send_displs[p] + send_counts[p]) * es);
  if (!ubParamForceKernels() && n == 1) {
    size_t b = std::min(send_counts[0], recv_counts[0]) * es;
    if (b) UB_CUDA(cudaMemcpyAsync((char*)out + recv_displs[0] * es, (const char*)in + send_displs[0] * es, b,
                                   cudaMemcpyDeviceToDevice, stream));
    return;
  }
  CollArgs a = base_args();
  a.out = out;
  a.in = in;
  if (in_heap(in, in_total)) {
    a.in_off = heap_offset(in);
  } else {
    // stage the send buffer once into the heap staging area (must fit)
    UB_CHECK(in_total <= layout_.stage_bytes,
             "alltoallv: non-symmetric send buffer (%zu B) exceeds the staging area (%lu B); allocate it from the "
             "symmetric heap or raise stage_bytes",
             in_total, (unsigned long)layout_.stage_bytes);
    if (in_total)
      UB_CUDA(cudaMemcpyAsync(fabric_->local() + layout_.stage_in_off, in, in_total, cudaMemcpyDeviceToDevice,
                              stream));
    a.in_off = layout_.stage_in_off;
  }
  A2AvArgs v;
  memset(&v, 0, sizeof(v));
  size_t maxb = 0;
  for (int p = 0; p < n; ++p) {
    v.send_off[p] = send_displs[p] * es;
    v.send_bytes[p] = send_counts[p] * es;
    v.recv_off[p] = recv_displs[p] * es;
    v.recv_bytes[p] = recv_counts[p] * es;
    maxb = std::max(maxb, (size_t)v.recv_bytes[p]);
  }
  v.table_off = layout_.a2av_tab_off;
  int ctas = ctas_for(maxb, max_ctas_, 32 << 10);
  cudaError_t e = launch_alltoallv(dev_, a, v, ctas, 512, stream);
  UB_CHECK(e == cudaSuccess, "alltoallv launch failed: %s", cudaGetErrorString(e));
  ++launches_;
}

void Comm::group_p2p(const std::vector<P2pOp>& ops, cudaStream_t stream) {
  if (ops.empty()) return;
  if (is_host()) {
    host_group_p2p(ops);
    return;
  }
  const int n = nranks();
  std::vector<std::vector<const P2pOp*>> sends(n), recvs(n);
  for (const auto& o : ops) {
    UB_CHECK(o.peer >= 0 && o.peer < n, "send/recv: bad peer %d", o.peer);
    UB_CHECK(o.buf != nullptr || o.bytes == 0, "send/recv: null buffer");
    UB_CHECK((((uintptr_t)o.buf) & 15) == 0, "send/recv: buffers must be 16-byte aligned");
    (o.is_send ? sends : recvs)[o.peer].push_back(&o);
  }
  size_t rounds = 0;
  for (int p = 0; p < n; ++p) rounds = std::max(rounds, std::max(sends[p].size(), recvs[p].size()));
  DeviceGuard g(device());
  for (size_t r = 0; r < rounds; ++r) {
    SendRecvArgs a;
    memset(&a, 0, sizeof(a));
    a.sr_flag_off = layout_.sr_flag_off;
    a.sr_stage_off = layout_.sr_stage_off;
    for (int p = 0; p < n; ++p) {
      const P2pOp* s = r < sends[p].size() ? sends[p][r] : nullptr;
      const P2pOp* v = r < recvs[p].size() ? recvs[p][r] : nullptr;
      if ((!s || s->bytes == 0) && (!v || v->bytes == 0)) continue;
      a.s_off[p] = kNoOff;
      if (s) {
        a.sbuf[p] = (const char*)s->buf;
        a.sbytes[p] = s->bytes;
        // a source inside the symmetric heap is pulled by the receiver straight from where it is (no staging)
        if (s->bytes && in_heap(s->buf, s->bytes)) a.s_off[p] = heap_offset(s->buf);
      }
      if (v) {
        a.rbuf[p] = (char*)v->buf;
        a.rbytes[p] = v->bytes;
      }
      if (p == rank()) UB_CHECK(s && v, "send/recv to self must be posted as a matching pair in one group");
      a.peers[a.npeers++] = p;
    }
    if (a.npeers == 0) continue;
    cudaError_t e = launch_sendrecv(dev_, a, stream);
    UB_CHECK(e == cudaSuccess, "send/recv launch failed: %s", cudaGetErrorString(e));
    ++launches_;
  }
}

void Comm::barrier(cudaStream_t stream) {
  if (is_host()) {
    host_barrier();
    return;
  }
  if (nranks() == 1) return;
  DeviceGuard g(device());
  cudaError_t e = launch_barrier(dev_, kDomUser0, stream);
  UB_CHECK(e == cudaSuccess, "barrier launch failed: %s", cudaGetErrorString(e));
  ++launches_;
}

}  // namespace ub
