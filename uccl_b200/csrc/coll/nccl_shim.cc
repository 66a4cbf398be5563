// NCCL-API drop-in: exports the nccl.h symbol set on top of the native communicator, so code
// written against NCCL (nccl-tests style harnesses, frameworks that dlopen/LD_PRELOAD libnccl)
// runs on the hand-written sm_90a kernels.
//
// Reference counterpart: experimental/lite/nccl/nccl.cu:1351-2430 (which falls back to a
// dlopen'd NCCL for ReduceScatter/Reduce and leaves AllToAll(v)/PreMulSum/CommAbort as stubs).
// Differences here: every collective incl. ReduceScatter / Reduce / Send / Recv is native; the
// buffers may be ordinary cudaMalloc memory (staged kernels) or come from ncclMemAlloc
// (symmetric heap -> zero-copy kernels); ncclCommInitAll supports ndev > 1 (single-process world).
//
// UCCL_B200_HOST_FAKE=1 selects the host backend (pointers are host memory, streams ignored):
// this is the GPU-less CI configuration "NCCL-API allreduce correctness world_size=2 on CPU".
#include <nccl.h>

#include <cmath>
#include <cstring>
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <vector>

#include "../common/log.h"
#include "../common/param.h"
#include "comm.h"
#include "multi_comm.h"
#include "nccl_fallback.h"
#include "../fabric/cu_api.h"
#include <algorithm>

using namespace ub;

UB_PARAM(ShimHeapMB, "NCCL_HEAP_MB", 2048)
UB_PARAM(ShimStageMB, "NCCL_STAGE_MB", 128)
UB_PARAM(ShimHostFake, "HOST_FAKE", 0)

struct ncclComm {
  std::shared_ptr<Comm> comm;        // one NVLink domain ...
  std::shared_ptr<MultiComm> multi;  // ... or a group that spans boxes (then `comm` is null)
  std::map<int, float> premul;  // user-created PreMulSum ops: op id -> scalar
  int next_op = (int)ncclNumOps;
  std::string last_error;
  ncclResult_t async_error = ncclSuccess;
  bool finalized = false;
  std::unique_ptr<NcclFallback> fallback;  // optional dlopen'd libnccl for the operations named in UCCL_B200_NCCL_FALLBACK_OPS
};

namespace {

std::mutex g_mu;
std::set<ncclComm*> g_comms;
thread_local int g_group_depth = 0;
struct PendingP2p {
  ncclComm* comm;
  Comm::P2pOp op;
  cudaStream_t stream;
  size_t count = 0;          // as given by the caller (forwarded verbatim when the communicator sends p2p to libnccl)
  ncclDataType_t dt = ncclChar;
};
thread_local std::vector<PendingP2p> g_pending;
thread_local std::string g_last_error;

CommConfig shim_config() {
  CommConfig cfg;
  cfg.heap_bytes = (size_t)ubParamShimHeapMB() << 20;
  cfg.stage_bytes = (size_t)ubParamShimStageMB() << 20;
  cfg.host_fake = ubParamShimHostFake() != 0;
  if (cfg.host_fake) {
    cfg.heap_bytes = std::min<size_t>(cfg.heap_bytes, 256ull << 20);
    cfg.stage_bytes = std::min<size_t>(cfg.stage_bytes, 8ull << 20);
  }
  return cfg;
}

template <typename F>
ncclResult_t guarded(ncclComm* c, F&& f) {
  try {
    f();
    return ncclSuccess;
  } catch (const std::exception& e) {
    g_last_error = e.what();
    if (c) c->last_error = e.what();
    const char* w = e.what();
    if (strstr(w, "bad ") || strstr(w, "null") || strstr(w, "must be") || strstr(w, "needs")) return ncclInvalidArgument;
    if (strstr(w, "cuda") || strstr(w, "CUDA") || strstr(w, "launch failed")) return ncclUnhandledCudaError;
    return ncclInternalError;
  }
}

bool valid(ncclComm_t c) { return c != nullptr && (c->comm != nullptr || c->multi != nullptr); }
// the NVLink-domain communicator behind a handle (for device / heap / error-word queries)
Comm* local_of(ncclComm_t c) { return c->multi ? c->multi->local().get() : c->comm.get(); }
int nranks_of(ncclComm_t c) { return c->multi ? c->multi->nranks() : c->comm->nranks(); }

// Ranks per NVLink domain when the job spans boxes: UCCL_B200_LOCAL_SIZE, else the launcher's hint.
int box_size_hint(int nranks) {
  int64_t v = param_load("LOCAL_SIZE", 0);
  if (v <= 0)
    for (const char* name : {"LOCAL_WORLD_SIZE", "OMPI_COMM_WORLD_LOCAL_SIZE", "SLURM_NTASKS_PER_NODE", "MPI_LOCALNRANKS"}) {
      const char* e = getenv(name);
      if (e && atoi(e) > 0) {
        v = atoi(e);
        break;
      }
    }
  if (v <= 0 && nranks > kMaxRanks) v = kMaxRanks;
  return (int)v;
}

// 128 bytes from rank 0 to everybody through the native communicator (device staging unless it is the host backend)
void share_from_rank0(Comm& c, void* buf128) {
  const int n = c.nranks();
  std::vector<char> all((size_t)n * 128);
  if (c.is_host()) {
    c.allgather(buf128, all.data(), 128, kU8, nullptr);
  } else {
    char *d_in = nullptr, *d_out = nullptr;
    UB_CUDA(cudaMalloc((void**)&d_in, 128));
    UB_CUDA(cudaMalloc((void**)&d_out, (size_t)n * 128));
    UB_CUDA(cudaMemcpy(d_in, buf128, 128, cudaMemcpyHostToDevice));
    c.allgather(d_in, d_out, 128, kU8, nullptr);
    UB_CUDA(cudaMemcpy(all.data(), d_out, (size_t)n * 128, cudaMemcpyDeviceToHost));
    cudaFree(d_in);
    cudaFree(d_out);
  }
  memcpy(buf128, all.data(), 128);
}

std::unique_ptr<NcclFallback> make_fallback(Comm& c) {
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  return NcclFallback::create(c.rank(), c.nranks(), [&](void* id) { share_from_rank0(c, id); });
}

ncclResult_t flush_group() {
  // launch queued send/recv per (comm, stream)
  std::vector<PendingP2p> pend;
  pend.swap(g_pending);
  ncclResult_t res = ncclSuccess;
  std::map<std::pair<ncclComm*, cudaStream_t>, std::vector<Comm::P2pOp>> by;
  std::map<ncclComm*, std::vector<PendingP2p*>> fwd;  // communicators whose send/recv go to the fallback library
  for (auto& p : pend) {
    if (p.comm->fallback && p.comm->fallback->takes(NcclFallback::kSendRecv, p.op.bytes)) fwd[p.comm].push_back(&p);
    else by[{p.comm, p.stream}].push_back(p.op);
  }
  for (auto& kv : fwd) {
    NcclFallback& fb = *kv.first->fallback;
    ncclResult_t r = fb.group_start();
    for (PendingP2p* p : kv.second) {
      if (r != ncclSuccess) break;
      r = p->op.is_send ? fb.send(p->op.buf, p->count, p->dt, p->op.peer, p->stream)
                        : fb.recv(p->op.buf, p->count, p->dt, p->op.peer, p->stream);
    }
    const ncclResult_t e = fb.group_end();
    if (r == ncclSuccess) r = e;
    if (r != ncclSuccess) res = r;
  }
  for (auto& kv : by) {
    ncclComm* c = kv.first.first;
    ncclResult_t r = guarded(c, [&] {
      if (c->multi) c->multi->group_p2p(kv.second, kv.first.second);
      else c->comm->group_p2p(kv.second, kv.first.second);
    });
    if (r != ncclSuccess) res = r;
  }
  return res;
}

// Does the communicator hand this collective to the fallback library?  `count` elements of `dt` is the message size
// NCCL's own tuning uses (all-gather / reduce-scatter: the whole buffer).  User-created PreMulSum operators only
// exist in this library, so they always stay native.
bool forwards(ncclComm_t c, NcclFallback::Op what, size_t count, ncclDataType_t dt, ncclRedOp_t op) {
  if (!c->fallback || (int)dt < 0 || (int)dt >= kNumDTypes || (int)op >= (int)ncclNumOps) return false;
  return c->fallback->takes(what, count * (size_t)dtype_size((int)dt));
}

}  // namespace

extern "C" {

#define UB_EXPORT __attribute__((visibility("default")))

UB_EXPORT ncclResult_t ncclGetVersion(int* version) {
  if (!version) return ncclInvalidArgument;
  *version = NCCL_VERSION_CODE;
  return ncclSuccess;
}

UB_EXPORT ncclResult_t ncclGetUniqueId(ncclUniqueId* uniqueId) {
  if (!uniqueId) return ncclInvalidArgument;
  static_assert(sizeof(ncclUniqueId) >= sizeof(UniqueId), "unique id does not fit");
  return guarded(nullptr, [&] {
    UniqueId id = Bootstrap::create_id();
    memset(uniqueId, 0, sizeof(*uniqueId));
    memcpy(uniqueId->internal, id.data, sizeof(id.data));
  });
}

// box_override: > 0 = ranks per box are known (ncclCommSplit derives them from the parent), 0 = use the hints
static ncclResult_t init_rank(ncclComm_t* comm, int nranks, ncclUniqueId commId, int rank, int box_override) {
  if (!comm || nranks < 1 || rank < 0 || rank >= nranks) return ncclInvalidArgument;
  const int box = box_override > 0 ? box_override : box_size_hint(nranks);
  const bool spans_boxes = box > 0 && box < nranks;
  if (spans_boxes && (nranks % box != 0 || box > kMaxRanks)) {
    g_last_error = "uccl_b200: " + std::to_string(nranks) + " ranks are not a multiple of the box size " + std::to_string(box);
    return ncclInvalidUsage;
  }
  *comm = nullptr;
  return guarded(nullptr, [&] {
    UniqueId id;
    memcpy(id.data, commId.internal, sizeof(id.data));
    CommConfig cfg = shim_config();
    int dev = -1;
    if (!cfg.host_fake) UB_CHECK(cudaGetDevice(&dev) == cudaSuccess, "cudaGetDevice failed");
    auto c = new ncclComm();
    try {
      // more ranks than one NVLink domain: NVLink kernels inside each box + datagram rails between boxes
      if (spans_boxes) c->multi = MultiComm::create(id, rank, nranks, box, dev, cfg);
      else c->comm = Comm::create(id, rank, nranks, dev, cfg);
    } catch (...) {
      delete c;
      throw;
    }
    if (c->comm) {
      try {
        c->fallback = make_fallback(*c->comm);
      } catch (...) {
        delete c;
        throw;
      }
    }
    std::lock_guard<std::mutex> g(g_mu);
    g_comms.insert(c);
    *comm = c;
  });
}

UB_EXPORT ncclResult_t ncclCommInitRankConfig(ncclComm_t* comm, int nranks, ncclUniqueId commId, int rank,
                                              ncclConfig_t* /*config*/) {
  return init_rank(comm, nranks, commId, rank, 0);
}

UB_EXPORT ncclResult_t ncclCommInitRank(ncclComm_t* comm, int nranks, ncclUniqueId commId, int rank) {
  return ncclCommInitRankConfig(comm, nranks, commId, rank, nullptr);
}

UB_EXPORT ncclResult_t ncclCommInitRankScalable(ncclComm_t* newcomm, int nranks, int myrank, int nId,
                                                ncclUniqueId* commIds, ncclConfig_t* config) {
  if (nId < 1 || !commIds) return ncclInvalidArgument;
  return ncclCommInitRankConfig(newcomm, nranks, commIds[0], myrank, config);
}

UB_EXPORT ncclResult_t ncclCommInitAll(ncclComm_t* comms, int ndev, const int* devlist) {
  if (!comms || ndev < 1 || ndev > kMaxRanks) return ncclInvalidArgument;
  return guarded(nullptr, [&] {
    CommConfig cfg = shim_config();
    std::vector<int> devs(ndev);
    for (int i = 0; i < ndev; ++i) devs[i] = cfg.host_fake ? -1 : (devlist ? devlist[i] : i);
    auto cs = Comm::create_local(devs, cfg);
    std::lock_guard<std::mutex> g(g_mu);
    for (int i = 0; i < ndev; ++i) {
      auto c = new ncclComm();
      c->comm = cs[i];
      g_comms.insert(c);
      comms[i] = c;
    }
  });
}

UB_EXPORT ncclResult_t ncclCommFinalize(ncclComm_t comm) {
  if (!valid(comm)) return ncclInvalidArgument;
  comm->finalized = true;
  return ncclSuccess;
}

UB_EXPORT ncclResult_t ncclCommDestroy(ncclComm_t comm) {
  if (!comm) return ncclSuccess;
  {
    std::lock_guard<std::mutex> g(g_mu);
    g_comms.erase(comm);
  }
  if (valid(comm) && !local_of(comm)->is_host()) {
    int prev = -1;
    cudaGetDevice(&prev);
    cudaSetDevice(local_of(comm)->device());
    cudaDeviceSynchronize();
    if (prev >= 0) cudaSetDevice(prev);
  }
  delete comm;
  return ncclSuccess;
}

UB_EXPORT ncclResult_t ncclCommAbort(ncclComm_t comm) { return ncclCommDestroy(comm); }

UB_EXPORT ncclResult_t ncclCommSplit(ncclComm_t comm, int color, int key, ncclComm_t* newcomm, ncclConfig_t* config) {
  if (!valid(comm) || !newcomm) return ncclInvalidArgument;
  *newcomm = nullptr;
  const bool multi = comm->multi != nullptr;
  Comm& c = *local_of(comm);
  const int n = nranks_of(comm), me = multi ? comm->multi->rank() : c.rank();
  auto gather = [&](const void* in, void* out, size_t bytes) {
    if (multi) comm->multi->allgather(in, out, bytes, kU8, nullptr);
    else c.allgather(in, out, bytes, kU8, nullptr);
  };
  struct Rec {
    int color, key, rank, pad;
    char uid[128];
  };
  std::vector<Rec> all(n);
  Rec mine;
  memset(&mine, 0, sizeof(mine));
  mine.color = color;
  mine.key = key;
  mine.rank = me;
  ncclResult_t r = guarded(comm, [&] {
    UniqueId id = Bootstrap::create_id();  // every rank offers one; the group leader's is used
    memcpy(mine.uid, id.data, sizeof(id.data));
    if (c.is_host()) {
      gather(&mine, all.data(), sizeof(Rec));
    } else {
      Rec *d_in = nullptr, *d_out = nullptr;
      UB_CUDA(cudaMalloc((void**)&d_in, sizeof(Rec)));
      UB_CUDA(cudaMalloc((void**)&d_out, sizeof(Rec) * n));
      UB_CUDA(cudaMemcpy(d_in, &mine, sizeof(Rec), cudaMemcpyHostToDevice));
      gather(d_in, d_out, sizeof(Rec));
      UB_CUDA(cudaMemcpy(all.data(), d_out, sizeof(Rec) * n, cudaMemcpyDeviceToHost));
      cudaFree(d_in);
      cudaFree(d_out);
    }
  });
  if (r != ncclSuccess) return r;
  if (color == NCCL_SPLIT_NOCOLOR) return ncclSuccess;
  std::vector<Rec> grp;
  for (auto& x : all)
    if (x.color == color) grp.push_back(x);
  std::sort(grp.begin(), grp.end(), [](const Rec& a, const Rec& b) { return a.key != b.key ? a.key < b.key : a.rank < b.rank; });
  int newrank = -1;
  for (size_t i = 0; i < grp.size(); ++i)
    if (grp[i].rank == me) newrank = (int)i;
  ncclUniqueId uid;
  memset(&uid, 0, sizeof(uid));
  memcpy(uid.internal, grp[0].uid, 128);
  (void)config;
  int box_override = (int)grp.size();  // a single-box parent: the group cannot span boxes
  if (multi) {
    // which boxes do the members live in?  The new communicator needs its ranks box-major with the same
    // number of members per box (that is what rails are built on); one box = a plain NVLink communicator.
    const int L = comm->multi->local_size();
    std::vector<int> per_box;
    int last_box = -1;
    bool ordered = true;
    for (auto& x : grp) {
      const int b = x.rank / L;
      if (b != last_box) {
        if (b < last_box) ordered = false;
        per_box.push_back(0);
        last_box = b;
      }
      ++per_box.back();
    }
    for (int cnt : per_box)
      if (cnt != per_box[0]) ordered = false;
    if (!ordered) {
      g_last_error = comm->last_error =
          "uccl_b200: ncclCommSplit across boxes needs the group's ranks ordered box by box with equally many members per box";
      return ncclInvalidUsage;
    }
    box_override = per_box[0];
  }
  return init_rank(newcomm, (int)grp.size(), uid, newrank, box_override);
}

UB_EXPORT ncclResult_t ncclCommShrink(ncclComm_t, int*, int, ncclComm_t*, ncclConfig_t*, int) {
  g_last_error = "uccl_b200: ncclCommShrink is not supported";
  return ncclInvalidUsage;
}

UB_EXPORT const char* ncclGetErrorString(ncclResult_t result) {
  switch (result) {
    case ncclSuccess: return "no error";
    case ncclUnhandledCudaError: return "unhandled cuda error (run with UCCL_B200_DEBUG=INFO for details)";
    case ncclSystemError: return "unhandled system error";
    case ncclInternalError: return "internal error";
    case ncclInvalidArgument: return "invalid argument";
    case ncclInvalidUsage: return "invalid usage";
    case ncclRemoteError: return "remote process exited or there was a network error";
    case ncclInProgress: return "operation in progress";
    default: return "unknown result code";
  }
}

UB_EXPORT const char* ncclGetLastError(ncclComm_t comm) {
  if (comm && !comm->last_error.empty()) return comm->last_error.c_str();
  return g_last_error.c_str();
}

UB_EXPORT ncclResult_t ncclCommGetAsyncError(ncclComm_t comm, ncclResult_t* asyncError) {
  if (!valid(comm) || !asyncError) return ncclInvalidArgument;
  *asyncError = local_of(comm)->error_word() ? ncclInternalError : ncclSuccess;
  return ncclSuccess;
}

UB_EXPORT ncclResult_t ncclCommCount(const ncclComm_t comm, int* count) {
  if (!valid(comm) || !count) return ncclInvalidArgument;
  *count = nranks_of(comm);
  return ncclSuccess;
}

UB_EXPORT ncclResult_t ncclCommCuDevice(const ncclComm_t comm, int* device) {
  if (!valid(comm) || !device) return ncclInvalidArgument;
  *device = local_of(comm)->device();
  return ncclSuccess;
}

UB_EXPORT ncclResult_t ncclCommUserRank(const ncclComm_t comm, int* rank) {
  if (!valid(comm) || !rank) return ncclInvalidArgument;
  *rank = comm->multi ? comm->multi->rank() : comm->comm->rank();
  return ncclSuccess;
}

// Registration is implicit: heap memory is already peer-mapped and multicast-bound.
UB_EXPORT ncclResult_t ncclCommRegister(const ncclComm_t comm, void* buff, size_t, void** handle) {
  if (!valid(comm)) return ncclInvalidArgument;
  if (handle) *handle = buff;
  return ncclSuccess;
}
UB_EXPORT ncclResult_t ncclCommDeregister(const ncclComm_t comm, void*) { return valid(comm) ? ncclSuccess : ncclInvalidArgument; }
UB_EXPORT ncclResult_t ncclCommWindowRegister(ncclComm_t comm, void* buff, size_t, ncclWindow_t* win, int) {
  if (!valid(comm)) return ncclInvalidArgument;
  if (win) *win = (ncclWindow_t)buff;
  return ncclSuccess;
}
UB_EXPORT ncclResult_t ncclCommWindowDeregister(ncclComm_t comm, ncclWindow_t) { return valid(comm) ? ncclSuccess : ncclInvalidArgument; }

// ncclMemAlloc hands out symmetric-heap memory of the (single) communicator of this process on
// the current device, falling back to cudaMalloc when there is none yet.
UB_EXPORT ncclResult_t ncclMemAlloc(void** ptr, size_t size) {
  if (!ptr) return ncclInvalidArgument;
  return guarded(nullptr, [&] {
    int dev = -1;
    cudaGetDevice(&dev);
    ncclComm* owner = nullptr;
    {
      std::lock_guard<std::mutex> g(g_mu);
      for (auto* c : g_comms)
        if (valid(c) && !local_of(c)->is_host() && local_of(c)->device() == dev) {
          owner = c;
          break;
        }
    }
    if (owner) {
      *ptr = local_of(owner)->alloc(size);
    } else {
      UB_CUDA(cudaMalloc(ptr, size));
    }
  });
}

UB_EXPORT ncclResult_t ncclMemFree(void* ptr) {
  if (!ptr) return ncclSuccess;
  return guarded(nullptr, [&] {
    std::lock_guard<std::mutex> g(g_mu);
    for (auto* c : g_comms)
      if (valid(c) && local_of(c)->in_heap(ptr, 1)) {
        local_of(c)->free(ptr);
        return;
      }
    UB_CUDA(cudaFree(ptr));
  });
}

// PreMulSum(s) = sum_r s * x_r.  With the same scalar on every rank -- the way it is used for
// averaging (torch's _make_nccl_premul_sum(1/world)) -- this is s * sum_r x_r, i.e. exactly the fused
// post-scale epilogue of the kernels (one multiply in fp32 before the single rounding).  Per-rank
// different scalars are not supported.  The scalar is read when the op is created.
UB_EXPORT ncclResult_t ncclRedOpCreatePreMulSum(ncclRedOp_t* op, void* scalar, ncclDataType_t datatype,
                                                ncclScalarResidence_t residence, ncclComm_t comm) {
  if (!valid(comm) || !op || !scalar) return ncclInvalidArgument;
  return guarded(comm, [&] {
    unsigned char raw[8] = {0};
    const size_t es = dtype_size((int)datatype);
    if (residence == ncclScalarDevice && !local_of(comm)->is_host()) {
      UB_CUDA(cudaMemcpy(raw, scalar, es, cudaMemcpyDeviceToHost));
    } else {
      memcpy(raw, scalar, es);
    }
    float v = 1.0f;
    switch ((int)datatype) {
      case kF32: memcpy(&v, raw, 4); break;
      case kF64: {
        double d;
        memcpy(&d, raw, 8);
        v = (float)d;
        break;
      }
      case kF16: {
        uint16_t h;
        memcpy(&h, raw, 2);
        const uint32_t sign = (h >> 15) & 1, ex = (h >> 10) & 0x1f, man = h & 0x3ff;
        if (ex == 0) v = (float)man * 5.9604644775390625e-08f;  // 2^-24
        else if (ex == 31) v = man ? NAN : INFINITY;
        else {
          const uint32_t bits = ((ex + 112) << 23) | (man << 13);
          memcpy(&v, &bits, 4);
        }
        if (sign) v = -v;
        break;
      }
      case kBF16: {
        uint16_t h;
        memcpy(&h, raw, 2);
        const uint32_t bits = (uint32_t)h << 16;
        memcpy(&v, &bits, 4);
        break;
      }
      default: UB_THROW("PreMulSum needs a floating-point datatype (got %d)", (int)datatype);
    }
    std::lock_guard<std::mutex> g(g_mu);
    const int id = comm->next_op++;
    comm->premul[id] = v;
    *op = (ncclRedOp_t)id;
  });
}
UB_EXPORT ncclResult_t ncclRedOpDestroy(ncclRedOp_t op, ncclComm_t comm) {
  if (!valid(comm)) return ncclInvalidArgument;
  std::lock_guard<std::mutex> g(g_mu);
  return comm->premul.erase((int)op) ? ncclSuccess : ncclInvalidArgument;
}

namespace {
// built-in op -> (op, 1); PreMulSum handle -> (sum, scalar)
bool resolve_op(ncclComm* c, ncclRedOp_t op, int* out_op, float* scale) {
  *scale = 1.0f;
  if ((int)op < (int)ncclNumOps) {
    *out_op = (int)op;
    return true;
  }
  std::lock_guard<std::mutex> g(g_mu);
  auto it = c->premul.find((int)op);
  if (it == c->premul.end()) return false;
  *out_op = kSum;
  *scale = it->second;
  return true;
}
}  // namespace

UB_EXPORT ncclResult_t ncclAllReduce(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t datatype,
                                     ncclRedOp_t op, ncclComm_t comm, cudaStream_t stream) {
  if (!valid(comm)) return ncclInvalidArgument;
  if (forwards(comm, NcclFallback::kAllReduce, count, datatype, op))
    return comm->fallback->all_reduce(sendbuff, recvbuff, count, datatype, op, stream);
  int rop;
  ArOpts o;
  if (!resolve_op(comm, op, &rop, &o.scale)) return ncclInvalidArgument;
  return guarded(comm, [&] {
    if (comm->multi) comm->multi->allreduce(sendbuff, recvbuff, count, (int)datatype, rop, stream, o.scale);
    else comm->comm->allreduce(sendbuff, recvbuff, count, (int)datatype, rop, stream, o);
  });
}

UB_EXPORT ncclResult_t ncclReduce(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t datatype,
                                  ncclRedOp_t op, int root, ncclComm_t comm, cudaStream_t stream) {
  if (!valid(comm)) return ncclInvalidArgument;
  if (forwards(comm, NcclFallback::kReduce, count, datatype, op))
    return comm->fallback->reduce(sendbuff, recvbuff, count, datatype, op, root, stream);
  int rop;
  float scale;
  if (!resolve_op(comm, op, &rop, &scale)) return ncclInvalidArgument;
  return guarded(comm, [&] {
    if (comm->multi) {
      UB_CHECK(scale == 1.0f, "PreMulSum reduce across boxes is not supported");
      comm->multi->reduce(sendbuff, recvbuff, count, (int)datatype, rop, root, stream);
    } else {
      comm->comm->reduce(sendbuff, recvbuff, count, (int)datatype, rop, root, stream, scale);
    }
  });
}

UB_EXPORT ncclResult_t ncclBroadcast(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t datatype,
                                     int root, ncclComm_t comm, cudaStream_t stream) {
  if (!valid(comm)) return ncclInvalidArgument;
  if (forwards(comm, NcclFallback::kBroadcast, count, datatype, ncclSum))
    return comm->fallback->broadcast(sendbuff, recvbuff, count, datatype, root, stream);
  return guarded(comm, [&] {
    if (comm->multi) comm->multi->broadcast(sendbuff, recvbuff, count, (int)datatype, root, stream);
    else comm->comm->broadcast(sendbuff, recvbuff, count, (int)datatype, root, stream);
  });
}

UB_EXPORT ncclResult_t ncclBcast(void* buff, size_t count, ncclDataType_t datatype, int root, ncclComm_t comm,
                                 cudaStream_t stream) {
  return ncclBroadcast(buff, buff, count, datatype, root, comm, stream);
}

UB_EXPORT ncclResult_t ncclReduceScatter(const void* sendbuff, void* recvbuff, size_t recvcount,
                                         ncclDataType_t datatype, ncclRedOp_t op, ncclComm_t comm,
                                         cudaStream_t stream) {
  if (!valid(comm)) return ncclInvalidArgument;
  if (forwards(comm, NcclFallback::kReduceScatter, recvcount * (size_t)nranks_of(comm), datatype, op))
    return comm->fallback->reduce_scatter(sendbuff, recvbuff, recvcount, datatype, op, stream);
  int rop;
  float scale;
  if (!resolve_op(comm, op, &rop, &scale)) return ncclInvalidArgument;
  return guarded(comm, [&] {
    if (comm->multi) {
      UB_CHECK(scale == 1.0f, "PreMulSum reduce_scatter across boxes is not supported");
      comm->multi->reduce_scatter(sendbuff, recvbuff, recvcount, (int)datatype, rop, stream);
    } else {
      comm->comm->reduce_scatter(sendbuff, recvbuff, recvcount, (int)datatype, rop, stream, scale);
    }
  });
}

UB_EXPORT ncclResult_t ncclAllGather(const void* sendbuff, void* recvbuff, size_t sendcount, ncclDataType_t datatype,
                                     ncclComm_t comm, cudaStream_t stream) {
  if (!valid(comm)) return ncclInvalidArgument;
  if (forwards(comm, NcclFallback::kAllGather, sendcount * (size_t)nranks_of(comm), datatype, ncclSum))
    return comm->fallback->all_gather(sendbuff, recvbuff, sendcount, datatype, stream);
  return guarded(comm, [&] {
    if (comm->multi) comm->multi->allgather(sendbuff, recvbuff, sendcount, (int)datatype, stream);
    else comm->comm->allgather(sendbuff, recvbuff, sendcount, (int)datatype, stream);
  });
}

// Not part of nccl.h 2.27 but exported by newer NCCL / the reference's shim (as stubs there).
UB_EXPORT ncclResult_t ncclAllToAll(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t datatype,
                                    ncclComm_t comm, cudaStream_t stream) {
  if (!valid(comm)) return ncclInvalidArgument;
  return guarded(comm, [&] {
    if (comm->multi) comm->multi->alltoall(sendbuff, recvbuff, count, (int)datatype, stream);
    else comm->comm->alltoall(sendbuff, recvbuff, count, (int)datatype, stream);
  });
}

UB_EXPORT ncclResult_t ncclAllToAllv(const void* sendbuff, const size_t sendcounts[], const size_t sdispls[],
                                     void* recvbuff, const size_t recvcounts[], const size_t rdispls[],
                                     ncclDataType_t datatype, ncclComm_t comm, cudaStream_t stream) {
  if (!valid(comm)) return ncclInvalidArgument;
  return guarded(comm, [&] {
    if (comm->multi) comm->multi->alltoallv(sendbuff, sendcounts, sdispls, recvbuff, recvcounts, rdispls, (int)datatype, stream);
    else comm->comm->alltoallv(sendbuff, sendcounts, sdispls, recvbuff, recvcounts, rdispls, (int)datatype, stream);
  });
}

// NCCL 2.28 spelling of the same operation
UB_EXPORT ncclResult_t ncclAlltoAll(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t datatype,
                                    ncclComm_t comm, cudaStream_t stream) {
  return ncclAllToAll(sendbuff, recvbuff, count, datatype, comm, stream);
}

namespace {
// rooted fan-in / fan-out (NCCL 2.28 ncclGather / ncclScatter) as one grouped send/recv launch plus the root's local copy
ncclResult_t rooted_p2p(bool gather, const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t dt, int root,
                        ncclComm_t comm, cudaStream_t stream) {
  if (!valid(comm)) return ncclInvalidArgument;
  const int n = nranks_of(comm);
  if ((int)dt < 0 || (int)dt >= kNumDTypes || root < 0 || root >= n) return ncclInvalidArgument;
  Comm* lc = local_of(comm);
  const int me = comm->multi ? comm->multi->rank() : lc->rank();
  const size_t bytes = count * (size_t)dtype_size((int)dt);
  return guarded(comm, [&] {
    std::vector<Comm::P2pOp> ops;
    if (me == root) {
      char* mine_dst = gather ? (char*)recvbuff + (size_t)root * bytes : (char*)recvbuff;
      const char* mine_src = gather ? (const char*)sendbuff : (const char*)sendbuff + (size_t)root * bytes;
      if (bytes && mine_dst != mine_src) {
        if (lc->is_host()) memcpy(mine_dst, mine_src, bytes);
        else UB_CUDA(cudaMemcpyAsync(mine_dst, mine_src, bytes, cudaMemcpyDeviceToDevice, stream));
      }
      for (int r = 0; r < n; ++r) {
        if (r == root) continue;
        if (gather) ops.push_back({false, (char*)recvbuff + (size_t)r * bytes, bytes, r});
        else ops.push_back({true, const_cast<char*>((const char*)sendbuff) + (size_t)r * bytes, bytes, r});
      }
    } else {
      if (gather) ops.push_back({true, const_cast<void*>(sendbuff), bytes, root});
      else ops.push_back({false, recvbuff, bytes, root});
    }
    if (ops.empty() || bytes == 0) return;
    if (comm->multi) comm->multi->group_p2p(ops, stream);
    else comm->comm->group_p2p(ops, stream);
  });
}
}  // namespace

UB_EXPORT ncclResult_t ncclGather(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t datatype, int root,
                                  ncclComm_t comm, cudaStream_t stream) {
  return rooted_p2p(true, sendbuff, recvbuff, count, datatype, root, comm, stream);
}

UB_EXPORT ncclResult_t ncclScatter(const void* sendbuff, void* recvbuff, size_t count, ncclDataType_t datatype, int root,
                                   ncclComm_t comm, cudaStream_t stream) {
  return rooted_p2p(false, sendbuff, recvbuff, count, datatype, root, comm, stream);
}

// NCCL 2.28: stop what is in flight and leave the communicator ready for destroy / split.  Every operation of this
// library is a kernel with a bounded spin, so quiescing is a device synchronisation.
UB_EXPORT ncclResult_t ncclCommRevoke(ncclComm_t comm, int revokeFlags) {
  if (!valid(comm) || revokeFlags != 0) return ncclInvalidArgument;
  Comm* lc = local_of(comm);
  if (!lc->is_host()) {
    int prev = -1;
    cudaGetDevice(&prev);
    cudaSetDevice(lc->device());
    cudaDeviceSynchronize();
    if (prev >= 0) cudaSetDevice(prev);
  }
  return ncclSuccess;
}

// NCCL 2.28 device-side communicators (nccl_device/core.h) belong to NCCL's own device API: kernels written against it
// cannot run on this library's communicators.  Exported so that a preloaded drop-in answers -- with an error -- instead
// of letting the call fall through to another libnccl with a foreign communicator handle.
UB_EXPORT ncclResult_t ncclDevCommCreate(ncclComm_t, const void*, void*) {
  g_last_error = "uccl_b200: NCCL device communicators (ncclDevCommCreate) are not provided by the drop-in";
  return ncclInvalidUsage;
}
UB_EXPORT ncclResult_t ncclDevCommDestroy(ncclComm_t, const void*) { return ncclInvalidUsage; }

UB_EXPORT ncclResult_t ncclGroupStart() {
  ++g_group_depth;
  return ncclSuccess;
}

UB_EXPORT ncclResult_t ncclGroupEnd() {
  if (g_group_depth <= 0) return ncclInvalidUsage;
  if (--g_group_depth > 0) return ncclSuccess;
  return flush_group();
}

UB_EXPORT ncclResult_t ncclGroupSimulateEnd(ncclSimInfo_t* simInfo) {
  if (simInfo) simInfo->estimatedTime = 0.f;
  return ncclSuccess;
}

static ncclResult_t post_p2p(bool is_send, void* buf, size_t count, ncclDataType_t dt, int peer, ncclComm_t comm,
                             cudaStream_t stream) {
  if (!valid(comm)) return ncclInvalidArgument;
  if ((int)dt < 0 || (int)dt >= kNumDTypes || peer < 0 || peer >= nranks_of(comm)) return ncclInvalidArgument;
  PendingP2p p;
  p.comm = comm;
  p.op.is_send = is_send;
  p.op.buf = buf;
  p.op.bytes = count * (size_t)dtype_size((int)dt);
  p.op.peer = peer;
  p.stream = stream;
  p.count = count;
  p.dt = dt;
  g_pending.push_back(p);
  if (g_group_depth == 0) return flush_group();
  return ncclSuccess;
}

UB_EXPORT ncclResult_t ncclSend(const void* sendbuff, size_t count, ncclDataType_t datatype, int peer, ncclComm_t comm,
                                cudaStream_t stream) {
  return post_p2p(true, const_cast<void*>(sendbuff), count, datatype, peer, comm, stream);
}

UB_EXPORT ncclResult_t ncclRecv(void* recvbuff, size_t count, ncclDataType_t datatype, int peer, ncclComm_t comm,
                                cudaStream_t stream) {
  return post_p2p(false, recvbuff, count, datatype, peer, comm, stream);
}

// pnccl* aliases (profiling entry points of nccl.h)
#define UB_ALIAS(ret, name, params, args) \
  UB_EXPORT ret p##name params { return name args; }
UB_ALIAS(ncclResult_t, ncclGetVersion, (int* v), (v))
UB_ALIAS(ncclResult_t, ncclGetUniqueId, (ncclUniqueId * u), (u))
UB_ALIAS(ncclResult_t, ncclCommInitRank, (ncclComm_t * c, int n, ncclUniqueId id, int r), (c, n, id, r))
UB_ALIAS(ncclResult_t, ncclCommInitAll, (ncclComm_t * c, int n, const int* d), (c, n, d))
UB_ALIAS(ncclResult_t, ncclCommDestroy, (ncclComm_t c), (c))
UB_ALIAS(ncclResult_t, ncclCommCount, (const ncclComm_t c, int* n), (c, n))
UB_ALIAS(ncclResult_t, ncclCommUserRank, (const ncclComm_t c, int* r), (c, r))
UB_ALIAS(ncclResult_t, ncclGroupStart, (), ())
UB_ALIAS(ncclResult_t, ncclGroupEnd, (), ())
UB_ALIAS(ncclResult_t, ncclAllReduce,
         (const void* s, void* r, size_t n, ncclDataType_t d, ncclRedOp_t o, ncclComm_t c, cudaStream_t st),
         (s, r, n, d, o, c, st))
UB_ALIAS(ncclResult_t, ncclAllGather, (const void* s, void* r, size_t n, ncclDataType_t d, ncclComm_t c, cudaStream_t st),
         (s, r, n, d, c, st))
UB_ALIAS(ncclResult_t, ncclReduceScatter,
         (const void* s, void* r, size_t n, ncclDataType_t d, ncclRedOp_t o, ncclComm_t c, cudaStream_t st),
         (s, r, n, d, o, c, st))
UB_ALIAS(ncclResult_t, ncclBroadcast,
         (const void* s, void* r, size_t n, ncclDataType_t d, int root, ncclComm_t c, cudaStream_t st),
         (s, r, n, d, root, c, st))
UB_ALIAS(ncclResult_t, ncclSend, (const void* s, size_t n, ncclDataType_t d, int p, ncclComm_t c, cudaStream_t st),
         (s, n, d, p, c, st))
UB_ALIAS(ncclResult_t, ncclRecv, (void* r, size_t n, ncclDataType_t d, int p, ncclComm_t c, cudaStream_t st),
         (r, n, d, p, c, st))
UB_ALIAS(ncclResult_t, ncclAlltoAll, (const void* s, void* r, size_t n, ncclDataType_t d, ncclComm_t c, cudaStream_t st),
         (s, r, n, d, c, st))
UB_ALIAS(ncclResult_t, ncclGather, (const void* s, void* r, size_t n, ncclDataType_t d, int root, ncclComm_t c, cudaStream_t st),
         (s, r, n, d, root, c, st))
UB_ALIAS(ncclResult_t, ncclScatter, (const void* s, void* r, size_t n, ncclDataType_t d, int root, ncclComm_t c, cudaStream_t st),
         (s, r, n, d, root, c, st))
UB_ALIAS(ncclResult_t, ncclCommRevoke, (ncclComm_t c, int f), (c, f))

}  // extern "C"
