// Communicator: symmetric heap + collective launchers + algorithm selection.
//
// Role in the reference: lite's Communicator/AlgorithmCollection/selector
// (experimental/lite/nccl/nccl.cu:1389-1547, collective/algorithm_selector.cc:63-155).
// Ours differs by design: one heap-backed fabric, block-sliced kernels, and a
// measured tuning table instead of hard-coded thresholds.
#pragma once
#include <cuda_runtime.h>

#include <initializer_list>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../fabric/fabric.h"
#include "../kernels/types.h"

namespace ub {

struct CommConfig {
  size_t heap_bytes = 1ull << 30;
  size_t stage_bytes = 64ull << 20;
  bool host_fake = false;
  int timeout_ms = -1;  // -1: from UCCL_B200_TIMEOUT_MS (default 20000)
  int max_ctas = -1;    // -1: from UCCL_B200_MAX_CTAS (default 128)
};

// algorithm ids (shared with Python)
enum ArAlgoId : int {
  ALGO_AUTO = 0,
  ALGO_ONESHOT_LL = 1,
  ALGO_ONESHOT_MC = 2,
  ALGO_TWOSHOT_P2P = 3,
  ALGO_TWOSHOT_NVLS = 4,
  ALGO_STAGED_P2P = 5,
  ALGO_STAGED_NVLS = 6,
  ALGO_STAGED_PIPE = 7  // staged + NVLS with copy-in / reduce / copy-out running concurrently on three CTA groups
};

struct ArOpts {
  int algo = ALGO_AUTO;
  float scale = 1.0f;   // fused post-scale (multiplies the reduced value)
  int out_dtype = -1;   // fused output cast (-1: same as input)
  int max_ctas = -1;    // per-call override
};

struct TuneEntry {  // "for messages up to max_bytes use (algo, ctas)"
  uint64_t max_bytes;
  int algo;
  int ctas;
};

class Comm {
 public:
  static std::shared_ptr<Comm> create(const UniqueId& id, int rank, int nranks, int device, const CommConfig& cfg);
  static std::vector<std::shared_ptr<Comm>> create_local(const std::vector<int>& devices, const CommConfig& cfg);
  ~Comm();

  int rank() const { return fabric_->rank(); }
  int nranks() const { return fabric_->nranks(); }
  int device() const { return fabric_->device(); }
  bool has_multicast() const { return fabric_->has_multicast(); }
  bool is_host() const { return fabric_->is_host(); }
  const Fabric& fabric() const { return *fabric_; }
  const HeapLayout& layout() const { return layout_; }
  DevComm dev() const { return dev_; }
  std::string describe() const;

  // symmetric heap allocation (collective: same sequence of calls on every rank)
  void* alloc(size_t bytes, size_t align = 256);
  void free(void* p);
  size_t heap_free_bytes() const;
  bool in_heap(const void* p, size_t bytes) const { return fabric_->contains(p, bytes); }
  uint64_t heap_offset(const void* p) const { return fabric_->offset_of(p); }
  void* peer_ptr(const void* local, int peer) const { return fabric_->heap(peer) + fabric_->offset_of(local); }
  void* mc_ptr(const void* local) const {
    return fabric_->mc() ? (void*)(fabric_->mc() + fabric_->offset_of(local)) : nullptr;
  }

  // collectives (asynchronous on `stream`; throw std::runtime_error on invalid arguments)
  void allreduce(const void* in, void* out, size_t count, int dtype, int op, cudaStream_t stream,
                 const ArOpts& opts = ArOpts());
  void allgather(const void* in, void* out, size_t count_per_rank, int dtype, cudaStream_t stream);
  // `scale`: fused post-scale of the result (float dtypes), multiplied with the 1/N of kAvg
  void reduce_scatter(const void* in, void* out, size_t recv_count, int dtype, int op, cudaStream_t stream,
                      float scale = 1.0f);
  void broadcast(const void* in, void* out, size_t count, int dtype, int root, cudaStream_t stream);
  void reduce(const void* in, void* out, size_t count, int dtype, int op, int root, cudaStream_t stream,
              float scale = 1.0f);
  void alltoall(const void* in, void* out, size_t count_per_peer, int dtype, cudaStream_t stream);
  void alltoallv(const void* in, const size_t* send_counts, const size_t* send_displs, void* out,
                 const size_t* recv_counts, const size_t* recv_displs, int dtype, cudaStream_t stream);
  void barrier(cudaStream_t stream);
  // In-place sum all-reduce of x [T, H], then residual_out = x + residual and out = rmsnorm(residual_out) * weight
  // (quant = 1: out is e4m3 with fp32 inverse scales per 128 channels in out_scales [T, H / 128]).  bf16 / fp16,
  // H % 8 == 0, H <= kRmsMaxH.  The fused one-shot kernel runs where AUTO picks a one-shot all-reduce (or
  // opts.algo forces one); otherwise the selected all-reduce runs, followed by the local epilogue kernel.
  void allreduce_rmsnorm(void* x, const void* residual, void* residual_out, const void* weight, void* out,
                         float* out_scales, size_t T, size_t H, int dtype, float eps, int quant, cudaStream_t stream,
                         const ArOpts& opts = ArOpts());
  // Sequence-parallel counterpart: x [T, H] (T % nranks == 0) is sum-reduce-scattered in place, so that rank r's row
  // block x[r*T/n, (r+1)*T/n) holds its rows of the sum; then the same epilogue on that block with residual,
  // residual_out, out [T/n, H] and out_scales [T/n, H / 128].  The fused LL kernel runs where the plain
  // reduce_scatter of T/n * H elements would take the LL kernel; otherwise reduce_scatter, then the epilogue kernel.
  void reduce_scatter_rmsnorm(void* x, const void* residual, void* residual_out, const void* weight, void* out,
                              float* out_scales, size_t T, size_t H, int dtype, float eps, int quant,
                              cudaStream_t stream);
  // grouped point-to-point (ncclGroupStart .. ncclSend/ncclRecv .. ncclGroupEnd)
  struct P2pOp {
    bool is_send;
    void* buf;
    size_t bytes;
    int peer;
  };
  void group_p2p(const std::vector<P2pOp>& ops, cudaStream_t stream);

  // which algorithm AUTO would pick (for tests / tuner)
  int select_allreduce(size_t bytes, bool symmetric, int dtype, int op, int* ctas) const;
  void set_tuning(bool symmetric, const std::vector<TuneEntry>& table);
  // LL-packet AllGather/AllToAll/ReduceScatter threshold (per-rank piece bytes): 0 default, <0 off
  void set_xchg_ll_max(int64_t bytes) { xchg_ll_max_ = bytes; }
  int64_t xchg_ll_max() const { return xchg_ll_max_; }
  // per-rank piece size up to which reduce_scatter and reduce_scatter_rmsnorm run the LL kernels (0: never)
  uint64_t rs_ll_max_bytes() const;
  // staged (plain-buffer) ReduceScatter: push pieces into the peers' stages instead of copy-in + pull.
  // Must be set identically on every rank.
  void set_rs_push(bool on) { rs_push_ = on; }
  bool rs_push() const { return rs_push_; }
  uint32_t error_word() const { return err_host_ ? *err_host_ : 0; }
  // in-kernel tracing (device timeline of every block's barriers / phases)
  struct TraceEvent {
    uint64_t t_ns;
    uint32_t code, block, aux;
  };
  void enable_trace(size_t max_events);
  void disable_trace();
  std::vector<TraceEvent> dump_trace(bool reset = true);
  uint64_t launches() const { return launches_; }

 private:
  Comm() = default;
  void init(std::shared_ptr<Fabric> f, const CommConfig& cfg);
  CollArgs base_args() const;
  int ctas_for(uint64_t bytes, int cap, int per_cta_bytes) const;
  int nvls_ctas() const;
  void check_buf(const void* p, const char* what) const;
  // the epilogue kernel of the unfused tails on r.T rows of an already reduced r.x
  void launch_add_rmsnorm(const RmsNormArgs& r, int dtype, bool fp8, cudaStream_t stream);
  // host fake implementations (host_coll.cc)
  void host_barrier();
  void host_allreduce(const void* in, void* out, size_t count, int dtype, int op, float scale, int out_dtype);
  void host_allgather(const void* in, void* out, size_t bytes);
  void host_reduce_scatter(const void* in, void* out, size_t count, int dtype, int op);
  void host_broadcast(const void* in, void* out, size_t bytes, int root);
  void host_reduce(const void* in, void* out, size_t count, int dtype, int op, int root);
  void host_alltoall(const void* in, void* out, size_t bytes);
  void host_group_p2p(const std::vector<P2pOp>& ops);
  void host_alltoallv(const void* in, const size_t* send_bytes, const size_t* send_off, void* out,
                      const size_t* recv_bytes, const size_t* recv_off);

  std::shared_ptr<Fabric> fabric_;
  HeapLayout layout_;
  DevComm dev_;
  CommConfig cfg_;
  int max_ctas_ = 64;
  int64_t xchg_ll_max_ = 0;
  bool rs_push_ = true;
  uint32_t* err_host_ = nullptr;
  uint64_t launches_ = 0;
  uint32_t host_epoch_ = 0;
  std::vector<uint64_t> host_send_seq_, host_recv_seq_;  // host send/recv mailboxes: chunks sent to / received from each peer
  unsigned long long* trace_dev_ = nullptr;
  size_t trace_cap_ = 0;
  std::vector<TuneEntry> tune_sym_, tune_unsym_;
  // heap allocator
  mutable std::mutex mu_;
  std::map<uint64_t, uint64_t> free_;   // offset -> size
  std::map<uint64_t, uint64_t> used_;   // offset -> size
};

const char* algo_name(int algo);

// CPU reference reduction used by the host backends: dst[i] = op_r srcs[r][i], then * scale (floats)
void host_reduce_n(void* dst, const void* const* srcs, int n, size_t count, int dtype, int op, float scale);
// CPU epilogue of allreduce_rmsnorm on an already reduced x (bf16 / fp16, fp32 arithmetic; e4m3 when out_scales)
void host_add_rmsnorm(const void* x, const void* residual, void* residual_out, const void* weight, void* out,
                      float* out_scales, size_t T, size_t H, int dtype, float eps);
// Checks of the fused residual add + RMSNorm layer tails (`op` names the call in messages): bf16 / fp16, H a multiple
// of `mult` in [mult, max_h], H % 128 == 0 for the e4m3 output (fp8), T < 2^32; for T > 0 residual, residual_out,
// weight, out (and out_scales with fp8) non-null; with `aligned` those, x and `extra` (optional inputs, may be null)
// 16-byte aligned.  Returns the epilogue arguments (out_scales only with fp8).
RmsNormArgs rmsnorm_tail_args(const char* op, void* x, const void* residual, void* residual_out, const void* weight,
                              void* out, float* out_scales, int64_t T, int64_t H, int dtype, float eps, bool fp8,
                              uint32_t max_h, uint32_t mult, bool aligned, std::initializer_list<const void*> extra = {});

// torch.cuda.MemPool backend (mem_pool.cc): which communicator serves `uccl_b200_pool_malloc`
void pool_install(std::shared_ptr<Comm> c);            // default for c->device()
void pool_set_thread_comm(std::shared_ptr<Comm> c);    // per-thread override (virtual ranks)
void pool_clear_thread_comm();
void pool_stats(uint64_t* allocs, uint64_t* frees, uint64_t* live_bytes, uint64_t* fallback_allocs);

}  // namespace ub
