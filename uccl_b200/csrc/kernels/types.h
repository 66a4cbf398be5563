// Host-safe shared types: constants, device communicator descriptor, dtype/op tables,
// heap control-region layout and collective launch arguments.  Included by both the
// CUDA kernels and the plain C++ runtime.
#pragma once
#include <stdint.h>
#ifdef __CUDACC__
#define UB_HD __host__ __device__
#else
#define UB_HD
#endif

namespace ub {

constexpr int kMaxRanks = 8;
constexpr int kMaxSyncBlocks = 512;   // max grid of any kernel that uses a cross-rank barrier
constexpr int kNumSyncDomains = 8;    // independent barrier domains (collectives, ep, p2p, ...)

// Passed by value to every kernel (fits in param space; __grid_constant__).
struct DevComm {
  int rank;
  int nranks;
  char* heap[kMaxRanks];  // heap[r] = VA (in *this* process/device) of rank r's symmetric heap
  char* mc;               // multicast VA of the heap (nullptr when NVLS is unavailable)
  uint64_t sig_off;       // offset of sync-domain signal slots inside each heap
  uint64_t epoch_off;     // offset of local per-block epoch counters
  uint64_t xchg_off;      // offset of the per-(domain, block, src) 16-byte exchange slots
  uint64_t timeout_ns;    // spin timeout (0 = infinite)
  uint32_t* err;          // host-mapped error word (set before trap)
  unsigned long long* trace;  // optional device trace buffer: [0] = write index, then {t_ns, tag} pairs
  uint32_t trace_cap;     // capacity in events (0 = tracing off)
};

// trace event codes (tag = code << 48 | block << 32 | aux)
enum TraceCode : uint32_t {
  TR_KERNEL_BEGIN = 1,
  TR_KERNEL_END = 2,
  TR_BARRIER_ENTER = 3,
  TR_BARRIER_EXIT = 4,
  TR_PHASE = 5,
};

enum DType : int {
  kI8 = 0,
  kU8 = 1,
  kI32 = 2,
  kU32 = 3,
  kI64 = 4,
  kU64 = 5,
  kF16 = 6,
  kF32 = 7,
  kF64 = 8,
  kBF16 = 9,
  kF8E4M3 = 10,
  kF8E5M2 = 11,
  kNumDTypes = 12
};
enum RedOp : int { kSum = 0, kProd = 1, kMax = 2, kMin = 3, kAvg = 4, kNumOps = 5 };

UB_HD inline int dtype_size(int dt) {
  switch (dt) {
    case kI8: case kU8: case kF8E4M3: case kF8E5M2: return 1;
    case kF16: case kBF16: return 2;
    case kI32: case kU32: case kF32: return 4;
    default: return 8;
  }
}

// Post-reduction epilogue parameters (fused scale / integer average).
struct Epilogue {
  float scale;  // multiplies floating accumulators (1.0f = none); avg => 1/nranks
  int idiv;     // divides integer accumulators (1 = none); avg => nranks
};

inline bool nvls_reduce_supported(int dtype, int op) {
  if (dtype == kF32) return op == kSum || op == kAvg;
  if (dtype == kBF16 || dtype == kF16) return op == kSum || op == kAvg || op == kMax || op == kMin;
  return false;
}

// Sync-domain assignment (independent barrier epochs so different subsystems may
// run concurrently on different streams).
enum SyncDomain : int { kDomColl = 0, kDomEp = 1, kDomEpLL = 2, kDomP2P = 3, kDomUser0 = 4 };

constexpr uint64_t kSigBytes = (uint64_t)kNumSyncDomains * kMaxSyncBlocks * kMaxRanks * sizeof(uint32_t);
constexpr uint64_t kEpochBytes = (uint64_t)kNumSyncDomains * kMaxSyncBlocks * sizeof(uint32_t);
constexpr uint64_t kMiscBytes = 4096;
constexpr uint64_t kXchgBytes = (uint64_t)kNumSyncDomains * kMaxSyncBlocks * kMaxRanks * 16;
constexpr uint64_t kA2AvTabBytes = (uint64_t)kMaxSyncBlocks * kMaxRanks * 2 * sizeof(uint64_t);
constexpr int kSrBlocks = 16;                        // CTAs per send/recv peer pair
constexpr int kSrSlots = 4;                          // staging slots per (peer, block)
constexpr uint64_t kSrChunkBytes = 64u << 10;        // bytes per staging slot
constexpr uint64_t kSrStageBytes = (uint64_t)kMaxRanks * kSrBlocks * kSrSlots * kSrChunkBytes;
constexpr uint64_t kSrFlagBytes = 4096;              // ready/ack/sseq/rseq words
constexpr uint64_t kLLMaxData = 1u << 20;           // max payload of the one-shot LL path
constexpr uint64_t kLLSlotBytes = 2 * kLLMaxData;     // 8 data bytes per 16-byte packet
constexpr uint64_t kLLBytes = 2 * kMaxRanks * kLLSlotBytes;  // 2 parities x src ranks

// misc words
enum MiscWord : int { kLLEpoch = 0, kLLDone = 1, kPipeIn = 8, kPipeRed = 9, kPipeOut = 10, kPipeExit = 11, kMiscWords = 64 };

struct HeapLayout {
  uint64_t sig_off, epoch_off, xchg_off, misc_off, a2av_tab_off, sr_flag_off, ll_off, sr_stage_off, stage_in_off, stage_out_off, user_off;
  uint64_t stage_bytes;
  static HeapLayout make(uint64_t stage_bytes) {
    HeapLayout l;
    l.sig_off = 0;
    l.epoch_off = l.sig_off + kSigBytes;
    l.xchg_off = l.epoch_off + kEpochBytes;
    l.misc_off = l.xchg_off + kXchgBytes;
    l.a2av_tab_off = l.misc_off + kMiscBytes;
    l.sr_flag_off = l.a2av_tab_off + kA2AvTabBytes;
    l.ll_off = (l.sr_flag_off + kSrFlagBytes + 4095) / 4096 * 4096;
    l.stage_bytes = (stage_bytes + 4095) / 4096 * 4096;
    l.sr_stage_off = l.ll_off + kLLBytes;
    l.stage_in_off = l.sr_stage_off + kSrStageBytes;
    l.stage_out_off = l.stage_in_off + l.stage_bytes;
    l.user_off = l.stage_out_off + l.stage_bytes;
    l.user_off = (l.user_off + (2u << 20) - 1) / (2u << 20) * (2u << 20);
    return l;
  }
  uint64_t ctrl_bytes() const { return sr_stage_off; }  // region that must start zeroed
};

constexpr uint64_t kNoOff = ~0ull;

struct CollArgs {
  const void* in;
  void* out;
  uint64_t in_off;   // offset of `in` inside the symmetric heap, kNoOff if it is a plain local buffer
  uint64_t out_off;  // same for `out`
  uint64_t count;    // elements (of the input dtype) per rank-visible buffer; see each kernel
  uint64_t bytes;    // count * sizeof(T)
  Epilogue ep;
  int root;
  int variant;  // kernel-specific algorithm switch (e.g. ReduceScatter staging: 0 = pull, 1 = push)
  uint64_t misc_off, ll_off, stage_in_off, stage_out_off, stage_bytes;
};

// Fused all-reduce + residual add + RMSNorm (allreduce_rmsnorm.cu).  One CTA of kRmsThreads threads holds a
// row in registers, at most kRmsUnits 16-byte units per thread, hence H <= kRmsMaxH for 16-bit dtypes.
constexpr int kRmsThreads = 512;
constexpr int kRmsUnits = 4;
constexpr uint32_t kRmsMaxH = (uint32_t)kRmsThreads * kRmsUnits * 8;
struct RmsNormArgs {
  void* x;                 // [T, H]: the reduced sum (stored by the fused kernel, read by the local one)
  const void* residual;    // [T, H]
  void* residual_out;      // [T, H] = x + residual; may equal residual
  const void* weight;      // [H]
  void* out;               // [T, H] of the input dtype, or e4m3 when out_scales != nullptr
  float* out_scales;       // [T, H / 128] inverse scales of the e4m3 output (nullptr: no quantisation)
  uint32_t T, H;
  float eps;
};

// Split [0, total) into `parts` nearly equal contiguous ranges whose boundaries are
// multiples of `gran` (except the final end).
UB_HD inline void split_range(uint64_t total, int parts, int idx, uint64_t& lo, uint64_t& hi,
                                            uint64_t gran = 1) {
  uint64_t units = (total + gran - 1) / gran;
  uint64_t per = (units + parts - 1) / parts * gran;
  lo = per * (uint64_t)idx;
  if (lo > total) lo = total;
  hi = lo + per;
  if (hi > total) hi = total;
}

// 16-byte units [lo, hi) of the current chunk (`cb` bytes) owned by part `idx` of `parts`.
// Boundaries are those of a FULL chunk (clamped to the current one), so a block touches the same
// range of the staging area in every chunk of a kernel; see chunk_slice() in coll_common.cuh.
UB_HD inline void chunk_slice_hd(uint64_t msg_bytes, uint64_t chunk_bytes, uint64_t cb, int parts, int idx,
                                               uint64_t& lo, uint64_t& hi, uint64_t gran = 1) {
  const uint64_t full = msg_bytes < chunk_bytes ? msg_bytes : chunk_bytes;
  const uint64_t cu = (cb + 15) / 16;
  split_range((full + 15) / 16, parts, idx, lo, hi, gran);
  if (lo > cu) lo = cu;
  if (hi > cu) hi = cu;
}

// Grouped send/recv launch arguments: at most one send and one recv per peer per launch.
struct SendRecvArgs {
  const char* sbuf[kMaxRanks];
  char* rbuf[kMaxRanks];
  uint64_t sbytes[kMaxRanks];  // 0 = no send to that peer
  uint64_t rbytes[kMaxRanks];  // 0 = no recv from that peer
  int peers[kMaxRanks];        // active peer list
  int npeers;
  uint64_t sr_flag_off, sr_stage_off;
  uint64_t s_off[kMaxRanks];   // heap offset of sbuf[p] if it lives in the symmetric heap (zero-copy pull), else kNoOff
};

// AllToAllv launch arguments.
struct A2AvArgs {
  uint64_t send_off[kMaxRanks];   // byte offsets inside `in`
  uint64_t send_bytes[kMaxRanks];
  uint64_t recv_off[kMaxRanks];   // byte offsets inside `out`
  uint64_t recv_bytes[kMaxRanks];
  uint64_t table_off;             // heap offset of a [kMaxRanks][2] u64 table (symmetric)
};

}  // namespace ub
