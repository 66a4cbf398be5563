#include "ep_buffer.h"

#include <sched.h>

#include <algorithm>
#include <chrono>
#include <cstring>

#include "../common/log.h"
#include "../common/param.h"
#include "../fabric/cu_api.h"

namespace ub {

UB_PARAM(EpCpuTimeoutSecs, "EP_CPU_TIMEOUT_SECS", 100)  // reference: UCCL_EP_CPU_TIMEOUT_SECS (ep/include/common.hpp:153-176)
UB_PARAM(EpImpl, "EP_IMPL", 0)                 // 0 auto, 1 register path, 2 TMA pipelines
UB_PARAM(EpLayoutMultiCta, "EP_LAYOUT_MC", 1)  // 0: single-CTA layout scan

namespace {
size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
struct DevGuard {
  int prev = -1;
  bool active = false;
  explicit DevGuard(int d) {
    if (d >= 0 && cudaGetDevice(&prev) == cudaSuccess && prev != d) {
      cudaSetDevice(d);
      active = true;
    }
  }
  ~DevGuard() {
    if (active) cudaSetDevice(prev);
  }
};
size_t per_token_bytes(int H, int mode, int K) {
  size_t row = (mode == EP_X_BF16) ? (size_t)H * 2 : (size_t)H;
  size_t sc = (mode == EP_X_BF16) ? 0 : (size_t)(H / 128) * 4;
  return row + sc + (size_t)K * 12 + 4;
}
}  // namespace

EpBuffer::EpBuffer(std::shared_ptr<Comm> comm, size_t num_nvl_bytes, int num_slots) : comm_(comm) {
  UB_CHECK(!comm->is_host(), "EpBuffer needs a CUDA communicator");
  UB_CHECK(num_slots >= 1 && num_slots <= 8, "num_slots must be in 1..8");
  num_slots_ = num_slots;
  DevGuard g(comm->device());
  ctrl_bytes_ = align_up((size_t)kEpMaxBlocks * kMaxRanks * kMaxRanks * 4 + (size_t)kMaxRanks * kEpMaxLocalExperts * 4, 4096);
  bytes_ = align_up(std::max(num_nvl_bytes, ctrl_bytes_ + (size_t)(num_slots + 1) * 4096), 4096);
  base_ = (char*)comm->alloc(bytes_, 4096);
  base_off_ = comm->heap_offset(base_);
  arena_bytes_ = (bytes_ - ctrl_bytes_) / (size_t)(num_slots_ + 1) / 256 * 256;
  UB_CUDA(cudaMemset(base_, 0, ctrl_bytes_));
  void* h = nullptr;
  UB_CUDA(cudaHostAlloc(&h, sizeof(int32_t) * (1 + kEpMaxLocalExperts), cudaHostAllocMapped));
  host_counts_ = (int32_t*)h;
  memset(host_counts_, 0, sizeof(int32_t) * (1 + kEpMaxLocalExperts));
  void* d = nullptr;
  UB_CUDA(cudaHostGetDevicePointer(&d, h, 0));
  host_counts_dev_ = (int32_t*)d;
  UB_CUDA(cudaMalloc((void**)&dev_counts_, sizeof(int32_t) * (1 + kEpMaxLocalExperts)));
  UB_CUDA(cudaMemset(dev_counts_, 0, sizeof(int32_t) * (1 + kEpMaxLocalExperts)));
  if (ubParamEpLayoutMultiCta()) {
    UB_CUDA(cudaMalloc((void**)&layout_scratch_, sizeof(uint32_t) * kEpLayoutScratchWords));
    UB_CUDA(cudaMemset(layout_scratch_, 0, sizeof(uint32_t) * kEpLayoutScratchWords));
  }
  set_impl((int)ubParamEpImpl());
  UB_CUDA(cudaDeviceSynchronize());
  UB_INFO(SUB_EP, "EpBuffer rank %d: %zu MiB, %d dispatch arenas + 1 combine arena of %zu MiB", comm->rank(),
          bytes_ >> 20, num_slots_, arena_bytes_ >> 20);
}

EpBuffer::~EpBuffer() {
  if (ll_send_cnt_) cudaFree(ll_send_cnt_);
  try {
    if (ll_base_) comm_->free(ll_base_);
  } catch (...) {
  }
  if (host_counts_) cudaFreeHost(host_counts_);
  if (dev_counts_) cudaFree(dev_counts_);
  if (layout_scratch_) cudaFree(layout_scratch_);
  try {
    if (base_) comm_->free(base_);
  } catch (...) {
  }
}

void EpBuffer::set_impl(int impl) {
  UB_CHECK(impl >= EP_IMPL_AUTO && impl <= EP_IMPL_TMA, "EP impl must be 0 (auto), 1 (register path) or 2 (TMA)");
  impl_ = impl;
}

// Across NVLink the TMA pipelines keep more bytes in flight per CTA than the register path; on ONE GPU (HBM-only
// permutation, nothing to hide) the register path's shorter per-token critical path is faster
// (benchmarks/ep_sweep.py times both).
int EpBuffer::pick_impl(int grid, bool combine) const {
  if (impl_ != EP_IMPL_AUTO) return impl_;
  if (nranks() == 1) return EP_IMPL_REG;
  // 2 GPUs, few CTAs: a token has two copies and one of them is local, so combine is bound by a CTA's own critical
  // path, not by bytes in flight -- the register path wins there; dispatch favours the pipelines at every CTA count
  if (combine && nranks() == 2 && grid <= 32) return EP_IMPL_REG;
  return EP_IMPL_TMA;
}

int EpBuffer::capacity_for(int hidden, int mode, int topk) const {
  size_t pt = per_token_bytes(hidden, mode, topk);
  if (arena_bytes_ < 5 * 256) return 0;
  return (int)std::min<size_t>((arena_bytes_ - 5 * 256) / pt, (size_t)INT32_MAX);
}

int EpBuffer::combine_capacity_for(int hidden, int topk) const {
  size_t pt = (size_t)hidden * 2 + (size_t)topk * 4;
  if (arena_bytes_ < 2 * 256) return 0;
  return (int)std::min<size_t>((arena_bytes_ - 2 * 256) / pt, (size_t)INT32_MAX);
}

EpArena EpBuffer::carve(int slot, int H, int mode, int K) const {
  EpArena a;
  const int cap = capacity_for(H, mode, K);
  const size_t row = (mode == EP_X_BF16) ? (size_t)H * 2 : (size_t)H;
  uint64_t off = base_off_ + ctrl_bytes_ + (uint64_t)slot * arena_bytes_;
  a.capacity = cap;
  a.x_off = off;
  off = align_up(off + (size_t)cap * row, 256);
  a.scales_off = off;
  if (mode != EP_X_BF16) off = align_up(off + (size_t)cap * (H / 128) * 4, 256);
  a.topk_idx_off = off;
  off = align_up(off + (size_t)cap * K * 8, 256);
  a.topk_w_off = off;
  off = align_up(off + (size_t)cap * K * 4, 256);
  a.src_idx_off = off;
  return a;
}

void EpBuffer::layout(uintptr_t topk_idx, int T, int K, int E, uintptr_t tokens_per_rank, uintptr_t tokens_per_expert,
                      uintptr_t is_token_in_rank, uintptr_t token_pos, cudaStream_t st) {
  const int R = nranks();
  UB_CHECK(E >= 0 && E <= kMaxRanks * kEpMaxLocalExperts, "layout: too many experts (%d)", E);
  UB_CHECK(E == 0 || E % R == 0, "layout: num_experts (%d) must be divisible by the EP size (%d)", E, R);
  UB_CHECK(topk_idx != 0 || is_token_in_rank != 0, "layout: need topk_idx or is_token_in_rank");
  UB_CHECK(token_pos != 0 && is_token_in_rank != 0, "layout: output buffers missing");
  DevGuard g(comm_->device());
  EpLayoutArgs a;
  a.topk_idx = (const int64_t*)topk_idx;
  a.T = T;
  a.K = K;
  a.E = E > 0 ? E : R;
  a.R = R;
  a.tokens_per_rank = (int32_t*)tokens_per_rank;
  a.tokens_per_expert = (int32_t*)tokens_per_expert;
  a.is_token_in_rank = (uint8_t*)is_token_in_rank;
  a.token_pos = (int32_t*)token_pos;
  a.scratch = layout_scratch_;
  a.tokens_per_block = 0;
  cudaError_t e = launch_ep_layout(a, st);
  UB_CHECK(e == cudaSuccess, "ep layout launch failed: %s", cudaGetErrorString(e));
  ++launches_;
}

EpDispatchOut EpBuffer::dispatch(uintptr_t x, uintptr_t x_scales, uintptr_t topk_idx, uintptr_t topk_w,
                                 uintptr_t token_pos, uintptr_t send_slot, uintptr_t tokens_per_rank,
                                 uintptr_t tokens_per_expert, int T, int H, int K, int E, int mode, bool cached,
                                 int reuse_slot, uintptr_t rank_prefix, int expert_alignment, int num_worst_tokens,
                                 bool round_scale, int num_sms, cudaStream_t st) {
  const int R = nranks();
  UB_CHECK(mode >= 0 && mode <= 2, "dispatch: bad mode %d", mode);
  UB_CHECK(H > 0 && H % 8 == 0, "dispatch: hidden (%d) must be a multiple of 8", H);
  if (mode != EP_X_BF16) UB_CHECK(H % 128 == 0 && H <= 8192, "dispatch: fp8 needs hidden %% 128 == 0 and <= 8192 (got %d)", H);
  if (mode == EP_X_FP8_SCALED) UB_CHECK(H % 16 == 0 && x_scales != 0, "dispatch: fp8 input needs scales");
  UB_CHECK(K >= 0 && K <= kEpMaxTopk, "dispatch: num_topk (%d) must be <= %d", K, kEpMaxTopk);
  UB_CHECK(send_slot != 0, "dispatch: send_slot buffer missing");
  UB_CHECK((x & 15) == 0, "dispatch: x must be 16-byte aligned");
  if (!cached) {
    UB_CHECK(token_pos != 0 && tokens_per_rank != 0, "dispatch: layout tensors missing");
    UB_CHECK(E > 0 && E % R == 0 && E / R <= kEpMaxLocalExperts, "dispatch: bad num_experts %d", E);
    UB_CHECK(tokens_per_expert != 0, "dispatch: num_tokens_per_expert missing");
  }
  DevGuard g(comm_->device());
  int slot = reuse_slot;
  if (slot < 0) {
    slot = next_slot_;
    next_slot_ = (next_slot_ + 1) % num_slots_;
  }
  UB_CHECK(slot < num_slots_, "dispatch: bad slot %d", slot);
  EpDispatchArgs a;
  memset(&a, 0, sizeof(a));
  a.x = (const void*)x;
  a.x_scales = (const float*)x_scales;
  a.topk_idx = (const int64_t*)topk_idx;
  a.topk_weights = (const float*)topk_w;
  a.token_pos = (const int32_t*)token_pos;
  a.send_slot = (int32_t*)send_slot;
  a.tokens_per_rank = (const int32_t*)tokens_per_rank;
  a.tokens_per_expert = (const int32_t*)tokens_per_expert;
  a.T = T;
  a.H = H;
  a.K = K;
  a.E = E > 0 ? E : R;
  a.mode = mode;
  a.cached = cached ? 1 : 0;
  a.arena = carve(slot, H, mode, K);
  UB_CHECK(a.arena.capacity > 0, "dispatch: buffer too small (arena %zu B)", arena_bytes_);
  a.cnt_tab_off = base_off_;
  a.exp_tab_off = base_off_ + (uint64_t)kEpMaxBlocks * kMaxRanks * kMaxRanks * 4;
  a.rank_prefix = (int32_t*)rank_prefix;
  a.dev_counts = dev_counts_;
  a.host_counts = (cached || num_worst_tokens > 0) ? nullptr : host_counts_dev_;
  a.expert_alignment = expert_alignment;
  a.num_worst_tokens = num_worst_tokens;
  a.round_scale = round_scale ? 1 : 0;
  if (num_worst_tokens > 0)
    UB_CHECK(num_worst_tokens <= a.arena.capacity, "dispatch: num_worst_tokens (%d) exceeds arena capacity (%d)",
             num_worst_tokens, a.arena.capacity);
  if (a.host_counts) {
    host_counts_[0] = -1;
    __atomic_thread_fence(__ATOMIC_SEQ_CST);
  }
  int grid = std::max(1, std::min(num_sms, kEpMaxBlocks));
  a.in_stages = st_in_;
  a.out_stages = st_out_;
  const bool tma = pick_impl(grid, false) == EP_IMPL_TMA && ep_dispatch_tma_supported(a);
  last_disp_impl_ = tma ? EP_IMPL_TMA : EP_IMPL_REG;
  cudaError_t e = tma ? launch_ep_dispatch_tma(comm_->dev(), a, grid, st) : launch_ep_dispatch(comm_->dev(), a, grid, st);
  UB_CHECK(e == cudaSuccess, "ep dispatch launch failed: %s", cudaGetErrorString(e));
  ++launches_;
  last_stream_ = st;
  EpDispatchOut o;
  char* heap = comm_->fabric().local();
  o.recv_x = (uintptr_t)(heap + a.arena.x_off);
  o.recv_scales = (mode == EP_X_BF16) ? 0 : (uintptr_t)(heap + a.arena.scales_off);
  o.recv_topk_idx = (uintptr_t)(heap + a.arena.topk_idx_off);
  o.recv_topk_w = (uintptr_t)(heap + a.arena.topk_w_off);
  o.recv_src_idx = (uintptr_t)(heap + a.arena.src_idx_off);
  o.slot = slot;
  o.capacity = a.arena.capacity;
  return o;
}

int EpBuffer::wait_counts(int E_local, std::vector<int>* per_expert, double timeout_s) {
  if (timeout_s <= 0) timeout_s = (double)ubParamEpCpuTimeoutSecs();
  auto t0 = std::chrono::steady_clock::now();
  volatile int32_t* hc = host_counts_;
  uint32_t spins = 0;
  while (hc[0] == -1) {
    if ((++spins & 0x3ff) == 0) {
      std::chrono::duration<double> dt = std::chrono::steady_clock::now() - t0;
      if (dt.count() > timeout_s)
        UB_THROW("EP dispatch: CPU timed out after %.1f s waiting for the receive counts (rank %d)", timeout_s, rank());
      if (comm_->error_word()) UB_THROW("EP dispatch: device reported error 0x%x", comm_->error_word());
      if ((spins & 0xfffff) == 0) {
        // a dead context (trap in any kernel of this process) never writes the counts: fail fast
        cudaError_t q = cudaStreamQuery(last_stream_);
        if (q != cudaSuccess && q != cudaErrorNotReady)
          UB_THROW("EP dispatch: CUDA error while waiting for the receive counts: %s", cudaGetErrorString(q));
      }
      sched_yield();
    }
  }
  __atomic_thread_fence(__ATOMIC_ACQUIRE);
  int total = hc[0];
  UB_CHECK(total != -2, "EP dispatch: receive arena overflow (raise num_nvl_bytes)");
  if (per_expert) {
    per_expert->resize(E_local);
    for (int e = 0; e < E_local; ++e) (*per_expert)[e] = hc[1 + e];
  }
  return total;
}

uintptr_t EpBuffer::combine_input_ptr(int num_tokens, int hidden, int topk) {
  UB_CHECK(num_tokens <= combine_capacity_for(hidden, topk), "combine buffer: %d tokens exceed the arena capacity %d",
           num_tokens, combine_capacity_for(hidden, topk));
  return (uintptr_t)(base_ + ctrl_bytes_ + (size_t)num_slots_ * arena_bytes_);
}

void EpBuffer::combine(uintptr_t x, int num_recv, uintptr_t topk_w, uintptr_t send_slot, uintptr_t bias0,
                       uintptr_t bias1, uintptr_t out, uintptr_t out_topk_w, int T, int H, int K, int num_sms,
                       cudaStream_t st) {
  UB_CHECK(H > 0 && H % 8 == 0, "combine: hidden (%d) must be a multiple of 8", H);
  UB_CHECK(K >= 0 && K <= kEpMaxTopk, "combine: bad num_topk %d", K);
  UB_CHECK(send_slot != 0 && out != 0, "combine: handle/out missing");
  DevGuard g(comm_->device());
  const int cap = combine_capacity_for(H, K);
  UB_CHECK(num_recv <= cap, "combine: %d tokens exceed the arena capacity %d", num_recv, cap);
  char* arena = base_ + ctrl_bytes_ + (size_t)num_slots_ * arena_bytes_;
  const size_t xbytes = (size_t)num_recv * H * 2;
  EpCombineArgs a;
  memset(&a, 0, sizeof(a));
  if (x != (uintptr_t)arena && xbytes) {
    if (comm_->in_heap((void*)x, xbytes)) {
      // any symmetric tensor works in place as long as every rank passes the same offset
      a.x_off = comm_->heap_offset((void*)x);
    } else {
      UB_CUDA(cudaMemcpyAsync(arena, (void*)x, xbytes, cudaMemcpyDeviceToDevice, st));
      a.x_off = comm_->heap_offset(arena);
    }
  } else {
    a.x_off = comm_->heap_offset(arena);
  }
  a.topk_w_off = kNoOff;
  if (topk_w && out_topk_w && K > 0) {
    char* wdst = arena + align_up((size_t)cap * H * 2, 256);
    UB_CUDA(cudaMemcpyAsync(wdst, (void*)topk_w, (size_t)num_recv * K * 4, cudaMemcpyDeviceToDevice, st));
    a.topk_w_off = comm_->heap_offset(wdst);
  }
  a.send_slot = (const int32_t*)send_slot;
  a.bias0 = (const void*)bias0;
  a.bias1 = (const void*)bias1;
  a.out = (void*)out;
  a.out_topk_w = (float*)out_topk_w;
  a.T = T;
  a.H = H;
  a.K = K;
  int grid = std::max(1, std::min(num_sms, kEpMaxBlocks));
  a.stages = st_comb_;
  const bool tma = pick_impl(grid, true) == EP_IMPL_TMA && ep_combine_tma_supported(a);
  last_comb_impl_ = tma ? EP_IMPL_TMA : EP_IMPL_REG;
  cudaError_t e = tma ? launch_ep_combine_tma(comm_->dev(), a, grid, st) : launch_ep_combine(comm_->dev(), a, grid, st);
  UB_CHECK(e == cudaSuccess, "ep combine launch failed: %s", cudaGetErrorString(e));
  ++launches_;
}

// ------------------------------------------------------------------ low latency
namespace {
size_t ll_cnt_tab_bytes(int E) { return align_up((size_t)kEpLLMaxBlocks * kMaxRanks * E * 4, 4096); }
size_t ll_half_bytes(int M, int H, int R, int E) {
  const size_t rows = (size_t)(E / R) * R * M;
  size_t b = 0;
  b += align_up(rows * (size_t)H * 2, 256);        // recv_x (bf16 worst case)
  b += align_up(rows * (size_t)(H / 128) * 4, 256);  // scales
  b += align_up(rows * 4, 256);                      // src info
  b += align_up(rows * (size_t)H * 2, 256);        // combine input (bf16 expert outputs)
  return b;
}
}  // namespace

size_t EpBuffer::ll_size_hint(int M, int H, int R, int E) {
  return ll_cnt_tab_bytes(E) + 2 * ll_half_bytes(M, H, R, E) + 4096;
}

void EpBuffer::ll_init(size_t ll_bytes) {
  if (ll_base_) return;
  DevGuard g(comm_->device());
  ll_bytes_ = align_up(ll_bytes, 4096);
  ll_base_ = (char*)comm_->alloc(ll_bytes_, 4096);
  UB_CUDA(cudaMemset(ll_base_, 0, std::min<size_t>(ll_bytes_, 8u << 20)));
  UB_CUDA(cudaMalloc((void**)&ll_send_cnt_, sizeof(int32_t) * 2 * kMaxRanks * kEpMaxLocalExperts));
  UB_CUDA(cudaMemset(ll_send_cnt_, 0, sizeof(int32_t) * 2 * kMaxRanks * kEpMaxLocalExperts));
  UB_CUDA(cudaDeviceSynchronize());
}

EpBuffer::LLLayout EpBuffer::ll_layout(int buffer_idx, int H, int E, int M) const {
  const int R = nranks();
  UB_CHECK(ll_base_ != nullptr, "low-latency buffer not initialised (construct Buffer with num_rdma_bytes > 0)");
  UB_CHECK(ll_size_hint(M, H, R, E) <= ll_bytes_, "low-latency buffer too small: need %zu bytes, have %zu",
           ll_size_hint(M, H, R, E), ll_bytes_);
  const size_t rows = (size_t)(E / R) * R * M;
  LLLayout l;
  uint64_t off = comm_->heap_offset(ll_base_);
  l.cnt_tab_off = off;
  off += ll_cnt_tab_bytes(E) + (uint64_t)buffer_idx * ll_half_bytes(M, H, R, E);
  l.recv_x_off = off;
  off += align_up(rows * (size_t)H * 2, 256);
  l.recv_scales_off = off;
  off += align_up(rows * (size_t)(H / 128) * 4, 256);
  l.recv_src_off = off;
  off += align_up(rows * 4, 256);
  l.comb_x_off = off;
  return l;
}

EpBuffer::LLOut EpBuffer::ll_dispatch(uintptr_t x, uintptr_t topk_idx, int T, int H, int K, int E, int M, bool use_fp8,
                                      bool round_scale, uintptr_t recv_count, uintptr_t layout_range,
                                      uintptr_t send_pos, int num_sms, cudaStream_t st, int phase, int scale_layout,
                                      uintptr_t wait_stats) {
  const int R = nranks();
  UB_CHECK(phase == EP_LL_FULL || phase == EP_LL_SEND, "ll_dispatch: phase must be FULL or SEND");
  UB_CHECK(ll_pending_grid_ == 0, "ll_dispatch: the receive hook of the previous dispatch has not been called");
  UB_CHECK(scale_layout >= EP_LL_SCALES_ROW_MAJOR && scale_layout <= EP_LL_SCALES_COL_UE8M0, "ll_dispatch: bad scale layout");
  if (scale_layout == EP_LL_SCALES_COL_UE8M0)
    UB_CHECK(use_fp8 && round_scale && H % 512 == 0, "ll_dispatch: UE8M0 scales need fp8, round_scale and hidden %% 512 == 0");
  UB_CHECK(E > 0 && E % R == 0 && E <= kMaxRanks * kEpMaxLocalExperts, "ll_dispatch: bad num_experts %d", E);
  UB_CHECK(H % 128 == 0 && H <= 8192, "ll_dispatch: hidden must be a multiple of 128 and <= 8192 (got %d)", H);
  UB_CHECK(K > 0 && K <= 32, "ll_dispatch: bad num_topk %d", K);
  UB_CHECK(T <= M, "ll_dispatch: %d tokens exceed num_max_dispatch_tokens_per_rank %d", T, M);
  UB_CHECK((x & 15) == 0, "ll_dispatch: x must be 16-byte aligned");
  DevGuard g(comm_->device());
  const int idx = ll_next_;
  ll_next_ ^= 1;
  LLLayout l = ll_layout(idx, H, E, M);
  EpLLDispatchArgs a;
  memset(&a, 0, sizeof(a));
  a.x = (const void*)x;
  a.topk_idx = (const int64_t*)topk_idx;
  a.T = T;
  a.H = H;
  a.K = K;
  a.E = E;
  a.M = M;
  a.use_fp8 = use_fp8 ? 1 : 0;
  a.round_scale = round_scale ? 1 : 0;
  a.recv_x_off = l.recv_x_off;
  a.recv_scales_off = l.recv_scales_off;
  a.recv_src_off = l.recv_src_off;
  a.cnt_tab_off = l.cnt_tab_off;
  a.send_cnt = ll_send_cnt_;
  a.parity = ll_parity_;
  ll_parity_ ^= 1;
  a.send_pos = (int64_t*)send_pos;
  a.recv_count = (int32_t*)recv_count;
  a.layout_range = (int64_t*)layout_range;
  a.phase = phase;
  a.scale_layout = use_fp8 ? scale_layout : EP_LL_SCALES_ROW_MAJOR;
  a.wait_stats = (long long*)wait_stats;
  int grid = std::max(1, std::min(std::min(num_sms, kEpLLMaxBlocks), std::max(T, 1)));  // one CTA per token
  cudaError_t e = launch_ep_ll_dispatch(comm_->dev(), a, grid, st);
  UB_CHECK(e == cudaSuccess, "ep ll_dispatch launch failed: %s", cudaGetErrorString(e));
  ++launches_;
  if (phase == EP_LL_SEND) ll_pending_grid_ = grid;
  char* heap = comm_->fabric().local();
  LLOut o;
  o.recv_x = (uintptr_t)(heap + l.recv_x_off);
  o.recv_scales = (uintptr_t)(heap + l.recv_scales_off);
  o.recv_src_info = (uintptr_t)(heap + l.recv_src_off);
  o.combine_x = (uintptr_t)(heap + l.comb_x_off);
  o.buffer_idx = idx;
  return o;
}

void EpBuffer::ll_dispatch_recv(int num_sms, uintptr_t wait_stats, cudaStream_t st) {
  UB_CHECK(ll_pending_grid_ > 0, "ll_dispatch_recv: no send-phase dispatch is pending");
  DevGuard g(comm_->device());
  EpLLDispatchArgs a;
  memset(&a, 0, sizeof(a));
  a.phase = EP_LL_RECV;
  a.H = 128;
  a.E = nranks();
  a.wait_stats = (long long*)wait_stats;
  const int grid = ll_pending_grid_;  // the same block indices that signalled
  (void)num_sms;
  cudaError_t e = launch_ep_ll_dispatch(comm_->dev(), a, grid, st);
  UB_CHECK(e == cudaSuccess, "ep ll_dispatch (receive half) launch failed: %s", cudaGetErrorString(e));
  ++launches_;
  ll_pending_grid_ = 0;
}

uintptr_t EpBuffer::ll_combine_buffer(int buffer_idx, int H, int E, int M) const {
  LLLayout l = ll_layout(buffer_idx, H, E, M);
  return (uintptr_t)(comm_->fabric().local() + l.comb_x_off);
}

void EpBuffer::ll_combine(uintptr_t x, int buffer_idx, uintptr_t topk_w, uintptr_t send_pos, uintptr_t out, int T,
                          int H, int K, int E, int M, int num_sms, cudaStream_t st, int phase, uintptr_t layout_range,
                          uintptr_t wait_stats, bool use_logfmt) {
  const int R = nranks();
  UB_CHECK(phase >= EP_LL_FULL && phase <= EP_LL_RECV, "ll_combine: bad phase %d", phase);
  DevGuard g(comm_->device());
  LLLayout l = ll_layout(buffer_idx, H, E, M);
  char* arena = comm_->fabric().local() + l.comb_x_off;
  if (use_logfmt && phase != EP_LL_RECV)
    UB_CHECK(layout_range != 0 && H % 128 == 0, "ll_combine: use_logfmt needs layout_range and hidden %% 128 == 0 (H = %d)", H);
  if ((x != (uintptr_t)arena || use_logfmt) && phase != EP_LL_RECV) {
    // expert outputs that do not live in the symmetric buffer: bring them in, occupied rows only; with use_logfmt
    // the same pass applies the reference's simulated LogFMT-10 cast (in place when x already is the buffer)
    if (layout_range) {
      EpLLPackArgs pa;
      pa.src = (const void*)x;
      pa.dst = arena;
      pa.layout_range = (const int64_t*)layout_range;
      pa.E_local = E / R;
      pa.R = R;
      pa.M = M;
      pa.H = H;
      pa.logfmt = use_logfmt ? 1 : 0;
      cudaError_t pe = launch_ep_ll_pack(pa, st);
      UB_CHECK(pe == cudaSuccess, "ep ll pack launch failed: %s", cudaGetErrorString(pe));
      ++launches_;
    } else {
      const size_t bytes = (size_t)(E / R) * R * M * H * 2;
      UB_CUDA(cudaMemcpyAsync(arena, (void*)x, bytes, cudaMemcpyDeviceToDevice, st));
    }
  }
  EpLLCombineArgs a;
  memset(&a, 0, sizeof(a));
  a.x_off = l.comb_x_off;
  a.send_pos = (const int64_t*)send_pos;
  a.topk_weights = (const float*)topk_w;
  a.out = (void*)out;
  a.T = T;
  a.H = H;
  a.K = K;
  a.phase = phase;
  a.wait_stats = (long long*)wait_stats;
  int grid = std::max(1, std::min(num_sms, kEpMaxBlocks));
  cudaError_t e = launch_ep_ll_combine(comm_->dev(), a, grid, st);
  UB_CHECK(e == cudaSuccess, "ep ll_combine launch failed: %s", cudaGetErrorString(e));
  ++launches_;
}

}  // namespace ub
