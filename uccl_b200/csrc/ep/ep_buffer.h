// Host runtime of the expert-parallel buffer (Hopper-native counterpart of the reference's
// `class Buffer`, ep/src/uccl_ep.cc:315-1600).  No IPC-handle exchange, proxies or ring
// buffers: the buffer is one block of the communicator's symmetric heap carved into
//   [ctrl | dispatch arena 0 .. S-1 | combine arena]
// and every kernel addresses peers through the fabric's mapped VAs.
#pragma once
#include <cuda_runtime.h>

#include <memory>
#include <vector>

#include "../coll/comm.h"
#include "ep_types.h"

namespace ub {

struct EpDispatchOut {
  uintptr_t recv_x, recv_scales, recv_topk_idx, recv_topk_w, recv_src_idx;
  int slot;
  int capacity;
};

class EpBuffer {
 public:
  EpBuffer(std::shared_ptr<Comm> comm, size_t num_nvl_bytes, int num_slots);
  ~EpBuffer();

  int rank() const { return comm_->rank(); }
  int nranks() const { return comm_->nranks(); }
  size_t arena_bytes() const { return arena_bytes_; }
  int num_slots() const { return num_slots_; }
  int capacity_for(int hidden, int mode, int topk) const;
  int combine_capacity_for(int hidden, int topk) const;
  uint64_t launches() const { return launches_; }
  uint64_t base_offset() const { return base_off_; }  // heap offset of the EP block (must match on every rank)
  // raw views for DeepEP's get_local_buffer_tensor: the arena area of the EP block (control words excluded) and
  // the low-latency block (0 / 0 before ll_init)
  uintptr_t arena_area_ptr() const { return (uintptr_t)(base_ + ctrl_bytes_); }
  size_t arena_area_bytes() const { return bytes_ - ctrl_bytes_; }
  uintptr_t ll_ptr() const { return (uintptr_t)ll_base_; }
  size_t ll_nbytes() const { return ll_bytes_; }
  // kernel implementation of dispatch / combine: EP_IMPL_AUTO (default, UCCL_B200_EP_IMPL), _REG or _TMA
  int impl() const { return impl_; }
  void set_impl(int impl);
  // TMA pipeline depths (0 = fill shared memory): dispatch in/out stages, combine stages
  void set_stages(int disp_in, int disp_out, int comb) { st_in_ = disp_in, st_out_ = disp_out, st_comb_ = comb; }
  int last_dispatch_impl() const { return last_disp_impl_; }
  int last_combine_impl() const { return last_comb_impl_; }

  // topk_idx != 0: full layout (counts + membership + positions); topk_idx == 0: positions only
  void layout(uintptr_t topk_idx, int T, int K, int E, uintptr_t tokens_per_rank, uintptr_t tokens_per_expert,
              uintptr_t is_token_in_rank, uintptr_t token_pos, cudaStream_t st);

  EpDispatchOut dispatch(uintptr_t x, uintptr_t x_scales, uintptr_t topk_idx, uintptr_t topk_w, uintptr_t token_pos,
                         uintptr_t send_slot, uintptr_t tokens_per_rank, uintptr_t tokens_per_expert, int T, int H,
                         int K, int E, int mode, bool cached, int reuse_slot, uintptr_t rank_prefix,
                         int expert_alignment, int num_worst_tokens, bool round_scale, int num_sms, cudaStream_t st);
  // CPU wait for the counts of the latest non-cached dispatch. Returns recv_total (>= 0),
  // throws on overflow (-2) / timeout.
  int wait_counts(int E_local, std::vector<int>* per_expert, double timeout_s);
  uintptr_t dev_counts_ptr() const { return (uintptr_t)dev_counts_; }

  // ---- low-latency mode (double-buffered region of `ll_bytes`, allocated on first use)
  void ll_init(size_t ll_bytes);
  struct LLOut {
    uintptr_t recv_x, recv_scales, recv_src_info, combine_x;
    int buffer_idx;
  };
  static size_t ll_size_hint(int M, int H, int R, int E);
  // phase: EP_LL_FULL, or EP_LL_SEND followed later by ll_dispatch_recv() (return_recv_hook)
  LLOut ll_dispatch(uintptr_t x, uintptr_t topk_idx, int T, int H, int K, int E, int M, bool use_fp8, bool round_scale,
                    uintptr_t recv_count, uintptr_t layout_range, uintptr_t send_pos, int num_sms, cudaStream_t st,
                    int phase = EP_LL_FULL, int scale_layout = EP_LL_SCALES_ROW_MAJOR, uintptr_t wait_stats = 0);
  void ll_dispatch_recv(int num_sms, uintptr_t wait_stats, cudaStream_t st);  // receive half of the last SEND-phase dispatch
  uintptr_t ll_combine_buffer(int buffer_idx, int H, int E, int M) const;
  // layout_range != 0: a non-arena `x` is packed (occupied rows only) instead of copied whole
  void ll_combine(uintptr_t x, int buffer_idx, uintptr_t topk_w, uintptr_t send_pos, uintptr_t out, int T, int H, int K,
                  int E, int M, int num_sms, cudaStream_t st, int phase = EP_LL_FULL, uintptr_t layout_range = 0,
                  uintptr_t wait_stats = 0, bool use_logfmt = false);

  // zero-copy combine input: a [num_tokens, hidden] bf16 view of the combine arena
  uintptr_t combine_input_ptr(int num_tokens, int hidden, int topk);
  void combine(uintptr_t x, int num_recv, uintptr_t topk_w, uintptr_t send_slot, uintptr_t bias0, uintptr_t bias1,
               uintptr_t out, uintptr_t out_topk_w, int T, int H, int K, int num_sms, cudaStream_t st);

 private:
  EpArena carve(int slot, int H, int mode, int K) const;
  std::shared_ptr<Comm> comm_;
  char* base_ = nullptr;      // local VA of the EP block
  uint64_t base_off_ = 0;     // its heap offset
  size_t bytes_ = 0;
  size_t ctrl_bytes_ = 0;
  size_t arena_bytes_ = 0;
  int num_slots_ = 2;
  int next_slot_ = 0;
  int32_t* host_counts_ = nullptr;  // pinned + mapped
  int32_t* host_counts_dev_ = nullptr;
  int32_t* dev_counts_ = nullptr;
  uint64_t launches_ = 0;
  cudaStream_t last_stream_ = nullptr;
  uint32_t* layout_scratch_ = nullptr;  // multi-CTA layout: epoch, flags, per-CTA counts
  int impl_ = EP_IMPL_AUTO;
  int st_in_ = 0, st_out_ = 0, st_comb_ = 0;
  int last_disp_impl_ = 0, last_comb_impl_ = 0;
  int pick_impl(int grid, bool combine) const;
  // low latency
  struct LLLayout {
    uint64_t cnt_tab_off, recv_x_off, recv_scales_off, recv_src_off, comb_x_off;
  };
  LLLayout ll_layout(int buffer_idx, int H, int E, int M) const;
  char* ll_base_ = nullptr;
  size_t ll_bytes_ = 0;
  int ll_next_ = 0;
  int32_t* ll_send_cnt_ = nullptr;
  int ll_parity_ = 0;
  int ll_pending_grid_ = 0;  // grid of a SEND-phase dispatch whose receive half has not run yet
};

cudaError_t launch_ep_layout(const EpLayoutArgs& a, cudaStream_t st);
cudaError_t launch_ep_dispatch(const DevComm& c, const EpDispatchArgs& a, int grid, cudaStream_t st);
cudaError_t launch_ep_combine(const DevComm& c, const EpCombineArgs& a, int grid, cudaStream_t st);
// TMA-pipelined implementations (ep_tma_kernels.cu)
bool ep_dispatch_tma_supported(const EpDispatchArgs& a);
bool ep_combine_tma_supported(const EpCombineArgs& a);
cudaError_t launch_ep_dispatch_tma(const DevComm& c, const EpDispatchArgs& a, int grid, cudaStream_t st);
cudaError_t launch_ep_combine_tma(const DevComm& c, const EpCombineArgs& a, int grid, cudaStream_t st);
cudaError_t launch_ep_ll_dispatch(const DevComm& c, const EpLLDispatchArgs& a, int grid, cudaStream_t st);
cudaError_t launch_ep_ll_combine(const DevComm& c, const EpLLCombineArgs& a, int grid, cudaStream_t st);
cudaError_t launch_ep_ll_pack(const EpLLPackArgs& a, cudaStream_t st);
constexpr int kEpLLMaxBlocks = 128;  // one CTA per token of a decode batch

}  // namespace ub
