// Expert-parallel dispatch / combine kernels for one NVSwitch node (sm_90a).
//
// What the reference does (ep/src/layout.cu:9-150, ep/src/intranode.cu:12-1152): a layout
// kernel, a notify kernel that all-to-alls the counts, then sender CTAs copy tokens into the
// *receiver's ring buffer* and receiver CTAs copy them again into recv_x (two passes over the
// payload, FP8 cast done beforehand by separate torch kernels, ep/bench/utils.py:666-675).
//
// Hopper-native design here -- direct placement, one pass, fused cast:
//   * counts are exchanged inside the dispatch kernel (peer stores + block barrier), every rank
//     then knows the full R x R matrix and therefore the exact slot of each of its tokens in each
//     destination arena: no ring, no receiver CTAs, no second copy;
//   * each warp loads a token once, (optionally) computes the per-128-channel amax, scales and
//     casts to e4m3 in registers, and stores the row + scales + remapped top-k metadata straight
//     into every destination rank's arena over NVLink;
//   * combine is a pull: the source rank reads the (<= R) expert-output rows it needs from the
//     peers' symmetric arenas, reduces in fp32 in a fixed order and writes bf16 once.
#include "../kernels/launch.h"
#include "../kernels/prims.cuh"
#include "ep_common.cuh"
#include "ep_types.h"

namespace ub {

// ----------------------------------------------------------------------------- layout
// Single CTA, 1024 threads: histogram per expert, per-rank membership and the exclusive
// per-rank running position of every token (needed for direct placement).
// If a.topk_idx == nullptr the membership is read from a.is_token_in_rank instead.
__global__ void __launch_bounds__(1024, 1) ep_layout_kernel(const EpLayoutArgs a) {
  extern __shared__ int s_dyn[];
  int* s_expert = s_dyn;                  // [E]
  __shared__ int s_warp_tot[32][kMaxRanks];
  __shared__ int s_warp_off[32][kMaxRanks];
  __shared__ int s_running[kMaxRanks];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int R = a.R, E_local = a.E / a.R;
  for (int e = tid; e < a.E; e += blockDim.x) s_expert[e] = 0;
  if (tid < kMaxRanks) s_running[tid] = 0;
  __syncthreads();
  for (int base = 0; base < a.T; base += blockDim.x) {
    const int t = base + tid;
    unsigned mask = 0;
    if (t < a.T) {
      if (a.topk_idx) {
        for (int k = 0; k < a.K; ++k) {
          long long e = a.topk_idx[(size_t)t * a.K + k];
          if (e >= 0 && e < a.E) {
            atomicAdd(&s_expert[(int)e], 1);
            mask |= 1u << ((int)e / E_local);
          }
        }
      } else {
        for (int r = 0; r < R; ++r) mask |= (a.is_token_in_rank[(size_t)t * R + r] ? 1u : 0u) << r;
      }
    }
    int pos_in_warp[kMaxRanks];
#pragma unroll
    for (int r = 0; r < kMaxRanks; ++r) {
      unsigned b = __ballot_sync(0xffffffffu, (mask >> r) & 1u);
      pos_in_warp[r] = __popc(b & ((1u << lane) - 1u));
      if (lane == 0) s_warp_tot[warp][r] = __popc(b);
    }
    __syncthreads();
    if (tid < 32 * kMaxRanks) {
      const int w = tid / kMaxRanks, r = tid % kMaxRanks;
      int off = 0;
      for (int i = 0; i < w; ++i) off += s_warp_tot[i][r];
      s_warp_off[w][r] = off;
    }
    __syncthreads();
    if (t < a.T) {
#pragma unroll
      for (int r = 0; r < kMaxRanks; ++r) {
        if (r < R) {
          const bool in = (mask >> r) & 1u;
          if (a.topk_idx) a.is_token_in_rank[(size_t)t * R + r] = in ? 1 : 0;
          a.token_pos[(size_t)t * R + r] = in ? (s_running[r] + s_warp_off[warp][r] + pos_in_warp[r]) : -1;
        }
      }
    }
    __syncthreads();
    if (tid < kMaxRanks) s_running[tid] += s_warp_off[31][tid] + s_warp_tot[31][tid];
    __syncthreads();
  }
  if (tid < R && a.tokens_per_rank) a.tokens_per_rank[tid] = s_running[tid];
  if (a.tokens_per_expert && a.topk_idx)
    for (int e = tid; e < a.E; e += blockDim.x) a.tokens_per_expert[e] = s_expert[e];
}

// Multi-CTA layout: every CTA owns `tokens_per_block` consecutive tokens.  It counts its tokens per
// rank, publishes the counts (flag = epoch of this call), waits for the counts of all lower-numbered
// CTAs (they were scheduled earlier, so the wait cannot deadlock even if the grid is not co-resident)
// and then writes the same stable positions as the single-CTA kernel.  The expert histogram is
// accumulated in shared memory and added to the global one, which CTA 0 zeroes before it publishes.
// Replaces a single-CTA scan that took a large share of an EP=1 step.
__global__ void __launch_bounds__(kEpLayoutThreads) ep_layout_mc_kernel(const EpLayoutArgs a) {
  extern __shared__ int s_dyn[];
  int* s_expert = s_dyn;                                               // [E]
  unsigned char* s_mask = reinterpret_cast<unsigned char*>(s_dyn + a.E);  // [tokens_per_block]
  constexpr int NW = kEpLayoutThreads / 32;
  __shared__ int s_warp_tot[NW][kMaxRanks];
  __shared__ int s_cnt[kMaxRanks];      // tokens of this CTA per rank
  __shared__ int s_running[kMaxRanks];  // positions handed out so far (prefix of lower CTAs + earlier steps)
  __shared__ uint32_t s_epoch;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int R = a.R, E_local = a.E / a.R;
  const int b = blockIdx.x, B = gridDim.x;
  uint32_t* flags = a.scratch + 16;
  uint32_t* cnts = a.scratch + 16 + kEpLayoutMaxBlocks;
  const bool want_experts = a.tokens_per_expert && a.topk_idx;
  if (tid == 0) s_epoch = ld_volatile(a.scratch) + 1;
  for (int e = tid; e < a.E; e += blockDim.x) s_expert[e] = 0;
  if (tid < kMaxRanks) {
    s_cnt[tid] = 0;
    s_running[tid] = 0;
  }
  __syncthreads();
  const uint32_t epoch = s_epoch;
  const int t_lo = min(a.T, b * a.tokens_per_block), t_hi = min(a.T, t_lo + a.tokens_per_block);

  // ---- pass A: membership masks, expert histogram, per-rank counts of this CTA
  for (int base = t_lo; base < t_hi; base += blockDim.x) {
    const int t = base + tid;
    unsigned mask = 0;
    if (t < t_hi) {
      if (a.topk_idx) {
        for (int k = 0; k < a.K; ++k) {
          const long long e = a.topk_idx[(size_t)t * a.K + k];
          if (e >= 0 && e < a.E) {
            if (want_experts) atomicAdd(&s_expert[(int)e], 1);
            mask |= 1u << ((int)e / E_local);
          }
        }
        for (int r = 0; r < R; ++r) a.is_token_in_rank[(size_t)t * R + r] = (mask >> r) & 1u;
      } else {
        for (int r = 0; r < R; ++r) mask |= (a.is_token_in_rank[(size_t)t * R + r] ? 1u : 0u) << r;
      }
      s_mask[t - t_lo] = (unsigned char)mask;
    }
#pragma unroll
    for (int r = 0; r < kMaxRanks; ++r) {
      const unsigned bal = __ballot_sync(0xffffffffu, (mask >> r) & 1u);
      if (lane == 0 && bal) atomicAdd(&s_cnt[r], __popc(bal));
    }
  }
  __syncthreads();
  // ---- publish my counts; CTA 0 zeroes the global expert histogram first
  if (b == 0 && want_experts)
    for (int e = tid; e < a.E; e += blockDim.x) a.tokens_per_expert[e] = 0;
  if (tid < kMaxRanks) cnts[b * kMaxRanks + tid] = s_cnt[tid];
  __threadfence();
  __syncthreads();
  if (tid == 0) st_release_gpu(&flags[b], epoch);
  // ---- wait for every lower CTA, accumulate its counts
  for (int q = tid; q < b; q += blockDim.x) {
    SpinGuard g(20ull * 1000 * 1000 * 1000);
    while (ld_acquire_gpu(&flags[q]) != epoch) {
      if (g.expired()) {
        printf("[uccl_b200] ep layout: block %d timed out waiting for block %d\n", b, q);
        __trap();
      }
    }
    for (int r = 0; r < R; ++r) {
      const int v = (int)cnts[q * kMaxRanks + r];
      if (v) atomicAdd(&s_running[r], v);
    }
  }
  __syncthreads();
  if (b == B - 1) {
    if (tid < R && a.tokens_per_rank) a.tokens_per_rank[tid] = s_running[tid] + s_cnt[tid];
    if (tid == 0) *reinterpret_cast<volatile uint32_t*>(a.scratch) = epoch;  // every CTA has read the old value
  }
  // ---- pass B: stable positions
  for (int base = t_lo; base < t_hi; base += blockDim.x) {
    const int t = base + tid;
    const unsigned mask = t < t_hi ? s_mask[t - t_lo] : 0u;
    int pos_in_warp[kMaxRanks];
#pragma unroll
    for (int r = 0; r < kMaxRanks; ++r) {
      const unsigned bal = __ballot_sync(0xffffffffu, (mask >> r) & 1u);
      pos_in_warp[r] = __popc(bal & ((1u << lane) - 1u));
      if (lane == 0) s_warp_tot[warp][r] = __popc(bal);
    }
    __syncthreads();
    if (t < t_hi) {
#pragma unroll
      for (int r = 0; r < kMaxRanks; ++r) {
        if (r < R) {
          int off = s_running[r];
          for (int w = 0; w < warp; ++w) off += s_warp_tot[w][r];
          a.token_pos[(size_t)t * R + r] = ((mask >> r) & 1u) ? off + pos_in_warp[r] : -1;
        }
      }
    }
    __syncthreads();
    if (tid < kMaxRanks) {
      int tot = 0;
      for (int w = 0; w < NW; ++w) tot += s_warp_tot[w][tid];
      s_running[tid] += tot;
    }
    __syncthreads();
  }
  // ---- expert histogram (CTA 0 zeroed it before any flag of this call was visible)
  if (want_experts)
    for (int e = tid; e < a.E; e += blockDim.x)
      if (s_expert[e]) atomicAdd(&a.tokens_per_expert[e], s_expert[e]);
}

// --------------------------------------------------------------------------- dispatch
// NR = number of ranks (1, 2, 4, 8): per-destination loops are unrolled to NR, so small EP degrees
// do not pay for predicated-off stores / address arithmetic of absent ranks.
template <int MODE, int NR>
__global__ void __launch_bounds__(512, 1) ep_dispatch_kernel(const __grid_constant__ DevComm c,
                                                             const __grid_constant__ EpDispatchArgs a) {
  const int R = c.nranks, me = c.rank;  // R <= NR
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int E_local = a.E / R;
  __shared__ int s_M[kMaxRanks][kMaxRanks];
  __shared__ int s_base[kMaxRanks];
  __shared__ int s_abort;
  __shared__ int s_recv_total;
  __shared__ float s_scales[16][64];

  BlockSync s = sync_begin(c, kDomEp, blockIdx.x);
  if (tid == 0) {
    s_abort = 0;
    s_recv_total = 0;
  }
  ep_dispatch_prologue(c, a, s, s_M, s_base, &s_abort, &s_recv_total);

  if (!s_abort) {
    const size_t in_row_bytes = (MODE == EP_X_FP8_SCALED) ? (size_t)a.H : (size_t)a.H * 2;
    const size_t out_row_bytes = (MODE == EP_X_BF16) ? (size_t)a.H * 2 : (size_t)a.H;
    const int n_scales = a.H / 128;
    const int warps_total = gridDim.x * (blockDim.x >> 5);
    for (int t = blockIdx.x * (blockDim.x >> 5) + warp; t < a.T; t += warps_total) {
      int my = -1;
      if (lane < R) {
        if (a.cached) {
          my = a.send_slot[(size_t)t * R + lane];
        } else {
          const int p = a.token_pos[(size_t)t * R + lane];
          my = p >= 0 ? s_base[lane] + p : -1;
          a.send_slot[(size_t)t * R + lane] = my;
        }
      }
      const unsigned mask = __ballot_sync(0xffffffffu, my >= 0);
      if (mask == 0) continue;
      char* dst_x[NR];
      int slots[NR];
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        slots[r] = __shfl_sync(0xffffffffu, my, r);
        dst_x[r] = ((mask >> r) & 1u) ? c.heap[r] + a.arena.x_off + (size_t)slots[r] * out_row_bytes : nullptr;
      }
      const char* src = reinterpret_cast<const char*>(a.x) + (size_t)t * in_row_bytes;

      if constexpr (MODE == EP_X_FUSED_FP8) {
        const int units = a.H / 16;  // 16 output bytes (16 channels) per lane-iteration
        constexpr int PF = 4;        // iterations whose loads are in flight together (8 x 16 B per lane; 7 spills)
        for (int ub = 0; ub < units; ub += 32 * PF) {
          uint4 v0[PF], v1[PF];
#pragma unroll
          for (int j = 0; j < PF; ++j) {
            const int u = ub + j * 32 + lane;
            v0[j] = make_uint4(0, 0, 0, 0);
            v1[j] = v0[j];
            if (u < units) {
              v0[j] = ld_nc_v4(src + (size_t)u * 32);
              v1[j] = ld_nc_v4(src + (size_t)u * 32 + 16);
            }
          }
#pragma unroll
          for (int j = 0; j < PF; ++j) {
            const int u = ub + j * 32 + lane;
            if (ub + j * 32 >= units) break;  // warp-uniform
            const bool valid = u < units;
            float f[16];
            bf16x8_to_float(v0[j], *reinterpret_cast<float(*)[8]>(&f[0]));
            bf16x8_to_float(v1[j], *reinterpret_cast<float(*)[8]>(&f[8]));
            float amax = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) amax = fmaxf(amax, fabsf(f[i]));
            // 128 channels = 8 consecutive lanes
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
            float scale, scale_inv;
            fp8_group_scale(amax, a.round_scale, scale, scale_inv);
            uint4 o;
            o.x = pack4_e4m3(f[0] * scale, f[1] * scale, f[2] * scale, f[3] * scale);
            o.y = pack4_e4m3(f[4] * scale, f[5] * scale, f[6] * scale, f[7] * scale);
            o.z = pack4_e4m3(f[8] * scale, f[9] * scale, f[10] * scale, f[11] * scale);
            o.w = pack4_e4m3(f[12] * scale, f[13] * scale, f[14] * scale, f[15] * scale);
            if (valid) {
#pragma unroll
              for (int r = 0; r < NR; ++r)
                if ((mask >> r) & 1u) st_v4(dst_x[r] + (size_t)u * 16, o);
              if ((lane & 7) == 0) s_scales[warp][u >> 3] = scale_inv;
            }
          }
        }
        __syncwarp();
#pragma unroll
        for (int r = 0; r < NR; ++r) {
          if ((mask >> r) & 1u) {
            float* ds = reinterpret_cast<float*>(c.heap[r] + a.arena.scales_off) + (size_t)slots[r] * n_scales;
            for (int j = lane; j < n_scales; j += 32) ds[j] = s_scales[warp][j];
          }
        }
        __syncwarp();
      } else {
        const int chunks = (int)(out_row_bytes / 16);
        for (int i0 = 0; i0 < chunks; i0 += 128) {
          uint4 v[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int i = i0 + j * 32 + lane;
            if (i < chunks) v[j] = ld_nc_v4(src + (size_t)i * 16);
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int i = i0 + j * 32 + lane;
            if (i < chunks) {
#pragma unroll
              for (int r = 0; r < NR; ++r)
                if ((mask >> r) & 1u) st_v4(dst_x[r] + (size_t)i * 16, v[j]);
            }
          }
        }
        if constexpr (MODE == EP_X_FP8_SCALED) {
          const float* ssrc = a.x_scales + (size_t)t * n_scales;
#pragma unroll
          for (int r = 0; r < NR; ++r) {
            if ((mask >> r) & 1u) {
              float* ds = reinterpret_cast<float*>(c.heap[r] + a.arena.scales_off) + (size_t)slots[r] * n_scales;
              for (int j = lane; j < n_scales; j += 32) ds[j] = ssrc[j];
            }
          }
        }
      }
      // ---- metadata: remapped top-k ids / weights + source token index
      long long idx = -1;
      float w = 0.f;
      if (a.topk_idx && lane < a.K) {
        idx = a.topk_idx[(size_t)t * a.K + lane];
        if (a.topk_weights) w = a.topk_weights[(size_t)t * a.K + lane];
      }
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        if ((mask >> r) & 1u) {
          const int slot = slots[r];
          if (a.topk_idx && lane < a.K) {
            const bool mine = idx >= (long long)r * E_local && idx < (long long)(r + 1) * E_local;
            long long* di = reinterpret_cast<long long*>(c.heap[r] + a.arena.topk_idx_off) + (size_t)slot * a.K + lane;
            *di = mine ? idx - (long long)r * E_local : -1;
            if (a.topk_weights) {
              float* dw = reinterpret_cast<float*>(c.heap[r] + a.arena.topk_w_off) + (size_t)slot * a.K + lane;
              *dw = mine ? w : 0.f;
            }
          }
          if (lane == 0) reinterpret_cast<int*>(c.heap[r] + a.arena.src_idx_off)[slot] = t;
        }
      }
    }
    // CUDA-graph friendly mode: pad the tail of recv_topk_idx with -1 (local writes)
    if (!a.cached && a.num_worst_tokens > 0 && a.topk_idx) {
      long long* ti = reinterpret_cast<long long*>(c.heap[me] + a.arena.topk_idx_off);
      const size_t lo = (size_t)s_recv_total * a.K, hi = (size_t)a.num_worst_tokens * a.K;
      for (size_t i = lo + (size_t)blockIdx.x * blockDim.x + tid; i < hi; i += (size_t)gridDim.x * blockDim.x) ti[i] = -1;
    }
  }
  sync_barrier(c, s);  // all my stores are visible at every destination; all inbound rows have landed
  sync_end(s);
}

// ---------------------------------------------------------------------------- combine
// NR = rank-count bucket (1, 2, 4, 8): source loops are unrolled to NR.  NR <= 2 takes a deeper
// chunk pipeline (few rows per token).  BIAS = false drops the bias code from the hot loop.
template <int NR, bool BIAS>
__global__ void __launch_bounds__(512, 1) ep_combine_kernel(const __grid_constant__ DevComm c,
                                                            const __grid_constant__ EpCombineArgs a) {
  const int R = c.nranks;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  BlockSync s = sync_begin(c, kDomEp, blockIdx.x);
  sync_barrier(c, s);  // every rank's expert outputs are in its combine arena
  const size_t row_bytes = (size_t)a.H * 2;
  const int chunks = (int)(row_bytes / 16);
  const int warps_total = gridDim.x * (blockDim.x >> 5);
  for (int t = blockIdx.x * (blockDim.x >> 5) + warp; t < a.T; t += warps_total) {
    const int my = lane < R ? a.send_slot[(size_t)t * R + lane] : -1;
    const unsigned mask = __ballot_sync(0xffffffffu, my >= 0);
    const char* src[NR];
    int slots[NR];
#pragma unroll
    for (int r = 0; r < NR; ++r) {
      slots[r] = __shfl_sync(0xffffffffu, my, r);
      src[r] = ((mask >> r) & 1u) ? c.heap[r] + a.x_off + (size_t)slots[r] * row_bytes : nullptr;
    }
    char* out = reinterpret_cast<char*>(a.out) + (size_t)t * row_bytes;
    const char* b0 = a.bias0 ? reinterpret_cast<const char*>(a.bias0) + (size_t)t * row_bytes : nullptr;
    const char* b1 = a.bias1 ? reinterpret_cast<const char*>(a.bias1) + (size_t)t * row_bytes : nullptr;
    auto add_bias = [&](float (&acc)[8], int i) {
      if constexpr (!BIAS) return;
      if (b0) {
        float f[8];
        bf16x8_to_float(ld_nc_v4(b0 + (size_t)i * 16), f);
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] += f[q];
      }
      if (b1) {
        float f[8];
        bf16x8_to_float(ld_nc_v4(b1 + (size_t)i * 16), f);
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] += f[q];
      }
    };
    auto store_acc = [&](const float (&acc)[8], int i) {
      uint4 o;
      __nv_bfloat162* oh = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
      for (int q = 0; q < 4; ++q) oh[q] = __floats2bfloat162_rn(acc[2 * q], acc[2 * q + 1]);
      st_v4(out + (size_t)i * 16, o);
    };
    if constexpr (NR <= 2) {
      // few sources (small EP degree / sparse routing): trade width for depth -- 8 chunks of up
      // to 2 rows in flight per lane instead of 2 chunks of up to 8 rows
      const int r0 = mask ? __ffs(mask) - 1 : -1;
      const unsigned m1 = mask & (mask - 1);
      const int r1 = m1 ? __ffs(m1) - 1 : -1;
      const int sl0 = __shfl_sync(0xffffffffu, my, r0 < 0 ? 0 : r0);
      const int sl1 = __shfl_sync(0xffffffffu, my, r1 < 0 ? 0 : r1);
      const char* p0 = r0 >= 0 ? c.heap[r0] + a.x_off + (size_t)sl0 * row_bytes : nullptr;
      const char* p1 = r1 >= 0 ? c.heap[r1] + a.x_off + (size_t)sl1 * row_bytes : nullptr;
      constexpr int D = 8;
      for (int i0 = 0; i0 < chunks; i0 += 32 * D) {
        uint4 v0[D], v1[D];
#pragma unroll
        for (int j = 0; j < D; ++j) {
          const int i = i0 + j * 32 + lane;
          if (i < chunks) {
            if (p0) v0[j] = ld_nc_v4(p0 + (size_t)i * 16);
            if constexpr (NR == 2) {
              if (p1) v1[j] = ld_nc_v4(p1 + (size_t)i * 16);
            }
          }
        }
#pragma unroll
        for (int j = 0; j < D; ++j) {
          const int i = i0 + j * 32 + lane;
          if (i < chunks) {
            float acc[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] = 0.f;
            add_bias(acc, i);
            if (p0) {
              float f[8];
              bf16x8_to_float(v0[j], f);
#pragma unroll
              for (int q = 0; q < 8; ++q) acc[q] += f[q];
            }
            if constexpr (NR == 2) {
              if (p1) {
                float f[8];
                bf16x8_to_float(v1[j], f);
#pragma unroll
                for (int q = 0; q < 8; ++q) acc[q] += f[q];
              }
            }
            store_acc(acc, i);
          }
        }
      }
    } else {
      for (int i0 = 0; i0 < chunks; i0 += 64) {
        uint4 v[2][NR];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int i = i0 + j * 32 + lane;
#pragma unroll
          for (int r = 0; r < NR; ++r)
            if (i < chunks && ((mask >> r) & 1u)) v[j][r] = ld_nc_v4(src[r] + (size_t)i * 16);
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int i = i0 + j * 32 + lane;
          if (i < chunks) {
            float acc[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] = 0.f;
            add_bias(acc, i);
#pragma unroll
            for (int r = 0; r < NR; ++r) {
              if ((mask >> r) & 1u) {
                float f[8];
                bf16x8_to_float(v[j][r], f);
#pragma unroll
                for (int q = 0; q < 8; ++q) acc[q] += f[q];
              }
            }
            store_acc(acc, i);
          }
        }
      }
    }
    if (a.out_topk_w && a.topk_w_off != kNoOff && lane < a.K) {
      float w = 0.f;
#pragma unroll
      for (int r = 0; r < NR; ++r)
        if ((mask >> r) & 1u)
          w += reinterpret_cast<const float*>(c.heap[r] + a.topk_w_off)[(size_t)slots[r] * a.K + lane];
      a.out_topk_w[(size_t)t * a.K + lane] = w;
    }
  }
  sync_barrier_relaxed(c, s);  // nobody still reads my arena when I return
  sync_end(s);
}

// --------------------------------------------------------------------------- launchers
cudaError_t launch_ep_layout(const EpLayoutArgs& a0, cudaStream_t st) {
  EpLayoutArgs a = a0;
  size_t smem = (size_t)a.E * sizeof(int);
  if (a.scratch) {
    // at most kEpLayoutMaxBlocks CTAs of >= kEpLayoutThreads consecutive tokens each
    int per = (a.T + kEpLayoutMaxBlocks - 1) / kEpLayoutMaxBlocks;
    per = (per + kEpLayoutThreads - 1) / kEpLayoutThreads * kEpLayoutThreads;
    if (per < kEpLayoutThreads) per = kEpLayoutThreads;
    const int grid = a.T > 0 ? (a.T + per - 1) / per : 1;
    smem += (size_t)(per + 3) / 4 * 4;
    if (smem <= (48u << 10)) {
      a.tokens_per_block = per;
      UB_LAUNCH((ep_layout_mc_kernel), grid, kEpLayoutThreads, smem, st, a);
      return cudaGetLastError();
    }
    smem = (size_t)a.E * sizeof(int);  // huge token counts: single-CTA scan below
  }
  UB_LAUNCH((ep_layout_kernel), 1, 1024, smem, st, a);
  return cudaGetLastError();
}

template <int NR>
static cudaError_t launch_ep_dispatch_nr(const DevComm& c, const EpDispatchArgs& a, int grid, cudaStream_t st) {
  switch (a.mode) {
    case EP_X_BF16: UB_LAUNCH((ep_dispatch_kernel<EP_X_BF16, NR>), grid, 512, 0, st, c, a); break;
    case EP_X_FP8_SCALED: UB_LAUNCH((ep_dispatch_kernel<EP_X_FP8_SCALED, NR>), grid, 512, 0, st, c, a); break;
    case EP_X_FUSED_FP8: UB_LAUNCH((ep_dispatch_kernel<EP_X_FUSED_FP8, NR>), grid, 512, 0, st, c, a); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

cudaError_t launch_ep_dispatch(const DevComm& c, const EpDispatchArgs& a, int grid, cudaStream_t st) {
  switch (c.nranks) {
    case 1: return launch_ep_dispatch_nr<1>(c, a, grid, st);
    case 2: return launch_ep_dispatch_nr<2>(c, a, grid, st);
    case 3: case 4: return launch_ep_dispatch_nr<4>(c, a, grid, st);
    default: return launch_ep_dispatch_nr<8>(c, a, grid, st);
  }
}

template <int NR>
static cudaError_t launch_ep_combine_nr(const DevComm& c, const EpCombineArgs& a, int grid, cudaStream_t st) {
  if (a.bias0 || a.bias1) UB_LAUNCH((ep_combine_kernel<NR, true>), grid, 512, 0, st, c, a);
  else UB_LAUNCH((ep_combine_kernel<NR, false>), grid, 512, 0, st, c, a);
  return cudaGetLastError();
}

cudaError_t launch_ep_combine(const DevComm& c, const EpCombineArgs& a, int grid, cudaStream_t st) {
  switch (c.nranks) {
    case 1: return launch_ep_combine_nr<1>(c, a, grid, st);
    case 2: return launch_ep_combine_nr<2>(c, a, grid, st);
    case 3: case 4: return launch_ep_combine_nr<4>(c, a, grid, st);
    default: return launch_ep_combine_nr<8>(c, a, grid, st);
  }
}

}  // namespace ub
