// TMA-pipelined expert-parallel dispatch / combine for one NVSwitch node (sm_90a).
//
// Why a second implementation next to ep_kernels.cu: the register-path kernels keep one row per
// warp in flight (LDG.128 -> registers -> STG.128), so the number of bytes in flight -- and with
// it the NVLink bandwidth -- scales with the number of CTAs (96 CTAs to saturate the links).
// The reference budgets 20-24 SMs for communication so that expert GEMMs can run beside it
// (ep/bench/buffer.py:56, ep/bench/test_intranode.py:571) and gets there with TMA staging through
// shared memory (ep/src/intranode.cu:460-575: receiver warps cp.async.bulk a ring slot into smem
// and bulk-store it to recv_x).  Here the same hardware path is used for the *direct placement*
// design of this library (no ring, no receiver CTAs, one pass):
//
//   dispatch   loader warp      cp.async.bulk  x[t] (HBM)            -> smem stage   (mbarrier tx)
//              14 cast warps    per-128-channel amax / scale / e4m3  -> smem out stage (fp8 fused mode)
//              storer warp      lane r: cp.async.bulk smem -> arena slot of rank r over NVLink
//              metadata warp    remapped top-k ids / weights / source index (register stores)
//   combine    loader warp      lane r: cp.async.bulk  peer r's expert-output row slice -> smem
//              14 reduce warps  fp32 sum of the <= R staged slices in rank order, bf16 store
//              weights warp     sums the routed top-k weights
//
// A CTA therefore keeps in_stages x row bytes of loads and several bulk stores in flight from
// three elected lanes; bytes in flight no longer depend on the number of resident warps, so
// 24 CTAs reach the bandwidth the register path needs 96 for.  Same results bit for bit (same
// quantiser, same summation order), same arenas, same cross-rank barriers.
#include "../kernels/launch.h"
#include "../kernels/prims.cuh"
#include "ep_common.cuh"
#include "ep_types.h"

namespace ub {

namespace {

constexpr int kTmaMaxStages = 12;
constexpr int kMetaRing = 32;    // > in_stages + out_stages + kStoreLag + 2
constexpr int kStoreLag = 2;     // bulk-store groups a storer lane leaves in flight before recycling a stage
constexpr int kWorkWarps = 14;   // cast warps (dispatch) / reduce warps (combine): 448 threads = 7168 B of 16-byte chunks
constexpr int kCastGroupWarps = kWorkWarps / 2;  // dispatch: two cast groups work on alternate tokens
constexpr int kDispThreads = (kWorkWarps + 3) * 32;  // loader | cast x14 | storer | metadata
constexpr int kCombThreads = (kWorkWarps + 2) * 32;  // loader | reduce x14 | weights
constexpr uint32_t kSliceBytes = kWorkWarps * 32 * 16;  // combine: bytes of one row slice handled per pipeline item
constexpr size_t kSmemLimit = 227u << 10;  // opt-in maximum of dynamic shared memory per CTA

struct alignas(16) EpItemMeta {
  int slot[kMaxRanks];  // dispatch: destination slot per rank (-1 = not routed there)
  int t;                // token index, -1 = end of stream
  int aux;              // combine: slice index
  unsigned mask;        // combine: ranks that hold a row of this token
  int pad;
};

struct alignas(128) EpPipeShared {
  uint64_t in_full[kTmaMaxStages];
  uint64_t in_empty[kTmaMaxStages];
  uint64_t out_full[kTmaMaxStages];
  uint64_t out_empty[kTmaMaxStages];
  EpItemMeta meta[kMetaRing];
  int M[kMaxRanks][kMaxRanks];
  int base[kMaxRanks];
  int abort_flag;
  int recv_total;
};

__host__ __device__ constexpr uint32_t align128(uint32_t x) { return (x + 127u) & ~127u; }

__device__ __forceinline__ uint4 lds128(const void* p) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(smem_u32(p)));
  return v;
}
__device__ __forceinline__ void sts128(void* p, const uint4& v) {
  asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(smem_u32(p)), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
// One lane polls the mbarrier, the warp then reconverges: 32x fewer try_wait operations on the shared-memory
// pipe that the TMA engine and the cast / reduce warps are using at the same time.
__device__ __forceinline__ void warp_mbar_wait(uint64_t* bar, uint32_t phase, int lane) {
  if (lane == 0) mbar_wait(bar, phase);
  __syncwarp();
}
// orders earlier generic-proxy accesses of this thread with later async-proxy (TMA) accesses
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

}  // namespace

// =========================================================================== dispatch
template <int MODE>
__global__ void __launch_bounds__(kDispThreads, 1) ep_dispatch_tma_kernel(const __grid_constant__ DevComm c,
                                                                         const __grid_constant__ EpDispatchArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  EpPipeShared& sh = *reinterpret_cast<EpPipeShared*>(smem);
  const int R = c.nranks;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int E_local = a.E / R;
  const int IN_ST = a.in_stages, OUT_ST = a.out_stages;
  const uint32_t n_scales = (uint32_t)a.H / 128;
  const uint32_t sc_bytes = (MODE == EP_X_BF16) ? 0u : n_scales * 4u;
  const uint32_t in_row = (MODE == EP_X_FP8_SCALED) ? (uint32_t)a.H : (uint32_t)a.H * 2u;
  const uint32_t out_row = (MODE == EP_X_BF16) ? (uint32_t)a.H * 2u : (uint32_t)a.H;
  const uint32_t in_stage_bytes = align128(in_row + ((MODE == EP_X_FP8_SCALED) ? sc_bytes : 0u));
  const uint32_t out_stage_bytes = align128(out_row + sc_bytes);
  unsigned char* in_base = smem + align128((uint32_t)sizeof(EpPipeShared));
  unsigned char* out_base = in_base + (size_t)IN_ST * in_stage_bytes;

  BlockSync s = sync_begin(c, kDomEp, blockIdx.x);
  if (tid == 0) {
    sh.abort_flag = 0;
    sh.recv_total = 0;
    for (int i = 0; i < IN_ST; ++i) {
      mbar_init(&sh.in_full[i], 1);
      mbar_init(&sh.in_empty[i], MODE == EP_X_FUSED_FP8 ? kCastGroupWarps : 1);
    }
    for (int i = 0; i < OUT_ST; ++i) {
      mbar_init(&sh.out_full[i], kCastGroupWarps);
      mbar_init(&sh.out_empty[i], 1);
    }
    mbar_fence_init();
  }
  ep_dispatch_prologue(c, a, s, sh.M, sh.base, &sh.abort_flag, &sh.recv_total);  // contains block-wide syncs

  if (!sh.abort_flag) {
    if (warp == 0) {
      // ------------------------------------------------------------------ loader
      // Slots are fetched for kGroup tokens at once (lane = token-in-group * kMaxRanks + rank) and one group
      // ahead, so the L2 latency of that lookup never sits between two bulk loads.
      uint32_t j = 0;
      constexpr int kGroup = 32 / kMaxRanks;
      const int gq = lane / kMaxRanks, gr = lane % kMaxRanks;
      auto fetch = [&](int t0) -> int {  // slot of token t0 + gq * grid at rank gr (-1: none / out of range)
        const long long t = (long long)t0 + (long long)gq * gridDim.x;
        if (t >= a.T || gr >= R) return -1;
        if (a.cached) return a.send_slot[(size_t)t * R + gr];
        const int p = a.token_pos[(size_t)t * R + gr];
        const int v = p >= 0 ? sh.base[gr] + p : -1;
        a.send_slot[(size_t)t * R + gr] = v;
        return v;
      };
      int nxt = fetch(blockIdx.x);
      for (int t0 = blockIdx.x; t0 < a.T; t0 += kGroup * gridDim.x) {
        const int cur = nxt;
        nxt = fetch(t0 + kGroup * (int)gridDim.x);
#pragma unroll
        for (int q = 0; q < kGroup; ++q) {
          const int t = t0 + q * (int)gridDim.x;
          if (t >= a.T) break;  // warp-uniform
          const int my = __shfl_sync(0xffffffffu, cur, q * kMaxRanks + (lane % kMaxRanks));
          if (__ballot_sync(0xffffffffu, my >= 0) == 0) continue;
          const int st = j % IN_ST;
          warp_mbar_wait(&sh.in_empty[st], ((j / IN_ST) & 1) ^ 1, lane);
          EpItemMeta& m = sh.meta[j % kMetaRing];
          if (lane < kMaxRanks) m.slot[lane] = my;
          if (lane == 0) m.t = t;
          __syncwarp();
          if (lane == 0) {
            unsigned char* dst = in_base + (size_t)st * in_stage_bytes;
            mbar_expect_tx(&sh.in_full[st], in_row + ((MODE == EP_X_FP8_SCALED) ? sc_bytes : 0u));
            tma_load_1d(dst, reinterpret_cast<const char*>(a.x) + (size_t)t * in_row, in_row, &sh.in_full[st]);
            if constexpr (MODE == EP_X_FP8_SCALED)
              tma_load_1d(dst + in_row, a.x_scales + (size_t)t * n_scales, sc_bytes, &sh.in_full[st]);
          }
          ++j;
        }
      }
      // end of stream: one sentinel per consumer chain (fused mode: one for each of the two cast groups; the
      // first one, aux = 0, is forwarded to the storer)
      for (int sidx = 0; sidx < (MODE == EP_X_FUSED_FP8 ? 2 : 1); ++sidx, ++j) {
        const int st = j % IN_ST;
        warp_mbar_wait(&sh.in_empty[st], ((j / IN_ST) & 1) ^ 1, lane);
        if (lane == 0) {
          sh.meta[j % kMetaRing].t = -1;
          sh.meta[j % kMetaRing].aux = sidx;
          mbar_arrive(&sh.in_full[st]);
        }
      }
    } else if (warp <= kWorkWarps) {
      // ------------------------------------------------------------- cast warps (fused fp8 only)
      if constexpr (MODE == EP_X_FUSED_FP8) {
        // two groups of 7 warps take alternate tokens: while one group waits for its row / its output stage
        // or runs the amax -> scale -> cast dependency chain, the other one is converting the next token
        const int grp = (warp - 1) / kCastGroupWarps;
        const int gtid = tid - 32 - grp * kCastGroupWarps * 32;
        const int units = a.H / 16;  // 16 channels (32 B in, 16 B out) per thread-iteration
        for (uint32_t j = grp;; j += 2) {
          const int st = j % IN_ST;
          warp_mbar_wait(&sh.in_full[st], (j / IN_ST) & 1, lane);
          const int t = sh.meta[j % kMetaRing].t;
          if (t < 0 && sh.meta[j % kMetaRing].aux != 0) break;  // the other group forwards the end of stream
          const int o = j % OUT_ST;
          warp_mbar_wait(&sh.out_empty[o], ((j / OUT_ST) & 1) ^ 1, lane);
          if (t >= 0) {
            const unsigned char* src = in_base + (size_t)st * in_stage_bytes;
            unsigned char* dst = out_base + (size_t)o * out_stage_bytes;
            float* dsc = reinterpret_cast<float*>(dst + out_row);
            for (int ub = 0; ub < units; ub += kCastGroupWarps * 32) {
              const int u = ub + gtid;
              const bool valid = u < units;
              uint4 v0 = make_uint4(0, 0, 0, 0), v1 = v0;
              if (valid) {
                v0 = lds128(src + (size_t)u * 32);
                v1 = lds128(src + (size_t)u * 32 + 16);
              }
              float f[16];
              bf16x8_to_float(v0, *reinterpret_cast<float(*)[8]>(&f[0]));
              bf16x8_to_float(v1, *reinterpret_cast<float(*)[8]>(&f[8]));
              float amax = 0.f;
#pragma unroll
              for (int i = 0; i < 16; ++i) amax = fmaxf(amax, fabsf(f[i]));
              // 128 channels = 8 consecutive lanes
              amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
              amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
              amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
              float scale, scale_inv;
              fp8_group_scale(amax, a.round_scale, scale, scale_inv);
              uint4 q;
              q.x = pack4_e4m3(f[0] * scale, f[1] * scale, f[2] * scale, f[3] * scale);
              q.y = pack4_e4m3(f[4] * scale, f[5] * scale, f[6] * scale, f[7] * scale);
              q.z = pack4_e4m3(f[8] * scale, f[9] * scale, f[10] * scale, f[11] * scale);
              q.w = pack4_e4m3(f[12] * scale, f[13] * scale, f[14] * scale, f[15] * scale);
              if (valid) {
                sts128(dst + (size_t)u * 16, q);
                if ((lane & 7) == 0) dsc[u >> 3] = scale_inv;
              }
            }
          }
          fence_proxy_async_smem();  // my smem writes -> visible to the bulk stores of the storer
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(&sh.in_empty[st]);
            mbar_arrive(&sh.out_full[o]);
          }
          if (t < 0) break;
        }
      }
    } else if (warp == kWorkWarps + 1) {
      // ------------------------------------------------------------------ storer
      constexpr bool kFused = MODE == EP_X_FUSED_FP8;
      unsigned char* ring = kFused ? out_base : in_base;
      const uint32_t stage_bytes = kFused ? out_stage_bytes : in_stage_bytes;
      const int NST = kFused ? OUT_ST : IN_ST;
      uint64_t* full = kFused ? sh.out_full : sh.in_full;
      uint64_t* empty = kFused ? sh.out_empty : sh.in_empty;
      char* my_heap = lane < R ? c.heap[lane] : nullptr;
      for (uint32_t j = 0;; ++j) {
        const int st = j % NST;
        warp_mbar_wait(&full[st], (j / NST) & 1, lane);
        const EpItemMeta& m = sh.meta[j % kMetaRing];
        if (m.t < 0) break;
        const int my = lane < kMaxRanks ? m.slot[lane] : -1;
        if (my >= 0) {
          const unsigned char* src = ring + (size_t)st * stage_bytes;
          tma_store_1d(my_heap + a.arena.x_off + (size_t)my * out_row, src, out_row);
          if (sc_bytes) tma_store_1d(my_heap + a.arena.scales_off + (size_t)my * sc_bytes, src + out_row, sc_bytes);
        }
        tma_store_commit();
        if (j >= (uint32_t)kStoreLag) {
          tma_store_wait_read<kStoreLag>();  // the stores of item j - kStoreLag have left shared memory
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[(j - kStoreLag) % NST]);
        }
      }
      tma_store_wait<0>();  // every row has been written at its destination before the exit barrier
    } else {
      // ---------------------------------------------------------------- metadata
      // remapped top-k ids / weights and the source token index of every routed copy; two tokens per
      // iteration so the (L2-latency-bound) loads of both are in flight together
      const bool has_topk = a.topk_idx != nullptr && a.K > 0;
      for (int t0 = blockIdx.x; t0 < a.T; t0 += 2 * gridDim.x) {
        int tt[2] = {t0, t0 + (int)gridDim.x};
        int my[2] = {-1, -1};
        long long idx[2] = {-1, -1};
        float w[2] = {0.f, 0.f};
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          if (tt[q] >= a.T) continue;
          if (lane < R) {
            if (a.cached) {
              my[q] = a.send_slot[(size_t)tt[q] * R + lane];
            } else {
              const int p = a.token_pos[(size_t)tt[q] * R + lane];
              my[q] = p >= 0 ? sh.base[lane] + p : -1;
            }
          }
          if (has_topk && lane < a.K) {
            idx[q] = a.topk_idx[(size_t)tt[q] * a.K + lane];
            if (a.topk_weights) w[q] = a.topk_weights[(size_t)tt[q] * a.K + lane];
          }
        }
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          if (tt[q] >= a.T) continue;  // warp-uniform
          const unsigned mask = __ballot_sync(0xffffffffu, my[q] >= 0);
          for (int r = 0; r < R; ++r) {
            const int slot = __shfl_sync(0xffffffffu, my[q], r);
            if (!((mask >> r) & 1u)) continue;
            if (has_topk && lane < a.K) {
              const bool mine = idx[q] >= (long long)r * E_local && idx[q] < (long long)(r + 1) * E_local;
              long long* di = reinterpret_cast<long long*>(c.heap[r] + a.arena.topk_idx_off) + (size_t)slot * a.K + lane;
              *di = mine ? idx[q] - (long long)r * E_local : -1;
              if (a.topk_weights) {
                float* dw = reinterpret_cast<float*>(c.heap[r] + a.arena.topk_w_off) + (size_t)slot * a.K + lane;
                *dw = mine ? w[q] : 0.f;
              }
            }
            if (lane == 0) reinterpret_cast<int*>(c.heap[r] + a.arena.src_idx_off)[slot] = tt[q];
          }
        }
      }
    }
    // CUDA-graph friendly mode: pad the tail of recv_topk_idx with -1 (local writes, rows nobody sends to)
    if (!a.cached && a.num_worst_tokens > 0 && a.topk_idx) {
      long long* ti = reinterpret_cast<long long*>(c.heap[c.rank] + a.arena.topk_idx_off);
      const size_t lo = (size_t)sh.recv_total * a.K, hi = (size_t)a.num_worst_tokens * a.K;
      for (size_t i = lo + (size_t)blockIdx.x * blockDim.x + tid; i < hi; i += (size_t)gridDim.x * blockDim.x) ti[i] = -1;
    }
  }
  sync_barrier(c, s);  // all my stores are visible at every destination; all inbound rows have landed
  sync_end(s);
}

// ============================================================================ combine
template <bool BIAS>
__global__ void __launch_bounds__(kCombThreads, 1) ep_combine_tma_kernel(const __grid_constant__ DevComm c,
                                                                        const __grid_constant__ EpCombineArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  EpPipeShared& sh = *reinterpret_cast<EpPipeShared*>(smem);
  const int R = c.nranks;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ST = a.stages;
  const uint32_t row_bytes = (uint32_t)a.H * 2u;
  const uint32_t SB = row_bytes < kSliceBytes ? row_bytes : kSliceBytes;  // bytes of one slice (multiple of 16)
  const int n_slices = (int)((row_bytes + SB - 1) / SB);
  const uint32_t src_stride = align128(SB);
  const uint32_t stage_bytes = (uint32_t)R * src_stride;
  unsigned char* stages = smem + align128((uint32_t)sizeof(EpPipeShared));
  uint64_t* full = sh.in_full;
  uint64_t* empty = sh.in_empty;

  BlockSync s = sync_begin(c, kDomEp, blockIdx.x);
  if (tid == 0) {
    for (int i = 0; i < ST; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], kWorkWarps);
    }
    mbar_fence_init();
  }
  sync_barrier(c, s);  // every rank's expert outputs are in its combine arena

  if (warp == 0) {
    // -------------------------------------------------------------------- loader
    fence_proxy_async_all();
    uint32_t j = 0;
    // slots of kGroup tokens per lookup, one group ahead (see the dispatch loader)
    constexpr int kGroup = 32 / kMaxRanks;
    const int gq = lane / kMaxRanks, gr = lane % kMaxRanks;
    auto fetch = [&](int t0) -> int {
      const long long t = (long long)t0 + (long long)gq * gridDim.x;
      return (t < a.T && gr < R) ? a.send_slot[(size_t)t * R + gr] : -1;
    };
    int nxt = fetch(blockIdx.x);
    for (int t0 = blockIdx.x; t0 < a.T; t0 += kGroup * gridDim.x) {
      const int cur = nxt;
      nxt = fetch(t0 + kGroup * (int)gridDim.x);
#pragma unroll
      for (int q = 0; q < kGroup; ++q) {
        const int t = t0 + q * (int)gridDim.x;
        if (t >= a.T) break;  // warp-uniform
        int my = __shfl_sync(0xffffffffu, cur, q * kMaxRanks + (lane % kMaxRanks));
        if (lane >= kMaxRanks) my = -1;
        const unsigned mask = __ballot_sync(0xffffffffu, my >= 0);
        const char* src = my >= 0 ? c.heap[lane] + a.x_off + (size_t)my * row_bytes : nullptr;
        for (int sl = 0; sl < n_slices; ++sl, ++j) {
          const int st = j % ST;
          warp_mbar_wait(&empty[st], ((j / ST) & 1) ^ 1, lane);
          const uint32_t bytes = min(SB, row_bytes - (uint32_t)sl * SB);
          if (lane == 0) {
            EpItemMeta& m = sh.meta[j % kMetaRing];
            m.t = t;
            m.aux = sl;
            m.mask = mask;
            mbar_expect_tx(&full[st], (uint32_t)__popc(mask) * bytes);
          }
          __syncwarp();
          if (my >= 0)
            tma_load_1d(stages + (size_t)st * stage_bytes + (size_t)lane * src_stride, src + (size_t)sl * SB, bytes, &full[st]);
        }
      }
    }
    const int st = j % ST;
    warp_mbar_wait(&empty[st], ((j / ST) & 1) ^ 1, lane);
    if (lane == 0) {
      sh.meta[j % kMetaRing].t = -1;
      mbar_arrive(&full[st]);
    }
  } else if (warp <= kWorkWarps) {
    // ------------------------------------------------------------------- reduce warps
    const uint32_t off = (uint32_t)(tid - 32) * 16u;
    for (uint32_t j = 0;; ++j) {
      const int st = j % ST;
      warp_mbar_wait(&full[st], (j / ST) & 1, lane);
      const EpItemMeta& m = sh.meta[j % kMetaRing];
      const int t = m.t;
      if (t < 0) break;
      const int sl = m.aux;
      const unsigned mask = m.mask;
      const uint32_t bytes = min(SB, row_bytes - (uint32_t)sl * SB);
      if (off < bytes) {
        const size_t goff = (size_t)t * row_bytes + (size_t)sl * SB + off;
        float acc[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = 0.f;
        if constexpr (BIAS) {
          if (a.bias0) {
            float f[8];
            bf16x8_to_float(ld_nc_v4(reinterpret_cast<const char*>(a.bias0) + goff), f);
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] += f[q];
          }
          if (a.bias1) {
            float f[8];
            bf16x8_to_float(ld_nc_v4(reinterpret_cast<const char*>(a.bias1) + goff), f);
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] += f[q];
          }
        }
        const unsigned char* sp = stages + (size_t)st * stage_bytes + off;
#pragma unroll
        for (int r = 0; r < kMaxRanks; ++r) {
          if ((mask >> r) & 1u) {
            float f[8];
            bf16x8_to_float(lds128(sp + (size_t)r * src_stride), f);
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] += f[q];
          }
        }
        uint4 o;
        __nv_bfloat162* oh = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
        for (int q = 0; q < 4; ++q) oh[q] = __floats2bfloat162_rn(acc[2 * q], acc[2 * q + 1]);
        st_v4(reinterpret_cast<char*>(a.out) + goff, o);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[st]);
    }
  } else {
    // ------------------------------------------------------------------ weights warp
    if (a.out_topk_w && a.topk_w_off != kNoOff && a.K > 0) {
      int Kp = 1;
      while (Kp < a.K) Kp <<= 1;   // a.K <= 32
      const int G = 32 / Kp;        // tokens per pass
      const int g = lane / Kp, k = lane % Kp;
      for (int i0 = 0;; i0 += G) {
        const long long t0 = (long long)blockIdx.x + (long long)i0 * gridDim.x;
        if (t0 >= a.T) break;  // warp-uniform
        const long long t = t0 + (long long)g * gridDim.x;
        if (t < a.T && k < a.K) {
          float vals[kMaxRanks];
#pragma unroll
          for (int r = 0; r < kMaxRanks; ++r) {
            vals[r] = 0.f;
            if (r < R) {
              const int slot = a.send_slot[(size_t)t * R + r];
              if (slot >= 0) vals[r] = reinterpret_cast<const float*>(c.heap[r] + a.topk_w_off)[(size_t)slot * a.K + k];
            }
          }
          float wsum = 0.f;
#pragma unroll
          for (int r = 0; r < kMaxRanks; ++r) wsum += vals[r];
          a.out_topk_w[(size_t)t * a.K + k] = wsum;
        }
      }
    }
  }
  sync_barrier_relaxed(c, s);  // nobody still reads my arena when I return
  sync_end(s);
}

// =========================================================================== launchers
namespace {
template <typename K>
cudaError_t set_smem(K kern, size_t bytes) {
  return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}
}  // namespace

bool ep_dispatch_tma_supported(const EpDispatchArgs& a) {
  if (a.H <= 0 || a.H % 8 != 0) return false;
  if (a.mode != EP_X_BF16 && (a.H % 512 != 0 || a.H > 8192)) return false;  // scale rows must be 16-byte multiples
  if (((uintptr_t)a.x & 15) != 0) return false;
  if (a.mode == EP_X_FP8_SCALED && ((uintptr_t)a.x_scales & 15) != 0) return false;
  return (size_t)a.H * 2 <= 32768;
}

bool ep_combine_tma_supported(const EpCombineArgs& a) {
  return a.H > 0 && a.H % 8 == 0 && ((uintptr_t)a.out & 15) == 0 && ((uintptr_t)a.bias0 & 15) == 0 &&
         ((uintptr_t)a.bias1 & 15) == 0;
}

template <int MODE>
static cudaError_t launch_dispatch_mode(const DevComm& c, EpDispatchArgs a, int grid, cudaStream_t st) {
  const uint32_t n_scales = (uint32_t)a.H / 128;
  const uint32_t sc = (MODE == EP_X_BF16) ? 0u : n_scales * 4u;
  const uint32_t in_row = (MODE == EP_X_FP8_SCALED) ? (uint32_t)a.H : (uint32_t)a.H * 2u;
  const uint32_t out_row = (MODE == EP_X_BF16) ? (uint32_t)a.H * 2u : (uint32_t)a.H;
  const size_t in_stage = align128(in_row + ((MODE == EP_X_FP8_SCALED) ? sc : 0u));
  const size_t out_stage = (MODE == EP_X_FUSED_FP8) ? align128(out_row + sc) : 0;
  const size_t ctrl = align128((uint32_t)sizeof(EpPipeShared));
  const size_t avail = kSmemLimit - ctrl;
  int in_st = a.in_stages, out_st = a.out_stages;
  if (MODE == EP_X_FUSED_FP8) {
    if (in_st <= 0 || out_st <= 0) in_st = out_st = (int)(avail / (in_stage + out_stage));
    in_st = in_st < 2 ? 2 : (in_st > kTmaMaxStages ? kTmaMaxStages : in_st);
    out_st = out_st < kStoreLag + 2 ? kStoreLag + 2 : (out_st > kTmaMaxStages ? kTmaMaxStages : out_st);
  } else {
    if (in_st <= 0) in_st = (int)(avail / in_stage);
    in_st = in_st < kStoreLag + 2 ? kStoreLag + 2 : (in_st > kTmaMaxStages ? kTmaMaxStages : in_st);
    out_st = 0;
  }
  const size_t smem = ctrl + (size_t)in_st * in_stage + (size_t)out_st * out_stage;
  if (smem > (227u << 10)) return cudaErrorInvalidConfiguration;
  a.in_stages = in_st;
  a.out_stages = out_st;
  if (!g_preload) {
    cudaError_t e = set_smem(ep_dispatch_tma_kernel<MODE>, smem);
    if (e != cudaSuccess) return e;
  }
  UB_LAUNCH((ep_dispatch_tma_kernel<MODE>), grid, kDispThreads, smem, st, c, a);
  return cudaGetLastError();
}

cudaError_t launch_ep_dispatch_tma(const DevComm& c, const EpDispatchArgs& a, int grid, cudaStream_t st) {
  switch (a.mode) {
    case EP_X_BF16: return launch_dispatch_mode<EP_X_BF16>(c, a, grid, st);
    case EP_X_FP8_SCALED: return launch_dispatch_mode<EP_X_FP8_SCALED>(c, a, grid, st);
    case EP_X_FUSED_FP8: return launch_dispatch_mode<EP_X_FUSED_FP8>(c, a, grid, st);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_ep_combine_tma(const DevComm& c, const EpCombineArgs& a0, int grid, cudaStream_t st) {
  EpCombineArgs a = a0;
  const uint32_t row_bytes = (uint32_t)a.H * 2u;
  const uint32_t SB = row_bytes < kSliceBytes ? row_bytes : kSliceBytes;
  const size_t stage = (size_t)c.nranks * align128(SB);
  const size_t ctrl = align128((uint32_t)sizeof(EpPipeShared));
  int stg = a.stages;
  if (stg <= 0) stg = (int)((kSmemLimit - ctrl) / stage);
  stg = stg < 2 ? 2 : (stg > kTmaMaxStages ? kTmaMaxStages : stg);
  const size_t smem = ctrl + (size_t)stg * stage;
  if (smem > (227u << 10)) return cudaErrorInvalidConfiguration;
  a.stages = stg;
  if (a.bias0 || a.bias1) {
    if (!g_preload) {
      cudaError_t e = set_smem(ep_combine_tma_kernel<true>, smem);
      if (e != cudaSuccess) return e;
    }
    UB_LAUNCH((ep_combine_tma_kernel<true>), grid, kCombThreads, smem, st, c, a);
  } else {
    if (!g_preload) {
      cudaError_t e = set_smem(ep_combine_tma_kernel<false>, smem);
      if (e != cudaSuccess) return e;
    }
    UB_LAUNCH((ep_combine_tma_kernel<false>), grid, kCombThreads, smem, st, c, a);
  }
  return cudaGetLastError();
}

}  // namespace ub
