// Low-latency (decode) expert-parallel kernels, sm_90a.
//
// Reference behaviour (ep/src/internode_ll.cu:50-731, 735-1304): dispatch casts each token to
// fp8, atomically claims a slot per (expert, source-rank) region at the destination, stores the
// message there, then a RECV phase waits for per-(expert, rank) count flags and *re-packs* the
// regions into the contiguous per-expert layout; combine pushes expert outputs back into a
// [token][topk] staging area at the source and a RECV phase does the weighted reduction.
//
// Hopper-native design: ONE pass each way.
//   dispatch: every rank all-gathers its per-expert histogram first (E ints to each peer + one
//     block barrier), so each sender knows the exact packed offset of its tokens inside every
//     remote expert's contiguous block.  A warp stages the (fp8-cast) token + scales in shared
//     memory once and one elected lane issues cp.async.bulk (TMA) stores straight into the final
//     packed position on each destination GPU -- no staging regions, no re-pack kernel phase.
//   combine: the token's home rank pulls its K expert-output rows from the peers' symmetric
//     buffers and does the top-k weighted sum in fp32 -- no [token][topk] staging, no recv phase.
#include "../kernels/launch.h"
#include "../kernels/prims.cuh"
#include "ep_common.cuh"
#include "ep_logfmt.h"
#include "ep_types.h"

namespace ub {

constexpr int kLLWarps = 8;  // 256 threads cooperate on one token (one staged row per CTA)

__global__ void __launch_bounds__(kLLWarps * 32, 1) ep_ll_dispatch_kernel(const __grid_constant__ DevComm c,
                                                                          const __grid_constant__ EpLLDispatchArgs a) {
  extern __shared__ __align__(128) unsigned char ll_smem[];
  const int R = c.nranks, me = c.rank;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int E = a.E, E_local = E / R;
  const int n_scales = a.H / 128;
  const size_t row_bytes = a.use_fp8 ? (size_t)a.H : (size_t)a.H * 2;
  const size_t scale_bytes = a.use_fp8 ? (size_t)n_scales * 4 : 0;
  const size_t stage_stride = (row_bytes + scale_bytes + 127) / 128 * 128;
  int* s_cnt = reinterpret_cast<int*>(ll_smem);         // [E] my histogram, then reused
  int* s_begin = s_cnt + E;                             // [E] packed offset of my tokens at each expert
  (void)stage_stride;

  BlockSync s = sync_begin(c, kDomEpLL, blockIdx.x);
  if (a.phase == EP_LL_RECV) {
    // receive half of a hook-split dispatch: the send half has published its epoch; wait until every
    // peer's rows (and counts) have landed here
    sync_wait(c, s, blockIdx.x == 0 ? a.wait_stats : nullptr);
    sync_end(s);
    return;
  }
  // ---- phase A: histogram + all-gather of the [R][E] count matrix
  for (int e = tid; e < E; e += blockDim.x) s_cnt[e] = 0;
  if (blockIdx.x == 0)
    for (int e = tid; e < E; e += blockDim.x) a.send_cnt[(1 - a.parity) * E + e] = 0;  // for the next call
  __syncthreads();
  for (int i = tid; i < a.T * a.K; i += blockDim.x) {
    const long long e = a.topk_idx[i];
    if (e >= 0 && e < E) atomicAdd(&s_cnt[(int)e], 1);
  }
  __syncthreads();
  if ((E & 3) == 0) {  // 16-byte stores: E / 4 per peer
    const int E4 = E >> 2;
    for (int i = tid; i < R * E4; i += blockDim.x) {
      const int dst = i / E4, q = i % E4;
      int* p = reinterpret_cast<int*>(c.heap[dst] + a.cnt_tab_off) + ((size_t)blockIdx.x * kMaxRanks + me) * E + q * 4;
      st_v4(p, *reinterpret_cast<const uint4*>(s_cnt + q * 4));
    }
  } else {
    for (int i = tid; i < R * E; i += blockDim.x) {
      const int dst = i / E, e = i % E;
      int* p = reinterpret_cast<int*>(c.heap[dst] + a.cnt_tab_off) + ((size_t)blockIdx.x * kMaxRanks + me) * E + e;
      *p = s_cnt[e];
    }
  }
  sync_signal(c, s);
  sync_wait(c, s, blockIdx.x == 0 ? a.wait_stats : nullptr);
  const int* tab = reinterpret_cast<const int*>(c.heap[me] + a.cnt_tab_off) + (size_t)blockIdx.x * kMaxRanks * E;
  for (int e = tid; e < E; e += blockDim.x) {
    int b = 0;
    for (int q = 0; q < me; ++q) b += tab[(size_t)q * E + e];
    s_begin[e] = b;
  }
  if (blockIdx.x == 0) {
    for (int el = tid; el < E_local; el += blockDim.x) {
      int run = 0;
      for (int q = 0; q < R; ++q) {
        const int cnt = tab[(size_t)q * E + me * E_local + el];
        a.layout_range[(size_t)el * R + q] = ((int64_t)run << 32) | (int64_t)cnt;
        run += cnt;
      }
      a.recv_count[el] = run;
    }
  }
  __syncthreads();

  // ---- phase B: one CTA per token.  A decode batch has about as many tokens as the GPU has SMs, so the
  // latency of ONE token is what matters: all 256 threads load the row at once (every 16-byte load of the
  // row is in flight together), the slot claims (global atomics) overlap those loads, and the K copies are
  // issued by K different warps.
  int* s_slot = s_begin + E;             // [kEpMaxTopk] claimed slot per top-k entry
  int* s_exp = s_slot + kEpMaxTopk;      // [kEpMaxTopk] expert id per top-k entry (-1: none)
  unsigned char* stage = ll_smem + ((((size_t)2 * E + 2 * kEpMaxTopk) * 4 + 127) / 128 * 128);
  const bool bulk_ok = (row_bytes % 16 == 0) && (scale_bytes % 16 == 0);
  const size_t rows_per_expert = (size_t)R * a.M;
  const float* sc_stage = reinterpret_cast<const float*>(stage + row_bytes);
  bool pending = false;  // this lane has bulk stores in flight that still read the stage
  for (int t = blockIdx.x; t < a.T; t += gridDim.x) {
    const char* src = reinterpret_cast<const char*>(a.x) + (size_t)t * a.H * 2;
    // slot claim first: its latency hides behind the row loads
    if (tid < a.K) {
      const long long e = a.topk_idx[(size_t)t * a.K + tid];
      int slot = -1;
      if (e >= 0 && e < E) slot = s_begin[(int)e] + atomicAdd(&a.send_cnt[a.parity * E + (int)e], 1);
      s_exp[tid] = (e >= 0 && e < E) ? (int)e : -1;
      s_slot[tid] = slot;
      int64_t pos = -1;
      if (slot >= 0) pos = ((int64_t)((int)e / E_local) << 32) | (int64_t)((size_t)((int)e % E_local) * R * a.M + slot);
      a.send_pos[(size_t)t * a.K + tid] = pos;
    }
    if (a.use_fp8) {
      const int units = a.H / 16;  // 16 channels per unit; 8 consecutive lanes share a 128-channel scale
      float* sc = reinterpret_cast<float*>(stage + row_bytes);
      constexpr int U = 2;  // units per thread per pass: 512 units (H = 8192) in one pass
      for (int ub = 0; ub < units; ub += U * kLLWarps * 32) {
        uint4 v0[U], v1[U];
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const int u = ub + j * kLLWarps * 32 + tid;
          v0[j] = make_uint4(0, 0, 0, 0);
          v1[j] = v0[j];
          if (u < units) {
            v0[j] = ld_nc_v4(src + (size_t)u * 32);
            v1[j] = ld_nc_v4(src + (size_t)u * 32 + 16);
          }
        }
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const int u = ub + j * kLLWarps * 32 + tid;
          if (ub + j * kLLWarps * 32 + (tid & ~31) >= units) break;  // warp-uniform
          const bool valid = u < units;
          float f[16];
          bf16x8_to_float(v0[j], *reinterpret_cast<float(*)[8]>(&f[0]));
          bf16x8_to_float(v1[j], *reinterpret_cast<float(*)[8]>(&f[8]));
          float amax = 0.f;
#pragma unroll
          for (int i = 0; i < 16; ++i) amax = fmaxf(amax, fabsf(f[i]));
          amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
          amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
          amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
          float scale, scale_inv;
          fp8_group_scale(amax, a.round_scale, scale, scale_inv);
          if (valid) {
            uint4 o;
            o.x = pack4_e4m3(f[0] * scale, f[1] * scale, f[2] * scale, f[3] * scale);
            o.y = pack4_e4m3(f[4] * scale, f[5] * scale, f[6] * scale, f[7] * scale);
            o.z = pack4_e4m3(f[8] * scale, f[9] * scale, f[10] * scale, f[11] * scale);
            o.w = pack4_e4m3(f[12] * scale, f[13] * scale, f[14] * scale, f[15] * scale);
            *reinterpret_cast<uint4*>(stage + (size_t)u * 16) = o;
            if ((lane & 7) == 0) sc[u >> 3] = scale_inv;
          }
        }
      }
    } else {
      const int chunks = (int)(row_bytes / 16);
      constexpr int U = 4;
      for (int cb = 0; cb < chunks; cb += U * kLLWarps * 32) {
        uint4 v[U];
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const int i = cb + j * kLLWarps * 32 + tid;
          if (i < chunks) v[j] = ld_nc_v4(src + (size_t)i * 16);
        }
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const int i = cb + j * kLLWarps * 32 + tid;
          if (i < chunks) *reinterpret_cast<uint4*>(stage + (size_t)i * 16) = v[j];
        }
      }
    }
    fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the bulk-copy (async) proxy
    __syncthreads();
    // one top-k entry per warp (round robin): bulk-store the staged row (+ scales) to its packed position
    for (int k = warp; k < a.K; k += kLLWarps) {
      const int ek = s_exp[k], sk = s_slot[k];
      if (ek < 0 || sk < 0) continue;
      const int r = ek / E_local, el = ek % E_local;
      const size_t row = (size_t)el * R * a.M + sk;
      char* dx = c.heap[r] + a.recv_x_off + row * row_bytes;
      char* ds = c.heap[r] + a.recv_scales_off + row * scale_bytes;
      if (scale_bytes && a.scale_layout != EP_LL_SCALES_ROW_MAJOR) {
        // column-major forms: element (row, j) of expert el lives at [el][j][row] -- strided 4-byte stores
        if (a.scale_layout == EP_LL_SCALES_COL_MAJOR) {
          float* base = reinterpret_cast<float*>(c.heap[r] + a.recv_scales_off) + (size_t)el * n_scales * rows_per_expert + sk;
          for (int jx = lane; jx < n_scales; jx += 32) base[(size_t)jx * rows_per_expert] = sc_stage[jx];
        } else {
          const int n_words = n_scales / 4;  // H % 512 == 0 (checked on the host)
          uint32_t* base = reinterpret_cast<uint32_t*>(c.heap[r] + a.recv_scales_off) + (size_t)el * n_words * rows_per_expert + sk;
          for (int jx = lane; jx < n_words; jx += 32) {
            uint32_t wv = 0;
#pragma unroll
            for (int b = 0; b < 4; ++b) wv |= ((__float_as_uint(sc_stage[jx * 4 + b]) >> 23) & 0xffu) << (8 * b);
            base[(size_t)jx * rows_per_expert] = wv;
          }
        }
        if (bulk_ok && lane == 0) tma_store_1d(dx, stage, (uint32_t)row_bytes);
        if (!bulk_ok)
          for (size_t i = lane * 4; i < row_bytes; i += 128) *reinterpret_cast<uint32_t*>(dx + i) = *reinterpret_cast<const uint32_t*>(stage + i);
      } else if (bulk_ok) {
        if (lane == 0) {
          tma_store_1d(dx, stage, (uint32_t)row_bytes);
          if (scale_bytes) tma_store_1d(ds, stage + row_bytes, (uint32_t)scale_bytes);
        }
      } else {
        for (size_t i = lane * 4; i < row_bytes + scale_bytes; i += 128) {
          const uint32_t w = *reinterpret_cast<const uint32_t*>(stage + i);
          if (i < row_bytes) *reinterpret_cast<uint32_t*>(dx + i) = w;
          else *reinterpret_cast<uint32_t*>(ds + (i - row_bytes)) = w;
        }
      }
      if (lane == 0) {
        reinterpret_cast<int*>(c.heap[r] + a.recv_src_off)[row] = t;
        pending = true;
      }
    }
    if (lane == 0 && pending) {
      tma_store_commit();
      if (t + (int)gridDim.x < a.T) tma_store_wait_read<0>();  // the stage is overwritten by the next token
    }
    __syncthreads();
  }
  if (lane == 0) tma_store_wait<0>();  // all bulk stores of this thread are globally visible before the barrier
  sync_signal(c, s);  // "everything I send has been written"
  if (a.phase == EP_LL_FULL) sync_wait(c, s, blockIdx.x == 0 ? a.wait_stats : nullptr);  // else: the hook's kernel waits
  sync_end(s);
}

__global__ void __launch_bounds__(512, 1) ep_ll_combine_kernel(const __grid_constant__ DevComm c,
                                                               const __grid_constant__ EpLLCombineArgs a) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  BlockSync s = sync_begin(c, kDomEpLL, blockIdx.x);
  // pull design: the "send" of a combine is just announcing that my expert outputs are in place; the
  // receive half waits for every peer's announcement, pulls the rows and reduces
  if (a.phase != EP_LL_RECV) sync_signal(c, s);
  if (a.phase == EP_LL_SEND) {
    sync_end(s);
    return;
  }
  sync_wait(c, s, blockIdx.x == 0 ? a.wait_stats : nullptr);
  const size_t row_bytes = (size_t)a.H * 2;
  const int chunks = (int)(row_bytes / 16);
  // One CTA per token, its warps split the row: the K source rows of a token live in K different
  // expert blocks (different 2 MiB pages, possibly on K different GPUs); keeping a CTA on ONE
  // token keeps the SM's TLB working set at K pages and gives 16 warps x K loads in flight per token.
  const int nwarps = blockDim.x >> 5;
  for (int t = blockIdx.x; t < a.T; t += gridDim.x) {
    long long pos = -1;
    float w = 0.f;
    if (lane < a.K) {
      pos = a.send_pos[(size_t)t * a.K + lane];
      w = a.topk_weights[(size_t)t * a.K + lane];
    }
    // per-top-k row pointers / weights in registers (K <= 9 fast path, generic tail below)
    const char* rowp[9];
    float wk[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const long long pk = __shfl_sync(0xffffffffu, pos, k);
      wk[k] = __shfl_sync(0xffffffffu, w, k);
      rowp[k] = nullptr;
      if (k < a.K && pk >= 0)
        rowp[k] = c.heap[(int)(pk >> 32)] + a.x_off + (size_t)(pk & 0xffffffffll) * row_bytes;
    }
    char* out = reinterpret_cast<char*>(a.out) + (size_t)t * row_bytes;
    // two 16-byte chunks per thread per pass: with 512 threads a 14 KB row is covered by ONE pass, so all
    // K x 2 loads of a thread are in flight together (one NVLink round trip per token instead of two)
    constexpr int PF = 2;
    for (int i0 = warp * 32; i0 < chunks; i0 += PF * nwarps * 32) {  // warp-uniform trip count
      uint4 v[PF][9];
      bool valid[PF];
#pragma unroll
      for (int j = 0; j < PF; ++j) {
        const int i = i0 + j * nwarps * 32 + lane;
        valid[j] = i < chunks;
#pragma unroll
        for (int k = 0; k < 9; ++k)
          if (rowp[k] && valid[j]) v[j][k] = ld_nc_v4(rowp[k] + (size_t)i * 16);
      }
#pragma unroll
      for (int j = 0; j < PF; ++j) {
        const int i = i0 + j * nwarps * 32 + lane;
        float acc[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = 0.f;
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          if (rowp[k] && valid[j]) {
            float f[8];
            bf16x8_to_float(v[j][k], f);
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] += wk[k] * f[q];
          }
        }
        for (int k = 9; k < a.K; ++k) {  // DeepEP's LL limit is 9; keep larger top-k correct
          const long long pk = __shfl_sync(0xffffffffu, pos, k);
          const float wkk = __shfl_sync(0xffffffffu, w, k);
          if (pk >= 0 && valid[j]) {
            float f[8];
            bf16x8_to_float(ld_nc_v4(c.heap[(int)(pk >> 32)] + a.x_off + (size_t)(pk & 0xffffffffll) * row_bytes + (size_t)i * 16), f);
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] += wkk * f[q];
          }
        }
        uint4 o;
        __nv_bfloat162* oh = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
        for (int q = 0; q < 4; ++q) oh[q] = __floats2bfloat162_rn(acc[2 * q], acc[2 * q + 1]);
        if (valid[j]) st_v4(out + (size_t)i * 16, o);
      }
    }
  }
  sync_barrier_relaxed(c, s);
  sync_end(s);
}

// Copies only the occupied rows of every local expert (contiguous: rows [0, recv_count[e]) of expert e).
__global__ void __launch_bounds__(256) ep_ll_pack_kernel(const EpLLPackArgs a) {
  const size_t row16 = (size_t)a.H * 2 / 16;
  for (int e = blockIdx.y; e < a.E_local; e += gridDim.y) {
    int rows = 0;
    for (int q = 0; q < a.R; ++q) rows += (int)(a.layout_range[(size_t)e * a.R + q] & 0xffffffffll);
    const size_t n16 = (size_t)rows * row16;
    const uint4* src = reinterpret_cast<const uint4*>(a.src) + (size_t)e * a.R * a.M * row16;
    uint4* dst = reinterpret_cast<uint4*>(a.dst) + (size_t)e * a.R * a.M * row16;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x)
      dst[i] = ld_nc_v4(src + i);
  }
}

// LogFMT-10 "simulated cast" of the reference's low-latency combine (ep/src/internode_ll.cu:934-995): every group of
// 128 channels whose |max| <= 1 is snapped to a 9-bit logarithmic grid between its smallest and largest magnitude
// (range clipped to 2^-32 of the maximum) and stays bf16 on the wire -- use_logfmt only changes the numerics, which
// is what a consumer that was tuned with it expects.  Sixteen consecutive lanes hold one group (8 channels each):
// all 32 lanes of the warp must call this.
__device__ __forceinline__ void logfmt10_simulate(uint4& v) {
  uint32_t* w = reinterpret_cast<uint32_t*>(&v);
  float la[8];
  float amax = 0.f, lmax = -INFINITY, lmin = INFINITY;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float av = fabsf(bf16_bits_to_f32((uint16_t)(w[q >> 1] >> ((q & 1) * 16))));
    la[q] = log2f(av);  // -inf for 0
    amax = fmaxf(amax, av);
    lmax = fmaxf(lmax, la[q]);
    if (av != 0.f) lmin = fminf(lmin, la[q]);
  }
#pragma unroll
  for (int o = 1; o < 16; o <<= 1) {
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
    lmin = fminf(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
  }
  const LogFmtParams p = logfmt10_params(amax, lmax, lmin);  // identical on the 16 lanes of the group
  if (!p.use) return;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const int sh = (q & 1) * 16;
    const uint32_t nb = logfmt10_quantize_bits((uint16_t)(w[q >> 1] >> sh), la[q], p);
    w[q >> 1] = (w[q >> 1] & ~(0xffffu << sh)) | (nb << sh);
  }
}

// pack + simulated LogFMT cast of the occupied rows (src may equal dst: every thread rewrites only what it read)
__global__ void __launch_bounds__(256) ep_ll_pack_logfmt_kernel(const EpLLPackArgs a) {
  const size_t row16 = (size_t)a.H * 2 / 16;  // H % 128 == 0 (host check): 16-lane groups never straddle rows
  const int lane = threadIdx.x & 31;
  for (int e = blockIdx.y; e < a.E_local; e += gridDim.y) {
    int rows = 0;
    for (int q = 0; q < a.R; ++q) rows += (int)(a.layout_range[(size_t)e * a.R + q] & 0xffffffffll);
    const size_t n16 = (size_t)rows * row16;
    const uint4* src = reinterpret_cast<const uint4*>(a.src) + (size_t)e * a.R * a.M * row16;
    uint4* dst = reinterpret_cast<uint4*>(a.dst) + (size_t)e * a.R * a.M * row16;
    // warp-uniform trip count: the shuffles inside need all 32 lanes
    for (size_t i0 = (size_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); i0 < n16; i0 += (size_t)gridDim.x * blockDim.x) {
      const size_t i = i0 + lane;
      const bool valid = i < n16;
      uint4 v = make_uint4(0, 0, 0, 0);
      if (valid) v = ld_v4(reinterpret_cast<const char*>(src + i));
      logfmt10_simulate(v);
      if (valid) st_v4(reinterpret_cast<char*>(dst + i), v);
    }
  }
}

cudaError_t launch_ep_ll_pack(const EpLLPackArgs& a, cudaStream_t st) {
  dim3 grid(16, (unsigned)(a.E_local < 1 ? 1 : (a.E_local > 64 ? 64 : a.E_local)));
  if (a.logfmt) {
    if (a.H % 128 != 0) return cudaErrorInvalidValue;
    UB_LAUNCH((ep_ll_pack_logfmt_kernel), grid, 256, 0, st, a);
  } else {
    UB_LAUNCH((ep_ll_pack_kernel), grid, 256, 0, st, a);
  }
  return cudaGetLastError();
}

// ------------------------------------------------------------------ launchers
cudaError_t launch_ep_ll_dispatch(const DevComm& c, const EpLLDispatchArgs& a, int grid, cudaStream_t st) {
  const size_t row_bytes = a.use_fp8 ? (size_t)a.H : (size_t)a.H * 2;
  const size_t scale_bytes = a.use_fp8 ? (size_t)(a.H / 128) * 4 : 0;
  const size_t stage_stride = (row_bytes + scale_bytes + 127) / 128 * 128;
  const size_t smem = ((((size_t)2 * a.E + 2 * kEpMaxTopk) * 4 + 127) / 128 * 128) + stage_stride;  // one staged row per CTA
  static bool attr_done[64] = {false};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr_done[dev & 63]) {
    cudaError_t e = cudaFuncSetAttribute(ep_ll_dispatch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return e;
    attr_done[dev & 63] = true;
  }
  if (smem > 200 * 1024) return cudaErrorInvalidValue;
  UB_LAUNCH((ep_ll_dispatch_kernel), grid, kLLWarps * 32, smem, st, c, a);
  return cudaGetLastError();
}

cudaError_t launch_ep_ll_combine(const DevComm& c, const EpLLCombineArgs& a, int grid, cudaStream_t st) {
  UB_LAUNCH((ep_ll_combine_kernel), grid, 512, 0, st, c, a);
  return cudaGetLastError();
}

}  // namespace ub
