// AllReduce kernels for one NVSwitch node (2/4/8 ranks), all sm_90a, all operating
// directly on NVLink-mapped peer memory from the symmetric heap.
//
//   ar_oneshot<MC>     small messages: every rank pushes LL16 packets {data,flag,data,flag}
//                      into every peer's scratch (P2P stores, or ONE multimem.st through the
//                      switch), then reduces the N slots locally.  No barrier at all.
//                      (reference counterparts: allreducePacket / allreduceNvlsPacket,
//                       experimental/lite/collective/allreduce_packet.cu:14-168,
//                       allreduce_nvls_packet.cu:13-61)
//   ar_twoshot<NVLS>   zero-copy on symmetric buffers: reduce my 1/N shard straight from the
//                      peers' inputs (8 P2P loads, or one multimem.ld_reduce) and broadcast it
//                      into the peers' outputs (P2P stores, or one multimem.st).
//                      (reference: allreduceRsAgZeroCopy / allreduceNvls,
//                       allreduce_rsag_zero_copy.cu:40-109, allreduce_nvls_zero_copy.cu:16-74)
//   ar_staged<NVLS>    arbitrary (non-symmetric) user buffers: copy-in -> reduce -> gather
//                      through heap staging, chunked, with block-sliced dependencies so only
//                      same-index blocks of different ranks ever synchronise (no grid barrier).
//                      (reference: allreduceRsAg / allreduceNvlsBlockPipeline)
// Fused epilogue everywhere: post-scale (avg / user scale) and output dtype cast happen in
// registers before the result is stored -- the reference has no such fusion (SURVEY 2.4).
#pragma once
#include <type_traits>

#include "launch.h"
#include "coll_common.cuh"

namespace ub {

// ------------------------------------------------------------------ one-shot LL
template <typename T, int OP, bool MC>
__global__ void __launch_bounds__(512) ar_oneshot(const __grid_constant__ DevComm c,
                                                  const __grid_constant__ CollArgs a) {
  uint32_t* misc = reinterpret_cast<uint32_t*>(c.heap[c.rank] + a.misc_off);
  __shared__ uint32_t s_flag;
  if (threadIdx.x == 0) s_flag = ld_volatile(misc + kLLEpoch) + 1;
  __syncthreads();
  const uint32_t flag = s_flag;
  const uint64_t parity_off = a.ll_off + (uint64_t)(flag & 1u) * (kMaxRanks * kLLSlotBytes);
  const uint64_t nunits = (a.bytes + 15) / 16;
  const uint64_t gtid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t gstride = (uint64_t)gridDim.x * blockDim.x;
  const int n = c.nranks, rank = c.rank;

  // phase 1: publish my data as packets into every peer's slot[rank] (4 loads in flight per thread)
  {
    constexpr int B = 4;
    for (uint64_t u0 = gtid; u0 < nunits; u0 += gstride * B) {
      uint4 d[B];
#pragma unroll
      for (int j = 0; j < B; ++j) {
        const uint64_t u = u0 + (uint64_t)j * gstride;
        if (u < nunits) d[j] = load16_partial(a.in, u * 16, a.bytes);
      }
#pragma unroll
      for (int j = 0; j < B; ++j) {
        const uint64_t u = u0 + (uint64_t)j * gstride;
        if (u >= nunits) continue;
        uint4 p0 = make_uint4(d[j].x, flag, d[j].y, flag);
        uint4 p1 = make_uint4(d[j].z, flag, d[j].w, flag);
        const uint64_t off = parity_off + (uint64_t)rank * kLLSlotBytes + u * 32;
        if constexpr (MC) {
          multimem_st_v4(c.mc + off, p0);
          multimem_st_v4(c.mc + off + 16, p1);
        } else {
          for (int k = 1; k < n; ++k) {
            int p = rank + k;
            if (p >= n) p -= n;
            st_v4(c.heap[p] + off, p0);
            st_v4(c.heap[p] + off + 16, p1);
          }
        }
      }
    }
  }
  // phase 2: wait for the peers' packets in my own scratch, reduce in rank order
  // (identical order on every rank => bitwise identical results everywhere)
  char* my_ll = c.heap[rank] + parity_off;
  for (uint64_t u = gtid; u < nunits; u += gstride) {
    Vec16<T, OP> acc;
    for (int s = 0; s < n; ++s) {
      uint4 d;
      if (s == rank) {
        d = load16_partial(a.in, u * 16, a.bytes);
      } else {
        const char* slot = my_ll + (uint64_t)s * kLLSlotBytes + u * 32;
        uint4 p0, p1;
        SpinGuard g(c.timeout_ns);
        while (true) {
          p0 = ld_volatile_v4(slot);
          p1 = ld_volatile_v4(slot + 16);
          if (p0.y == flag && p0.w == flag && p1.y == flag && p1.w == flag) break;
          if (g.expired()) comm_abort(c, 10, s, (int)flag);
        }
        d = make_uint4(p0.x, p0.z, p1.x, p1.z);
      }
      if (s == 0) acc.init(d);
      else acc.accum(d);
    }
    acc.epilogue(a.ep);
    store16_partial(a.out, u * 16, a.bytes, acc.pack_same());
  }
  // last block to finish bumps the epoch (graph-replay safe: no host-side counter)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    uint32_t old = atomicAdd(misc + kLLDone, 1u);
    if (old == gridDim.x - 1) {
      misc[kLLDone] = 0;
      misc[kLLEpoch] = flag;
      __threadfence();
    }
  }
}

// ------------------------------------------------------------ two-shot zero-copy
// in/out live in the symmetric heap; bytes % 16 == 0.  The ranks exchange their actual heap
// offsets in the entry barrier, so buffers need not sit at identical offsets on every rank
// (the NVLS variant needs identical offsets for the multicast address and silently takes the
// P2P data path of the same kernel when they differ).
template <typename T, int OP, typename TO>
__device__ __forceinline__ void twoshot_p2p_body(const DevComm& c, const CollArgs& a, const uint64_t* s_off,
                                                 uint64_t lo, uint64_t hi) {
  constexpr int N = Vec16<T, OP>::N;
  constexpr int U = 2;
  const int n = c.nranks, rank = c.rank;
  const char* src[kMaxRanks];
  TO* dst[kMaxRanks];
#pragma unroll
  for (int q = 0; q < kMaxRanks; ++q) {
    src[q] = q < n ? c.heap[q] + s_off[q] : nullptr;
    int p = rank + q;
    if (p >= n) p -= n;
    dst[q] = q < n ? reinterpret_cast<TO*>(c.heap[p] + s_off[kMaxRanks + p]) : nullptr;
  }
  for (uint64_t v = lo + threadIdx.x; v < hi; v += (uint64_t)blockDim.x * U) {
    uint4 r[U][kMaxRanks];
#pragma unroll
    for (int j = 0; j < U; ++j) {
      uint64_t vv = v + (uint64_t)j * blockDim.x;
      if (vv < hi) {
#pragma unroll
        for (int q = 0; q < kMaxRanks; ++q)
          if (q < n) r[j][q] = ld_v4(src[q] + vv * 16);
      }
    }
#pragma unroll
    for (int j = 0; j < U; ++j) {
      uint64_t vv = v + (uint64_t)j * blockDim.x;
      if (vv < hi) {
        // accumulate in global rank order so the rounding is independent of who reduces
        Vec16<T, OP> acc;
        acc.init(r[j][0]);
#pragma unroll
        for (int q = 1; q < kMaxRanks; ++q)
          if (q < n) acc.accum(r[j][q]);
        acc.epilogue(a.ep);
#pragma unroll
        for (int k = 0; k < kMaxRanks; ++k)
          if (k < n) store_out<T, OP, TO, false>(dst[k], vv * N, acc);
      }
    }
  }
}

template <typename T, int OP, typename TO, bool NVLS>
__global__ void __launch_bounds__(512, 1) ar_twoshot(const __grid_constant__ DevComm c,
                                                     const __grid_constant__ CollArgs a) {
  constexpr int N = Vec16<T, OP>::N;
  const int n = c.nranks, rank = c.rank;
  __shared__ uint64_t s_off[2 * kMaxRanks];
  BlockSync s = sync_begin(c, kDomColl, blockIdx.x);
  // every rank's input is complete (and nobody still reads my output); learn the peers' offsets
  sync_exchange(c, s, kDomColl, a.in_off, a.out_off, s_off);

  const uint64_t nvec = a.bytes / 16;
  uint64_t blo, bhi, lo, hi;
  split_range(nvec, gridDim.x, blockIdx.x, blo, bhi);
  split_range(bhi - blo, n, rank, lo, hi);
  lo += blo;
  hi += blo;

  bool use_mc = false;
  if constexpr (NVLS) use_mc = all_equal(s_off, n) && all_equal(s_off + kMaxRanks, n);
  if (use_mc) {
    if constexpr (NVLS) {
      const char* in_mc = c.mc + a.in_off;
      TO* out_mc = reinterpret_cast<TO*>(c.mc + a.out_off);
      // in-switch reductions in flight per thread: a.variant = 8 doubles the default of 4 (UCCL_B200_NVLS_UNROLL)
      auto body = [&](auto uc) {
        constexpr int U = decltype(uc)::value;
        for (uint64_t v = lo + threadIdx.x; v < hi; v += (uint64_t)blockDim.x * U) {
          uint4 r[U];
#pragma unroll
          for (int j = 0; j < U; ++j) {
            uint64_t vv = v + (uint64_t)j * blockDim.x;
            if (vv < hi) r[j] = MmLdRed<T, OP>::ld(in_mc + vv * 16);
          }
#pragma unroll
          for (int j = 0; j < U; ++j) {
            uint64_t vv = v + (uint64_t)j * blockDim.x;
            if (vv < hi) {
              Vec16<T, OP> acc;
              acc.init(r[j]);
              acc.epilogue(a.ep);
              store_out<T, OP, TO, true>(out_mc, vv * N, acc);
            }
          }
        }
      };
      if (a.variant == 8) body(std::integral_constant<int, 8>{});
      else body(std::integral_constant<int, 4>{});
    }
  } else {
    twoshot_p2p_body<T, OP, TO>(c, a, s_off, lo, hi);
  }
  sync_barrier(c, s);  // every rank's output is complete
  sync_end(s);
}

// ------------------------------------------------------------------- staged
// Arbitrary local in/out (16-byte aligned, bytes % 16 == 0). Works chunk by chunk
// through stage_in / stage_out in the heap. Block b of every rank owns slice b of
// each chunk in all three phases, so a block only depends on same-index peer blocks.
template <typename T, int OP, typename TO, bool NVLS>
__global__ void __launch_bounds__(512, 1) ar_staged(const __grid_constant__ DevComm c,
                                                    const __grid_constant__ CollArgs a) {
  constexpr int N = Vec16<T, OP>::N;
  constexpr uint64_t kOutVecBytes = (uint64_t)N * sizeof(TO);  // output bytes per input vector
  // slice boundaries must keep the 16-byte bulk copies of phase 3 aligned
  constexpr uint64_t G = kOutVecBytes >= 16 ? 1 : 16 / kOutVecBytes;
  const int n = c.nranks, rank = c.rank;
  BlockSync s = sync_begin(c, kDomColl, blockIdx.x);

  const uint64_t nvec_total = a.bytes / 16;
  // vectors per chunk limited by both stages
  uint64_t cap_in = a.stage_bytes / 16, cap_out = a.stage_bytes / kOutVecBytes;
  const uint64_t chunk_vec = (cap_in < cap_out ? cap_in : cap_out) / G * G;
  const char* in = reinterpret_cast<const char*>(a.in);
  char* out = reinterpret_cast<char*>(a.out);
  char* my_stage_in = c.heap[rank] + a.stage_in_off;
  char* my_stage_out = c.heap[rank] + a.stage_out_off;

  for (uint64_t base = 0; base < nvec_total; base += chunk_vec) {
    const uint64_t cvec = (nvec_total - base) < chunk_vec ? (nvec_total - base) : chunk_vec;
    uint64_t blo, bhi;
    // slice boundaries of a full chunk, clamped: every block keeps the same stage range in every
    // chunk (see chunk_slice in coll_common.cuh)
    split_range(nvec_total < chunk_vec ? nvec_total : chunk_vec, gridDim.x, blockIdx.x, blo, bhi, G);
    if (blo > cvec) blo = cvec;
    if (bhi > cvec) bhi = cvec;
    // 1. copy-in my slice
    copy_units16(my_stage_in, in + base * 16, blo, bhi);
    sync_barrier(c, s);
    // 2. reduce my shard of the slice
    uint64_t lo, hi;
    split_range(bhi - blo, n, rank, lo, hi, G);
    lo += blo;
    hi += blo;
    if constexpr (NVLS) {
      const char* in_mc = c.mc + a.stage_in_off;
      TO* out_mc = reinterpret_cast<TO*>(c.mc + a.stage_out_off);
      constexpr int U = 4;
      for (uint64_t v0 = lo + threadIdx.x; v0 < hi; v0 += (uint64_t)U * blockDim.x) {
        uint4 r[U];
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const uint64_t v = v0 + (uint64_t)j * blockDim.x;
          if (v < hi) r[j] = MmLdRed<T, OP>::ld(in_mc + v * 16);
        }
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const uint64_t v = v0 + (uint64_t)j * blockDim.x;
          if (v < hi) {
            Vec16<T, OP> acc;
            acc.init(r[j]);
            acc.epilogue(a.ep);
            store_out<T, OP, TO, true>(out_mc, v * N, acc);
          }
        }
      }
    } else {
      constexpr int U = 2;
      for (uint64_t v0 = lo + threadIdx.x; v0 < hi; v0 += (uint64_t)U * blockDim.x) {
        uint4 r[U][kMaxRanks];
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const uint64_t v = v0 + (uint64_t)j * blockDim.x;
          if (v < hi) {
#pragma unroll
            for (int q = 0; q < kMaxRanks; ++q)
              if (q < n) r[j][q] = ld_v4(c.heap[q] + a.stage_in_off + v * 16);
          }
        }
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const uint64_t v = v0 + (uint64_t)j * blockDim.x;
          if (v < hi) {
            Vec16<T, OP> acc;
            acc.init(r[j][0]);
#pragma unroll
            for (int q = 1; q < kMaxRanks; ++q)
              if (q < n) acc.accum(r[j][q]);
            acc.epilogue(a.ep);
            store_out<T, OP, TO, false>(reinterpret_cast<TO*>(my_stage_out), v * N, acc);
            store_out<T, OP, TO, false>(reinterpret_cast<TO*>(out) + base * N, v * N, acc);
          }
        }
      }
    }
    sync_barrier(c, s);
    // 3. gather the slice into the user output
    if constexpr (NVLS) {
      copy_units16(out + base * kOutVecBytes, my_stage_out, blo * kOutVecBytes / 16, bhi * kOutVecBytes / 16);
    } else {
      for (int k = 1; k < n; ++k) {
        int p = rank + k;
        if (p >= n) p -= n;
        uint64_t plo, phi;
        split_range(bhi - blo, n, p, plo, phi, G);
        copy_units16(out + base * kOutVecBytes, c.heap[p] + a.stage_out_off, (plo + blo) * kOutVecBytes / 16,
                     (phi + blo) * kOutVecBytes / 16);
      }
    }
  }
  sync_barrier(c, s);  // peers are done pulling from my stage_out before anyone reuses it
  sync_end(s);
}

// ------------------------------------------------------- staged, block-pipelined (NVLS)
// Large ordinary (cudaMalloc / torch) buffers.  ar_staged runs copy-in -> in-switch reduce -> copy-out
// strictly one after the other per chunk, so the two HBM passes (2 x S read + 2 x S written) are added to
// the NVLink time and the kernel loses to NCCL from 256 MiB up.  Here the three phases run CONCURRENTLY on
// three groups of CTAs, two chunks deep:
//     group A (copy-in)   user input  -> stage_in[k & 1]                       local HBM
//     group B (reduce)    multimem.ld_reduce my shard of stage_in[k & 1] over all ranks, multimem.st the result
//                         into every rank's stage_out[k & 1]                    NVLink / NVSwitch
//     group C (copy-out)  stage_out[k & 1] -> user output                       local HBM
// Inside a rank the groups hand chunks to each other through three monotonic device counters (zeroed by the last
// CTA to leave); across ranks only the B CTAs of equal index synchronise (two barriers per chunk, as before).
//   A(k) needs red >= (k-1) nB   (all ranks finished reading stage_in slot k&1 for chunk k-2)
//   B(k) reduces, then needs in >= (k+2) nA and out >= k nC before the barrier that ends chunk k and opens k+1
//   C(k) needs red >= (k+1) nB   (every shard of chunk k has been written into my stage_out)
// a.variant = nB | nA << 8 | nC << 16; grid = nA + nB + nC (<= SM count: the groups wait for each other).
template <typename T, int OP>
__global__ void __launch_bounds__(512, 1) ar_staged_pipe(const __grid_constant__ DevComm c,
                                                         const __grid_constant__ CollArgs a) {
  constexpr int N = Vec16<T, OP>::N;
  const int n = c.nranks, rank = c.rank;
  const int nB = a.variant & 0xff, nA = (a.variant >> 8) & 0xff, nC = (a.variant >> 16) & 0xff;
  const int bid = blockIdx.x;
  const int role = bid < nB ? 1 : (bid < nB + nA ? 0 : 2);  // 0 copy-in, 1 reduce, 2 copy-out
  const int idx = role == 1 ? bid : (role == 0 ? bid - nB : bid - nB - nA);
  uint32_t* misc = reinterpret_cast<uint32_t*>(c.heap[rank] + a.misc_off);
  uint32_t* in_cnt = misc + kPipeIn;
  uint32_t* red_cnt = misc + kPipeRed;
  uint32_t* out_cnt = misc + kPipeOut;

  const uint64_t nvec_total = a.bytes / 16;
  const uint64_t slot_vec = (a.stage_bytes / 2) / 16;
  // chunk: about a tenth of the message (fill / drain of the pipeline vs. one barrier per chunk), 512 KiB granules,
  // at most one slot
  uint64_t chunk_vec = (nvec_total + 9) / 10;
  const uint64_t gran = (512u << 10) / 16;
  chunk_vec = (chunk_vec + gran - 1) / gran * gran;
  if (chunk_vec < (8u << 20) / 16) chunk_vec = (8u << 20) / 16;
  if (chunk_vec > slot_vec) chunk_vec = slot_vec / gran * gran;
  const uint64_t nchunks = (nvec_total + chunk_vec - 1) / chunk_vec;
  const char* in = reinterpret_cast<const char*>(a.in);
  char* out = reinterpret_cast<char*>(a.out);

  auto wait_ge = [&](uint32_t* p, uint64_t target) {
    if (threadIdx.x == 0) {
      SpinGuard g(c.timeout_ns);
      while ((uint64_t)ld_acquire_gpu(p) < target) {
        if (g.expired()) comm_abort(c, 30 + role, (int)target, (int)ld_acquire_gpu(p));
      }
    }
    __syncthreads();
  };
  auto bump = [&](uint32_t* p) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) atomicAdd(p, 1u);
  };

  BlockSync s;
  if (role == 1) {
    s = sync_begin(c, kDomColl, idx);
    wait_ge(in_cnt, (uint64_t)nA);
    sync_barrier(c, s);  // every rank has staged chunk 0
  }
  for (uint64_t k = 0; k < nchunks; ++k) {
    const uint64_t base = k * chunk_vec;
    const uint64_t cvec = (nvec_total - base) < chunk_vec ? (nvec_total - base) : chunk_vec;
    const uint64_t slot_off = (k & 1) * slot_vec * 16;
    if (role == 0) {
      if (k >= 2) wait_ge(red_cnt, (k - 1) * (uint64_t)nB);
      uint64_t lo, hi;
      split_range(cvec, nA, idx, lo, hi);
      copy_units16(c.heap[rank] + a.stage_in_off + slot_off, in + base * 16, lo, hi);
      bump(in_cnt);
    } else if (role == 1) {
      uint64_t blo, bhi, lo, hi;
      split_range(cvec, nB, idx, blo, bhi);
      split_range(bhi - blo, n, rank, lo, hi);
      lo += blo;
      hi += blo;
      const char* in_mc = c.mc + a.stage_in_off + slot_off;
      T* out_mc = reinterpret_cast<T*>(c.mc + a.stage_out_off + slot_off);
      constexpr int U = 8;  // 8 multimem.ld_reduce in flight per thread
      for (uint64_t v0 = lo + threadIdx.x; v0 < hi; v0 += (uint64_t)U * blockDim.x) {
        uint4 r[U];
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const uint64_t v = v0 + (uint64_t)j * blockDim.x;
          if (v < hi) r[j] = MmLdRed<T, OP>::ld(in_mc + v * 16);
        }
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const uint64_t v = v0 + (uint64_t)j * blockDim.x;
          if (v < hi) {
            Vec16<T, OP> acc;
            acc.init(r[j]);
            acc.epilogue(a.ep);
            store_out<T, OP, T, true>(out_mc, v * N, acc);
          }
        }
      }
      // ONE barrier per chunk: it says "my shard of chunk k is written everywhere" and, because the local
      // conditions of chunk k + 1 are checked first, also "my stage_in holds chunk k + 1 and my stage_out slot of
      // chunk k + 1 has been drained"
      if (k + 1 < nchunks) {
        wait_ge(in_cnt, (k + 2) * (uint64_t)nA);
        if (k >= 1) wait_ge(out_cnt, k * (uint64_t)nC);
      }
      sync_barrier(c, s);
      bump(red_cnt);
    } else {
      wait_ge(red_cnt, (k + 1) * (uint64_t)nB);
      uint64_t lo, hi;
      split_range(cvec, nC, idx, lo, hi);
      copy_units16(out + base * 16, c.heap[rank] + a.stage_out_off + slot_off, lo, hi);
      bump(out_cnt);
    }
  }
  if (role == 1) sync_end(s);
  // the last CTA to leave zeroes the hand-off counters for the next launch (graph-replay safe: no host state)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const uint32_t old = atomicAdd(misc + kPipeExit, 1u);
    if (old == gridDim.x - 1) {
      *reinterpret_cast<volatile uint32_t*>(in_cnt) = 0;
      *reinterpret_cast<volatile uint32_t*>(red_cnt) = 0;
      *reinterpret_cast<volatile uint32_t*>(out_cnt) = 0;
      *reinterpret_cast<volatile uint32_t*>(misc + kPipeExit) = 0;
      __threadfence();
    }
  }
}

// ------------------------------------------------------------------ launchers
enum ArAlgo : int {
  AR_AUTO = 0,
  AR_ONESHOT_LL = 1,
  AR_ONESHOT_MC = 2,
  AR_TWOSHOT_P2P = 3,
  AR_TWOSHOT_NVLS = 4,
  AR_STAGED_P2P = 5,
  AR_STAGED_NVLS = 6,
  AR_STAGED_PIPE = 7,
  AR_NUM_ALGOS = 8
};

template <typename T, int OP, typename TO>
cudaError_t launch_ar_typed(int algo, const DevComm& c, const CollArgs& a, int grid, int block, cudaStream_t st) {
  constexpr bool same = std::is_same<T, TO>::value;
  switch (algo) {
    case AR_ONESHOT_LL:
      if constexpr (same) { UB_LAUNCH((ar_oneshot<T, OP, false>), grid, block, 0, st, c, a); break; }
      return cudaErrorInvalidValue;
    case AR_ONESHOT_MC:
      if constexpr (same) { UB_LAUNCH((ar_oneshot<T, OP, true>), grid, block, 0, st, c, a); break; }
      return cudaErrorInvalidValue;
    case AR_TWOSHOT_P2P: UB_LAUNCH((ar_twoshot<T, OP, TO, false>), grid, block, 0, st, c, a); break;
    case AR_STAGED_P2P: UB_LAUNCH((ar_staged<T, OP, TO, false>), grid, block, 0, st, c, a); break;
    case AR_TWOSHOT_NVLS:
      if constexpr (MmLdRed<T, OP>::ok) { UB_LAUNCH((ar_twoshot<T, OP, TO, true>), grid, block, 0, st, c, a); break; }
      return cudaErrorInvalidValue;
    case AR_STAGED_NVLS:
      if constexpr (MmLdRed<T, OP>::ok) { UB_LAUNCH((ar_staged<T, OP, TO, true>), grid, block, 0, st, c, a); break; }
      return cudaErrorInvalidValue;
    case AR_STAGED_PIPE:
      if constexpr (MmLdRed<T, OP>::ok && same) { UB_LAUNCH((ar_staged_pipe<T, OP>), grid, block, 0, st, c, a); break; }
      return cudaErrorInvalidValue;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

template <typename T>
cudaError_t launch_ar_ops(int algo, int op, const DevComm& c, const CollArgs& a, int grid, int block,
                          cudaStream_t st) {
  switch (op) {
    case kSum: case kAvg: return launch_ar_typed<T, kSum, T>(algo, c, a, grid, block, st);
    case kProd: return launch_ar_typed<T, kProd, T>(algo, c, a, grid, block, st);
    case kMax: return launch_ar_typed<T, kMax, T>(algo, c, a, grid, block, st);
    case kMin: return launch_ar_typed<T, kMin, T>(algo, c, a, grid, block, st);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace ub
