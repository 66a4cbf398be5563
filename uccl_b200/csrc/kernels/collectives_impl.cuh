// AllGather / ReduceScatter / Broadcast / Reduce / AllToAll(v) kernels over the
// symmetric heap.  The reference only ships native AllGather + AllReduce (+ one
// broadcast); ReduceScatter, Reduce and AllToAll fall back to NCCL or are stubs
// (experimental/lite/nccl/nccl.cu:1747,1952-1966,2069-2102).  Here they are all native.
//
// Rule used everywhere: block b of every rank owns slice b of the data in every phase,
// so cross-rank dependencies only exist between same-index blocks and the per-block
// cross-rank barrier (prims.cuh) is sufficient -- no grid-wide sync is ever needed.
//
// "Source resolution": a collective that reads peers' inputs needs them in the heap.
// If the user input is symmetric (in_off != kNoOff) peers read it in place (zero copy);
// otherwise each block first copies its slice into stage_in and peers read that.
#pragma once
#include "coll_common.cuh"

namespace ub {

__device__ __forceinline__ void copy_bytes16(char* dst, const char* src, uint64_t lo, uint64_t hi,
                                             uint64_t total_bytes_src, uint64_t total_bytes_dst) {
  // copies 16-byte units [lo, hi) (unit index), partial-tail aware on both sides;
  // degrades to a byte loop when either side is not 16-byte aligned (odd segment sizes).
  // Loads are issued in batches of 8 before the dependent stores: with one load per store the
  // loop is bound by the (NVLink) load latency instead of the bandwidth.
  if ((((uintptr_t)src | (uintptr_t)dst) & 15) == 0) {
    constexpr int B = 8;
    const uint64_t full_src = total_bytes_src / 16, full_dst = total_bytes_dst / 16;
    const uint64_t full = full_src < full_dst ? full_src : full_dst;  // units that need no tail handling
    const uint64_t fhi = hi < full ? hi : full;
    uint64_t u = lo + threadIdx.x;
    for (; u + (uint64_t)(B - 1) * blockDim.x < fhi; u += (uint64_t)B * blockDim.x) {
      uint4 v[B];
#pragma unroll
      for (int j = 0; j < B; ++j) v[j] = ld_v4(src + (u + (uint64_t)j * blockDim.x) * 16);
#pragma unroll
      for (int j = 0; j < B; ++j) st_v4(dst + (u + (uint64_t)j * blockDim.x) * 16, v[j]);
    }
    for (; u < hi; u += blockDim.x) {
      uint4 v = load16_partial(src, u * 16, total_bytes_src);
      store16_partial(dst, u * 16, total_bytes_dst, v);
    }
  } else {
    uint64_t total = total_bytes_src < total_bytes_dst ? total_bytes_src : total_bytes_dst;
    uint64_t b0 = lo * 16, b1 = hi * 16 < total ? hi * 16 : total;
    for (uint64_t i = b0 + threadIdx.x; i < b1; i += blockDim.x) dst[i] = src[i];
  }
}

// Pull one 16-byte-unit range [lo, hi) from each of `n` sources into `n` destinations, issuing the
// loads of ALL sources before the dependent stores (n x 2 loads in flight per thread): a loop over
// peers with an inner copy loop would expose one NVLink round trip per peer.
template <typename SrcFn, typename DstFn>
__device__ __forceinline__ void gather_units16(int n, uint64_t lo, uint64_t hi, uint64_t src_bytes, uint64_t dst_bytes,
                                               SrcFn src_of, DstFn dst_of) {
  bool aligned = true;
  for (int k = 0; k < n; ++k) aligned = aligned && ((((uintptr_t)src_of(k) | (uintptr_t)dst_of(k)) & 15) == 0);
  if (!aligned) {
    for (int k = 0; k < n; ++k) copy_bytes16(dst_of(k), src_of(k), lo, hi, src_bytes, dst_bytes);
    return;
  }
  constexpr int B = 2;
  for (uint64_t u0 = lo + threadIdx.x; u0 < hi; u0 += (uint64_t)B * blockDim.x) {
    uint4 v[B][kMaxRanks];
#pragma unroll
    for (int j = 0; j < B; ++j) {
      const uint64_t u = u0 + (uint64_t)j * blockDim.x;
      if (u < hi) {
#pragma unroll
        for (int k = 0; k < kMaxRanks; ++k)
          if (k < n) v[j][k] = load16_partial(src_of(k), u * 16, src_bytes);
      }
    }
#pragma unroll
    for (int j = 0; j < B; ++j) {
      const uint64_t u = u0 + (uint64_t)j * blockDim.x;
      if (u < hi) {
#pragma unroll
        for (int k = 0; k < kMaxRanks; ++k)
          if (k < n) store16_partial(dst_of(k), u * 16, dst_bytes, v[j][k]);
      }
    }
  }
}

// ------------------------------------------------------------------ AllGather
// a.bytes = bytes contributed by each rank. out holds n * bytes.
// MODE 0: push P2P (out symmetric)   MODE 1: push multicast (out symmetric, NVLS)
// MODE 2: pull (in symmetric or staged copy-in; out arbitrary)
template <int MODE>
__global__ void __launch_bounds__(512, 1) ag_kernel(const __grid_constant__ DevComm c,
                                                    const __grid_constant__ CollArgs a) {
  const int n = c.nranks, rank = c.rank;
  __shared__ uint64_t s_off[2 * kMaxRanks];
  BlockSync s = sync_begin(c, kDomColl, blockIdx.x);
  const uint64_t units = (a.bytes + 15) / 16;
  const char* in = reinterpret_cast<const char*>(a.in);
  // entry barrier: peers have entered (their `out` may be overwritten / their `in` is complete)
  // and everybody learns everybody's heap offsets
  sync_exchange(c, s, kDomColl, a.in_off, a.out_off, s_off);
  if constexpr (MODE == 0 || MODE == 1) {
    uint64_t blo, bhi;
    split_range(units, gridDim.x, blockIdx.x, blo, bhi);
    const bool use_mc = (MODE == 1) && all_equal(s_off + kMaxRanks, n);
    constexpr int B = 4;
    for (uint64_t u0 = blo + threadIdx.x; u0 < bhi; u0 += (uint64_t)B * blockDim.x) {
      uint4 v[B];
#pragma unroll
      for (int j = 0; j < B; ++j) {
        const uint64_t u = u0 + (uint64_t)j * blockDim.x;
        if (u < bhi) v[j] = load16_partial(in, u * 16, a.bytes);
      }
#pragma unroll
      for (int j = 0; j < B; ++j) {
        const uint64_t u = u0 + (uint64_t)j * blockDim.x;
        if (u >= bhi) continue;
        if (use_mc && u * 16 + 16 <= a.bytes) {
          multimem_st_v4(c.mc + a.out_off + (uint64_t)rank * a.bytes + u * 16, v[j]);
        } else {
          for (int k = 0; k < n; ++k) {
            int p = rank + k;
            if (p >= n) p -= n;
            store16_partial(c.heap[p] + s_off[kMaxRanks + p] + (uint64_t)rank * a.bytes, u * 16, a.bytes, v[j]);
          }
        }
      }
    }
    sync_barrier(c, s);
  } else {
    bool staged = false;
    for (int q = 0; q < n; ++q) staged = staged || (s_off[q] == kNoOff);  // consensus: any plain input => stage
    char* out = reinterpret_cast<char*>(a.out);
    const uint64_t chunk_bytes = staged ? (a.stage_bytes / 16 * 16) : a.bytes;
    for (uint64_t base = 0; base < a.bytes; base += chunk_bytes) {
      const uint64_t cb = (a.bytes - base) < chunk_bytes ? (a.bytes - base) : chunk_bytes;
      uint64_t blo, bhi;
      chunk_slice(a.bytes, chunk_bytes, cb, blo, bhi);
      if (staged) {
        copy_bytes16(c.heap[rank] + a.stage_in_off, in + base, blo, bhi, cb, cb);
        sync_barrier(c, s);
      }
      gather_units16(
          n, blo, bhi, cb, cb,
          [&](int k) -> const char* {
            int p = rank + k;
            if (p >= n) p -= n;
            if (p == rank) return in + base;
            return c.heap[p] + (staged ? a.stage_in_off : (s_off[p] + base));
          },
          [&](int k) -> char* {
            int p = rank + k;
            if (p >= n) p -= n;
            return out + (uint64_t)p * a.bytes + base;
          });
      sync_barrier_relaxed(c, s);  // peers finished reading my stage / input
    }
  }
  sync_end(s);
}

// ------------------------------------------------------------- ReduceScatter
// a.count = elements each rank receives; input holds n * count elements of T.
// NVLS requires a symmetric input. Output is a plain local buffer.
// In place (out = in + rank * bytes, NCCL's in-place reduce-scatter; reduce_scatter_rmsnorm relies on it) is safe in
// every variant.  Push: block b writes its slice of a chunk only after the barrier that follows its own push of that
// slice of every piece, own piece included, and later chunks read other bytes.  Pull / zero-copy: peer q only reads
// piece q of my input (or of my stage, which holds a copy made before the barrier), never my own piece, and each
// thread reads my own units before it stores their sum.
template <typename T, int OP, bool NVLS>
__global__ void __launch_bounds__(512, 1) rs_kernel(const __grid_constant__ DevComm c,
                                                    const __grid_constant__ CollArgs a) {
  const int n = c.nranks, rank = c.rank;
  __shared__ uint64_t s_off[2 * kMaxRanks];
  BlockSync s = sync_begin(c, kDomColl, blockIdx.x);
  sync_exchange(c, s, kDomColl, a.in_off, a.out_off, s_off);
  bool staged = false;
  for (int q = 0; q < n; ++q) staged = staged || (s_off[q] == kNoOff);
  const bool same = all_equal(s_off, n);
  const char* in = reinterpret_cast<const char*>(a.in);
  char* out = reinterpret_cast<char*>(a.out);
  if (staged && a.variant == 1) {
    // Push staging: every rank stores piece d of its (plain) input straight into slot[rank] of
    // rank d's stage over NVLink, then each rank reduces its n slots from *local* memory.  Compared
    // with the pull scheme below (copy all n pieces into the own stage, peers read them) this
    // drops the local copy of the whole input: the only bytes moved besides the NVLink traffic are
    // the 1/n that end up in the result.  stage_in / stage_out alternate as halves, so the barrier
    // of chunk k+1 doubles as "everybody is done reading chunk k-1's half".
    const uint64_t chunk_bytes = a.stage_bytes / n / 16 * 16;
    int k = 0;
    for (uint64_t base = 0; base < a.bytes; base += chunk_bytes, ++k) {
      const uint64_t cb = (a.bytes - base) < chunk_bytes ? (a.bytes - base) : chunk_bytes;
      uint64_t blo, bhi;
      chunk_slice(a.bytes, chunk_bytes, cb, blo, bhi);
      const uint64_t half = (k & 1) ? a.stage_out_off : a.stage_in_off;
      gather_units16(
          n, blo, bhi, cb, cb,
          [&](int j) -> const char* {
            int d = rank + j;
            if (d >= n) d -= n;
            return in + (uint64_t)d * a.bytes + base;
          },
          [&](int j) -> char* {
            int d = rank + j;
            if (d >= n) d -= n;
            return c.heap[d] + half + (uint64_t)rank * chunk_bytes;
          });
      sync_barrier(c, s);  // every peer's slice b of this chunk has landed in my stage
      const char* my = c.heap[rank] + half;
      constexpr int U = 2;
      for (uint64_t u0 = blo + threadIdx.x; u0 < bhi; u0 += (uint64_t)U * blockDim.x) {
        uint4 r[U][kMaxRanks];
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const uint64_t u = u0 + (uint64_t)j * blockDim.x;
          if (u >= bhi) continue;
#pragma unroll
          for (int q = 0; q < kMaxRanks; ++q)
            if (q < n) r[j][q] = ld_v4(my + (uint64_t)q * chunk_bytes + u * 16);
        }
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const uint64_t u = u0 + (uint64_t)j * blockDim.x;
          if (u >= bhi) continue;
          Vec16<T, OP> acc;
          acc.init(r[j][0]);
#pragma unroll
          for (int q = 1; q < kMaxRanks; ++q)
            if (q < n) acc.accum(r[j][q]);
          acc.epilogue(a.ep);
          store16_partial(out + base, u * 16, cb, acc.pack_same());
        }
      }
    }
    sync_barrier_relaxed(c, s);  // the next collective may overwrite the stage halves
    sync_end(s);
    return;
  }
  // per-destination chunk so that n chunks fit the stage
  const uint64_t chunk_bytes = staged ? (a.stage_bytes / n / 16 * 16) : a.bytes;
  for (uint64_t base = 0; base < a.bytes; base += chunk_bytes) {
    const uint64_t cb = (a.bytes - base) < chunk_bytes ? (a.bytes - base) : chunk_bytes;
    uint64_t blo, bhi;
    chunk_slice(a.bytes, chunk_bytes, cb, blo, bhi);
    if (staged) {
      for (int d = 0; d < n; ++d)
        copy_bytes16(c.heap[rank] + a.stage_in_off + (uint64_t)d * chunk_bytes, in + (uint64_t)d * a.bytes + base,
                     blo, bhi, cb, cb);
      sync_barrier(c, s);
    }
    const uint64_t rel = staged ? (uint64_t)rank * chunk_bytes : ((uint64_t)rank * a.bytes + base);
    constexpr int U = 2;
    const bool use_mc = NVLS && (staged || same);
    for (uint64_t u0 = blo + threadIdx.x; u0 < bhi; u0 += (uint64_t)U * blockDim.x) {
      uint4 r[U][kMaxRanks];
#pragma unroll
      for (int j = 0; j < U; ++j) {
        const uint64_t u = u0 + (uint64_t)j * blockDim.x;
        if (u >= bhi) continue;
        if constexpr (NVLS) {
          if (use_mc) {
            r[j][0] = MmLdRed<T, OP>::ld(c.mc + (staged ? a.stage_in_off : a.in_off) + rel + u * 16);
            continue;
          }
        }
#pragma unroll
        for (int q = 0; q < kMaxRanks; ++q)
          if (q < n) r[j][q] = ld_v4(c.heap[q] + (staged ? a.stage_in_off : s_off[q]) + rel + u * 16);
      }
#pragma unroll
      for (int j = 0; j < U; ++j) {
        const uint64_t u = u0 + (uint64_t)j * blockDim.x;
        if (u >= bhi) continue;
        Vec16<T, OP> acc;
        acc.init(r[j][0]);
        if (!use_mc) {
#pragma unroll
          for (int q = 1; q < kMaxRanks; ++q)
            if (q < n) acc.accum(r[j][q]);
        }
        acc.epilogue(a.ep);
        store16_partial(out + base, u * 16, cb, acc.pack_same());
      }
    }
    sync_barrier_relaxed(c, s);  // peers finished reading my input / stage
  }
  sync_end(s);
}

// ------------------------------------------------------------------ Broadcast
// Only `out` is meaningful on every rank (non-roots may pass any `in`), so the variant is
// chosen from `out` alone: symmetric out -> root pushes (MODE 1 multicast, MODE 2 P2P);
// otherwise MODE 0: root copies into its stage and everyone pulls.
template <int MODE>
__global__ void __launch_bounds__(512, 1) bcast_kernel(const __grid_constant__ DevComm c,
                                                       const __grid_constant__ CollArgs a) {
  const int n = c.nranks, rank = c.rank, root = a.root;
  BlockSync s = sync_begin(c, kDomColl, blockIdx.x);
  const char* in = reinterpret_cast<const char*>(a.in);
  char* out = reinterpret_cast<char*>(a.out);
  if constexpr (MODE == 1 || MODE == 2) {
    __shared__ uint64_t s_off[2 * kMaxRanks];
    sync_exchange(c, s, kDomColl, a.in_off, a.out_off, s_off);
    if (rank == root) {
      const bool use_mc = (MODE == 1) && all_equal(s_off + kMaxRanks, n);
      const uint64_t units = (a.bytes + 15) / 16;
      uint64_t blo, bhi;
      split_range(units, gridDim.x, blockIdx.x, blo, bhi);
      for (uint64_t u = blo + threadIdx.x; u < bhi; u += blockDim.x) {
        uint4 v = load16_partial(in, u * 16, a.bytes);
        if (use_mc && u * 16 + 16 <= a.bytes) {
          multimem_st_v4(c.mc + a.out_off + u * 16, v);
        } else {
          for (int p = 0; p < n; ++p) store16_partial(c.heap[p] + s_off[kMaxRanks + p], u * 16, a.bytes, v);
        }
      }
    }
    sync_barrier(c, s);
  } else if constexpr (MODE == 3) {
    // ordinary output buffers + NVLS: the root stores every 16-byte word ONCE into the multicast address of the
    // staging area (the switch replicates it to all ranks), everybody copies its stage to the user buffer.  A pull from
    // the root's stage would be bound by the root's egress (N - 1 copies of the message over one GPU's links).  Stage halves alternate, so one barrier per chunk suffices: the root
    // rewrites half k & 1 only after the barrier of chunk k - 1, which every peer enters after copying chunk k - 2 out.
    const uint64_t half = (a.stage_bytes / 2) / 16 * 16;
    uint64_t k = 0;
    for (uint64_t base = 0; base < a.bytes; base += half, ++k) {
      const uint64_t cb = (a.bytes - base) < half ? (a.bytes - base) : half;
      const uint64_t hoff = a.stage_out_off + (k & 1) * half;
      uint64_t blo, bhi;
      chunk_slice(a.bytes, half, cb, blo, bhi);
      if (rank == root) {
        constexpr int B = 4;
        for (uint64_t u0 = blo + threadIdx.x; u0 < bhi; u0 += (uint64_t)B * blockDim.x) {
          uint4 v[B];
#pragma unroll
          for (int q = 0; q < B; ++q) {
            const uint64_t u = u0 + (uint64_t)q * blockDim.x;
            if (u < bhi) v[q] = load16_partial(in + base, u * 16, cb);
          }
#pragma unroll
          for (int q = 0; q < B; ++q) {
            const uint64_t u = u0 + (uint64_t)q * blockDim.x;
            if (u < bhi) {
              multimem_st_v4(c.mc + hoff + u * 16, v[q]);
              // the root's own output comes straight from the registers: no second pass over its stage, so after the
              // barrier it starts on chunk k + 1 while the peers are still copying chunk k out
              if (out != in) store16_partial(out + base, u * 16, cb, v[q]);
            }
          }
        }
      }
      sync_barrier(c, s);
      if (rank != root) copy_bytes16(out + base, c.heap[rank] + hoff, blo, bhi, cb, cb);
    }
    sync_barrier_relaxed(c, s);  // the next collective may reuse the stage
  } else {
    const uint64_t chunk_bytes = a.stage_bytes / 16 * 16;
    for (uint64_t base = 0; base < a.bytes; base += chunk_bytes) {
      const uint64_t cb = (a.bytes - base) < chunk_bytes ? (a.bytes - base) : chunk_bytes;
      uint64_t blo, bhi;
      chunk_slice(a.bytes, chunk_bytes, cb, blo, bhi);
      if (rank == root) copy_bytes16(c.heap[rank] + a.stage_in_off, in + base, blo, bhi, cb, cb);
      sync_barrier(c, s);
      if (rank != root) {
        copy_bytes16(out + base, c.heap[root] + a.stage_in_off, blo, bhi, cb, cb);
      } else if (out != in) {
        copy_bytes16(out + base, in + base, blo, bhi, cb, cb);
      }
      sync_barrier_relaxed(c, s);
    }
  }
  sync_end(s);
}

// --------------------------------------------------------------------- Reduce
template <typename T, int OP, bool NVLS>
__global__ void __launch_bounds__(512, 1) reduce_kernel(const __grid_constant__ DevComm c,
                                                        const __grid_constant__ CollArgs a) {
  const int n = c.nranks, rank = c.rank, root = a.root;
  __shared__ uint64_t s_off[2 * kMaxRanks];
  BlockSync s = sync_begin(c, kDomColl, blockIdx.x);
  sync_exchange(c, s, kDomColl, a.in_off, a.out_off, s_off);
  bool staged = false;
  for (int q = 0; q < n; ++q) staged = staged || (s_off[q] == kNoOff);
  const bool same = all_equal(s_off, n);
  const char* in = reinterpret_cast<const char*>(a.in);
  char* out = reinterpret_cast<char*>(a.out);
  const uint64_t chunk_bytes = staged ? (a.stage_bytes / 16 * 16) : a.bytes;
  for (uint64_t base = 0; base < a.bytes; base += chunk_bytes) {
    const uint64_t cb = (a.bytes - base) < chunk_bytes ? (a.bytes - base) : chunk_bytes;
    uint64_t blo, bhi;
    chunk_slice(a.bytes, chunk_bytes, cb, blo, bhi);
    if (staged) {
      copy_bytes16(c.heap[rank] + a.stage_in_off, in + base, blo, bhi, cb, cb);
      sync_barrier(c, s);
    }
    if (rank == root) {
      for (uint64_t u = blo + threadIdx.x; u < bhi; u += blockDim.x) {
        Vec16<T, OP> acc;
        bool done = false;
        if constexpr (NVLS) {
          if (staged || same) {
            acc.init(MmLdRed<T, OP>::ld(c.mc + (staged ? a.stage_in_off : a.in_off + base) + u * 16));
            done = true;
          }
        }
        if (!done) {
          uint4 r[kMaxRanks];
#pragma unroll
          for (int q = 0; q < kMaxRanks; ++q)
            if (q < n) r[q] = ld_v4(c.heap[q] + (staged ? a.stage_in_off : s_off[q] + base) + u * 16);
          acc.init(r[0]);
#pragma unroll
          for (int q = 1; q < kMaxRanks; ++q)
            if (q < n) acc.accum(r[q]);
        }
        acc.epilogue(a.ep);
        store16_partial(out + base, u * 16, cb, acc.pack_same());
      }
    }
    sync_barrier_relaxed(c, s);
  }
  sync_end(s);
}

// ------------------------------------------------------------------- AllToAll
// a.bytes = bytes exchanged with each peer. in/out hold n * bytes.
// MODE 0: pull (in symmetric or staged)   MODE 1: push (out symmetric)
template <int MODE>
__global__ void __launch_bounds__(512, 1) a2a_kernel(const __grid_constant__ DevComm c,
                                                     const __grid_constant__ CollArgs a) {
  const int n = c.nranks, rank = c.rank;
  __shared__ uint64_t s_off[2 * kMaxRanks];
  BlockSync s = sync_begin(c, kDomColl, blockIdx.x);
  const char* in = reinterpret_cast<const char*>(a.in);
  char* out = reinterpret_cast<char*>(a.out);
  sync_exchange(c, s, kDomColl, a.in_off, a.out_off, s_off);
  if constexpr (MODE == 1) {
    const uint64_t units = (a.bytes + 15) / 16;
    uint64_t blo, bhi;
    split_range(units, gridDim.x, blockIdx.x, blo, bhi);
    gather_units16(
        n, blo, bhi, a.bytes, a.bytes,
        [&](int k) -> const char* {
          int p = rank + k;
          if (p >= n) p -= n;
          return in + (uint64_t)p * a.bytes;
        },
        [&](int k) -> char* {
          int p = rank + k;
          if (p >= n) p -= n;
          return c.heap[p] + s_off[kMaxRanks + p] + (uint64_t)rank * a.bytes;
        });
    sync_barrier(c, s);
  } else {
    bool staged = false;
    for (int q = 0; q < n; ++q) staged = staged || (s_off[q] == kNoOff);
    const uint64_t chunk_bytes = staged ? (a.stage_bytes / n / 16 * 16) : a.bytes;
    for (uint64_t base = 0; base < a.bytes; base += chunk_bytes) {
      const uint64_t cb = (a.bytes - base) < chunk_bytes ? (a.bytes - base) : chunk_bytes;
      uint64_t blo, bhi;
      chunk_slice(a.bytes, chunk_bytes, cb, blo, bhi);
      if (staged) {
        for (int d = 0; d < n; ++d)
          copy_bytes16(c.heap[rank] + a.stage_in_off + (uint64_t)d * chunk_bytes,
                       in + (uint64_t)d * a.bytes + base, blo, bhi, cb, cb);
        sync_barrier(c, s);
      }
      gather_units16(
          n, blo, bhi, cb, cb,
          [&](int k) -> const char* {
            int p = rank + k;
            if (p >= n) p -= n;
            return c.heap[p] + (staged ? (a.stage_in_off + (uint64_t)rank * chunk_bytes)
                                       : (s_off[p] + (uint64_t)rank * a.bytes + base));
          },
          [&](int k) -> char* {
            int p = rank + k;
            if (p >= n) p -= n;
            return out + (uint64_t)p * a.bytes + base;
          });
      sync_barrier_relaxed(c, s);
    }
  }
  sync_end(s);
}

// ------------------------------------------------------------------ AllToAllv
// Variable counts: every rank publishes its (send offset, send bytes) row for each
// destination into the heap (misc area), then each rank pulls its column.
static __global__ void __launch_bounds__(512, 1) a2av_kernel(const __grid_constant__ DevComm c,
                                                      const __grid_constant__ CollArgs a,
                                                      const __grid_constant__ A2AvArgs v) {
  // input must be symmetric (host stages it otherwise): peers read in_off + send_off[me].
  const int n = c.nranks, rank = c.rank;
  BlockSync s = sync_begin(c, kDomColl, blockIdx.x);
  // per-block private copy of the table so that same-index blocks suffice for ordering
  uint64_t* my_tab = reinterpret_cast<uint64_t*>(c.heap[rank] + v.table_off) + (uint64_t)blockIdx.x * kMaxRanks * 2;
  if (threadIdx.x < n) {
    my_tab[threadIdx.x * 2 + 0] = a.in_off + v.send_off[threadIdx.x];  // absolute heap offset of the segment
    my_tab[threadIdx.x * 2 + 1] = v.send_bytes[threadIdx.x];
  }
  sync_barrier(c, s);
  char* out = reinterpret_cast<char*>(a.out);
  for (int k = 0; k < n; ++k) {
    int p = rank + k;
    if (p >= n) p -= n;
    const uint64_t* ptab =
        reinterpret_cast<const uint64_t*>(c.heap[p] + v.table_off) + (uint64_t)blockIdx.x * kMaxRanks * 2;
    const uint64_t soff = ptab[rank * 2 + 0];
    uint64_t sbytes = ptab[rank * 2 + 1];
    if (sbytes > v.recv_bytes[p]) sbytes = v.recv_bytes[p];
    const uint64_t units = (sbytes + 15) / 16;
    uint64_t blo, bhi;
    split_range(units, gridDim.x, blockIdx.x, blo, bhi);
    const char* src = c.heap[p] + soff;
    char* dst = out + v.recv_off[p];
    // offsets may be only element-aligned: fall back to byte copies when not 16-byte aligned
    if ((((uintptr_t)src | (uintptr_t)dst) & 15) == 0) {
      copy_bytes16(dst, src, blo, bhi, sbytes, sbytes);
    } else {
      uint64_t lo = blo * 16, hi = bhi * 16 < sbytes ? bhi * 16 : sbytes;
      for (uint64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) dst[i] = src[i];
    }
  }
  sync_barrier_relaxed(c, s);
  sync_end(s);
}

}  // namespace ub

namespace ub {
// ------------------------------------------------------------------ Send / Recv
// ncclSend/ncclRecv.  Grid = npeers * kSrBlocks CTAs; in each CTA warps 0-7 run the send flow and
// warps 8-15 the receive flow of one (peer, sub-block), so both directions always make progress (no
// deadlock for symmetric exchanges).  Two data paths, chosen per message by the SENDER and announced in
// a header word that travels with the first "ready" signal:
//   * zero-copy: the source lives in the symmetric heap -> the receiver pulls its slice straight from
//     the sender's buffer with a TMA pipeline (cp.async.bulk peer -> smem -> local) and acks; the sender
//     only waits for that ack (its buffer may be reused when the kernel returns, NCCL semantics);
//   * staged: arbitrary user buffers -> the sender stages chunks in its own heap and publishes a
//     sequence number in the receiver's heap; the receiver pulls the chunk over NVLink and acks.
// Sequence counters are persistent and monotonic per (peer, sub-block): no reset, graph-replay safe.
// (reference: lite's host-staged ncclSend/Recv, experimental/lite/nccl/nccl.cu:1145-1350,2033-2067;
//  the first version of this kernel moved 512 KB slots with one 16-byte load in flight per thread, far too
//  few bytes in flight for NVLink)
__device__ __forceinline__ void half_sync(int id) { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }

constexpr int kSrTmaStages = 8;      // receive half: bulk loads in flight (zero-copy pull and staged copy-out)
constexpr int kSrSendStages = 4;     // send half (staged push)
constexpr uint32_t kSrTmaChunk = 16u << 10;
constexpr int kSrPiecesPerSlot = (int)(kSrChunkBytes / kSrTmaChunk);

static __global__ void __launch_bounds__(512, 1) sendrecv_kernel(const __grid_constant__ DevComm c,
                                                                const __grid_constant__ SendRecvArgs a) {
  extern __shared__ __align__(128) unsigned char sr_smem[];  // [recv: kSrTmaStages | send: kSrSendStages] x kSrTmaChunk
  __shared__ __align__(8) uint64_t sr_full[kSrTmaStages];
  __shared__ __align__(8) uint64_t sr_sfull[kSrSendStages];
  __shared__ uint32_t s_send_done;  // staged push: slots whose bulk stores have completed (pump thread -> announcer thread)
  unsigned char* send_smem = sr_smem + (size_t)kSrTmaStages * kSrTmaChunk;
  if (threadIdx.x == 0) s_send_done = 0;
  __syncthreads();
  __shared__ uint64_t s_hdr;
  const int me = c.rank;
  // the staging area is sized for kMaxRanks peers x kSrBlocks x kSrSlots slots: with fewer ranks every (peer, sub-block)
  // pair gets a proportionally deeper window (2 ranks: 16 slots = 1 MiB in flight per pair), which is what hides the
  // NVLink round trip of the ready / ack handshake when ONE peer must take the whole link bandwidth
  int npow2 = 1;
  while (npow2 < c.nranks) npow2 <<= 1;
  const int nslots_pair = kSrSlots * (kMaxRanks / npow2);
  const int pi = blockIdx.x / kSrBlocks, j = blockIdx.x % kSrBlocks;
  const int peer = a.peers[pi];
  // sub-blocks that take part in a message: one per 64 KiB, so a small message costs one handshake, not sixteen
  // (both ends derive the count from the byte count they were given, which NCCL semantics require to match)
  auto active_blocks = [](uint64_t bytes) -> int {
    const uint64_t nb = (bytes + (64u << 10) - 1) / (64u << 10);
    return nb < 1 ? 1 : (nb > (uint64_t)kSrBlocks ? kSrBlocks : (int)nb);
  };
  const bool is_send = threadIdx.x < 256;
  const int t = threadIdx.x & 255;
  // flag words (u32) inside every heap: ready[src][j], ack[dst][j], sseq[dst][j], rseq[src][j], then u64 hdr[src][j]
  auto flags = [&](int rank) { return reinterpret_cast<uint32_t*>(c.heap[rank] + a.sr_flag_off); };
  const int W = kMaxRanks * kSrBlocks;
  auto hdrs = [&](int rank) { return reinterpret_cast<uint64_t*>(flags(rank) + 4 * W); };
  uint32_t* my_flags = flags(me);
  if (peer == me) {
    // self send/recv: plain local copy by the whole CTA slice
    const uint64_t bytes = a.sbytes[me] < a.rbytes[me] ? a.sbytes[me] : a.rbytes[me];
    uint64_t lo, hi;
    split_range((bytes + 15) / 16, kSrBlocks, j, lo, hi);
    copy_bytes16(a.rbuf[me], a.sbuf[me], lo, hi, bytes, bytes);
    return;
  }
  if (is_send) {
    const uint64_t bytes = a.sbytes[peer];
    if (bytes == 0) return;
    const int nb = active_blocks(bytes);
    if (j >= nb) return;
    uint64_t lo, hi;
    split_range((bytes + 15) / 16, nb, j, lo, hi);
    uint32_t seq = my_flags[2 * W + peer * kSrBlocks + j];
    uint32_t* my_ack = my_flags + 1 * W + peer * kSrBlocks + j;
    uint32_t* peer_ready = flags(peer) + 0 * W + me * kSrBlocks + j;
    uint64_t* peer_hdr = hdrs(peer) + me * kSrBlocks + j;
    const bool direct = a.s_off[peer] != kNoOff && (bytes % 16) == 0;
    if (direct) {
      // announce where the data is and wait until the receiver has pulled my slice
      if (t == 0) {
        ++seq;
        *reinterpret_cast<volatile uint64_t*>(peer_hdr) = a.s_off[peer];
        st_release_sys(peer_ready, seq);  // also orders the (earlier) writes of the source buffer
        SpinGuard g(c.timeout_ns);
        while ((int32_t)(ld_acquire_sys(my_ack) - seq) < 0) {
          if (g.expired()) comm_abort(c, 22, peer, (int)seq);
        }
        my_flags[2 * W + peer * kSrBlocks + j] = seq;
      }
      return;
    }
    // staged: the chunks go straight into the RECEIVER's staging slots (push: remote stores are posted, a pull
    // would pay the NVLink round trip per slot), the receiver copies them out locally
    char* stage = c.heap[peer] + a.sr_stage_off + ((uint64_t)(me * kSrBlocks + j) * nslots_pair) * kSrChunkBytes;
    const uint64_t cu = kSrChunkBytes / 16;
    if (lo >= hi) {  // an empty slice still announces the mode once (the receiver waits for one header)
      if (t == 0) {
        ++seq;
        *reinterpret_cast<volatile uint64_t*>(peer_hdr) = kNoOff;
        st_release_sys(peer_ready, seq);
        my_flags[2 * W + peer * kSrBlocks + j] = seq;
      }
      return;
    }
    if ((bytes % 16) == 0) {
      // ---- two elected threads.  The PUMP (t == 0) moves sbuf -> smem -> peer slot with bulk copies, kSrSendStages
      //      pieces in flight, and publishes in shared memory how many slots have completed.  The ANNOUNCER (t == 32)
      //      turns that into ready flags for the receiver: each announcement needs a system-scope release fence
      //      (~3 us; without it the flag can overtake the data on another NVLink), and on its own thread the fence
      //      overlaps the next slots' copies and batches itself: while it is fencing, more slots complete.
      const uint32_t seq0 = seq;
      const uint64_t b0 = lo * 16, b1 = hi * 16;
      const uint64_t npieces = (b1 - b0 + kSrTmaChunk - 1) / kSrTmaChunk;
      const uint64_t nslots = (npieces + kSrPiecesPerSlot - 1) / kSrPiecesPerSlot;
      if (t == 32) {
        uint32_t announced = 0;
        SpinGuard g(c.timeout_ns);
        while (announced < (uint32_t)nslots) {
          uint32_t d;
          asm volatile("ld.acquire.cta.shared.u32 %0, [%1];" : "=r"(d) : "r"(smem_u32(&s_send_done)) : "memory");
          if (d > announced) {
            if (announced == 0) *reinterpret_cast<volatile uint64_t*>(peer_hdr) = kNoOff;
            st_release_sys(peer_ready, seq0 + d);
            announced = d;
          } else if (g.expired()) {
            comm_abort(c, 23, peer, (int)announced);
          }
        }
        return;
      }
      if (t != 0) return;
      for (int st = 0; st < kSrSendStages; ++st) mbar_init(&sr_sfull[st], 1);
      mbar_fence_init();
      asm volatile("fence.proxy.async;" ::: "memory");
      uint64_t issued = 0, stored = 0;
      uint32_t phase_bits = 0;
      auto publish = [&](uint64_t upto) {  // slots [0, upto) have completed at the receiver's memory system
        asm volatile("st.release.cta.shared.u32 [%0], %1;" ::"r"(smem_u32(&s_send_done)), "r"((uint32_t)upto) : "memory");
      };
      while (stored < npieces) {
        // a stage is refilled one iteration after its store was committed: wait_group.read 1 then covers that store
        // (everything but the newest group has left shared memory) without ever blocking on the store just issued
        while (issued < npieces && issued < stored + kSrSendStages - 1) {
          const int st = (int)(issued % kSrSendStages);
          if (issued >= (uint64_t)kSrSendStages) tma_store_wait_read<1>();
          const uint64_t off = b0 + issued * kSrTmaChunk;
          const uint32_t nb = (uint32_t)((b1 - off) < kSrTmaChunk ? (b1 - off) : kSrTmaChunk);
          mbar_expect_tx(&sr_sfull[st], nb);
          tma_load_1d(send_smem + (size_t)st * kSrTmaChunk, a.sbuf[peer] + off, nb, &sr_sfull[st]);
          ++issued;
        }
        const uint64_t slot_i = stored / kSrPiecesPerSlot, piece = stored % kSrPiecesPerSlot;
        const uint32_t sseq = seq0 + 1 + (uint32_t)slot_i;
        // the slot must have been drained by the receiver -- also by its kernel of the PREVIOUS message on this
        // (peer, sub-block) pair, which may still be copying out while this launch already runs: sequence numbers are global
        if (piece == 0 && sseq > (uint32_t)nslots_pair) {
          SpinGuard g(c.timeout_ns);
          while ((int32_t)(ld_acquire_sys(my_ack) - (sseq - (uint32_t)nslots_pair)) < 0) {
            if (g.expired()) comm_abort(c, 20, peer, (int)sseq);
          }
        }
        const int st = (int)(stored % kSrSendStages);
        mbar_wait(&sr_sfull[st], (phase_bits >> st) & 1u);
        phase_bits ^= 1u << st;
        const uint64_t off = b0 + stored * kSrTmaChunk;
        const uint32_t nb = (uint32_t)((b1 - off) < kSrTmaChunk ? (b1 - off) : kSrTmaChunk);
        char* dst = stage + (uint64_t)(sseq % (uint32_t)nslots_pair) * kSrChunkBytes + piece * kSrTmaChunk;
        tma_store_1d(dst, send_smem + (size_t)st * kSrTmaChunk, nb);
        tma_store_commit();
        ++stored;
        if (piece == kSrPiecesPerSlot - 1 && slot_i >= 1) {
          tma_store_wait<kSrPiecesPerSlot>();  // everything but the newest slot's pieces has completed
          publish(slot_i);
        }
      }
      tma_store_wait<0>();
      publish(nslots);
      my_flags[2 * W + peer * kSrBlocks + j] = seq0 + (uint32_t)nslots;
      return;
    }
    // ---- odd sizes: register path (partial last vector)
  } else {
    const uint64_t bytes = a.rbytes[peer];
    if (bytes == 0) return;
    const int nb = active_blocks(bytes);
    if (j >= nb) return;
    uint64_t lo, hi;
    split_range((bytes + 15) / 16, nb, j, lo, hi);
    uint32_t seq = my_flags[3 * W + peer * kSrBlocks + j];
    uint32_t* my_ready = my_flags + 0 * W + peer * kSrBlocks + j;
    uint32_t* peer_ack = flags(peer) + 1 * W + me * kSrBlocks + j;
    const uint64_t* my_hdr = hdrs(me) + peer * kSrBlocks + j;
    // first signal of the message: learn the mode
    ++seq;
    if (t == 0) {
      SpinGuard g(c.timeout_ns);
      while ((int32_t)(ld_acquire_sys(my_ready) - seq) < 0) {
        if (g.expired()) comm_abort(c, 21, peer, (int)seq);
      }
      s_hdr = *reinterpret_cast<const volatile uint64_t*>(my_hdr);
      for (int st = 0; st < kSrTmaStages; ++st) mbar_init(&sr_full[st], 1);
      mbar_fence_init();
    }
    half_sync(2);
    const uint64_t hdr = s_hdr;
    if (hdr != kNoOff) {
      // ---- zero-copy: pull my slice [lo, hi) of the peer's buffer; one elected thread runs the pipeline
      if (t == 0) {
        asm volatile("fence.proxy.async;" ::: "memory");
        const char* src = c.heap[peer] + hdr;
        char* dst = a.rbuf[peer];
        const uint64_t b0 = lo * 16, b1 = hi * 16 < bytes ? hi * 16 : bytes;
        const uint64_t total = b1 > b0 ? (b1 - b0 + kSrTmaChunk - 1) / kSrTmaChunk : 0;
        uint64_t issued = 0, stored = 0;
        uint32_t phase_bits = 0;
        while (stored < total) {
          while (issued < total && issued < stored + kSrTmaStages - 1) {  // refill lags the store by one iteration (see the send pump)
            const int st = (int)(issued % kSrTmaStages);
            if (issued >= (uint64_t)kSrTmaStages) tma_store_wait_read<1>();
            const uint64_t off = b0 + issued * kSrTmaChunk;
            const uint32_t nb = (uint32_t)((b1 - off) < kSrTmaChunk ? (b1 - off) : kSrTmaChunk);
            mbar_expect_tx(&sr_full[st], nb);
            tma_load_1d(sr_smem + (size_t)st * kSrTmaChunk, src + off, nb, &sr_full[st]);
            ++issued;
          }
          const int st = (int)(stored % kSrTmaStages);
          mbar_wait(&sr_full[st], (phase_bits >> st) & 1u);
          phase_bits ^= 1u << st;
          const uint64_t off = b0 + stored * kSrTmaChunk;
          const uint32_t nb = (uint32_t)((b1 - off) < kSrTmaChunk ? (b1 - off) : kSrTmaChunk);
          tma_store_1d(dst + off, sr_smem + (size_t)st * kSrTmaChunk, nb);
          tma_store_commit();
          ++stored;
        }
        tma_store_wait<0>();
        st_release_sys(peer_ack, seq);
        my_flags[3 * W + peer * kSrBlocks + j] = seq;
      }
      return;
    }
    // ---- staged: the sender pushed the chunks into MY slots
    const char* stage = c.heap[me] + a.sr_stage_off + ((uint64_t)(peer * kSrBlocks + j) * nslots_pair) * kSrChunkBytes;
    const uint64_t cu = kSrChunkBytes / 16;
    if (lo >= hi) {
      if (t == 0) my_flags[3 * W + peer * kSrBlocks + j] = seq;
      return;
    }
    if ((bytes % 16) == 0) {
      // ---- one elected thread: my slot -> smem -> rbuf; a slot is acked as soon as its pieces sit in smem
      if (t != 0) return;
      asm volatile("fence.proxy.async;" ::: "memory");
      const uint32_t seq0 = seq - 1;  // seq already names the first slot (its ready flag has been seen)
      const uint64_t b0 = lo * 16, b1 = hi * 16;
      const uint64_t npieces = (b1 - b0 + kSrTmaChunk - 1) / kSrTmaChunk;
      const uint64_t nslots = (npieces + kSrPiecesPerSlot - 1) / kSrPiecesPerSlot;
      uint64_t issued = 0, stored = 0, ready_slots = 1;
      uint32_t phase_bits = 0;
      char* dst = a.rbuf[peer];
      while (stored < npieces) {
        while (issued < npieces && issued < stored + kSrTmaStages - 1) {  // refill lags the store by one iteration
          const uint64_t slot_i = issued / kSrPiecesPerSlot, piece = issued % kSrPiecesPerSlot;
          if (slot_i >= ready_slots) {
            if (issued > stored) break;  // drain what is in flight before blocking on the sender
            SpinGuard g(c.timeout_ns);
            while ((int32_t)(ld_acquire_sys(my_ready) - (seq0 + 1 + (uint32_t)slot_i)) < 0) {
              if (g.expired()) comm_abort(c, 21, peer, (int)(seq0 + 1 + slot_i));
            }
            ready_slots = slot_i + 1;
            asm volatile("fence.proxy.async;" ::: "memory");
          }
          const int st = (int)(issued % kSrTmaStages);
          if (issued >= (uint64_t)kSrTmaStages) tma_store_wait_read<1>();
          const uint64_t off = b0 + issued * kSrTmaChunk;
          const uint32_t nb = (uint32_t)((b1 - off) < kSrTmaChunk ? (b1 - off) : kSrTmaChunk);
          const char* src = stage + (uint64_t)((seq0 + 1 + (uint32_t)slot_i) % (uint32_t)nslots_pair) * kSrChunkBytes + piece * kSrTmaChunk;
          mbar_expect_tx(&sr_full[st], nb);
          tma_load_1d(sr_smem + (size_t)st * kSrTmaChunk, src, nb, &sr_full[st]);
          ++issued;
        }
        const int st = (int)(stored % kSrTmaStages);
        mbar_wait(&sr_full[st], (phase_bits >> st) & 1u);
        phase_bits ^= 1u << st;
        const uint64_t off = b0 + stored * kSrTmaChunk;
        const uint32_t nb = (uint32_t)((b1 - off) < kSrTmaChunk ? (b1 - off) : kSrTmaChunk);
        tma_store_1d(dst + off, sr_smem + (size_t)st * kSrTmaChunk, nb);
        tma_store_commit();
        const uint64_t slot_i = stored / kSrPiecesPerSlot;
        ++stored;
        // last piece of a slot has left the slot (it is in shared memory): hand the slot back
        // (relaxed: the slot's bytes already sit in shared memory -- the mbarrier waits above -- nothing to order)
        if (stored % kSrPiecesPerSlot == 0 || stored == npieces) st_relaxed_sys(peer_ack, seq0 + 1 + (uint32_t)slot_i);
      }
      tma_store_wait<0>();
      my_flags[3 * W + peer * kSrBlocks + j] = seq0 + (uint32_t)nslots;
      return;
    }
    // ---- odd sizes: register path
    bool first = true;
    for (uint64_t u0 = lo; u0 < hi; u0 += cu) {
      const uint64_t u1 = (u0 + cu < hi) ? u0 + cu : hi;
      if (!first) {
        ++seq;
        if (t == 0) {
          SpinGuard g(c.timeout_ns);
          while ((int32_t)(ld_acquire_sys(my_ready) - seq) < 0) {
            if (g.expired()) comm_abort(c, 21, peer, (int)seq);
          }
        }
        half_sync(2);
      }
      first = false;
      const char* slot = stage + (uint64_t)(seq % (uint32_t)nslots_pair) * kSrChunkBytes;
      constexpr int B = 8;
      for (uint64_t ub = u0; ub < u1; ub += (uint64_t)B * 256) {
        uint4 v[B];
#pragma unroll
        for (int q = 0; q < B; ++q) {
          const uint64_t u = ub + (uint64_t)q * 256 + t;
          if (u < u1) v[q] = ld_v4(slot + (u - u0) * 16);
        }
#pragma unroll
        for (int q = 0; q < B; ++q) {
          const uint64_t u = ub + (uint64_t)q * 256 + t;
          if (u < u1) store16_partial(a.rbuf[peer], u * 16, bytes, v[q]);
        }
      }
      half_sync(2);
      if (t == 0) st_release_sys(peer_ack, seq);
    }
    if (t == 0) my_flags[3 * W + peer * kSrBlocks + j] = seq;
  }
}
}  // namespace ub
