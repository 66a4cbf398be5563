// Host ("fake GPU") backend of the communicator: the same symmetric-heap protocol
// (epoch barriers in shared memory + peers reading each other's staging area), run
// by CPU threads/processes over POSIX shm or malloc heaps.  It exists so that the
// control plane (bootstrap, heap layout, allocator, barrier protocol, argument
// checking, NCCL shim, Python bindings) is exercised by CI on GPU-less machines;
// the pattern follows ukernel's MockBackend idea
// (experimental/ukernel/src/ccl/test/common/backend_test_utils.h:211).
#include <sched.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <vector>

#include "../common/log.h"
#include "comm.h"

namespace ub {

namespace {

inline float bf16_to_f32(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
inline uint16_t f32_to_bf16(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
  uint32_t lsb = (u >> 16) & 1u;
  u += 0x7fffu + lsb;
  return (uint16_t)(u >> 16);
}
inline float f16_to_f32(uint16_t h) {
  uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
  uint32_t exp = (h >> 10) & 0x1fu, man = h & 0x3ffu;
  uint32_t u;
  if (exp == 0) {
    if (man == 0) u = sign;
    else {
      int e = -1;
      do {
        ++e;
        man <<= 1;
      } while (!(man & 0x400u));
      u = sign | ((uint32_t)(127 - 15 - e) << 23) | ((man & 0x3ffu) << 13);
    }
  } else if (exp == 31) {
    u = sign | 0x7f800000u | (man << 13);
  } else {
    u = sign | ((exp + 112) << 23) | (man << 13);
  }
  float f;
  memcpy(&f, &u, 4);
  return f;
}
inline uint16_t f32_to_f16(float f) {
  uint32_t x;
  memcpy(&x, &f, 4);
  uint32_t sign = (x >> 16) & 0x8000u;
  int32_t exp = (int32_t)((x >> 23) & 0xff) - 127 + 15;
  uint32_t man = x & 0x7fffffu;
  if (((x >> 23) & 0xff) == 0xff) return (uint16_t)(sign | 0x7c00u | (man ? 0x200u : 0));
  if (exp >= 31) return (uint16_t)(sign | 0x7c00u);
  if (exp <= 0) {
    if (exp < -10) return (uint16_t)sign;
    man |= 0x800000u;
    uint32_t shift = (uint32_t)(14 - exp);
    uint32_t half = man >> shift;
    uint32_t rem = man & ((1u << shift) - 1), halfway = 1u << (shift - 1);
    if (rem > halfway || (rem == halfway && (half & 1))) ++half;
    return (uint16_t)(sign | half);
  }
  uint32_t half = ((uint32_t)exp << 10) | (man >> 13);
  uint32_t rem = man & 0x1fffu;
  if (rem > 0x1000u || (rem == 0x1000u && (half & 1))) ++half;
  return (uint16_t)(sign | half);
}

template <typename A>
inline A apply(int op, A a, A b) {
  switch (op) {
    case kSum: case kAvg: return a + b;
    case kProd: return a * b;
    case kMax: return a > b ? a : b;
    default: return a < b ? a : b;
  }
}

// dst[i] = op over r of srcs[r][i]  (count elements of dtype), then scale / int-average
void reduce_n(void* dst, const void* const* srcs, int n, size_t count, int dtype, int op, float scale) {
  auto loop = [&](auto load, auto store, auto acc_zero, bool is_float) {
    using A = decltype(acc_zero);
    for (size_t i = 0; i < count; ++i) {
      A acc = load(srcs[0], i);
      for (int r = 1; r < n; ++r) acc = apply<A>(op, acc, load(srcs[r], i));
      if (is_float) {
        if (scale != 1.0f) acc = (A)(acc * (A)scale);
      } else if (op == kAvg) {
        acc = (A)(acc / (A)n);
      }
      store(dst, i, acc);
    }
  };
#define UB_PLAIN(T, FL)                                                                         \
  loop([](const void* p, size_t i) { return ((const T*)p)[i]; },                                \
       [](void* p, size_t i, T v) { ((T*)p)[i] = v; }, (T)0, FL)
  switch (dtype) {
    case kI8: UB_PLAIN(int8_t, false); break;
    case kU8: UB_PLAIN(uint8_t, false); break;
    case kI32: UB_PLAIN(int32_t, false); break;
    case kU32: UB_PLAIN(uint32_t, false); break;
    case kI64: UB_PLAIN(int64_t, false); break;
    case kU64: UB_PLAIN(uint64_t, false); break;
    case kF32: UB_PLAIN(float, true); break;
    case kF64: UB_PLAIN(double, true); break;
    case kBF16:
      loop([](const void* p, size_t i) { return bf16_to_f32(((const uint16_t*)p)[i]); },
           [](void* p, size_t i, float v) { ((uint16_t*)p)[i] = f32_to_bf16(v); }, 0.0f, true);
      break;
    case kF16:
      loop([](const void* p, size_t i) { return f16_to_f32(((const uint16_t*)p)[i]); },
           [](void* p, size_t i, float v) { ((uint16_t*)p)[i] = f32_to_f16(v); }, 0.0f, true);
      break;
    default: UB_THROW("host backend: dtype %d unsupported", dtype);
  }
#undef UB_PLAIN
}

// float family with a different output type: accumulate in fp32 over the ranks, round once
// (same arithmetic as the fused-cast epilogue of the CUDA kernels)
void reduce_n_cast(void* dst, const void* const* srcs, int n, size_t count, int in_dtype, int out_dtype, int op,
                   float scale) {
  auto load = [&](const void* p, size_t i) -> float {
    switch (in_dtype) {
      case kF32: return ((const float*)p)[i];
      case kBF16: return bf16_to_f32(((const uint16_t*)p)[i]);
      default: return f16_to_f32(((const uint16_t*)p)[i]);
    }
  };
  for (size_t i = 0; i < count; ++i) {
    float acc = load(srcs[0], i);
    for (int r = 1; r < n; ++r) acc = apply<float>(op, acc, load(srcs[r], i));
    if (scale != 1.0f) acc *= scale;
    switch (out_dtype) {
      case kF32: ((float*)dst)[i] = acc; break;
      case kBF16: ((uint16_t*)dst)[i] = f32_to_bf16(acc); break;
      default: ((uint16_t*)dst)[i] = f32_to_f16(acc); break;
    }
  }
}

}  // namespace

namespace {
// Two-source, unscaled reductions are the inner loop of every inter-box ring step (MultiComm::rail_*): the
// operator is a template parameter so that the compiler vectorises the loop (the generic reduce_n switches on
// `op` per element).  dst may alias a.
template <typename T, int OP>
void reduce2_plain(T* __restrict__ dst, const T* a, const T* __restrict__ b, size_t n) {
#pragma GCC ivdep
  for (size_t i = 0; i < n; ++i) {
    const T x = a[i], y = b[i];
    dst[i] = OP == kSum ? (T)(x + y) : OP == kProd ? (T)(x * y) : OP == kMax ? (x > y ? x : y) : (x < y ? x : y);
  }
}
template <int OP>
void reduce2_bf16(uint16_t* __restrict__ dst, const uint16_t* a, const uint16_t* __restrict__ b, size_t n) {
#pragma GCC ivdep
  for (size_t i = 0; i < n; ++i) {
    const float x = bf16_to_f32(a[i]), y = bf16_to_f32(b[i]);
    dst[i] = f32_to_bf16(OP == kSum ? x + y : OP == kProd ? x * y : OP == kMax ? (x > y ? x : y) : (x < y ? x : y));
  }
}
template <typename T>
bool reduce2_dispatch(T* dst, const T* a, const T* b, size_t n, int op) {
  switch (op) {
    case kSum: reduce2_plain<T, kSum>(dst, a, b, n); return true;
    case kProd: reduce2_plain<T, kProd>(dst, a, b, n); return true;
    case kMax: reduce2_plain<T, kMax>(dst, a, b, n); return true;
    case kMin: reduce2_plain<T, kMin>(dst, a, b, n); return true;
    default: return false;
  }
}
bool reduce2_fast(void* dst, const void* a, const void* b, size_t n, int dtype, int op) {
  switch (dtype) {
    case kF32: return reduce2_dispatch((float*)dst, (const float*)a, (const float*)b, n, op);
    case kF64: return reduce2_dispatch((double*)dst, (const double*)a, (const double*)b, n, op);
    case kI32: return reduce2_dispatch((int32_t*)dst, (const int32_t*)a, (const int32_t*)b, n, op);
    case kU32: return reduce2_dispatch((uint32_t*)dst, (const uint32_t*)a, (const uint32_t*)b, n, op);
    case kI64: return reduce2_dispatch((int64_t*)dst, (const int64_t*)a, (const int64_t*)b, n, op);
    case kU64: return reduce2_dispatch((uint64_t*)dst, (const uint64_t*)a, (const uint64_t*)b, n, op);
    case kBF16:
      switch (op) {
        case kSum: reduce2_bf16<kSum>((uint16_t*)dst, (const uint16_t*)a, (const uint16_t*)b, n); return true;
        case kMax: reduce2_bf16<kMax>((uint16_t*)dst, (const uint16_t*)a, (const uint16_t*)b, n); return true;
        case kMin: reduce2_bf16<kMin>((uint16_t*)dst, (const uint16_t*)a, (const uint16_t*)b, n); return true;
        default: return false;
      }
    default: return false;
  }
}
}  // namespace

void host_reduce_n(void* dst, const void* const* srcs, int n, size_t count, int dtype, int op, float scale) {
  if (n == 2 && scale == 1.0f && reduce2_fast(dst, srcs[0], srcs[1], count, dtype, op)) return;
  reduce_n(dst, srcs, n, count, dtype, op, scale);
}

namespace {
// fp32 -> e4m3 (finite-only format, max 448): round to nearest even, saturating like the device conversion
uint8_t f32_to_e4m3(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  const uint8_t sign = (uint8_t)((u >> 24) & 0x80u);
  const float a = std::fabs(f);
  if (std::isnan(f)) return sign | 0x7f;
  if (a >= 448.0f) return sign | 0x7e;
  if (a < 0.015625f) return sign | (uint8_t)std::nearbyint(a * 512.0f);  // subnormals: multiples of 2^-9
  int e = (int)((u >> 23) & 0xff) - 127;                                  // -6 .. 8
  int q = (int)std::nearbyint(std::ldexp(a, 3 - e));                       // 8 .. 16
  if (q == 16) {
    q = 8;
    ++e;
  }
  return sign | (uint8_t)(((e + 7) << 3) | (q - 8));
}
}  // namespace

void host_add_rmsnorm(const void* x, const void* residual, void* residual_out, const void* weight, void* out,
                      float* out_scales, size_t T, size_t H, int dtype, float eps) {
  const bool bf = dtype == kBF16;
  auto ld = [bf](const void* p, size_t i) {
    const uint16_t h = static_cast<const uint16_t*>(p)[i];
    return bf ? bf16_to_f32(h) : f16_to_f32(h);
  };
  auto rnd = [bf](float v) { return bf ? f32_to_bf16(v) : f32_to_f16(v); };
  std::vector<float> r(H), y(H);
  for (size_t t = 0; t < T; ++t) {
    const size_t o = t * H;
    float ss = 0.f;
    for (size_t i = 0; i < H; ++i) {  // read the whole row first: residual_out may alias residual
      const uint16_t h = rnd(ld(x, o + i) + ld(residual, o + i));
      r[i] = bf ? bf16_to_f32(h) : f16_to_f32(h);
      ss += r[i] * r[i];
    }
    for (size_t i = 0; i < H; ++i) static_cast<uint16_t*>(residual_out)[o + i] = rnd(r[i]);
    const float inv = 1.0f / std::sqrt(ss / (float)H + eps);
    for (size_t i = 0; i < H; ++i) {
      const uint16_t h = rnd(r[i] * inv * ld(weight, i));
      if (!out_scales) static_cast<uint16_t*>(out)[o + i] = h;
      y[i] = bf ? bf16_to_f32(h) : f16_to_f32(h);
    }
    if (!out_scales) continue;
    for (size_t g = 0; g < H / 128; ++g) {
      float amax = 0.f;
      for (size_t i = 0; i < 128; ++i) amax = std::max(amax, std::fabs(y[g * 128 + i]));
      amax = std::max(amax, 1e-4f);
      const float scale = (1.0f / amax) * 448.0f;  // rounded like per_token_cast_to_fp8 (see fp8_quant.cuh)
      out_scales[t * (H / 128) + g] = amax / 448.0f;
      for (size_t i = 0; i < 128; ++i) static_cast<uint8_t*>(out)[o + g * 128 + i] = f32_to_e4m3(y[g * 128 + i] * scale);
    }
  }
}

void Comm::host_barrier() {
  const int n = nranks(), me = rank();
  ++host_epoch_;
  const uint32_t e = host_epoch_;
  const uint64_t off = layout_.sig_off + ((uint64_t)kDomColl * kMaxSyncBlocks + 0) * kMaxRanks * sizeof(uint32_t);
  for (int p = 0; p < n; ++p) {
    if (p == me) continue;
    uint32_t* slot = reinterpret_cast<uint32_t*>(fabric_->heap(p) + off) + me;
    __atomic_store_n(slot, e, __ATOMIC_RELEASE);
  }
  auto t0 = std::chrono::steady_clock::now();
  for (int p = 0; p < n; ++p) {
    if (p == me) continue;
    uint32_t* slot = reinterpret_cast<uint32_t*>(fabric_->local() + off) + p;
    uint32_t spins = 0;
    while ((int32_t)(__atomic_load_n(slot, __ATOMIC_ACQUIRE) - e) < 0) {
      if ((++spins & 0xff) == 0) {
        sched_yield();
        if (dev_.timeout_ns) {
          auto dt = std::chrono::steady_clock::now() - t0;
          if ((uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(dt).count() > dev_.timeout_ns)
            UB_THROW("host barrier timeout: rank %d waiting for rank %d (epoch %u)", me, p, e);
        }
      }
    }
  }
}

// All host collectives: copy my input into my stage (chunked), barrier, read peers' stages.
void Comm::host_allreduce(const void* in, void* out, size_t count, int dtype, int op, float scale, int out_dtype) {
  const int n = nranks(), me = rank();
  const size_t es = dtype_size(dtype);
  const size_t eo = dtype_size(out_dtype);
  const bool cast = out_dtype != dtype;
  if (cast) {
    auto fl = [](int d) { return d == kF32 || d == kBF16 || d == kF16; };
    UB_CHECK(fl(dtype) && fl(out_dtype), "host backend: fused cast only between fp32 / bf16 / fp16");
  }
  const size_t chunk_elems = layout_.stage_bytes / std::max(es, eo);
  for (size_t base = 0; base < count; base += chunk_elems) {
    const size_t c = std::min(chunk_elems, count - base);
    memcpy(fabric_->local() + layout_.stage_in_off, (const char*)in + base * es, c * es);
    host_barrier();
    // two-shot: reduce my shard into my stage_out, then gather all shards
    uint64_t lo, hi;
    split_range(c, n, me, lo, hi);
    const void* srcs[kMaxRanks];
    for (int r = 0; r < n; ++r) srcs[r] = fabric_->heap(r) + layout_.stage_in_off + lo * es;
    if (cast) reduce_n_cast(fabric_->local() + layout_.stage_out_off + lo * eo, srcs, n, hi - lo, dtype, out_dtype, op, scale);
    else reduce_n(fabric_->local() + layout_.stage_out_off + lo * es, srcs, n, hi - lo, dtype, op, scale);
    host_barrier();
    for (int r = 0; r < n; ++r) {
      uint64_t l2, h2;
      split_range(c, n, r, l2, h2);
      memcpy((char*)out + (base + l2) * eo, fabric_->heap(r) + layout_.stage_out_off + l2 * eo, (h2 - l2) * eo);
    }
    host_barrier();
  }
}

void Comm::host_allgather(const void* in, void* out, size_t bytes) {
  const int n = nranks();
  const size_t chunk = layout_.stage_bytes;
  for (size_t base = 0; base < bytes; base += chunk) {
    const size_t c = std::min(chunk, bytes - base);
    memcpy(fabric_->local() + layout_.stage_in_off, (const char*)in + base, c);
    host_barrier();
    for (int r = 0; r < n; ++r)
      memcpy((char*)out + (size_t)r * bytes + base, fabric_->heap(r) + layout_.stage_in_off, c);
    host_barrier();
  }
}

void Comm::host_reduce_scatter(const void* in, void* out, size_t count, int dtype, int op) {
  const int n = nranks(), me = rank();
  const size_t es = dtype_size(dtype);
  const size_t chunk_elems = layout_.stage_bytes / n / es;
  const float scale = (op == kAvg) ? 1.0f / (float)n : 1.0f;
  for (size_t base = 0; base < count; base += chunk_elems) {
    const size_t c = std::min(chunk_elems, count - base);
    for (int d = 0; d < n; ++d)
      memcpy(fabric_->local() + layout_.stage_in_off + (size_t)d * chunk_elems * es,
             (const char*)in + ((size_t)d * count + base) * es, c * es);
    host_barrier();
    const void* srcs[kMaxRanks];
    for (int r = 0; r < n; ++r) srcs[r] = fabric_->heap(r) + layout_.stage_in_off + (size_t)me * chunk_elems * es;
    reduce_n((char*)out + base * es, srcs, n, c, dtype, op, scale);
    host_barrier();
  }
}

void Comm::host_broadcast(const void* in, void* out, size_t bytes, int root) {
  const size_t chunk = layout_.stage_bytes;
  for (size_t base = 0; base < bytes; base += chunk) {
    const size_t c = std::min(chunk, bytes - base);
    if (rank() == root) memcpy(fabric_->local() + layout_.stage_in_off, (const char*)in + base, c);
    host_barrier();
    if (rank() != root) memcpy((char*)out + base, fabric_->heap(root) + layout_.stage_in_off, c);
    else if (in != out) memcpy((char*)out + base, (const char*)in + base, c);
    host_barrier();
  }
}

void Comm::host_reduce(const void* in, void* out, size_t count, int dtype, int op, int root) {
  const int n = nranks();
  const size_t es = dtype_size(dtype);
  const size_t chunk_elems = layout_.stage_bytes / es;
  const float scale = (op == kAvg) ? 1.0f / (float)n : 1.0f;
  for (size_t base = 0; base < count; base += chunk_elems) {
    const size_t c = std::min(chunk_elems, count - base);
    memcpy(fabric_->local() + layout_.stage_in_off, (const char*)in + base * es, c * es);
    host_barrier();
    if (rank() == root) {
      const void* srcs[kMaxRanks];
      for (int r = 0; r < n; ++r) srcs[r] = fabric_->heap(r) + layout_.stage_in_off;
      reduce_n((char*)out + base * es, srcs, n, c, dtype, op, scale);
    }
    host_barrier();
  }
}

void Comm::host_alltoall(const void* in, void* out, size_t bytes) {
  const int n = nranks(), me = rank();
  const size_t chunk = layout_.stage_bytes / n;
  for (size_t base = 0; base < bytes; base += chunk) {
    const size_t c = std::min(chunk, bytes - base);
    for (int d = 0; d < n; ++d)
      memcpy(fabric_->local() + layout_.stage_in_off + (size_t)d * chunk, (const char*)in + (size_t)d * bytes + base, c);
    host_barrier();
    for (int r = 0; r < n; ++r)
      memcpy((char*)out + (size_t)r * bytes + base, fabric_->heap(r) + layout_.stage_in_off + (size_t)me * chunk, c);
    host_barrier();
  }
}

// Variable-size all-to-all: rounds of (stage one slice per destination, barrier, read my slice from
// every peer's stage, barrier).  The number of rounds is not known locally (a rank only knows its own
// counts), so every rank publishes a "more data after this round" flag next to its stage and all ranks
// continue while anybody's flag is set -- they all read the same flags, hence run the same rounds.
void Comm::host_alltoallv(const void* in, const size_t* send_bytes, const size_t* send_off, void* out,
                          const size_t* recv_bytes, const size_t* recv_off) {
  const int n = nranks(), me = rank();
  const size_t chunk = (layout_.stage_bytes / n) / 16 * 16;
  UB_CHECK(chunk > 0, "host alltoallv: staging area too small");
  for (size_t base = 0;; base += chunk) {
    bool more = false;
    for (int d = 0; d < n; ++d) {
      if (send_bytes[d] > base) {
        const size_t c = std::min(chunk, send_bytes[d] - base);
        memcpy(fabric_->local() + layout_.stage_in_off + (size_t)d * chunk, (const char*)in + send_off[d] + base, c);
        more = more || send_bytes[d] > base + chunk;
      }
      more = more || recv_bytes[d] > base + chunk;
    }
    __atomic_store_n(reinterpret_cast<uint32_t*>(fabric_->local() + layout_.stage_out_off), more ? 1u : 0u,
                     __ATOMIC_RELEASE);
    host_barrier();
    bool any_more = false;
    for (int r = 0; r < n; ++r) {
      if (recv_bytes[r] > base) {
        const size_t c = std::min(chunk, recv_bytes[r] - base);
        memcpy((char*)out + recv_off[r] + base, fabric_->heap(r) + layout_.stage_in_off + (size_t)me * chunk, c);
      }
      any_more = any_more ||
                 __atomic_load_n(reinterpret_cast<uint32_t*>(fabric_->heap(r) + layout_.stage_out_off), __ATOMIC_ACQUIRE);
    }
    host_barrier();
    if (!any_more) break;
  }
}

// Grouped point-to-point on the host backend.  Every ordered pair (src -> dst) owns a mailbox in the
// *destination's* heap (inside the send/recv staging area): {ready seq, acked seq, chunk}.  The sender
// fills the chunk when the previous one has been acknowledged and publishes its sequence number; the
// receiver copies the chunk out and acknowledges.  One rank usually has sends and receives in the same
// group (ring step, all-to-all pattern), so all of its operations are progressed round-robin -- nothing
// blocks on a single peer.  Only the two ranks of a pair synchronise (no global barrier), like the
// send/recv kernel of the CUDA backend.
void Comm::host_group_p2p(const std::vector<P2pOp>& ops) {
  const int n = nranks(), me = rank();
  const uint64_t box_bytes = kSrStageBytes / kMaxRanks;  // data area per source rank
  const uint64_t chunk = box_bytes;
  struct Prog {
    const P2pOp* op;
    size_t done = 0;
  };
  // operations towards one peer complete in posting order
  std::vector<std::vector<Prog>> sends(n), recvs(n);
  for (const auto& o : ops) {
    UB_CHECK(o.peer >= 0 && o.peer < n, "send/recv: bad peer %d", o.peer);
    (o.is_send ? sends : recvs)[o.peer].push_back(Prog{&o, 0});
  }
  if (host_send_seq_.empty()) {
    host_send_seq_.assign(n, 0);
    host_recv_seq_.assign(n, 0);
  }
  auto box = [&](int dst, int src) { return fabric_->heap(dst) + layout_.sr_stage_off + (uint64_t)src * box_bytes; };
  // {ready, acked} of the pair live in the flag area, which is part of the zero-initialised control region
  auto flags = [&](int dst, int src) {
    return reinterpret_cast<uint64_t*>(fabric_->heap(dst) + layout_.sr_flag_off) + (uint64_t)src * 2;
  };
  std::vector<size_t> si(n, 0), ri(n, 0);  // index of the operation in progress per peer
  auto t0 = std::chrono::steady_clock::now();
  uint32_t idle = 0;
  while (true) {
    bool pending = false, progressed = false;
    for (int p = 0; p < n; ++p) {
      // skip zero-byte operations
      while (si[p] < sends[p].size() && sends[p][si[p]].op->bytes == 0) ++si[p];
      while (ri[p] < recvs[p].size() && recvs[p][ri[p]].op->bytes == 0) ++ri[p];
      if (si[p] < sends[p].size()) {
        pending = true;
        Prog& s = sends[p][si[p]];
        char* b = box(p, me);
        uint64_t* ready = flags(p, me);
        uint64_t* acked = flags(p, me) + 1;
        if (__atomic_load_n(acked, __ATOMIC_ACQUIRE) == host_send_seq_[p]) {  // mailbox free
          const size_t c = std::min<size_t>(chunk, s.op->bytes - s.done);
          memcpy(b, (const char*)s.op->buf + s.done, c);
          __atomic_store_n(ready, ++host_send_seq_[p], __ATOMIC_RELEASE);
          s.done += c;
          if (s.done == s.op->bytes) ++si[p];
          progressed = true;
        }
      }
      if (ri[p] < recvs[p].size()) {
        pending = true;
        Prog& r = recvs[p][ri[p]];
        char* b = box(me, p);
        uint64_t* ready = flags(me, p);
        uint64_t* acked = flags(me, p) + 1;
        if (__atomic_load_n(ready, __ATOMIC_ACQUIRE) == host_recv_seq_[p] + 1) {
          const size_t c = std::min<size_t>(chunk, r.op->bytes - r.done);
          memcpy((char*)r.op->buf + r.done, b, c);
          __atomic_store_n(acked, ++host_recv_seq_[p], __ATOMIC_RELEASE);
          r.done += c;
          if (r.done == r.op->bytes) ++ri[p];
          progressed = true;
        }
      }
    }
    if (!pending) break;
    if (progressed) {
      idle = 0;
      continue;
    }
    if ((++idle & 0xff) == 0) {
      sched_yield();
      if (dev_.timeout_ns) {
        auto dt = std::chrono::steady_clock::now() - t0;
        if ((uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(dt).count() > dev_.timeout_ns)
          UB_THROW("host send/recv timeout on rank %d (a peer did not post the matching operation)", me);
      }
    }
  }
  // my last chunks must be consumed before the buffers may be reused: wait for the acknowledgements
  for (int p = 0; p < n; ++p) {
    if (sends[p].empty()) continue;
    uint64_t* acked = flags(p, me) + 1;
    uint32_t spins = 0;
    while (__atomic_load_n(acked, __ATOMIC_ACQUIRE) != host_send_seq_[p]) {
      if ((++spins & 0xff) == 0) {
        sched_yield();
        if (dev_.timeout_ns) {
          auto dt = std::chrono::steady_clock::now() - t0;
          if ((uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(dt).count() > dev_.timeout_ns)
            UB_THROW("host send/recv timeout on rank %d waiting for rank %d to drain", me, p);
        }
      }
    }
  }
}

}  // namespace ub
