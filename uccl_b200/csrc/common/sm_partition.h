// SM partitions: a fixed set of SMs carved out of a GPU as a CUDA green context, plus streams bound to it.
//
// Why it exists here: the communication kernels of this library run on an SM budget (the expert-parallel kernels on
// 24 of the 132 SMs of an H100, like the reference's DeepEP configuration), but a budget expressed as a grid size only limits how
// many CTAs the kernel brings -- not WHERE they land, and a GEMM launched first can leave them queued behind its waves.
// A partition makes the budget physical: kernels launched on a partition's stream only ever occupy that partition's
// SMs, and the complementary partition keeps compute off them.  The reference probes the same mechanism as a
// stand-alone experiment (experimental/misc/cuda_greenctx.cu: split, create, list the SM ids a kernel lands on).
//
// Contract for this library's kernels: they synchronise CTAs of one launch with each other (and with the same CTA
// index on peer GPUs), so every CTA of a launch must be resident at once -- keep the kernel's SM budget
// (Buffer.set_num_sms, Communicator max_ctas) at or below sm_count() of the partition it is launched on.
#pragma once
#include <cuda_runtime.h>

#include <memory>
#include <mutex>
#include <string>
#include <vector>

namespace ub {

class SmPartition {
 public:
  struct Pair {
    std::shared_ptr<SmPartition> part;  // >= the requested SM count (rounded up to the device's granularity)
    std::shared_ptr<SmPartition> rest;  // every other SM of the device; null when nothing is left
  };
  // false (and a reason) where the driver has no green contexts or no device is usable
  static bool supported(int device, std::string* why = nullptr);
  // SM count of the whole device as the partitioning API sees it
  static int device_sm_count(int device);
  // Splits `device` into a partition of at least `sm_count` SMs and the rest.  `fine_grained` lowers the granularity
  // (2 SMs instead of 8 on sm_90+) at the cost of large thread-block clusters inside the partition.
  static Pair split(int device, int sm_count, bool fine_grained = false);

  ~SmPartition();
  SmPartition(const SmPartition&) = delete;
  SmPartition& operator=(const SmPartition&) = delete;

  int device() const { return device_; }
  int sm_count() const { return sm_count_; }
  // a non-blocking stream whose kernels run on this partition's SMs only; created on first use per priority and
  // owned by the partition (valid until it is destroyed)
  cudaStream_t stream(int priority = 0);

 private:
  SmPartition() = default;
  static std::shared_ptr<SmPartition> make(int device, void* resource);
  int device_ = 0;
  int sm_count_ = 0;
  void* green_ = nullptr;  // CUgreenCtx
  std::mutex mu_;
  std::vector<std::pair<int, cudaStream_t>> streams_;
};

}  // namespace ub
