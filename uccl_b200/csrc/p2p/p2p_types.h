// Host-safe structs of the P2P copy kernel and wire descriptors.
#pragma once
#include <stdint.h>

namespace ub {

constexpr int kP2PStages = 3;        // bulk loads in flight per warp pipeline
constexpr int kP2PWarps = 4;         // independent TMA pipelines per CTA (one elected lane each)
constexpr int kP2PMaxEntries = 64;   // entries that travel in the kernel parameters
constexpr int kP2PTableEntries = 8192;  // entries of one pinned descriptor table (larger batches: several launches)

struct P2PCopyEntry {
  const char* src;
  char* dst;
  uint64_t bytes;
  uint64_t bulk_bytes;  // 16-byte aligned prefix moved by TMA (0 if src/dst are not 16-byte aligned)
};

struct P2PCopyBatch {
  P2PCopyEntry e[kP2PMaxEntries];
  uint32_t chunk_prefix[kP2PMaxEntries + 1];  // exclusive prefix of per-entry bulk chunk counts
  int n;
  uint32_t chunk_bytes;
  // n > kP2PMaxEntries: the descriptors live in a DEVICE table instead (filled through a pinned staging copy; a
  // first version let the kernel read the pinned table itself and paid a PCIe round trip per block); one launch moves thousands of KV blocks.  `table_prefix` has n + 1 words
  const P2PCopyEntry* table;
  const uint32_t* table_prefix;
  int any_tail;  // some entry is not a 16-byte multiple / aligned: the non-issuing lanes copy those bytes
};

// A registered/advertised memory window, shipped between endpoints (128 bytes on the wire).
// Role of the reference's FifoItem / IpcTransferInfo (p2p/include/common.h:40-49, p2p/engine.h:82-90).
struct XferDesc {
  unsigned char ipc_handle[64];  // cudaIpcMemHandle_t of the allocation base
  uint64_t base;                 // allocation base VA in the owner process
  uint64_t addr;                 // window start VA in the owner process
  uint64_t size;                 // window bytes
  int32_t pid;                   // owner process
  int32_t dev;                   // owner CUDA device
  uint32_t kind;                 // 0 = CUDA IPC, 1 = pinned host (same process only), 2 = same-process device ptr
  uint32_t mr_id;
  uint64_t host_id;              // which machine owns the window (0 = unknown / legacy): other hosts use the wire
  unsigned char pad[16];
};
static_assert(sizeof(XferDesc) == 128, "XferDesc must be 128 bytes");

}  // namespace ub
