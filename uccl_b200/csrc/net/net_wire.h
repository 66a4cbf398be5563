// Wire format of the inter-node datagram transport (uccl_b200::net).
//
// Role in the reference: the UCCL-Tran packet formats -- `IMMData{FID,RID,CSN,HINT}` + the ACK/SACK
// control header of the RDMA transport (collective/rdma/transport.h:122, transport_header.h) and the
// `ucclh`/`ucclsackh` headers of the AF_XDP / DPDK / EFA transports.  Inside one NVSwitch node none of
// this is needed (peers are load/store reachable); this is the scale-OUT path between H100 boxes.
//
// One datagram = PktHdr (+ type specific body) (+ payload).  All fields little endian (x86-64 / aarch64
// hosts of H100 systems are both LE).  A flow is bidirectional; each direction numbers its reliable
// packets independently.
#pragma once
#include <cstdint>

namespace ub {
namespace net {

constexpr uint32_t kMagic = 0x4e324255u;  // "UB2N"
constexpr int kMaxPaths = 32;             // UDP source ports per engine ("paths": ECMP entropy)
constexpr int kSackWords = 4;
constexpr int kSackBits = 64 * kSackWords;  // receive window / SACK span in packets
constexpr int kTxRing = 2 * kSackBits;      // in-flight descriptor ring (power of two)

enum PktType : uint8_t {
  PKT_SYN = 1,     // connect request (unsequenced, retried by the client)
  PKT_SYNACK = 2,  // connect reply
  PKT_DATA = 3,    // sequenced, reliable; carries exactly one frame
  PKT_ACK = 4,     // unsequenced; cumulative ack + SACK bitmap + timestamp echo + credit
  PKT_RST = 5,     // "no such flow" / aborted
};

enum FrameKind : uint8_t {
  FR_MSG = 1,  // a slice of message `msg_id`: bytes [offset, offset+len) of msg_len
  FR_RTR = 2,  // receiver -> sender: "recvs [0, msg_id) are posted" (rendezvous credit for large messages)
  FR_FIN = 3,  // orderly close of this direction
};

struct PktHdr {
  uint32_t magic;
  uint8_t type;      // PktType
  uint8_t kind;      // FrameKind (DATA only)
  uint16_t path;     // index of the path this datagram was sent on
  uint32_t dst_flow; // flow id at the destination (0 in SYN)
  uint32_t seq;      // DATA: packet sequence number.  ACK: cumulative ack = next sequence expected
  uint64_t ts_ns;    // DATA: sender clock at (re)transmission.  ACK: echo of the newest DATA timestamp seen
  uint32_t msg_id;   // MSG: message index.  RTR and ACK: number of receives posted so far
  uint32_t len;      // payload bytes after the header (MSG) / body bytes (SYN, ACK)
  uint64_t offset;   // MSG: byte offset of this slice
  uint64_t msg_len;  // MSG: total message length
  uint64_t aux;      // DATA: sender backlog in bytes (EQDS demand).  ACK: cumulative credit granted (bytes)
};
static_assert(sizeof(PktHdr) == 56, "PktHdr layout");

struct AckBody {
  uint64_t sack[kSackWords];  // bit i <=> packet (ack + i) has been received (bit 0 is always 0)
  uint16_t echo_path;         // path of the DATA packet whose timestamp is echoed
  uint16_t reserved;
  uint32_t dup_cum;           // duplicates this receiver has seen so far (low 32 bits): the sender's spurious-rexmit signal
};

struct SynBody {
  uint64_t nonce;      // identifies the connect attempt (duplicate SYNs map to the same flow)
  uint32_t src_flow;   // sender's flow id: what the peer must put into dst_flow
  uint32_t listen_id;  // SYN: which listener at the destination
  uint16_t npaths;
  uint16_t ports[kMaxPaths];  // network byte order UDP ports of the sender's paths
  uint16_t pad[3];
};

}  // namespace net
}  // namespace ub
