// uccl_b200::net -- software multipath reliable datagram transport between nodes.
//
// What the reference builds for scale-out (SURVEY N2 "UCCL-Tran", N6 AF_XDP, N7 DPDK, N5 EFA): messages
// are cut into chunks, every chunk is sprayed over one of P paths picked by power-of-two choices, the
// receiver places chunks at their final offset as they arrive (no reorder buffer), and reliability is
// software: cumulative ACK + SACK bitmap, RACK-style fast retransmit, RTO with backoff and abort, and a
// pluggable congestion controller (Swift window, Timely rate pacing, EQDS receiver credits from
// csrc/common/cc).  Reference: collective/rdma/transport.{h,cc} (engine threads, `senderCC_tx_message`,
// `select_qpidx_pot`, `uc_rx_chunk/uc_rx_ack`), collective/afxdp/transport.{h,cc}.
//
// Re-designed rather than ported: the packet I/O here is plain UDP sockets (P sockets = P source ports =
// P ECMP paths) driven with sendmmsg/recvmmsg from ONE engine thread per NIC; the engine is the same
// whether the bytes are host memory or a pinned staging buffer of the symmetric heap.  Inside an H100 box
// nothing here is used -- NVLink peers are load/store reachable -- this is the path *between* boxes, and
// what the NCCL net plugin (csrc/net/nccl_net_plugin.cc) and `uccl_b200.net` are built on.
//
// Message semantics (NCCL-net compatible): per flow and direction, the i-th send matches the i-th recv.
// Small messages are eager (buffered if the recv is not posted yet); large ones wait for the receiver's
// RTR ("recv i is posted") so data always lands in place.
#pragma once
#include <netinet/in.h>

#include <atomic>
#include <cstddef>
#include <cstdint>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <random>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../common/cc/eqds.h"
#include "../common/cc/swift.h"
#include "../common/cc/timely.h"
#include "net_wire.h"

namespace ub {
namespace net {

enum CcKind : int { CC_NONE = 0, CC_SWIFT = 1, CC_TIMELY = 2, CC_EQDS = 3 };

struct EngineConfig {
  std::string bind_ip = "0.0.0.0";  // local address of the NIC this engine drives
  int paths = 8;                    // UDP sockets / source ports
  int payload = 8192;               // bytes of message data per datagram (jumbo-frame sized by default)
  int max_inflight = 192;           // packets in flight per flow (< kSackBits)
  size_t eager_max = 16384;         // messages up to this size do not wait for the receiver's RTR
  int eager_ahead = 32;             // eager messages allowed beyond the receiver's posted count
  int cc = CC_SWIFT;
  double drop_prob = 0.0;           // fault injection: probability of dropping any outgoing datagram
  int rto_min_us = 4000;
  int rto_max_us = 400000;
  int rto_abort = 50;               // consecutive RTOs before the flow is declared dead
  int syn_retry_ms = 50;
  int connect_timeout_ms = 30000;
  double link_gbps = 400.0;         // pacing ceiling / EQDS receiver line rate
  double swift_target_us = 400.0;   // kernel UDP sockets: base delay target
  bool busy_poll = false;           // never sleep in epoll (lowest latency, one core)
  int sockbuf_bytes = 8 << 20;
  static EngineConfig from_env();
};

struct Request {
  std::atomic<int> done{0};
  std::atomic<int> err{0};
  size_t bytes = 0;
  uint32_t flow = 0;
  bool is_send = false;
};

struct FlowStats {
  uint64_t tx_pkts = 0, tx_bytes = 0, rx_pkts = 0, rx_bytes = 0, rx_dup = 0;
  uint64_t fast_rexmit = 0, rto_rexmit = 0, tlp = 0, acks_tx = 0, acks_rx = 0, unexpected_msgs = 0;
  uint64_t path_tx[kMaxPaths] = {0};
  uint64_t path_bans = 0;
  double srtt_us = 0, min_rtt_us = 0, cwnd = 0, rate_gbps = 0;
  int state = 0;
};

struct EngineStats {
  uint64_t tx_pkts = 0, rx_pkts = 0, tx_bytes = 0, rx_bytes = 0, dropped_tx = 0, bad_pkts = 0;
  uint64_t fast_rexmit = 0, rto_rexmit = 0, loops = 0, sleeps = 0;
  int flows = 0;
};

enum FlowState : int { FL_SYN_SENT = 1, FL_ESTABLISHED = 2, FL_CLOSING = 3, FL_CLOSED = 4, FL_ERROR = 5 };

class Engine {
 public:
  explicit Engine(const EngineConfig& cfg = EngineConfig::from_env());
  ~Engine();
  Engine(const Engine&) = delete;
  Engine& operator=(const Engine&) = delete;

  const EngineConfig& config() const { return cfg_; }
  uint16_t port() const { return ports_[0]; }  // path-0 port: the address peers connect to
  int paths() const { return cfg_.paths; }

  // ---- connection management (all non-blocking unless noted)
  uint32_t listen();
  void close_listen(uint32_t listen_id);
  uint32_t connect_async(const std::string& ip, uint16_t port, uint32_t listen_id);
  int flow_state(uint32_t flow) const;                   // FlowState, 0 if unknown
  bool accept_nb(uint32_t listen_id, uint32_t* flow);    // true if a connection was dequeued
  uint32_t connect(const std::string& ip, uint16_t port, uint32_t listen_id, int timeout_ms = -1);  // blocking
  uint32_t accept(uint32_t listen_id, int timeout_ms = -1);                                         // blocking
  void close_flow(uint32_t flow);
  // Graceful stop (also run by the destructor): close every flow, then linger -- like TCP's TIME_WAIT -- until
  // our FINs are acknowledged and the wire has been quiet for a few RTOs, so that a peer whose last packets or
  // whose ACKs were lost still gets its retransmissions answered.  Bounded by linger_ms
  // (UCCL_B200_NET_LINGER_MS, default 2000).
  void shutdown(int linger_ms = -1);

  // ---- data path: the i-th send of a flow matches the i-th recv of its peer
  Request* send_async(uint32_t flow, const void* data, size_t bytes);
  Request* recv_async(uint32_t flow, void* data, size_t capacity);
  // true when complete (the request is freed); *bytes = message size; *err != 0 on failure
  bool test(Request* r, size_t* bytes, int* err);
  // Blocking completion.  Returns WAIT_OK / WAIT_ERROR (request freed in both cases) or WAIT_TIMEOUT: the
  // request is then still owned by the engine, which may yet read / write the caller's buffer -- call
  // cancel() before that buffer goes away (or keep waiting).
  enum WaitResult : int { WAIT_OK = 0, WAIT_ERROR = 1, WAIT_TIMEOUT = 2 };
  WaitResult wait3(Request* r, size_t* bytes, int timeout_ms = -1);
  // Fails the request's flow (every request queued on it completes with an error, the peer gets a reset) and
  // waits until the engine has dropped `r`; afterwards neither the request nor its buffer is referenced.
  // Returns false if the engine thread did not react within grace_ms (the request is then leaked, not freed).
  bool cancel(Request* r, int grace_ms = 5000);
  void abort_flow(uint32_t flow);  // application-initiated failure of one flow
  // wait3 + cancel on timeout: true only on success; the request is always released and the buffer is free again
  bool wait(Request* r, size_t* bytes, int timeout_ms = -1);

  void set_drop_prob(double p) { drop_prob_.store(p); }
  // fault injection: hold back a fraction of the outgoing datagrams for `delay_us` (reordering inside and across paths)
  void set_reorder(double prob, int delay_us) {
    reorder_delay_us_.store(delay_us);
    reorder_prob_.store(prob);
  }
  // fault injection on ONE local path (models a black-holed ECMP route); path < 0 clears
  void set_path_drop(int path, double p) {
    path_drop_idx_.store(path);
    path_drop_prob_.store(p);
  }
  EngineStats stats() const;
  bool flow_stats(uint32_t flow, FlowStats* out) const;

 private:
  struct TxMsg {
    Request* req = nullptr;
    const uint8_t* ptr = nullptr;
    size_t len = 0, next_off = 0, acked = 0;
    uint32_t id = 0;
    uint32_t pkts_out = 0, pkts_acked = 0;
    bool all_queued = false;
  };
  struct RxMsg {
    Request* req = nullptr;
    uint8_t* ptr = nullptr;
    size_t cap = 0, got = 0, total = 0;
    bool have_total = false, overflow = false;
  };
  struct Unexpected {
    std::vector<uint8_t> buf;
    size_t total = 0, got = 0;
  };
  struct TxPkt {
    uint32_t seq = 0;
    uint8_t kind = 0;
    bool in_use = false, acked = false, lost = false;
    uint16_t path = 0;
    uint32_t msg_id = 0, len = 0, rexmits = 0;
    uint64_t offset = 0, msg_len = 0, ts_send = 0;
    const uint8_t* payload = nullptr;
    TxMsg* msg = nullptr;
  };
  struct PathState {
    double srtt_us = 0;
    uint32_t inflight = 0;
    uint64_t tx = 0;
    uint32_t loss_streak = 0;      // consecutive packets declared lost on this path (reset by any ACK from it)
    uint32_t bans = 0;             // how often it was quarantined (quarantine time backs off)
    uint64_t banned_until_ns = 0;  // path quarantine: a black-holed ECMP path stops getting new packets
  };
  struct Flow {
    uint32_t id = 0, peer_flow = 0, listen_id = 0;
    std::atomic<int> state{0};
    uint64_t nonce = 0;
    in_addr peer_ip{};
    int npaths = 0;
    sockaddr_in peer_addr[kMaxPaths];
    // connect
    uint64_t syn_next_ns = 0, syn_deadline_ns = 0;
    uint16_t syn_port = 0;
    // tx reliability
    uint32_t snd_nxt = 0, snd_una = 0, isn = 0;  // isn: initial sequence number of OUR direction (random)
    TxPkt ring[kTxRing];
    uint32_t inflight = 0;  // sent, not acked, not marked lost
    std::deque<uint32_t> rexmit_q;
    uint64_t newest_acked_send_ts = 0;
    double srtt_us = 0, rttvar_us = 0, min_rtt_us = 0;
    uint64_t rto_ns = 0;
    int rto_count = 0;
    uint64_t last_progress_ns = 0;
    uint64_t close_start_ns = 0;  // when the flow entered FL_CLOSING: hard bound of the close handshake
    uint64_t last_tx_ns = 0;   // last (re)transmission of a DATA packet
    bool tlp_fired = false;    // one tail-loss probe per quiet period
    uint32_t peer_dup_seen = 0;   // last AckBody.dup_cum
    uint32_t reo_mult = 1;        // RACK reordering window = reo_mult * srtt/4 (adapts to observed spurious retransmissions)
    uint64_t reo_decay_ns = 0;
    PathState path[kMaxPaths];
    // congestion control
    cc::Swift swift;
    cc::Timely timely;
    uint64_t pace_next_ns = 0;
    uint64_t credit_cum = 0, sent_payload_cum = 0;  // EQDS (sender side)
    uint64_t grant_cum = 0, demand_seen = 0;        // EQDS (receiver side)
    bool credit_dirty = false;
    bool credit_starved = false;  // sender: blocked on EQDS credit in the last pump
    // tx messages
    std::deque<TxMsg*> txq;       // not yet fully acked, in id order
    size_t tx_cursor = 0;         // index into txq of the message being cut into packets
    uint32_t next_tx_msg = 0;
    uint32_t peer_posted = 0;     // receives the peer has posted (from RTR frames / ACK hints)
    bool rtr_pending = false, fin_pending = false, fin_sent = false;
    // rx reliability
    uint32_t rcv_nxt = 0;
    uint64_t rx_bits[kSackWords] = {0, 0, 0, 0};
    bool need_ack = false;
    uint64_t echo_ts = 0;
    uint16_t echo_path = 0;
    // rx messages
    std::deque<RxMsg> rxq;  // posted receives; front has id rx_base
    uint32_t rx_base = 0, rx_posted = 0;
    std::map<uint32_t, Unexpected> unexpected;
    std::atomic<bool> peer_fin{false};  // the peer's FIN and everything before it has arrived
    bool have_fin = false;
    uint32_t fin_seq = 0;
    FlowStats st;
    Flow() : swift(cc::SwiftConfig()), timely(cc::TimelyConfig()) {}
  };
  struct Listener {
    std::deque<uint32_t> ready;
  };
  struct Cmd {
    int op = 0;  // 1 connect, 2 send, 3 recv, 4 close flow
    uint32_t flow = 0;
    Request* req = nullptr;
    void* ptr = nullptr;
    size_t len = 0;
  };

  void run();
  void wake();
  void drain_cmds();
  bool rx_poll();
  void on_packet(int sock_idx, const sockaddr_in& from, uint8_t* buf, size_t n);
  void on_syn(int sock_idx, const sockaddr_in& from, const PktHdr& h, const SynBody& b);
  void on_synack(const sockaddr_in& from, const PktHdr& h, const SynBody& b);
  void on_data(Flow& f, const PktHdr& h, const uint8_t* payload);
  void on_ack(Flow& f, const PktHdr& h, const AckBody& b);
  void deliver_frame(Flow& f, const PktHdr& h, const uint8_t* payload);
  void mark_acked(Flow& f, TxPkt& p, uint64_t now);
  void detect_loss(Flow& f, uint64_t now);
  bool tx_pump(Flow& f, uint64_t now);
  bool can_send_new(Flow& f, uint64_t now);
  void emit_data(Flow& f, TxPkt& p, uint64_t now, bool is_rexmit);
  int pick_path(Flow& f, int avoid);
  void send_ack(Flow& f);
  void send_syn(Flow& f, bool synack, int sock_idx, const sockaddr_in* to);
  void send_rst(int sock_idx, const sockaddr_in& to, uint32_t dst_flow);
  void raw_send(int path, const sockaddr_in& to, const void* hdr, size_t hlen, const void* body, size_t blen);
  void timers(uint64_t now);
  void fail_flow(Flow& f, const char* why);
  void complete(Request* r, size_t bytes, int err);
  void post_recv(Flow& f, Request* r, void* ptr, size_t cap);
  void post_send(Flow& f, Request* r, const void* ptr, size_t len);
  void fill_syn_body(SynBody* b, const Flow& f) const;
  std::shared_ptr<Flow> find(uint32_t id) const;
  void eqds_tick(uint64_t now);
  void apply_peer_fin(Flow& f);

  EngineConfig cfg_;
  int socks_[kMaxPaths];
  uint16_t ports_[kMaxPaths];
  int epfd_ = -1, evfd_ = -1;
  std::thread thr_;
  std::atomic<bool> stop_{false};
  std::atomic<double> drop_prob_{0.0}, path_drop_prob_{0.0};
  std::atomic<int> path_drop_idx_{-1};
  std::atomic<double> reorder_prob_{0.0};
  std::atomic<int> reorder_delay_us_{300};
  struct Held {
    uint64_t release_ns;
    int path;
    sockaddr_in to;
    std::vector<char> bytes;  // header + payload, copied: the user buffer may be gone when the datagram finally leaves
  };
  std::deque<Held> held_;
  void release_held(uint64_t now);
  void note_path_loss(Flow& f, int path, uint64_t now);
  std::atomic<uint32_t> next_flow_{1}, next_listen_{1};
  std::atomic<uint64_t> last_rx_ns_{0};
  bool shut_ = false;

  mutable std::mutex mu_;  // flows_, listeners_, cmds_, syn_index_
  std::unordered_map<uint32_t, std::shared_ptr<Flow>> flows_;
  std::unordered_map<uint32_t, Listener> listeners_;
  std::map<std::pair<uint64_t, uint64_t>, uint32_t> syn_index_;  // (peer addr, nonce) -> flow
  std::vector<Cmd> cmds_;
  std::vector<std::shared_ptr<Flow>> active_;  // engine thread's working set
  std::unordered_map<uint32_t, Flow*> index_;  // id -> flow of active_ (engine thread only)
  bool active_dirty_ = true;

  cc::EqdsPacer pacer_;
  std::mt19937_64 rng_;
  EngineStats est_;
  mutable std::mutex st_mu_;
  // rx scratch
  std::vector<uint8_t> rx_buf_;
  // tx batching: datagrams queued per path during one loop iteration leave in one sendmmsg
  static constexpr int kTxBatch = 32;
  struct TxSlot {
    PktHdr hdr;
    uint8_t body[96];  // AckBody / SynBody (payload of DATA packets is referenced in place)
    sockaddr_in to;
    const void* payload;
    uint32_t blen;
  };
  struct TxBatch {
    TxSlot slot[kTxBatch];
    int n = 0;
  };
  std::vector<TxBatch> txb_;
  bool gro_ok_ = true;  // UDP_GRO on the receive sockets (coalesced trains are split in rx_poll)
  bool gso_ok_ = true;  // UDP_SEGMENT super-datagrams (cleared at the first EINVAL/EIO from the kernel)
  void flush_path(int path);
  void flush_all();
};

std::vector<std::pair<std::string, std::string>> list_interfaces();  // (name, ipv4) of usable NICs

}  // namespace net
}  // namespace ub
