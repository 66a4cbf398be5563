#include "endpoint.h"

#include <atomic>

#include <arpa/inet.h>
#include <errno.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <poll.h>
#include <sys/eventfd.h>
#include <sys/socket.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <cstring>

#include "../common/log.h"
#include "../common/param.h"
#include "../fabric/cu_api.h"

namespace ub {

UB_PARAM(P2PCtas, "P2P_CTAS", 0)       // 0: by transfer size (8 / 32 / 64 CTAs)
UB_PARAM(P2PChunkKB, "P2P_CHUNK_KB", 16)  // bytes per bulk copy; 4 pipelines x 3 stages of it per CTA
UB_PARAM(P2PUseKernel, "P2P_USE_KERNEL", 1)
// a handful of very large blocks is what the copy engines are best at: up to 8
// blocks of at least this many MiB each go through cudaMemcpyAsync, everything else through the TMA copy kernel
UB_PARAM(P2PMemcpyMinMB, "P2P_MEMCPY_MIN_MB", 32)
// engine status line every N seconds at INFO level (reference: per-engine stats thread every 2 s unless
// UCCL_ENGINE_QUIET, collective/rdma/transport.cc:1797-1825); 0 = off
UB_PARAM(P2PStatsSec, "ENGINE_STATS_SEC", 0)

cudaError_t launch_p2p_copy(const P2PCopyBatch& b, int grid, cudaStream_t st);

namespace {
enum MsgType : uint32_t {
  MSG_HELLO = 1, MSG_ADV = 2, MSG_DONE = 3, MSG_NOTIF = 4, MSG_BYE = 5,
  // host mode between processes: the payload itself travels on the connection (TCP data path)
  MSG_WRITE = 6,      // {u64 dst_addr, u64 bytes, data}: the target's engine copies data to dst_addr
  MSG_FLUSH = 7,      // seq = initiator transfer id; answered by MSG_FLUSH_ACK once every earlier WRITE is applied
  MSG_FLUSH_ACK = 8,
  MSG_READ_REQ = 9,   // seq = initiator transfer id; payload = {u64 src_addr, u64 bytes} per buffer
  MSG_READ_RESP = 10  // seq = same id; payload = the concatenated data
};
struct MsgHdr {
  uint32_t type;
  uint32_t len;
  uint64_t seq;
};
struct Hello {
  int32_t gpu;
  int32_t pid;
};
bool write_full(int fd, const void* p, size_t n) {
  const char* c = (const char*)p;
  while (n) {
    ssize_t w = ::send(fd, c, n, MSG_NOSIGNAL);
    if (w < 0) {
      if (errno == EINTR || errno == EAGAIN) continue;
      return false;
    }
    c += w;
    n -= (size_t)w;
  }
  return true;
}
bool read_full(int fd, void* p, size_t n) {
  char* c = (char*)p;
  while (n) {
    ssize_t r = ::recv(fd, c, n, 0);
    if (r < 0) {
      if (errno == EINTR || errno == EAGAIN) continue;
      return false;
    }
    if (r == 0) return false;
    c += r;
    n -= (size_t)r;
  }
  return true;
}
}  // namespace

struct Endpoint::Conn {
  uint64_t id = 0;
  int fd = -1;
  int remote_gpu = -1;
  int remote_pid = -1;
  std::string ip;
  std::mutex send_mu;
  std::map<uint64_t, std::vector<XferDesc>> advs;  // seq -> advertised windows (from the peer's recv)
  std::map<uint64_t, bool> dones;                  // seq -> DONE received
  std::map<uint64_t, bool> acks;                   // transfer id -> FLUSH_ACK received (TCP data path)
  uint64_t next_send_seq = 0, next_recv_seq = 0;
  // written by the engine thread (EOF / BYE) and by remove_remote_endpoint(); read everywhere
  std::atomic<bool> alive{true};
};

struct Endpoint::Transfer {
  enum State { SEND_WAIT_ADV, COPYING, RECV_WAIT_DONE, DONE, FAILED, WAIT_ACK, WAIT_RESP, TCP_SENDING };
  uint64_t id = 0;
  // written by the engine thread under mu_ and by the polling caller; read without the lock on the poll path
  std::atomic<State> state{DONE};
  std::shared_ptr<Conn> conn;
  uint64_t seq = 0;
  bool notify_done = false;  // send DONE{seq} to the peer when the copy finishes
  std::vector<const char*> src;
  std::vector<char*> dst;  // read over the TCP data path: where the response is scattered to
  std::vector<size_t> sizes;
  cudaEvent_t ev = nullptr;
};

// local_gpu_idx < 0 selects the host mode: buffers are ordinary host memory of this process, copies are
// memcpy and complete immediately.  Everything else (TCP control plane, send/recv matching, transfer
// tables, notifications, polling) is the production code, which is what the GPU-less CI exercises.
Endpoint::Endpoint(int local_gpu_idx, int num_streams) : gpu_(local_gpu_idx) {
  if (gpu_ >= 0) {
    UB_CUDA(cudaSetDevice(gpu_));
    UB_CUDA(cudaFree(0));
    for (int i = 0; i < std::max(1, num_streams); ++i) {
      cudaStream_t s;
      UB_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
      streams_.push_back(s);
    }
  }
  ip_ = param_load_str("P2P_IP", "127.0.0.1");
  listen_fd_ = ::socket(AF_INET, SOCK_STREAM, 0);
  UB_CHECK(listen_fd_ >= 0, "socket failed: %s", strerror(errno));
  int one = 1;
  setsockopt(listen_fd_, SOL_SOCKET, SO_REUSEADDR, &one, sizeof(one));
  sockaddr_in addr;
  memset(&addr, 0, sizeof(addr));
  addr.sin_family = AF_INET;
  addr.sin_addr.s_addr = htonl(INADDR_ANY);
  addr.sin_port = 0;
  UB_CHECK(::bind(listen_fd_, (sockaddr*)&addr, sizeof(addr)) == 0, "bind failed: %s", strerror(errno));
  UB_CHECK(::listen(listen_fd_, 128) == 0, "listen failed: %s", strerror(errno));
  socklen_t al = sizeof(addr);
  getsockname(listen_fd_, (sockaddr*)&addr, &al);
  port_ = ntohs(addr.sin_port);
  wake_fd_ = eventfd(0, EFD_NONBLOCK);
  engine_ = std::thread([this] { engine_loop(); });
  UB_INFO(SUB_P2P, "p2p endpoint gpu %d listening on %s:%u", gpu_, ip_.c_str(), (unsigned)port_);
}

Endpoint::~Endpoint() {
  stop_ = true;
  wake();
  if (engine_.joinable()) engine_.join();
  {
    std::lock_guard<std::mutex> g(mu_);
    for (auto& kv : conns_)
      if (kv.second->fd >= 0) ::shutdown(kv.second->fd, SHUT_RDWR);  // unblock helper threads stuck in send()
  }
  {
    std::lock_guard<std::mutex> g(helpers_mu_);
    for (auto& t : helpers_)
      if (t.joinable()) t.join();
    helpers_.clear();
  }
  {
    std::lock_guard<std::mutex> g(mu_);
    retire_closed_locked();
    for (auto& kv : conns_)
      if (kv.second->fd >= 0) ::close(kv.second->fd);
    conns_.clear();
  }
  if (listen_fd_ >= 0) ::close(listen_fd_);
  if (wake_fd_ >= 0) ::close(wake_fd_);
  if (gpu_ < 0) return;
  cudaSetDevice(gpu_);
  for (auto& kv : ipc_open_) cudaIpcCloseMemHandle(kv.second);
  for (auto s : streams_) {
    cudaStreamSynchronize(s);  // descriptor-table callbacks reference this object
    cudaStreamDestroy(s);
  }
  for (auto e : event_pool_) cudaEventDestroy(e);
  for (auto* t : tables_all_) {
    cudaFreeHost(t->host);
    cudaFree(t->dev);
    delete t;
  }
}

void Endpoint::wake() {
  uint64_t one = 1;
  if (wake_fd_ >= 0) (void)!::write(wake_fd_, &one, sizeof(one));
}

std::string Endpoint::get_metadata() const {
  // 4-byte IPv4 + 2-byte port (network order) + 4-byte gpu index (like the reference's 10-byte blob)
  std::string md(10, '\0');
  in_addr a;
  inet_pton(AF_INET, ip_.c_str(), &a);
  memcpy(&md[0], &a, 4);
  uint16_t p = htons(port_);
  memcpy(&md[4], &p, 2);
  int32_t g = gpu_;
  memcpy(&md[6], &g, 4);
  return md;
}

bool Endpoint::parse_metadata(const std::string& md, std::string* ip, uint16_t* port, int* gpu_idx) {
  if (md.size() != 10) return false;
  char buf[INET_ADDRSTRLEN];
  in_addr a;
  memcpy(&a, &md[0], 4);
  if (!inet_ntop(AF_INET, &a, buf, sizeof(buf))) return false;
  uint16_t p;
  memcpy(&p, &md[4], 2);
  int32_t g;
  memcpy(&g, &md[6], 4);
  if (ip) *ip = buf;
  if (port) *port = ntohs(p);
  if (gpu_idx) *gpu_idx = g;
  return true;
}

std::shared_ptr<Endpoint::Conn> Endpoint::find_conn(uint64_t id) {
  std::lock_guard<std::mutex> g(mu_);
  auto it = conns_.find(id);
  return it == conns_.end() ? nullptr : it->second;
}

bool Endpoint::connect(const std::string& ip, int remote_gpu_idx, uint16_t remote_port, uint64_t* conn_id) {
  int fd = -1;
  sockaddr_in addr;
  memset(&addr, 0, sizeof(addr));
  addr.sin_family = AF_INET;
  addr.sin_port = htons(remote_port);
  if (inet_pton(AF_INET, ip.c_str(), &addr.sin_addr) != 1) return false;
  // retry loop like the reference's connect (p2p/engine.cc:1322-1357)
  for (int attempt = 0; attempt < 200; ++attempt) {
    fd = ::socket(AF_INET, SOCK_STREAM, 0);
    if (fd < 0) return false;
    if (::connect(fd, (sockaddr*)&addr, sizeof(addr)) == 0) break;
    ::close(fd);
    fd = -1;
    std::this_thread::sleep_for(std::chrono::milliseconds(25));
  }
  if (fd < 0) {
    UB_WARN("p2p connect to %s:%u failed", ip.c_str(), (unsigned)remote_port);
    return false;
  }
  int one = 1;
  setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof(one));
  MsgHdr h{MSG_HELLO, sizeof(Hello), 0};
  Hello me{gpu_, (int32_t)getpid()};
  Hello peer;
  MsgHdr rh;
  if (!write_full(fd, &h, sizeof(h)) || !write_full(fd, &me, sizeof(me)) || !read_full(fd, &rh, sizeof(rh)) ||
      rh.type != MSG_HELLO || !read_full(fd, &peer, sizeof(peer))) {
    ::close(fd);
    return false;
  }
  auto c = std::make_shared<Conn>();
  c->fd = fd;
  c->remote_gpu = peer.gpu;
  c->remote_pid = peer.pid;
  c->ip = ip;
  {
    std::lock_guard<std::mutex> g(mu_);
    c->id = next_conn_++;
    conns_[c->id] = c;
  }
  if (conn_id) *conn_id = c->id;
  (void)remote_gpu_idx;
  wake();
  return true;
}

bool Endpoint::add_remote_endpoint(const std::string& metadata, uint64_t* conn_id) {
  std::string ip;
  uint16_t port;
  int gpu;
  if (!parse_metadata(metadata, &ip, &port, &gpu)) return false;
  return connect(ip, gpu, port, conn_id);
}

bool Endpoint::accept(std::string* ip, int* remote_gpu_idx, uint64_t* conn_id, int timeout_ms) {
  std::unique_lock<std::mutex> lk(mu_);
  auto pred = [this] { return !accepted_.empty() || stop_.load(); };
  if (timeout_ms < 0) accept_cv_.wait(lk, pred);
  else if (!accept_cv_.wait_for(lk, std::chrono::milliseconds(timeout_ms), pred)) return false;
  if (accepted_.empty()) return false;
  uint64_t id = accepted_.front();
  accepted_.pop_front();
  auto c = conns_[id];
  if (ip) *ip = c->ip;
  if (remote_gpu_idx) *remote_gpu_idx = c->remote_gpu;
  if (conn_id) *conn_id = id;
  return true;
}

bool Endpoint::remove_remote_endpoint(uint64_t conn_id) {
  std::shared_ptr<Conn> c;
  {
    std::lock_guard<std::mutex> g(mu_);
    auto it = conns_.find(conn_id);
    if (it == conns_.end()) return false;
    c = it->second;
    conns_.erase(it);
    for (auto& kv : transfers_)
      if (kv.second->conn == c && kv.second->state != Transfer::DONE) kv.second->state = Transfer::FAILED;
  }
  send_msg(*c, MSG_BYE, 0, nullptr, 0);
  c->alive = false;
  // The engine thread may be inside read() on this descriptor: shut the socket down (that wakes it with EOF) but
  // leave close() to the engine thread, which retires the connection at the top of its next iteration -- closing
  // here could hand the descriptor number to a new socket while the old read is still in flight.
  ::shutdown(c->fd, SHUT_RDWR);
  {
    std::lock_guard<std::mutex> g(mu_);
    closing_.push_back(c);
  }
  wake();
  return true;
}

void Endpoint::retire_closed_locked() {
  for (auto& c : closing_) {
    std::lock_guard<std::mutex> sg(c->send_mu);  // no sender is between its fd check and its write
    if (c->fd >= 0) ::close(c->fd);
    c->fd = -1;
  }
  closing_.clear();
}

bool Endpoint::send_msg(Conn& c, uint32_t type, uint64_t seq, const void* payload, uint32_t len) {
  std::lock_guard<std::mutex> g(c.send_mu);
  if (c.fd < 0) return false;
  MsgHdr h{type, len, seq};
  if (!write_full(c.fd, &h, sizeof(h))) return false;
  if (len && !write_full(c.fd, payload, len)) return false;
  return true;
}

// header + two payload parts as one frame (the connection is shared by several threads)
bool Endpoint::send_msg2(Conn& c, uint32_t type, uint64_t seq, const void* p1, uint32_t len1, const void* p2,
                         uint32_t len2) {
  std::lock_guard<std::mutex> g(c.send_mu);
  if (c.fd < 0) return false;
  MsgHdr h{type, len1 + len2, seq};
  if (!write_full(c.fd, &h, sizeof(h))) return false;
  if (len1 && !write_full(c.fd, p1, len1)) return false;
  if (len2 && !write_full(c.fd, p2, len2)) return false;
  return true;
}

// TCP data path (host mode, peer in another process): one MSG_WRITE frame per buffer, cut into pieces
// that fit the 32-bit frame length.
bool Endpoint::tcp_write_buffers(Conn& c, const std::vector<const char*>& src, const std::vector<uint64_t>& dst_addr,
                                 const std::vector<size_t>& sizes) {
  const size_t kPiece = gpu_ >= 0 ? (4u << 20) : (64u << 20);
  std::vector<char> bounce;  // GPU endpoints: the socket cannot read device memory
  if (gpu_ >= 0) bounce.resize(kPiece);
  for (size_t i = 0; i < src.size(); ++i)
    for (size_t off = 0; off < sizes[i]; off += kPiece) {
      const uint64_t n = std::min(kPiece, sizes[i] - off);
      const uint64_t pre[2] = {dst_addr[i] + off, n};
      const char* from = src[i] + off;
      if (gpu_ >= 0) {
        copy_any(bounce.data(), from, n);
        from = bounce.data();
      }
      if (!send_msg2(c, MSG_WRITE, 0, pre, sizeof(pre), from, (uint32_t)n)) return false;
    }
  return true;
}

namespace {
// Identity of this machine (hostname + boot id); UCCL_B200_P2P_HOST_ID overrides (tests emulate two hosts with it).
uint64_t local_host_id() {
  static const uint64_t id = [] {
    const int64_t forced = param_load("P2P_HOST_ID", 0);
    if (forced > 0) return (uint64_t)forced;
    char buf[320] = {0};
    gethostname(buf, 255);
    if (FILE* f = fopen("/proc/sys/kernel/random/boot_id", "r")) {
      const size_t at = strlen(buf);
      if (fgets(buf + at, (int)(sizeof(buf) - at), f) == nullptr) buf[at] = 0;
      fclose(f);
    }
    uint64_t h = 1469598103934665603ull;  // FNV-1a
    for (const char* p = buf; *p; ++p) h = (h ^ (unsigned char)*p) * 1099511628211ull;
    return h ? h : 1;
  }();
  return id;
}
}  // namespace

// Same host: GPU endpoints map each other's memory (CUDA IPC) and host endpoints of one process share an address
// space.  Everything else -- a host-mode peer in another process, any peer on another machine -- gets its payload
// over the (TCP) connection; GPU memory is staged through host bounce buffers on both sides.
bool Endpoint::remote_is_other_process(const XferDesc& d) const {
  if (d.host_id != 0 && d.host_id != local_host_id()) return true;
  return gpu_ < 0 && d.pid != (int32_t)getpid();
}

void Endpoint::copy_any(void* dst, const void* src, size_t n) {
  if (!n) return;
  if (gpu_ < 0) {
    memcpy(dst, src, n);
    return;
  }
  int prev = -1;
  cudaGetDevice(&prev);
  if (prev != gpu_) cudaSetDevice(gpu_);
  cudaError_t e = cudaMemcpy(dst, src, n, cudaMemcpyDefault);  // either side may be device or host memory
  if (e != cudaSuccess) UB_WARN("p2p: staged copy of %zu bytes failed: %s", n, cudaGetErrorString(e));
  if (prev >= 0 && prev != gpu_) cudaSetDevice(prev);
}

void Endpoint::run_helper(std::function<void()> fn) {
  std::lock_guard<std::mutex> g(helpers_mu_);
  helpers_.emplace_back(std::move(fn));
}

// ------------------------------------------------------------------ registration
bool Endpoint::reg(const void* ptr, size_t size, uint64_t* mr_id) {
  if (!ptr || !size) return false;
  XferDesc d;
  if (!describe(ptr, size, &d)) return false;  // also caches the IPC export of the allocation
  std::lock_guard<std::mutex> g(mu_);
  uint64_t id = next_mr_++;
  mrs_[id] = MR{ptr, size};
  if (mr_id) *mr_id = id;
  return true;
}

bool Endpoint::dereg(uint64_t mr_id) {
  MR gone;
  bool still_covered = false;
  {
    std::lock_guard<std::mutex> g(mu_);
    auto it = mrs_.find(mr_id);
    if (it == mrs_.end()) return false;
    gone = it->second;
    mrs_.erase(it);
    for (auto& kv : mrs_)  // another registration of the same window keeps it reachable
      if (kv.second.ptr == gone.ptr && kv.second.size >= gone.size) still_covered = true;
  }
  if (!still_covered) {
    // revoke the window: a peer on another host must not write into memory that was deregistered (and maybe freed)
    std::lock_guard<std::mutex> g(exp_mu_);
    for (auto it = exposed_.begin(); it != exposed_.end();)
      it = (it->first == (uint64_t)gone.ptr && it->second <= gone.size) ? exposed_.erase(it) : std::next(it);
  }
  return true;
}

void Endpoint::expose(uint64_t addr, uint64_t size) {
  std::lock_guard<std::mutex> g(exp_mu_);
  for (auto& r : exposed_)
    if (r.first == addr) {
      if (size > r.second) r.second = size;
      return;
    }
  if (exposed_.size() >= 65536) exposed_.erase(exposed_.begin(), exposed_.begin() + 32768);  // bounded; oldest go
  exposed_.emplace_back(addr, size);
}

bool Endpoint::is_exposed(uint64_t addr, uint64_t n) {
  std::lock_guard<std::mutex> g(exp_mu_);
  for (auto& r : exposed_)
    if (addr >= r.first && addr + n <= r.first + r.second && addr + n >= addr) return true;
  return false;
}

bool Endpoint::describe(const void* ptr, size_t size, XferDesc* out) {
  memset(out, 0, sizeof(*out));
  out->addr = (uint64_t)ptr;
  out->size = size;
  out->pid = (int32_t)getpid();
  out->dev = gpu_;
  out->host_id = local_host_id();
  if (gpu_ < 0) {  // host mode: plain memory of this process
    out->kind = 1;
    out->base = (uint64_t)ptr;
    expose((uint64_t)ptr, size);
    return true;
  }
  cudaPointerAttributes attr;
  memset(&attr, 0, sizeof(attr));
  cudaError_t e = cudaPointerGetAttributes(&attr, ptr);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    return false;
  }
  expose((uint64_t)ptr, size);  // a peer on another host may address this window through the wire
  if (attr.type == cudaMemoryTypeHost) {
    out->kind = 1;
    out->base = (uint64_t)ptr;
    return true;
  }
  if (attr.type != cudaMemoryTypeDevice) {
    UB_WARN("p2p: pointer %p is neither device nor pinned host memory", ptr);
    return false;
  }
  out->dev = attr.device;
  CUdeviceptr base = 0;
  size_t asz = 0;
  CUresult (*getRange)(CUdeviceptr*, size_t*, CUdeviceptr) = nullptr;
  {
    cudaDriverEntryPointQueryResult st;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", (void**)&getRange, cudaEnableDefault, &st) != cudaSuccess)
      getRange = nullptr;
  }
  if (!getRange || getRange(&base, &asz, (CUdeviceptr)ptr) != CUDA_SUCCESS) {
    (void)cudaGetLastError();
    base = (CUdeviceptr)ptr;
  }
  out->base = (uint64_t)base;
  std::lock_guard<std::mutex> g(mu_);
  auto it = ipc_export_.find((uint64_t)base);
  if (it == ipc_export_.end()) {
    cudaIpcMemHandle_t h;
    int prev = 0;
    cudaGetDevice(&prev);
    if (prev != attr.device) cudaSetDevice(attr.device);
    cudaError_t ie = cudaIpcGetMemHandle(&h, (void*)base);
    if (prev != attr.device) cudaSetDevice(prev);
    std::string hs;
    if (ie == cudaSuccess) hs.assign((const char*)&h, sizeof(h));
    else (void)cudaGetLastError();  // e.g. VMM memory: only usable by same-process peers
    it = ipc_export_.emplace((uint64_t)base, hs).first;
  }
  if (it->second.empty()) {
    out->kind = 2;
  } else {
    out->kind = 0;
    memcpy(out->ipc_handle, it->second.data(), 64);
  }
  return true;
}

bool Endpoint::advertise(uint64_t conn, const void* ptr, size_t size, XferDesc* out) {
  (void)conn;
  return describe(ptr, size, out);
}

void* Endpoint::map_remote(const XferDesc& d) {
  if (gpu_ < 0) {
    if (d.pid == (int32_t)getpid()) return (void*)d.addr;
    UB_WARN("p2p(host mode): descriptors of another process cannot be mapped");
    return nullptr;
  }
  if (d.pid == (int32_t)getpid()) {
    // same-process short-circuit (reference: direct_addr); a pointer of another device needs
    // peer access from ours (cudaMalloc memory is not peer-mapped by default)
    if (d.kind != 1 && d.dev != gpu_) {
      std::lock_guard<std::mutex> g(mu_);
      if (!(peer_enabled_mask_ & (1u << (d.dev & 31)))) {
        int prev = -1;
        cudaGetDevice(&prev);
        cudaSetDevice(gpu_);
        cudaError_t e = cudaDeviceEnablePeerAccess(d.dev, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
          UB_WARN("cudaDeviceEnablePeerAccess(%d -> %d) failed: %s", gpu_, d.dev, cudaGetErrorString(e));
        (void)cudaGetLastError();
        if (prev >= 0 && prev != gpu_) cudaSetDevice(prev);
        peer_enabled_mask_ |= 1u << (d.dev & 31);
      }
    }
    return (void*)d.addr;
  }
  if (d.kind != 0) {
    UB_WARN("p2p: descriptor kind %u from another process cannot be mapped", d.kind);
    return nullptr;
  }
  std::string key((const char*)d.ipc_handle, 64);
  void* base = nullptr;
  {
    std::lock_guard<std::mutex> g(mu_);
    auto it = ipc_open_.find(key);
    if (it != ipc_open_.end()) base = it->second;
  }
  if (!base) {
    cudaIpcMemHandle_t h;
    memcpy(&h, d.ipc_handle, sizeof(h));
    cudaError_t e = cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      UB_WARN("cudaIpcOpenMemHandle failed: %s", cudaGetErrorString(e));
      (void)cudaGetLastError();
      return nullptr;
    }
    std::lock_guard<std::mutex> g(mu_);
    ipc_open_[key] = base;
  }
  return (char*)base + (d.addr - d.base);
}

// ------------------------------------------------------------------ data path
static cudaEvent_t new_event();

bool Endpoint::is_device_ptr(const void* p) {
  const uint64_t key = (uint64_t)(uintptr_t)p >> 21;  // allocations are at least 2 MiB-granular in the VA space
  {
    std::lock_guard<std::mutex> g(mu_);
    auto it = ptr_is_device_.find(key);
    if (it != ptr_is_device_.end()) return it->second;
  }
  cudaPointerAttributes a;
  memset(&a, 0, sizeof(a));
  bool dev = cudaPointerGetAttributes(&a, p) == cudaSuccess && a.type == cudaMemoryTypeDevice;
  (void)cudaGetLastError();
  if (dev) {  // only positive answers are cached: host memory can be remapped, device VA ranges are not reused as host
    std::lock_guard<std::mutex> g(mu_);
    if (ptr_is_device_.size() > (1u << 16)) ptr_is_device_.clear();
    ptr_is_device_[key] = true;
  }
  return dev;
}

// Cuts a block vector into launches of the copy kernel: up to kP2PMaxEntries blocks ride in the kernel parameters,
// larger batches in pinned descriptor tables of kP2PTableEntries entries each.
bool Endpoint::build_launches(const std::vector<const char*>& src, const std::vector<char*>& dst,
                              const std::vector<size_t>& sizes, std::vector<CopyLaunch>* out, cudaStream_t st) {
  const size_t n = src.size();
  const uint32_t chunk = (uint32_t)std::max<int64_t>(4, std::min<int64_t>(16, ubParamP2PChunkKB())) * 1024;
  const size_t per_launch = n > (size_t)kP2PMaxEntries ? (size_t)kP2PTableEntries : (size_t)kP2PMaxEntries;
  for (size_t i0 = 0; i0 < n; i0 += per_launch) {
    out->emplace_back();
    CopyLaunch& l = out->back();
    P2PCopyBatch& b = l.b;
    memset(&b, 0, sizeof(b));
    b.chunk_bytes = chunk;
    const size_t m = std::min<size_t>(per_launch, n - i0);
    P2PCopyEntry* ents = b.e;
    uint32_t* pfx = b.chunk_prefix;
    if (m > (size_t)kP2PMaxEntries) {
      l.tab = acquire_table();
      if (!l.tab) {
        for (auto& r : *out)
          if (r.tab) release_table_cb(r.tab);
        out->clear();
        return false;
      }
      ents = (P2PCopyEntry*)l.tab->host;
      pfx = (uint32_t*)((char*)l.tab->host + sizeof(P2PCopyEntry) * kP2PTableEntries);
      b.table = (const P2PCopyEntry*)l.tab->dev;
      b.table_prefix = (const uint32_t*)((char*)l.tab->dev + sizeof(P2PCopyEntry) * kP2PTableEntries);
    }
    uint64_t total = 0, bytes_total = 0;
    for (size_t j = 0; j < m; ++j) {
      auto& e = ents[j];
      e.src = src[i0 + j];
      e.dst = dst[i0 + j];
      e.bytes = sizes[i0 + j];
      const bool al = ((((uintptr_t)e.src) | ((uintptr_t)e.dst)) & 15) == 0;
      e.bulk_bytes = al ? (e.bytes / 16 * 16) : 0;
      pfx[j] = (uint32_t)total;
      total += (e.bulk_bytes + chunk - 1) / chunk;
      bytes_total += e.bytes;
      if (e.bulk_bytes != e.bytes) b.any_tail = 1;
    }
    pfx[m] = (uint32_t)total;
    b.n = (int)m;
    if (l.tab) {  // upload the part of the table that is in use
      const size_t eb = sizeof(P2PCopyEntry) * m, pb = sizeof(uint32_t) * (m + 1);
      const size_t poff = sizeof(P2PCopyEntry) * kP2PTableEntries;
      if (cudaMemcpyAsync(l.tab->dev, l.tab->host, eb, cudaMemcpyHostToDevice, st) != cudaSuccess ||
          cudaMemcpyAsync((char*)l.tab->dev + poff, (char*)l.tab->host + poff, pb, cudaMemcpyHostToDevice, st) != cudaSuccess) {
        (void)cudaGetLastError();
        for (auto& r : *out)
          if (r.tab) release_table_cb(r.tab);
        out->clear();
        return false;
      }
    }
    // enough CTAs for the bytes in flight the link needs (4 pipelines x 3 stages x chunk each); small
    // transfers keep the launch small so they do not take SMs from a co-running kernel
    int64_t want = ubParamP2PCtas();
    if (want <= 0) want = bytes_total >= (8u << 20) ? 64 : (bytes_total >= (1u << 20) ? 32 : 8);
    l.grid = (int)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)((total + kP2PWarps - 1) / kP2PWarps)));
  }
  return true;
}

bool Endpoint::prepare(uint64_t conn, bool is_write, const std::vector<const void*>& local,
                       const std::vector<size_t>& sizes, const std::vector<XferDesc>& remote, uint64_t* prep_id) {
  auto c = find_conn(conn);
  if (!c || gpu_ < 0 || local.size() != sizes.size() || local.size() != remote.size() || local.empty()) return false;
  if (remote_is_other_process(remote[0])) return false;  // not load/store reachable: use write_async / read_async
  cudaSetDevice(gpu_);
  std::vector<const char*> s;
  std::vector<char*> d;
  auto p = std::make_shared<Prepared>();
  for (size_t i = 0; i < local.size(); ++i) {
    if (sizes[i] > remote[i].size) return false;
    void* r = map_remote(remote[i]);
    if (!r || !is_device_ptr(r) || !is_device_ptr(local[i])) return false;
    s.push_back(is_write ? (const char*)local[i] : (const char*)r);
    d.push_back(is_write ? (char*)r : (char*)local[i]);
    p->bytes += sizes[i];
  }
  bool few_large = local.size() <= 8 && ubParamP2PMemcpyMinMB() > 0;
  for (size_t i = 0; i < sizes.size() && few_large; ++i) few_large = sizes[i] >= ((size_t)ubParamP2PMemcpyMinMB() << 20);
  if (few_large || !ubParamP2PUseKernel()) {
    p->use_memcpy = true;
    p->src = s;
    p->dst = d;
    p->sizes = sizes;
  } else {
    cudaStream_t up = streams_[0];
    if (!build_launches(s, d, sizes, &p->launches, up)) return false;
    cudaStreamSynchronize(up);  // the tables are resident before the first post (which may use another stream)
  }
  p->conn = c;
  p->is_write = is_write;
  std::lock_guard<std::mutex> g(mu_);
  const uint64_t id = next_prep_++;
  prepared_[id] = p;
  if (prep_id) *prep_id = id;
  return true;
}

bool Endpoint::post(uint64_t prep_id, uint64_t* tid) {
  std::shared_ptr<Prepared> p;
  cudaStream_t st;
  {
    std::lock_guard<std::mutex> g(mu_);
    auto it = prepared_.find(prep_id);
    if (it == prepared_.end()) return false;
    p = it->second;
    st = streams_[next_stream_++ % streams_.size()];
  }
  cudaSetDevice(gpu_);
  if (p->use_memcpy)
    for (size_t i = 0; i < p->src.size(); ++i)
      if (cudaMemcpyAsync(p->dst[i], p->src[i], p->sizes[i], cudaMemcpyDefault, st) != cudaSuccess) return false;
  for (auto& l : p->launches) {
    cudaError_t e = launch_p2p_copy(l.b, l.grid, st);
    if (e != cudaSuccess) {
      UB_WARN("p2p copy kernel launch failed: %s", cudaGetErrorString(e));
      return false;
    }
  }
  auto t = std::make_shared<Transfer>();
  t->conn = p->conn;
  t->state = Transfer::COPYING;
  t->ev = new_event();
  if (cudaEventRecord(t->ev, st) != cudaSuccess) return false;
  std::lock_guard<std::mutex> g(mu_);
  t->id = next_tid_++;
  transfers_[t->id] = t;
  stats_.transfers++;
  stats_.kernel_launches += p->launches.size();
  (p->is_write ? stats_.bytes_written : stats_.bytes_read) += p->bytes;
  if (tid) *tid = t->id;
  return true;
}

bool Endpoint::release(uint64_t prep_id) {
  std::shared_ptr<Prepared> p;
  {
    std::lock_guard<std::mutex> g(mu_);
    auto it = prepared_.find(prep_id);
    if (it == prepared_.end()) return false;
    p = it->second;
    prepared_.erase(it);
  }
  // launches that still read the tables must finish before the tables are reused
  for (auto st : streams_) cudaStreamSynchronize(st);
  for (auto& l : p->launches)
    if (l.tab) release_table_cb(l.tab);
  return true;
}

bool Endpoint::launch_copy(const std::vector<const char*>& src, const std::vector<char*>& dst,
                           const std::vector<size_t>& sizes, cudaEvent_t ev) {
  if (gpu_ < 0) {
    for (size_t i = 0; i < src.size(); ++i) memmove(dst[i], src[i], sizes[i]);
    std::lock_guard<std::mutex> g(mu_);
    stats_.memcpy_fallbacks += src.size();
    return true;  // complete: transfers carry no event in host mode
  }
  cudaStream_t st;
  {
    std::lock_guard<std::mutex> g(mu_);
    st = streams_[next_stream_++ % streams_.size()];
  }
  const size_t n = src.size();
  bool any_host = false;
  for (size_t i = 0; i < n && !any_host; ++i) any_host = !is_device_ptr(src[i]) || !is_device_ptr(dst[i]);
  bool few_large = n <= 8 && ubParamP2PMemcpyMinMB() > 0;
  for (size_t i = 0; i < n && few_large; ++i) few_large = sizes[i] >= ((size_t)ubParamP2PMemcpyMinMB() << 20);
  if (any_host || few_large || !ubParamP2PUseKernel()) {
    for (size_t i = 0; i < n; ++i)
      if (cudaMemcpyAsync(dst[i], src[i], sizes[i], cudaMemcpyDefault, st) != cudaSuccess) return false;
    std::lock_guard<std::mutex> g(mu_);
    stats_.memcpy_fallbacks += n;
  } else {
    std::vector<CopyLaunch> ls;
    if (!build_launches(src, dst, sizes, &ls, st)) return false;
    for (auto& l : ls) {
      cudaError_t e = launch_p2p_copy(l.b, l.grid, st);
      if (e != cudaSuccess) {
        UB_WARN("p2p copy kernel launch failed: %s", cudaGetErrorString(e));
        for (auto& r : ls)
          if (r.tab) release_table_cb(r.tab);
        return false;
      }
      if (l.tab && cudaLaunchHostFunc(st, release_table_cb, l.tab) != cudaSuccess) {
        (void)cudaGetLastError();  // could not enqueue the callback: drain the stream and recycle by hand
        cudaStreamSynchronize(st);
        release_table_cb(l.tab);
      }
      l.tab = nullptr;
      std::lock_guard<std::mutex> g(mu_);
      stats_.kernel_launches++;
    }
  }
  return cudaEventRecord(ev, st) == cudaSuccess;
}

Endpoint::DescTable* Endpoint::acquire_table() {
  {
    std::lock_guard<std::mutex> g(mu_);
    if (!table_pool_.empty()) {
      DescTable* t = table_pool_.back();
      table_pool_.pop_back();
      return t;
    }
  }
  auto* t = new DescTable();
  t->owner = this;
  const size_t bytes = sizeof(P2PCopyEntry) * kP2PTableEntries + sizeof(uint32_t) * (kP2PTableEntries + 1);
  if (cudaHostAlloc(&t->host, bytes, cudaHostAllocDefault) != cudaSuccess || cudaMalloc(&t->dev, bytes) != cudaSuccess) {
    (void)cudaGetLastError();
    if (t->host) cudaFreeHost(t->host);
    delete t;
    UB_WARN("p2p: could not allocate a pinned descriptor table");
    return nullptr;
  }
  std::lock_guard<std::mutex> g(mu_);
  tables_all_.push_back(t);
  return t;
}

void Endpoint::release_table_cb(void* p) {
  auto* t = (DescTable*)p;
  std::lock_guard<std::mutex> g(t->owner->mu_);
  t->owner->table_pool_.push_back(t);
}

static cudaEvent_t new_event() {
  cudaEvent_t e = nullptr;
  cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
  return e;
}

bool Endpoint::send_async(uint64_t conn, const std::vector<const void*>& ptrs, const std::vector<size_t>& sizes,
                          uint64_t* tid) {
  auto c = find_conn(conn);
  if (!c || ptrs.size() != sizes.size() || ptrs.empty()) return false;
  for (size_t s : sizes)
    if (s > 0xffffffffull * 16) return false;
  auto t = std::make_shared<Transfer>();
  t->conn = c;
  t->state = Transfer::SEND_WAIT_ADV;
  t->notify_done = true;
  for (auto p : ptrs) t->src.push_back((const char*)p);
  t->sizes = sizes;
  {
    std::lock_guard<std::mutex> g(mu_);
    t->seq = c->next_send_seq++;
    t->id = next_tid_++;
    transfers_[t->id] = t;
    stats_.transfers++;
    for (size_t s : sizes) stats_.bytes_sent += s;
  }
  if (tid) *tid = t->id;
  wake();
  return true;
}

bool Endpoint::recv_async(uint64_t conn, const std::vector<void*>& ptrs, const std::vector<size_t>& sizes,
                          uint64_t* tid) {
  auto c = find_conn(conn);
  if (!c || ptrs.size() != sizes.size() || ptrs.empty()) return false;
  std::vector<XferDesc> descs(ptrs.size());
  for (size_t i = 0; i < ptrs.size(); ++i)
    if (!describe(ptrs[i], sizes[i], &descs[i])) return false;
  auto t = std::make_shared<Transfer>();
  t->conn = c;
  t->state = Transfer::RECV_WAIT_DONE;
  t->sizes = sizes;
  {
    std::lock_guard<std::mutex> g(mu_);
    t->seq = c->next_recv_seq++;
    t->id = next_tid_++;
    transfers_[t->id] = t;
    stats_.transfers++;
    for (size_t s : sizes) stats_.bytes_received += s;
  }
  if (!send_msg(*c, MSG_ADV, t->seq, descs.data(), (uint32_t)(descs.size() * sizeof(XferDesc)))) return false;
  if (tid) *tid = t->id;
  wake();
  return true;
}

bool Endpoint::write_async(uint64_t conn, const std::vector<const void*>& src, const std::vector<size_t>& sizes,
                           const std::vector<XferDesc>& remote, uint64_t* tid) {
  auto c = find_conn(conn);
  if (!c || src.size() != sizes.size() || src.size() != remote.size() || src.empty()) return false;
  if (remote_is_other_process(remote[0])) {
    // TCP data path: the caller's thread streams the payload, then asks for an acknowledgement
    std::vector<const char*> sp;
    std::vector<uint64_t> da;
    for (size_t i = 0; i < src.size(); ++i) {
      if (sizes[i] > remote[i].size) return false;
      sp.push_back((const char*)src[i]);
      da.push_back(remote[i].addr);
    }
    auto t = std::make_shared<Transfer>();
    t->conn = c;
    t->state = Transfer::WAIT_ACK;
    {
      std::lock_guard<std::mutex> g(mu_);
      t->id = next_tid_++;
      transfers_[t->id] = t;
      stats_.transfers++;
      for (size_t b : sizes) stats_.bytes_written += b;
    }
    if (!tcp_write_buffers(*c, sp, da, sizes) || !send_msg(*c, MSG_FLUSH, t->id, nullptr, 0)) {
      std::lock_guard<std::mutex> g(mu_);
      transfers_.erase(t->id);
      return false;
    }
    if (tid) *tid = t->id;
    return true;
  }
  if (gpu_ >= 0) cudaSetDevice(gpu_);
  std::vector<const char*> s;
  std::vector<char*> d;
  for (size_t i = 0; i < src.size(); ++i) {
    if (sizes[i] > remote[i].size) return false;
    void* r = map_remote(remote[i]);
    if (!r) return false;
    s.push_back((const char*)src[i]);
    d.push_back((char*)r);
  }
  auto t = std::make_shared<Transfer>();
  t->conn = c;
  t->state = Transfer::COPYING;
  t->ev = gpu_ >= 0 ? new_event() : nullptr;
  if (!launch_copy(s, d, sizes, t->ev)) return false;
  std::lock_guard<std::mutex> g(mu_);
  t->id = next_tid_++;
  transfers_[t->id] = t;
  stats_.transfers++;
  for (size_t b : sizes) stats_.bytes_written += b;
  if (tid) *tid = t->id;
  return true;
}

bool Endpoint::read_async(uint64_t conn, const std::vector<void*>& dst, const std::vector<size_t>& sizes,
                          const std::vector<XferDesc>& remote, uint64_t* tid) {
  auto c = find_conn(conn);
  if (!c || dst.size() != sizes.size() || dst.size() != remote.size() || dst.empty()) return false;
  if (remote_is_other_process(remote[0])) {
    std::vector<uint64_t> req;
    auto t = std::make_shared<Transfer>();
    for (size_t i = 0; i < dst.size(); ++i) {
      if (sizes[i] > remote[i].size) return false;
      req.push_back(remote[i].addr);
      req.push_back(sizes[i]);
      t->dst.push_back((char*)dst[i]);
    }
    t->conn = c;
    t->sizes = sizes;
    t->state = Transfer::WAIT_RESP;
    {
      std::lock_guard<std::mutex> g(mu_);
      t->id = next_tid_++;
      transfers_[t->id] = t;
      stats_.transfers++;
      for (size_t b : sizes) stats_.bytes_read += b;
    }
    if (!send_msg(*c, MSG_READ_REQ, t->id, req.data(), (uint32_t)(req.size() * sizeof(uint64_t)))) {
      std::lock_guard<std::mutex> g(mu_);
      transfers_.erase(t->id);
      return false;
    }
    if (tid) *tid = t->id;
    return true;
  }
  if (gpu_ >= 0) cudaSetDevice(gpu_);
  std::vector<const char*> s;
  std::vector<char*> d;
  for (size_t i = 0; i < dst.size(); ++i) {
    if (sizes[i] > remote[i].size) return false;
    void* r = map_remote(remote[i]);
    if (!r) return false;
    s.push_back((const char*)r);
    d.push_back((char*)dst[i]);
  }
  auto t = std::make_shared<Transfer>();
  t->conn = c;
  t->state = Transfer::COPYING;
  t->ev = gpu_ >= 0 ? new_event() : nullptr;
  if (!launch_copy(s, d, sizes, t->ev)) return false;
  std::lock_guard<std::mutex> g(mu_);
  t->id = next_tid_++;
  transfers_[t->id] = t;
  stats_.transfers++;
  for (size_t b : sizes) stats_.bytes_read += b;
  if (tid) *tid = t->id;
  return true;
}

bool Endpoint::poll_async(uint64_t tid, bool* done) {
  std::shared_ptr<Transfer> t;
  {
    std::lock_guard<std::mutex> g(mu_);
    auto it = transfers_.find(tid);
    if (it == transfers_.end()) return false;
    t = it->second;
  }
  if (t->state == Transfer::WAIT_ACK) {
    std::lock_guard<std::mutex> g(mu_);
    auto it = t->conn->acks.find(tid);
    if (it != t->conn->acks.end()) {
      t->conn->acks.erase(it);
      t->state = Transfer::DONE;
    } else if (!t->conn->alive) {
      t->state = Transfer::FAILED;
    }
  }
  if (t->state == Transfer::COPYING && !t->notify_done) {
    // one-sided ops are driven by the caller: no engine-thread latency on the hot path
    cudaError_t q = t->ev ? cudaEventQuery(t->ev) : cudaSuccess;
    if (q == cudaSuccess) t->state = Transfer::DONE;
    else if (q != cudaErrorNotReady) t->state = Transfer::FAILED;
    (void)cudaGetLastError();
  }
  const bool fin = t->state == Transfer::DONE || t->state == Transfer::FAILED;
  if (done) *done = fin;
  if (fin) {
    std::lock_guard<std::mutex> g(mu_);
    transfers_.erase(tid);
    if (t->ev) cudaEventDestroy(t->ev);
    t->ev = nullptr;
    return t->state == Transfer::DONE;
  }
  return true;
}

bool Endpoint::wait(uint64_t tid, int timeout_ms) {
  auto t0 = std::chrono::steady_clock::now();
  bool done = false;
  uint32_t spins = 0;
  while (true) {
    if (!poll_async(tid, &done)) return false;
    if (done) return true;
    if ((++spins & 0x3f) == 0) {
      if (timeout_ms >= 0 &&
          std::chrono::steady_clock::now() - t0 > std::chrono::milliseconds(timeout_ms))
        return false;
      std::this_thread::yield();
    }
  }
}

bool Endpoint::send_notif(uint64_t conn, const std::string& msg) {
  auto c = find_conn(conn);
  if (!c) return false;
  return send_msg(*c, MSG_NOTIF, 0, msg.data(), (uint32_t)msg.size());
}

std::vector<std::pair<uint64_t, std::string>> Endpoint::get_notifs() {
  std::lock_guard<std::mutex> g(mu_);
  std::vector<std::pair<uint64_t, std::string>> out(notifs_.begin(), notifs_.end());
  notifs_.clear();
  return out;
}

P2PStats Endpoint::stats() const {
  std::lock_guard<std::mutex> g(mu_);
  return stats_;
}

// ------------------------------------------------------------------ engine thread
void Endpoint::handle_message(Conn& c, uint32_t type, uint64_t seq, std::vector<char>& payload) {
  std::lock_guard<std::mutex> g(mu_);
  switch (type) {
    case MSG_ADV: {
      std::vector<XferDesc> d(payload.size() / sizeof(XferDesc));
      memcpy(d.data(), payload.data(), d.size() * sizeof(XferDesc));
      c.advs[seq] = std::move(d);
      break;
    }
    case MSG_DONE: c.dones[seq] = true; break;
    case MSG_WRITE: {
      if (payload.size() < 16) break;
      uint64_t pre[2];
      memcpy(pre, payload.data(), 16);
      if (pre[1] != payload.size() - 16) break;
      if (!is_exposed(pre[0], pre[1])) {
        UB_LOG_FIRST_N(5, LOG_WARN, SUB_P2P, "p2p: peer tried to write %llu bytes outside every exposed window: ignored",
                       (unsigned long long)pre[1]);
        break;
      }
      copy_any((void*)pre[0], payload.data() + 16, pre[1]);
      break;
    }
    case MSG_FLUSH: {
      // frames are processed in order, so every WRITE sent before this FLUSH has been applied
      MsgHdr h{MSG_FLUSH_ACK, 0, seq};
      std::lock_guard<std::mutex> sg(c.send_mu);
      if (c.fd >= 0) write_full(c.fd, &h, sizeof(h));
      break;
    }
    case MSG_FLUSH_ACK: c.acks[seq] = true; break;
    case MSG_READ_REQ: {
      const size_t nb = payload.size() / 16;
      auto data = std::make_shared<std::vector<char>>();
      for (size_t i = 0; i < nb; ++i) {
        uint64_t e[2];
        memcpy(e, payload.data() + i * 16, 16);
        if (!is_exposed(e[0], e[1])) {  // the short response makes the requester's transfer fail
          UB_LOG_FIRST_N(5, LOG_WARN, SUB_P2P, "p2p: peer tried to read outside every exposed window: refused");
          data->clear();
          break;
        }
        const size_t at = data->size();
        data->resize(at + e[1]);
        copy_any(data->data() + at, (const void*)e[0], e[1]);
      }
      std::shared_ptr<Conn> conn;
      for (auto& kv : conns_)
        if (kv.second.get() == &c) conn = kv.second;
      if (conn) run_helper([this, conn, data, seq] { send_msg(*conn, MSG_READ_RESP, seq, data->data(), (uint32_t)data->size()); });
      break;
    }
    case MSG_READ_RESP: {
      auto it = transfers_.find(seq);
      if (it == transfers_.end() || it->second->state != Transfer::WAIT_RESP) break;
      auto& t = it->second;
      size_t at = 0;
      bool ok = true;
      for (size_t i = 0; i < t->dst.size() && ok; ++i) {
        if (at + t->sizes[i] > payload.size()) ok = false;
        else copy_any(t->dst[i], payload.data() + at, t->sizes[i]);
        at += t->sizes[i];
      }
      t->state = ok ? Transfer::DONE : Transfer::FAILED;
      break;
    }
    case MSG_NOTIF: notifs_.emplace_back(c.id, std::string(payload.begin(), payload.end())); break;
    case MSG_BYE: c.alive = false; break;
    default: break;
  }
}

void Endpoint::progress_locked() {
  // called with mu_ held
  for (auto& kv : transfers_) {
    auto t = kv.second;
    Conn& c = *t->conn;
    switch (t->state) {
      case Transfer::SEND_WAIT_ADV: {
        auto it = c.advs.find(t->seq);
        if (it == c.advs.end()) {
          if (!c.alive) t->state = Transfer::FAILED;
          break;
        }
        std::vector<XferDesc> descs = std::move(it->second);
        c.advs.erase(it);
        if (descs.size() != t->src.size()) {
          UB_WARN("p2p send: receiver posted %zu buffers, sender has %zu", descs.size(), t->src.size());
          t->state = Transfer::FAILED;
          break;
        }
        if (remote_is_other_process(descs[0])) {
          // TCP data path: a helper thread streams the payload (the engine thread must keep reading),
          // then tells the receiver that the message is complete
          for (size_t i = 0; i < descs.size(); ++i)
            if (descs[i].size < t->sizes[i]) {
              t->state = Transfer::FAILED;
              break;
            }
          if (t->state == Transfer::FAILED) break;
          t->state = Transfer::TCP_SENDING;
          std::vector<uint64_t> da;
          for (auto& d : descs) da.push_back(d.addr);
          auto conn = t->conn;
          run_helper([this, t, conn, da] {
            bool ok = tcp_write_buffers(*conn, t->src, da, t->sizes) && send_msg(*conn, MSG_DONE, t->seq, nullptr, 0);
            std::lock_guard<std::mutex> g(mu_);
            t->state = ok ? Transfer::DONE : Transfer::FAILED;
          });
          break;
        }
        std::vector<char*> dst;
        bool ok = true;
        mu_.unlock();  // map_remote / launch_copy take mu_ themselves
        for (size_t i = 0; i < descs.size() && ok; ++i) {
          if (descs[i].size < t->sizes[i]) ok = false;
          void* r = ok ? map_remote(descs[i]) : nullptr;
          if (!r) ok = false;
          dst.push_back((char*)r);
        }
        cudaEvent_t ev = (ok && gpu_ >= 0) ? new_event() : nullptr;
        if (ok) ok = launch_copy(t->src, dst, t->sizes, ev);
        mu_.lock();
        t->ev = ev;
        t->state = ok ? Transfer::COPYING : Transfer::FAILED;
        return;  // tables may have changed while unlocked: restart the scan next tick
      }
      case Transfer::COPYING: {
        if (!t->notify_done) break;  // caller-driven
        cudaError_t q = t->ev ? cudaEventQuery(t->ev) : cudaSuccess;
        if (q == cudaSuccess) {
          mu_.unlock();
          bool ok = send_msg(c, MSG_DONE, t->seq, nullptr, 0);
          mu_.lock();
          t->state = ok ? Transfer::DONE : Transfer::FAILED;
          return;
        } else if (q != cudaErrorNotReady) {
          (void)cudaGetLastError();
          t->state = Transfer::FAILED;
        }
        break;
      }
      case Transfer::RECV_WAIT_DONE: {
        auto it = c.dones.find(t->seq);
        if (it != c.dones.end()) {
          c.dones.erase(it);
          t->state = Transfer::DONE;
        } else if (!c.alive) {
          t->state = Transfer::FAILED;
        }
        break;
      }
      default: break;
    }
  }
}

void Endpoint::engine_loop() {
  if (gpu_ >= 0) cudaSetDevice(gpu_);
  const int64_t stats_sec = ubParamP2PStatsSec();
  auto last_stats = std::chrono::steady_clock::now();
  while (!stop_) {
    if (stats_sec > 0 && std::chrono::steady_clock::now() - last_stats >= std::chrono::seconds(stats_sec)) {
      last_stats = std::chrono::steady_clock::now();
      std::lock_guard<std::mutex> g(mu_);
      UB_INFO(SUB_P2P,
              "p2p engine gpu %d: %zu conns, %zu transfers in flight, %llu done, sent %llu B, recv %llu B, written "
              "%llu B, read %llu B, %llu kernel launches, %llu memcpy fallbacks",
              gpu_, conns_.size(), transfers_.size(), (unsigned long long)stats_.transfers,
              (unsigned long long)stats_.bytes_sent, (unsigned long long)stats_.bytes_received,
              (unsigned long long)stats_.bytes_written, (unsigned long long)stats_.bytes_read,
              (unsigned long long)stats_.kernel_launches, (unsigned long long)stats_.memcpy_fallbacks);
    }
    std::vector<pollfd> fds;
    std::vector<std::shared_ptr<Conn>> cs;
    bool active = false;
    {
      std::lock_guard<std::mutex> g(mu_);
      retire_closed_locked();  // nothing of this thread is reading those descriptors now
      for (auto& kv : conns_)
        if (kv.second->fd >= 0 && kv.second->alive) {
          fds.push_back({kv.second->fd, POLLIN, 0});
          cs.push_back(kv.second);
        }
      for (auto& kv : transfers_)
        if (kv.second->state == Transfer::SEND_WAIT_ADV || kv.second->state == Transfer::RECV_WAIT_DONE ||
            (kv.second->state == Transfer::COPYING && kv.second->notify_done))
          active = true;
    }
    const size_t nconn = fds.size();
    fds.push_back({listen_fd_, POLLIN, 0});
    fds.push_back({wake_fd_, POLLIN, 0});
    int rc = ::poll(fds.data(), fds.size(), active ? 0 : 20);
    if (rc > 0) {
      for (size_t i = 0; i < nconn; ++i) {
        if (!(fds[i].revents & (POLLIN | POLLHUP | POLLERR))) continue;
        MsgHdr h;
        if (!read_full(cs[i]->fd, &h, sizeof(h))) {
          cs[i]->alive = false;
          continue;
        }
        std::vector<char> payload(h.len);
        if (h.len && !read_full(cs[i]->fd, payload.data(), h.len)) {
          cs[i]->alive = false;
          continue;
        }
        handle_message(*cs[i], h.type, h.seq, payload);
      }
      if (fds[nconn].revents & POLLIN) {
        sockaddr_in pa;
        socklen_t pl = sizeof(pa);
        int fd = ::accept(listen_fd_, (sockaddr*)&pa, &pl);
        if (fd >= 0) {
          int one = 1;
          setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof(one));
          MsgHdr h;
          Hello peer;
          if (read_full(fd, &h, sizeof(h)) && h.type == MSG_HELLO && read_full(fd, &peer, sizeof(peer))) {
            MsgHdr rh{MSG_HELLO, sizeof(Hello), 0};
            Hello me{gpu_, (int32_t)getpid()};
            write_full(fd, &rh, sizeof(rh));
            write_full(fd, &me, sizeof(me));
            auto c = std::make_shared<Conn>();
            c->fd = fd;
            c->remote_gpu = peer.gpu;
            c->remote_pid = peer.pid;
            char buf[INET_ADDRSTRLEN];
            inet_ntop(AF_INET, &pa.sin_addr, buf, sizeof(buf));
            c->ip = buf;
            std::lock_guard<std::mutex> g(mu_);
            c->id = next_conn_++;
            conns_[c->id] = c;
            accepted_.push_back(c->id);
            accept_cv_.notify_all();
          } else {
            ::close(fd);
          }
        }
      }
      if (fds[nconn + 1].revents & POLLIN) {
        uint64_t v;
        (void)!::read(wake_fd_, &v, sizeof(v));
      }
    }
    {
      std::lock_guard<std::mutex> g(mu_);
      progress_locked();
    }
  }
  accept_cv_.notify_all();
}

}  // namespace ub
