// NCCL network plugin (ncclNet v8 ABI) on top of the multipath datagram transport.
//
// Role in the reference: collective/rdma/nccl_plugin.cc:85-633 (and the afxdp / efa twins) -- the object
// NCCL loads through NCCL_NET_PLUGIN so that inter-node rings/trees run over UCCL's transport.  Inside a
// H100 NVSwitch box NCCL never calls a net plugin; between boxes this one carries the traffic:
//
//   NCCL_NET_PLUGIN=uccl_b200 LD_LIBRARY_PATH=$(python -c 'import uccl_b200;print(uccl_b200.lib_dir())') ...
//
// The ABI structs below are declared from the documented v8 layout (ext-net), not included from NCCL:
// this file has no build dependency on NCCL or CUDA.  Buffers are host pointers (NCCL_PTR_HOST): NCCL
// stages GPU data through its own pinned FIFOs, which is also what its socket transport does.
#include <arpa/inet.h>
#include <limits.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "net_engine.h"

extern "C" {
typedef enum {
  ncclSuccess = 0,
  ncclUnhandledCudaError = 1,
  ncclSystemError = 2,
  ncclInternalError = 3,
  ncclInvalidArgument = 4,
  ncclInvalidUsage = 5,
  ncclRemoteError = 6,
  ncclInProgress = 7
} ncclResult_t;
typedef enum {
  NCCL_LOG_NONE = 0,
  NCCL_LOG_VERSION = 1,
  NCCL_LOG_WARN = 2,
  NCCL_LOG_INFO = 3,
  NCCL_LOG_ABORT = 4,
  NCCL_LOG_TRACE = 5
} ncclDebugLogLevel;
typedef void (*ncclDebugLogger_t)(ncclDebugLogLevel level, unsigned long flags, const char* file, int line,
                                  const char* fmt, ...);
typedef enum { NCCL_NET_DEVICE_HOST = 0, NCCL_NET_DEVICE_UNPACK = 1 } ncclNetDeviceType;
typedef struct ncclNetDeviceHandle_v8 ncclNetDeviceHandle_v8_t;

typedef struct {       // layout of ncclNetProperties_v8_t (field names are ours; only the layout is ABI)
  char* dev_name;
  char* pci_path;
  uint64_t chip_guid;
  int ptr_kinds;         // NCCL_PTR_* bit mask
  int mr_is_global;
  int speed_mbps;
  int port_num;
  float latency_us;
  int max_comms;
  int max_grouped_recvs;
  ncclNetDeviceType offload_type;
  int offload_version;
} ncclNetProperties_v8_t;

typedef struct {       // ncclNet_v8_t: 19 entries in this order
  const char* plugin_name;
  ncclResult_t (*fn_init)(ncclDebugLogger_t);
  ncclResult_t (*fn_devices)(int*);
  ncclResult_t (*fn_properties)(int, ncclNetProperties_v8_t*);
  ncclResult_t (*fn_listen)(int, void*, void**);
  ncclResult_t (*fn_connect)(int, void*, void**, ncclNetDeviceHandle_v8_t**);
  ncclResult_t (*fn_accept)(void*, void**, ncclNetDeviceHandle_v8_t**);
  ncclResult_t (*fn_reg_mr)(void*, void*, size_t, int, void**);
  ncclResult_t (*fn_reg_mr_dmabuf)(void*, void*, size_t, int, uint64_t, int, void**);
  ncclResult_t (*fn_dereg_mr)(void*, void*);
  ncclResult_t (*fn_isend)(void*, void*, int, int, void*, void**);
  ncclResult_t (*fn_irecv)(void*, int, void**, int*, int*, void**, void**);
  ncclResult_t (*fn_iflush)(void*, int, void**, int*, void**, void**);
  ncclResult_t (*fn_test)(void*, int*, int*);
  ncclResult_t (*fn_close_send)(void*);
  ncclResult_t (*fn_close_recv)(void*);
  ncclResult_t (*fn_close_listen)(void*);
  ncclResult_t (*fn_device_mr)(void*, void*, void**);
  ncclResult_t (*fn_recv_consumed)(void*, int, void*);
} ncclNet_v8_t;
}

#define NCCL_PTR_HOST 0x1
#define NCCL_NET_HANDLE_MAXSIZE 128
#define NCCL_NET_SUBSYS 16ul

namespace {
using ub::net::Engine;
using ub::net::EngineConfig;

struct Device {
  std::string name, ip, pci;
  int speed_mbps = 10000;
  std::unique_ptr<Engine> engine;
};
struct Handle {  // what travels to the peer (<= NCCL_NET_HANDLE_MAXSIZE); the tail is connect()'s scratch
  uint32_t magic;
  uint32_t ip_be;
  uint16_t port;
  uint16_t pad;
  uint32_t listen_id;
  uint32_t stage_flow;  // connect in progress (NCCL re-calls connect with the same handle memory)
};
static_assert(sizeof(Handle) <= NCCL_NET_HANDLE_MAXSIZE, "handle too large");
struct ListenComm {
  int dev;
  uint32_t listen_id;
};
struct Comm {
  int dev;
  uint32_t flow;
  bool send;
};
struct Req {
  Engine* eng;
  ub::net::Request* r;
};

std::mutex g_mu;
std::vector<Device> g_devs;
ncclDebugLogger_t g_log = nullptr;

#define PLOG(level, ...)                                                          \
  do {                                                                            \
    if (g_log) g_log(level, NCCL_NET_SUBSYS, __FILE__, __LINE__, __VA_ARGS__);    \
  } while (0)

Engine* engine_of(int dev) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (dev < 0 || dev >= (int)g_devs.size()) return nullptr;
  Device& d = g_devs[dev];
  if (!d.engine) {
    EngineConfig c = EngineConfig::from_env();
    c.bind_ip = d.ip;
    if (d.speed_mbps > 0) c.link_gbps = d.speed_mbps / 1000.0;
    d.engine.reset(new Engine(c));
  }
  return d.engine.get();
}

ncclResult_t p_init(ncclDebugLogger_t logf) {
  g_log = logf;
  std::lock_guard<std::mutex> lk(g_mu);
  if (!g_devs.empty()) return ncclSuccess;
  for (auto& kv : ub::net::list_interfaces()) {
    Device d;
    d.name = kv.first;
    d.ip = kv.second;
    char path[PATH_MAX], real[PATH_MAX];
    snprintf(path, sizeof(path), "/sys/class/net/%s/device", d.name.c_str());
    if (realpath(path, real)) d.pci = real;
    snprintf(path, sizeof(path), "/sys/class/net/%s/speed", d.name.c_str());
    if (FILE* f = fopen(path, "r")) {
      int v = 0;
      if (fscanf(f, "%d", &v) == 1 && v > 0) d.speed_mbps = v;
      fclose(f);
    }
    g_devs.push_back(std::move(d));
  }
  PLOG(NCCL_LOG_INFO, "NET/uccl_b200: %zu device(s), multipath datagram transport", g_devs.size());
  return g_devs.empty() ? ncclSystemError : ncclSuccess;
}

ncclResult_t p_devices(int* ndev) {
  std::lock_guard<std::mutex> lk(g_mu);
  *ndev = (int)g_devs.size();
  return ncclSuccess;
}

ncclResult_t p_props(int dev, ncclNetProperties_v8_t* p) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (dev < 0 || dev >= (int)g_devs.size()) return ncclInvalidArgument;
  Device& d = g_devs[dev];
  memset(p, 0, sizeof(*p));
  p->dev_name = const_cast<char*>(d.name.c_str());
  p->pci_path = d.pci.empty() ? nullptr : const_cast<char*>(d.pci.c_str());
  p->chip_guid = (uint64_t)dev;
  p->ptr_kinds = NCCL_PTR_HOST;
  p->mr_is_global = 0;
  p->speed_mbps = d.speed_mbps;
  p->port_num = 0;
  p->latency_us = 0;
  p->max_comms = 65536;
  p->max_grouped_recvs = 1;
  p->offload_type = NCCL_NET_DEVICE_HOST;
  p->offload_version = 0;
  return ncclSuccess;
}

ncclResult_t p_listen(int dev, void* handle, void** listenComm) {
  Engine* e = engine_of(dev);
  if (!e) return ncclInvalidArgument;
  Handle h{};
  h.magic = ub::net::kMagic;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    inet_pton(AF_INET, g_devs[dev].ip.c_str(), &h.ip_be);
  }
  h.port = e->port();
  h.listen_id = e->listen();
  memset(handle, 0, NCCL_NET_HANDLE_MAXSIZE);
  memcpy(handle, &h, sizeof(h));
  *listenComm = new ListenComm{dev, h.listen_id};
  return ncclSuccess;
}

ncclResult_t p_connect(int dev, void* handle, void** sendComm, ncclNetDeviceHandle_v8_t** /*sendDevComm*/) {
  Engine* e = engine_of(dev);
  if (!e) return ncclInvalidArgument;
  Handle* h = static_cast<Handle*>(handle);
  if (h->magic != ub::net::kMagic) return ncclInvalidArgument;
  *sendComm = nullptr;
  if (h->stage_flow == 0) {
    char ip[INET_ADDRSTRLEN];
    inet_ntop(AF_INET, &h->ip_be, ip, sizeof(ip));
    try {
      h->stage_flow = e->connect_async(ip, h->port, h->listen_id);
    } catch (const std::exception& ex) {
      PLOG(NCCL_LOG_WARN, "NET/uccl_b200: connect: %s", ex.what());
      return ncclSystemError;
    }
  }
  const int st = e->flow_state(h->stage_flow);
  if (st == ub::net::FL_ESTABLISHED) {
    *sendComm = new Comm{dev, h->stage_flow, true};
    h->stage_flow = 0;
    return ncclSuccess;
  }
  if (st == ub::net::FL_SYN_SENT) return ncclSuccess;  // not yet: NCCL calls again
  PLOG(NCCL_LOG_WARN, "NET/uccl_b200: connect failed (flow state %d)", st);
  return ncclRemoteError;
}

ncclResult_t p_accept(void* listenComm, void** recvComm, ncclNetDeviceHandle_v8_t** /*recvDevComm*/) {
  ListenComm* l = static_cast<ListenComm*>(listenComm);
  Engine* e = engine_of(l->dev);
  *recvComm = nullptr;
  uint32_t flow = 0;
  if (e->accept_nb(l->listen_id, &flow)) *recvComm = new Comm{l->dev, flow, false};
  return ncclSuccess;
}

ncclResult_t p_regmr(void* /*comm*/, void* /*data*/, size_t /*size*/, int type, void** mhandle) {
  if (type != NCCL_PTR_HOST) return ncclInternalError;
  *mhandle = reinterpret_cast<void*>(uintptr_t(1));  // sockets need no registration
  return ncclSuccess;
}
ncclResult_t p_regmr_dmabuf(void*, void*, size_t, int, uint64_t, int, void**) { return ncclInternalError; }
ncclResult_t p_deregmr(void*, void*) { return ncclSuccess; }

ncclResult_t p_isend(void* sendComm, void* data, int size, int /*tag*/, void* /*mhandle*/, void** request) {
  Comm* c = static_cast<Comm*>(sendComm);
  Engine* e = engine_of(c->dev);
  *request = new Req{e, e->send_async(c->flow, data, (size_t)size)};
  return ncclSuccess;
}

ncclResult_t p_irecv(void* recvComm, int n, void** data, int* sizes, int* /*tags*/, void** /*mhandles*/, void** request) {
  if (n != 1) return ncclInternalError;
  Comm* c = static_cast<Comm*>(recvComm);
  Engine* e = engine_of(c->dev);
  *request = new Req{e, e->recv_async(c->flow, data[0], (size_t)sizes[0])};
  return ncclSuccess;
}

ncclResult_t p_iflush(void*, int, void**, int*, void**, void** request) {
  *request = nullptr;  // host memory: nothing to flush
  return ncclSuccess;
}

ncclResult_t p_test(void* request, int* done, int* sizes) {
  Req* q = static_cast<Req*>(request);
  size_t bytes = 0;
  int err = 0;
  *done = 0;
  if (!q->eng->test(q->r, &bytes, &err)) return ncclSuccess;
  *done = 1;
  if (sizes) sizes[0] = (int)bytes;
  delete q;
  if (err) {
    const char* why = err == 2 ? "message larger than the receive" : err == 3 ? "peer closed" : "flow error";
    PLOG(NCCL_LOG_WARN, "NET/uccl_b200: request failed (%s)", why);
    return ncclRemoteError;
  }
  return ncclSuccess;
}

ncclResult_t p_close_comm(void* comm) {
  Comm* c = static_cast<Comm*>(comm);
  if (!c) return ncclSuccess;
  if (Engine* e = engine_of(c->dev)) e->close_flow(c->flow);
  delete c;
  return ncclSuccess;
}

ncclResult_t p_close_listen(void* listenComm) {
  ListenComm* l = static_cast<ListenComm*>(listenComm);
  if (!l) return ncclSuccess;
  if (Engine* e = engine_of(l->dev)) e->close_listen(l->listen_id);
  delete l;
  return ncclSuccess;
}
}  // namespace

extern "C" {
__attribute__((visibility("default"))) ncclNet_v8_t ncclNetPlugin_v8 = {
    "uccl_b200", p_init,  p_devices, p_props,      p_listen,     p_connect,      p_accept, p_regmr, p_regmr_dmabuf, p_deregmr,
    p_isend,     p_irecv, p_iflush,  p_test,       p_close_comm, p_close_comm,   p_close_listen,    nullptr,        nullptr,
};
}
