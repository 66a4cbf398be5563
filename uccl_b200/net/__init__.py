"""``uccl_b200.net`` -- the scale-OUT transport: multipath reliable datagrams between H100 boxes.

Inside one NVSwitch domain every peer is load/store reachable and nothing in this module is used.
Between boxes the reference's core contribution applies (SURVEY N2 "UCCL-Tran", N6/N7 the AF_XDP / DPDK
variants, N1 the NCCL net plugin): messages are chunked, sprayed over many paths picked by
power-of-two-choices, placed out of order at the receiver, and made reliable in software (SACK, RACK-style
fast retransmit, RTO) under a pluggable congestion controller (Swift / Timely / EQDS credits).  The native
engine is ``csrc/net/net_engine.{h,cc}`` (one thread per NIC, UDP sockets = paths); this module adds

* :class:`Engine`        tensor-level send / recv on flows
* :class:`NetCommunicator`  a rank group over the engine with ring / pairwise collectives on host
  (or pinned) tensors -- the inter-node half of :class:`uccl_b200.parallel.MultiNodeCommunicator`
* :func:`nccl_net_plugin_path`  the ``ncclNet_v8`` plugin built from the same engine

Reference: collective/rdma/transport.{h,cc}, collective/afxdp/transport.{h,cc}, collective/rdma/nccl_plugin.cc.
"""
from __future__ import annotations

import os
from typing import Callable, Dict, List, Optional, Sequence

import torch

from .._native import C

CC = {"none": 0, "swift": 1, "timely": 2, "eqds": 3}


def list_interfaces():
    """[(name, ipv4)] of the NICs the transport may use (``UCCL_B200_NET_IFNAME`` filters by prefix)."""
    return C().net.list_interfaces()


def nccl_net_plugin_path() -> str:
    from .. import _build

    return str(_build.nccl_net_plugin_path())


class Work:
    """Handle of one asynchronous send / recv; keeps the tensor alive until completion."""

    def __init__(self, engine: "Engine", req: int, tensor: Optional[torch.Tensor]):
        self._e, self._req, self._t = engine, req, tensor
        self.bytes: Optional[int] = None

    def done(self) -> bool:
        if self._req is None:
            return True
        r = self._e._native.test(self._req)
        if r is None:
            return False
        self._req = None
        self.bytes, err = r
        self._t = None
        if err:
            raise RuntimeError("net: request failed: " + {2: "message larger than the posted receive",
                                                          3: "peer closed the flow"}.get(err, "flow error"))
        return True

    def wait(self, timeout_ms: int = -1) -> int:
        if self._req is not None:
            req, self._req = self._req, None
            try:
                self.bytes = self._e._native.wait(req, timeout_ms)
            except RuntimeError as e:
                if "timed out" in str(e):
                    # the engine still owns the request and may yet read / write the buffer: keep both alive
                    # for the lifetime of the engine instead of letting the tensor be freed under it
                    self._e._zombies.append((req, self._t))
                raise
            finally:
                self._t = None
        return self.bytes


class _MultiWork:
    """Completion of a message that was striped over several engines."""

    def __init__(self, parts: List[Work]):
        self._parts = parts
        self.bytes: Optional[int] = None

    def done(self) -> bool:
        return all(p.done() for p in self._parts)

    def wait(self, timeout_ms: int = -1) -> int:
        self.bytes = sum(p.wait(timeout_ms) for p in self._parts)
        return self.bytes


class Engine:
    """One transport engine (= one NIC, one engine thread, ``paths`` UDP source ports)."""

    def __init__(self, bind_ip: str = "", paths: int = 0, payload: int = 0, max_inflight: int = 0, eager_max: int = -1,
                 cc: Optional[str] = None, drop_prob: float = -1.0, rto_min_us: int = 0, rto_abort: int = 0,
                 link_gbps: float = 0.0, busy_poll: bool = False):
        self._native = C().net.Engine(bind_ip, paths, payload, max_inflight, eager_max, CC[cc] if cc else -1, drop_prob,
                                      rto_min_us, rto_abort, link_gbps, busy_poll)
        self._zombies: List = []  # (request, tensor) pairs whose wait timed out; see Work.wait

    # ---- addressing / connections
    @property
    def port(self) -> int:
        return self._native.port

    @property
    def paths(self) -> int:
        return self._native.paths

    @property
    def address(self) -> str:
        ip = self._native.bind_ip
        if ip == "0.0.0.0":
            ifs = list_interfaces()
            ip = ifs[0][1] if ifs else "127.0.0.1"
        return ip

    def listen(self) -> int:
        return self._native.listen()

    def close_listen(self, listen_id: int) -> None:
        self._native.close_listen(listen_id)

    def connect(self, ip: str, port: int, listen_id: int, timeout_ms: int = 30000) -> int:
        return self._native.connect(ip, port, listen_id, timeout_ms)

    def accept(self, listen_id: int, timeout_ms: int = 30000) -> int:
        return self._native.accept(listen_id, timeout_ms)

    def close(self, flow: int) -> None:
        self._native.close_flow(flow)

    def flow_state(self, flow: int) -> int:
        return self._native.flow_state(flow)

    # ---- data
    @staticmethod
    def _check(t: torch.Tensor) -> None:
        if t.is_cuda:
            raise ValueError("net: pass a host (ideally pinned) tensor; GPU data is staged by the caller "
                             "(MultiNodeCommunicator does it)")
        if not t.is_contiguous():
            raise ValueError("net: tensor must be contiguous")

    def isend(self, flow: int, t: torch.Tensor) -> Work:
        self._check(t)
        return Work(self, self._native.send_async(flow, t.data_ptr(), t.numel() * t.element_size()), t)

    def irecv(self, flow: int, t: torch.Tensor) -> Work:
        self._check(t)
        return Work(self, self._native.recv_async(flow, t.data_ptr(), t.numel() * t.element_size()), t)

    def send(self, flow: int, t: torch.Tensor, timeout_ms: int = -1) -> None:
        self.isend(flow, t).wait(timeout_ms)

    def recv(self, flow: int, t: torch.Tensor, timeout_ms: int = -1) -> int:
        return self.irecv(flow, t).wait(timeout_ms)

    # ---- introspection / fault injection
    def set_drop_prob(self, p: float) -> None:
        self._native.set_drop_prob(p)

    def set_reorder(self, prob: float, delay_us: int = 300) -> None:
        """Fault injection: hold back this fraction of the outgoing datagrams for ``delay_us`` (reordering)."""
        self._native.set_reorder(prob, delay_us)

    def set_path_drop(self, path: int, prob: float = 1.0) -> None:
        """Fault injection: black-hole one local path (``path < 0`` clears)."""
        self._native.set_path_drop(path, prob)

    def stats(self) -> Dict:
        return self._native.stats()

    def flow_stats(self, flow: int) -> Optional[Dict]:
        return self._native.flow_stats(flow)


_REDUCE = {
    "sum": lambda a, b: a.add_(b),
    "prod": lambda a, b: a.mul_(b),
    "max": lambda a, b: torch.maximum(a, b, out=a),
    "min": lambda a, b: torch.minimum(a, b, out=a),
}


class NetCommunicator:
    """A rank group over the datagram transport: full mesh of flows + collectives on host tensors.

    ``exchange`` is any all-gather of small python objects among the ``world_size`` members (used once,
    for the addresses): ``torch.distributed.all_gather_object`` on a gloo group, a TCPStore, or the
    bootstrap of a :class:`uccl_b200.Communicator`.  Use :meth:`from_store` / :meth:`from_process_group`.

    Algorithms: ring reduce-scatter + ring all-gather for AllReduce (bandwidth optimal: 2(n-1)/n of the
    bytes per rank), pairwise exchange for AllToAll, binomial tree for Broadcast -- every step is an
    ``isend`` + ``irecv`` pair on different flows, so both directions of the NIC stay busy.
    """

    def __init__(self, rank: int, world_size: int, exchange: Callable[[object], List[object]],
                 engine: Optional[Engine] = None, timeout_ms: int = 60000, chunk_bytes: int = 4 << 20,
                 extra_engines: Sequence[Engine] = (), stripe_min_bytes: int = 1 << 20):
        """``extra_engines``: more engine threads (each with its own sockets / paths) for the same rank; messages
        of at least ``stripe_min_bytes`` are cut into one contiguous slice per engine, so one rank can drive a
        NIC that a single engine thread cannot fill (the reference runs several engines per NIC for the same
        reason: collective/rdma NUM_ENGINES)."""
        self.rank, self.world_size = rank, world_size
        self.engine = engine or Engine()
        self.engines: List[Engine] = [self.engine] + list(extra_engines)
        self.timeout_ms = timeout_ms
        self.chunk_bytes = chunk_bytes
        self.stripe_min_bytes = stripe_min_bytes
        self.small_bytes = int(os.environ.get("UCCL_B200_NET_AR_SMALL_BYTES", str(32 << 10)))  # recursive doubling below
        self.flows: Dict[int, int] = {}                 # peer -> flow on the primary engine
        self.stripe_flows: Dict[int, List[int]] = {}    # peer -> one flow per engine (index 0 == self.flows[peer])
        lids = [e.listen() for e in self.engines]
        addrs = exchange([(e.address, e.port, lid) for e, lid in zip(self.engines, lids)])
        ne = min(len(a) for a in addrs)                 # engines every member has
        self.engines = self.engines[:ne]
        # pair (i < j): j connects to i and introduces itself with its rank, once per engine
        hello = torch.tensor([rank], dtype=torch.int64)
        per_engine: List[Dict[int, int]] = []
        for k, e in enumerate(self.engines):
            fl: Dict[int, int] = {}
            for peer in range(rank):
                ip, port, plid = addrs[peer][k]
                f = e.connect(ip, port, plid, timeout_ms)
                e.send(f, hello, timeout_ms)
                fl[peer] = f
            for _ in range(rank + 1, world_size):
                f = e.accept(lids[k], timeout_ms)
                who = torch.zeros(1, dtype=torch.int64)
                e.recv(f, who, timeout_ms)
                fl[int(who.item())] = f
            assert sorted(fl) == [p for p in range(world_size) if p != rank]
            per_engine.append(fl)
        for e, lid in zip([self.engine] + list(extra_engines), lids):
            e.close_listen(lid)
        self.flows = per_engine[0]
        self.stripe_flows = {p: [fl[p] for fl in per_engine] for p in self.flows}

    # ---- constructors
    @classmethod
    def from_store(cls, store, rank: int, world_size: int, prefix: str = "uccl_b200_net", **kw) -> "NetCommunicator":
        import pickle

        def exchange(obj):
            store.set(f"{prefix}/{rank}", pickle.dumps(obj))
            return [pickle.loads(store.get(f"{prefix}/{r}")) for r in range(world_size)]

        return cls(rank, world_size, exchange, **kw)

    @classmethod
    def from_process_group(cls, group=None, **kw) -> "NetCommunicator":
        import torch.distributed as dist

        rank, world = dist.get_rank(group), dist.get_world_size(group)

        def exchange(obj):
            out = [None] * world
            dist.all_gather_object(out, obj, group=group)
            return out

        return cls(rank, world, exchange, **kw)

    # ---- point to point
    def _striped(self, t: torch.Tensor, peer: int, post) -> "Work":
        ne = len(self.engines)
        nbytes = t.numel() * t.element_size()
        if ne == 1 or nbytes < self.stripe_min_bytes or not t.is_contiguous():
            return post(self.engine, self.flows[peer], t)
        b = t.view(-1).view(torch.uint8)
        step = -(-nbytes // ne)
        step += (-step) % 64  # slice boundaries on 64-byte lines
        parts = [post(self.engines[k], self.stripe_flows[peer][k], b[k * step: min((k + 1) * step, nbytes)])
                 for k in range(ne) if k * step < nbytes]
        return _MultiWork(parts)

    def isend(self, t: torch.Tensor, dst: int) -> Work:
        return self._striped(t, dst, lambda e, f, x: e.isend(f, x))

    def irecv(self, t: torch.Tensor, src: int) -> Work:
        return self._striped(t, src, lambda e, f, x: e.irecv(f, x))

    def send(self, t: torch.Tensor, dst: int) -> None:
        self.isend(t, dst).wait(self.timeout_ms)

    def _wait_recv(self, w, t: torch.Tensor) -> None:
        """A receive of a collective must fill its buffer exactly: a short message means the two ends disagree
        on the message size, and silently continuing would reduce stale bytes."""
        got = w.wait(self.timeout_ms)
        want = t.numel() * t.element_size()
        if got != want:
            raise RuntimeError(f"net: received {got} bytes into a {want}-byte receive (size mismatch between ranks)")

    def recv(self, t: torch.Tensor, src: int) -> None:
        self._wait_recv(self.irecv(t, src), t)

    def _sendrecv(self, s: torch.Tensor, dst: int, r: torch.Tensor, src: int) -> None:
        wr = self.irecv(r, src)
        ws = self.isend(s, dst)
        self._wait_recv(wr, r)
        ws.wait(self.timeout_ms)

    # ---- collectives (in place on contiguous host tensors)
    def barrier(self) -> None:
        n, r = self.world_size, self.rank
        tok, got = torch.zeros(1, dtype=torch.uint8), torch.zeros(1, dtype=torch.uint8)
        d = 1
        while d < n:  # dissemination barrier: ceil(log2 n) rounds
            self._sendrecv(tok, (r + d) % n, got, (r - d) % n)
            d *= 2

    def _segments(self, numel: int) -> List[slice]:
        n = self.world_size
        base, rem = divmod(numel, n)
        out, lo = [], 0
        for i in range(n):
            hi = lo + base + (1 if i < rem else 0)
            out.append(slice(lo, hi))
            lo = hi
        return out

    def all_reduce(self, t: torch.Tensor, op: str = "sum") -> torch.Tensor:
        n, r = self.world_size, self.rank
        if n == 1:
            return t
        avg = op == "avg"
        red = _REDUCE["sum" if avg else op]
        flat = t.view(-1)
        if n & (n - 1) == 0 and flat.numel() * t.element_size() <= self.small_bytes:
            # latency bound: recursive doubling, log2(n) exchanges of the whole (small) vector
            tmp = torch.empty_like(flat)
            d = 1
            while d < n:
                self._sendrecv(flat, r ^ d, tmp, r ^ d)
                red(flat, tmp)
                d <<= 1
            if avg:
                flat.div_(n) if t.is_floating_point() else flat.copy_(torch.div(flat, n, rounding_mode="trunc"))
            return t
        seg = self._segments(flat.numel())
        nxt, prv = (r + 1) % n, (r - 1) % n
        tmp = torch.empty(max(s.stop - s.start for s in seg), dtype=t.dtype)
        # reduce-scatter: after n-1 steps rank r owns the full reduction of segment (r+1) % n
        es = t.element_size()
        for step in range(n - 1):
            s_idx, r_idx = (r - step) % n, (r - step - 1) % n
            s_seg, r_seg = flat[seg[s_idx]], flat[seg[r_idx]]
            rbuf = tmp[: r_seg.numel()]
            # channels: the segment travels as K slices posted back to back; slice k is reduced while slices
            # > k are still on the wire, so only 1/K of the reduction time is exposed per step
            # K must be the same on both ends of every step: derive it from numel // n, not from the local
            # segment (segments differ by one element when numel % n != 0 and could straddle a chunk multiple)
            K = max(1, min(8, ((flat.numel() // n) * es) // self.chunk_bytes))
            if K == 1:
                self._sendrecv(s_seg, nxt, rbuf, prv)
                red(r_seg, rbuf)
                continue
            rb = [(k * r_seg.numel() // K, (k + 1) * r_seg.numel() // K) for k in range(K)]
            sb = [(k * s_seg.numel() // K, (k + 1) * s_seg.numel() // K) for k in range(K)]
            rws = [self.irecv(rbuf[lo:hi], prv) for lo, hi in rb]
            sws = [self.isend(s_seg[lo:hi], nxt) for lo, hi in sb]
            for (lo, hi), w in zip(rb, rws):
                self._wait_recv(w, rbuf[lo:hi])
                red(r_seg[lo:hi], rbuf[lo:hi])
            for w in sws:
                w.wait(self.timeout_ms)
        if avg:
            own = flat[seg[(r + 1) % n]]
            own.div_(n) if t.is_floating_point() else own.copy_(torch.div(own, n, rounding_mode="trunc"))
        # all-gather of the reduced segments
        for step in range(n - 1):
            s_idx, r_idx = (r + 1 - step) % n, (r - step) % n
            self._sendrecv(flat[seg[s_idx]], nxt, flat[seg[r_idx]], prv)
        return t

    def all_gather(self, out: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        n, r = self.world_size, self.rank
        parts = out.view(n, -1)
        parts[r].copy_(t.view(-1))
        nxt, prv = (r + 1) % n, (r - 1) % n
        for step in range(n - 1):
            self._sendrecv(parts[(r - step) % n], nxt, parts[(r - step - 1) % n], prv)
        return out

    def reduce_scatter(self, out: torch.Tensor, t: torch.Tensor, op: str = "sum") -> torch.Tensor:
        n, r = self.world_size, self.rank
        red = _REDUCE["sum" if op == "avg" else op]
        parts = t.view(n, -1).clone()
        tmp = torch.empty_like(parts[0])
        nxt, prv = (r + 1) % n, (r - 1) % n
        # ring shifted so that the segment completed at rank r is segment r
        for step in range(n - 1):
            s_idx, r_idx = (r - step - 1) % n, (r - step - 2) % n
            self._sendrecv(parts[s_idx], nxt, tmp, prv)
            red(parts[r_idx], tmp)
        res = parts[r]
        if op == "avg":
            res = res / n if t.is_floating_point() else torch.div(res, n, rounding_mode="trunc")
        out.view(-1).copy_(res)
        return out

    def broadcast(self, t: torch.Tensor, root: int = 0) -> torch.Tensor:
        n = self.world_size
        vr = (self.rank - root) % n  # binomial tree on ranks relative to the root
        mask = 1
        while mask < n:
            if vr & mask:
                self.recv(t, (vr - mask + root) % n)
                break
            mask <<= 1
        mask >>= 1
        while mask > 0:
            if vr + mask < n:
                self.send(t, (vr + mask + root) % n)
            mask >>= 1
        return t

    def all_to_all(self, out: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        n, r = self.world_size, self.rank
        src, dst = t.view(n, -1), out.view(n, -1)
        dst[r].copy_(src[r])
        for d in range(1, n):  # pairwise exchange: step d talks to r+d / r-d
            self._sendrecv(src[(r + d) % n], (r + d) % n, dst[(r - d) % n], (r - d) % n)
        return out

    def stats(self) -> Dict:
        return {"engine": self.engine.stats(), "flows": {p: self.engine.flow_stats(f) for p, f in self.flows.items()},
                "engines": [e.stats() for e in self.engines]}

    def close(self) -> None:
        for fl in self.stripe_flows.values():
            for e, f in zip(self.engines, fl):
                e.close(f)
        self.flows.clear()
        self.stripe_flows.clear()


__all__ = ["Engine", "NetCommunicator", "Work", "list_interfaces", "nccl_net_plugin_path", "CC"]
