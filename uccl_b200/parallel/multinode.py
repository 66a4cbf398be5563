"""Collectives across several H100 boxes: NVLink inside a box, the datagram transport between boxes.

The reference scales out by plugging its transport under NCCL's rings.  With a full-bandwidth NVSwitch
inside every box the better shape is hierarchical and *rail aligned*: local rank ``l`` of every node owns
NIC ``l``; a collective is (1) an NVLink kernel inside the box that leaves each local rank with 1/L of the
node's data, (2) L independent inter-node collectives, one per rail, running concurrently on L NICs through
:class:`uccl_b200.net.NetCommunicator`, (3) an NVLink kernel that re-assembles.  Every byte crosses the
network exactly once per remote node and all NICs of a box are busy.

``local`` is a :class:`uccl_b200.Communicator` (GPU symmetric heap, or the host backend on a CPU-only
machine -- that is how ``tests/test_net_transport.py`` runs 2 "nodes" x 2 ranks on one box).  GPU data is
staged through pinned host buffers (the transport is socket based; a GPUDirect verbs backend would slot in
under the same ``NetCommunicator`` API).

Reference: NCCL's net transport + collective/rdma (inter-node rings); thirdparty NCCL proxy staging.
"""
from __future__ import annotations

import os
import queue
import threading
from typing import Dict, Optional, Tuple

import torch

from ..net import NetCommunicator
from .comm import Communicator


class MultiNodeCommunicator:
    def __init__(self, local: Communicator, net: NetCommunicator):
        self.local, self.net = local, net
        self.local_rank, self.local_size = local.rank, local.world_size
        self.node_rank, self.num_nodes = net.rank, net.world_size
        self.rank = self.node_rank * self.local_size + self.local_rank
        self.world_size = self.num_nodes * self.local_size
        self.device = local.device
        self._pinned: Dict[Tuple[int, torch.dtype, int], torch.Tensor] = {}
        # all_reduce of more than this many bytes per rank-shard runs as a 3-stage pipeline over chunks
        self.pipeline_bytes = int(os.environ.get("UCCL_B200_MN_PIPELINE_BYTES", str(8 << 20)))
        self.small_bytes = int(os.environ.get("UCCL_B200_MN_SMALL_BYTES", str(16 << 10)))

    @staticmethod
    def _rail_engine(local_rank: int, device: Optional[int]):
        """Engine bound to the NIC closest to this rank's GPU (round robin by local rank without PCI data);
        ``UCCL_B200_NET_BIND_IP`` overrides."""
        from ..net import Engine
        from ..net.topology import nic_for_gpu

        if os.environ.get("UCCL_B200_NET_BIND_IP"):
            return Engine()
        gpu = device if (device is not None and device >= 0) else (torch.cuda.current_device() if torch.cuda.is_available() else None)
        _, ip = nic_for_gpu(gpu, local_rank)
        return Engine(bind_ip=ip)

    @classmethod
    def _extra_engines(cls, local_rank: int, device: Optional[int]):
        """``UCCL_B200_NET_ENGINES`` engine threads per rail (default 1): large messages are striped over them."""
        n = int(os.environ.get("UCCL_B200_NET_ENGINES", "1"))
        return [cls._rail_engine(local_rank, device) for _ in range(max(0, n - 1))]

    @classmethod
    def from_torch_dist(cls, local_size: int, device: Optional[int] = None, engine=None, **comm_kw) -> "MultiNodeCommunicator":
        """Build from an initialised ``torch.distributed`` world (any backend; only used for bootstrap):
        ranks ``[k*local_size, (k+1)*local_size)`` form node ``k``."""
        import torch.distributed as dist

        world, rank = dist.get_world_size(), dist.get_rank()
        assert world % local_size == 0
        nodes = world // local_size
        node_groups = [dist.new_group(list(range(k * local_size, (k + 1) * local_size))) for k in range(nodes)]
        rail_groups = [dist.new_group(list(range(l, world, local_size))) for l in range(local_size)]
        local = Communicator.from_torch_dist(group=node_groups[rank // local_size], device=device, **comm_kw)
        engine = engine or cls._rail_engine(rank % local_size, device)
        net = NetCommunicator.from_process_group(rail_groups[rank % local_size], engine=engine,
                                                 extra_engines=cls._extra_engines(rank % local_size, device))
        return cls(local, net)

    @classmethod
    def from_store(cls, store, rank: int, world_size: int, local_size: int, prefix: str = "uccl_b200/mn",
                   engine=None, **comm_kw) -> "MultiNodeCommunicator":
        """Bootstrap through a c10d-style store (``set`` / ``get``): one unique id per node, one address
        exchange per rail.  This is what the ``"uccl_b200"`` torch backend uses for multi-node groups."""
        assert world_size % local_size == 0
        node, lrank = divmod(rank, local_size)
        key = f"{prefix}/uid/{node}"
        if lrank == 0:
            store.set(key, Communicator.create_unique_id())
        uid = bytes(store.get(key))
        local = Communicator.init(uid, lrank, local_size, **comm_kw)
        engine = engine or cls._rail_engine(lrank, comm_kw.get("device"))
        net = NetCommunicator.from_store(store, node, world_size // local_size, prefix=f"{prefix}/rail{lrank}", engine=engine,
                                         extra_engines=cls._extra_engines(lrank, comm_kw.get("device")))
        return cls(local, net)

    @property
    def is_host(self) -> bool:
        return self.local.is_host

    # ------------------------------------------------------------------ staging
    def _host(self, like: torch.Tensor, numel: int, slot: int = 0) -> torch.Tensor:
        key = (slot, like.dtype, numel)
        buf = self._pinned.get(key)
        if buf is None:
            pin = like.is_cuda
            buf = torch.empty(numel, dtype=like.dtype, pin_memory=pin)
            if len(self._pinned) > 16:
                self._pinned.clear()
            self._pinned[key] = buf
        return buf

    def _down(self, dev: torch.Tensor, slot: int = 0) -> torch.Tensor:
        """device -> host staging (identity for host tensors)."""
        if not dev.is_cuda:
            return dev
        h = self._host(dev, dev.numel(), slot)
        h.copy_(dev.view(-1), non_blocking=True)
        torch.cuda.current_stream(dev.device).synchronize()
        return h

    def _up(self, dev: torch.Tensor, host: torch.Tensor) -> None:
        if dev.is_cuda:
            dev.view(-1).copy_(host, non_blocking=True)
        elif dev.data_ptr() != host.data_ptr():
            dev.view(-1).copy_(host)

    def _sync_local(self) -> None:
        if self.device.type == "cuda":
            torch.cuda.current_stream(self.device).synchronize()

    # -------------------------------------------------------------- collectives
    def barrier(self) -> None:
        self.local.barrier()
        self._sync_local()
        self.net.barrier()
        self.local.barrier()
        self._sync_local()

    def all_reduce(self, t: torch.Tensor, op: str = "sum", out: Optional[torch.Tensor] = None, scale: float = 1.0,
                   **_ignored) -> torch.Tensor:
        """reduce-scatter over NVLink -> per-rail all-reduce over the network -> all-gather over NVLink.
        In place unless ``out`` is given (which may have another float dtype: the cast happens once, at the end);
        ``scale`` multiplies the result (same contract as :meth:`Communicator.all_reduce`)."""
        if out is not None and out is not t:
            tmp = t.clone()
            self.all_reduce(tmp, op, scale=scale)
            out.view(-1).copy_(tmp.view(-1))
            return out
        if scale != 1.0:
            if not t.is_floating_point():
                raise ValueError("uccl_b200: all_reduce scale needs a floating-point tensor")
            self.all_reduce(t, op)
            t.mul_(scale)
            return t
        L, N = self.local_size, self.num_nodes
        if N == 1:
            self.local.all_reduce(t, op)
            return t
        inner = "sum" if op == "avg" else op
        flat = t.view(-1)
        n = flat.numel()
        if n * t.element_size() <= self.small_bytes:
            # latency bound: one NVLink all-reduce, then every local rank all-reduces the whole (tiny) vector along
            # its rail -- two phases instead of three
            if L > 1:
                self.local.all_reduce(flat, inner)
            h = self._down(flat)
            self.net.all_reduce(h, inner)
            if op == "avg":
                h.div_(self.world_size) if t.is_floating_point() else h.copy_(torch.div(h, self.world_size, rounding_mode="trunc"))
            self._up(flat, h)
            return t
        per = (n + L - 1) // L
        if per * L != n:  # pad to a multiple of the node size
            work = torch.zeros(per * L, dtype=t.dtype, device=t.device)
            work[:n].copy_(flat)
        else:
            work = flat
        if L > 1 and per * t.element_size() > self.pipeline_bytes:
            self._all_reduce_pipelined(work, per, inner, op)
            if work.data_ptr() != flat.data_ptr():
                flat.copy_(work[:n])
            return t
        if L > 1:
            shard = torch.empty(per, dtype=t.dtype, device=t.device)
            self.local.reduce_scatter(shard, work, inner)
        else:
            shard = work
        h = self._down(shard)
        self.net.all_reduce(h, inner)
        if op == "avg":
            h.div_(self.world_size) if t.is_floating_point() else h.copy_(torch.div(h, self.world_size, rounding_mode="trunc"))
        self._up(shard, h)
        if L > 1:
            self.local.all_gather(work, shard)
        if work.data_ptr() != flat.data_ptr():
            flat.copy_(work[:n])
        return t

    def _all_reduce_pipelined(self, work: torch.Tensor, per: int, inner: str, op: str) -> None:
        """Chunked 3-stage pipeline: while chunk k is on the network (helper thread, one rail per local rank),
        the NVLink reduce-scatter of chunk k+1 and the NVLink all-gather of chunk k-1 run on this thread.

        A chunk is a column block: ``work`` viewed as [L, per], chunk c = columns [lo, hi) of every row, so the
        local reduce-scatter of the block leaves this rank with its own row's columns -- the same bytes the
        unchunked algorithm would send over this rank's rail."""
        L = self.local_size
        es = work.element_size()
        cols = max(1, self.pipeline_bytes // es)
        bounds = [(lo, min(lo + cols, per)) for lo in range(0, per, cols)]
        rows = work.view(L, per)
        cuda = work.is_cuda
        todo: "queue.Queue" = queue.Queue()
        done: "queue.Queue" = queue.Queue()

        def network():
            while True:
                item = todo.get()
                if item is None:
                    return
                k, h, ev = item
                try:
                    if ev is not None:
                        ev.synchronize()
                    self.net.all_reduce(h, inner)
                    if op == "avg":
                        h.div_(self.world_size) if h.is_floating_point() else h.copy_(
                            torch.div(h, self.world_size, rounding_mode="trunc"))
                    done.put((k, None))
                except Exception as e:  # surface in the caller
                    done.put((k, e))

        th = threading.Thread(target=network, daemon=True)
        th.start()
        state = {}

        def stage_a(k):
            lo, hi = bounds[k]
            blk = rows[:, lo:hi].contiguous().view(-1)          # [L * w]
            shard = torch.empty(hi - lo, dtype=work.dtype, device=work.device)
            self.local.reduce_scatter(shard, blk, inner)
            if cuda:
                h = self._host(shard, cols, slot=10 + k % 3)[: hi - lo]
                h.copy_(shard, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(torch.cuda.current_stream(work.device))
            else:
                h, ev = shard, None
            state[k] = (shard, h)
            todo.put((k, h, ev))

        def stage_c(k):
            lo, hi = bounds[k]
            shard, h = state.pop(k)
            self._up(shard, h)
            full = torch.empty(L * (hi - lo), dtype=work.dtype, device=work.device)
            self.local.all_gather(full, shard)
            rows[:, lo:hi].copy_(full.view(L, hi - lo))

        depth = 2
        try:
            for k in range(min(depth, len(bounds))):
                stage_a(k)
            for k in range(len(bounds)):
                kk, err = done.get()
                if err is not None:
                    raise err
                assert kk == k
                stage_c(k)
                if k + depth < len(bounds):
                    stage_a(k + depth)
        finally:
            todo.put(None)
            th.join()

    def all_gather(self, out: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """out[g] = t of global rank g (node major).  Rail all-gather first (each NIC carries only its own
        rank's rows), then one NVLink all-gather and a local transpose."""
        L, N = self.local_size, self.num_nodes
        c = t.numel()
        rail = torch.empty(N * c, dtype=t.dtype, device=t.device)
        if N > 1:
            h_in = self._down(t.contiguous().view(-1), slot=0)
            h_out = self._host(t, N * c, slot=1)
            self.net.all_gather(h_out, h_in)
            self._up(rail, h_out)
        else:
            rail.copy_(t.view(-1))
        if L > 1:
            g = torch.empty(L * N * c, dtype=t.dtype, device=t.device)
            self.local.all_gather(g, rail)
            out.view(N, L, c).copy_(g.view(L, N, c).transpose(0, 1))
        else:
            out.view(-1).copy_(rail)
        return out

    def reduce_scatter(self, out: torch.Tensor, t: torch.Tensor, op: str = "sum") -> torch.Tensor:
        """out = reduction over all ranks of segment ``rank`` of t ([world_size * out.numel()])."""
        L, N = self.local_size, self.num_nodes
        c = out.numel()
        inner = "sum" if op == "avg" else op
        if L > 1:
            # bring the N segments that belong to local rank l of every node together, then reduce over NVLink
            src = t.view(N, L, c).transpose(0, 1).contiguous().view(-1)
            part = torch.empty(N * c, dtype=t.dtype, device=t.device)
            self.local.reduce_scatter(part, src, inner)
        else:
            part = t.contiguous().view(-1)
        if N > 1:
            h_in = self._down(part, slot=0)
            h_out = self._host(t, c, slot=1)
            self.net.reduce_scatter(h_out, h_in, inner)
            res = h_out
        else:
            res = part
        if op == "avg":
            res = res / self.world_size if t.is_floating_point() else torch.div(res, self.world_size, rounding_mode="trunc")
        self._up(out, res)
        return out

    def broadcast(self, t: torch.Tensor, root: int = 0) -> torch.Tensor:
        """Root's node fans out over NVLink; every rail then carries 1/L of the tensor to the other nodes,
        which re-assemble with an NVLink all-gather."""
        L, N = self.local_size, self.num_nodes
        root_node, root_local = divmod(root, L)
        if self.node_rank == root_node and L > 1:
            self.local.broadcast(t, root_local)
        if N == 1:
            return t
        flat = t.view(-1)
        n = flat.numel()
        per = (n + L - 1) // L
        lo = min(self.local_rank * per, n)
        hi = min(lo + per, n)
        piece = torch.zeros(per, dtype=t.dtype, device=t.device)
        if self.node_rank == root_node:
            piece[: hi - lo].copy_(flat[lo:hi])
        h = self._down(piece)
        self.net.broadcast(h, root_node)
        if self.node_rank != root_node:
            self._up(piece, h)
            if L > 1:
                full = torch.empty(per * L, dtype=t.dtype, device=t.device)
                self.local.all_gather(full, piece)
                flat.copy_(full[:n])
            else:
                flat.copy_(piece[:n])
        elif L > 1:
            # keep the node's ranks in step with the other nodes' all-gather (same number of local collectives)
            full = torch.empty(per * L, dtype=t.dtype, device=t.device)
            self.local.all_gather(full, piece)
        return t

    def all_to_all(self, out: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """Equal-split all-to-all in two hops (the shape of DeepEP's internode dispatch): NVLink moves every
        chunk to the local rank that owns the destination's rail, then one all-to-all per rail."""
        L, N = self.local_size, self.num_nodes
        c = t.numel() // self.world_size
        if L > 1:
            hop1_in = t.view(N, L, c).transpose(0, 1).contiguous().view(-1)  # [dst local][dst node][c]
            hop1 = torch.empty_like(hop1_in)
            self.local.all_to_all(hop1, hop1_in)  # [src local][dst node][c]
            rail_in = hop1.view(L, N, c).transpose(0, 1).contiguous().view(-1)  # [dst node][src local][c]
        else:
            rail_in = t.contiguous().view(-1)
        if N > 1:
            h_in = self._down(rail_in, slot=0)
            h_out = self._host(t, rail_in.numel(), slot=1)
            self.net.all_to_all(h_out, h_in)  # [src node][src local][c] == global source order
            self._up(out, h_out)
        else:
            out.view(-1).copy_(rail_in)
        return out

    def reduce(self, t: torch.Tensor, root: int = 0, op: str = "sum") -> torch.Tensor:
        """Result only at ``root`` (the other ranks keep their input, like NCCL)."""
        tmp = t.clone()
        self.all_reduce(tmp, op)
        if self.rank == root:
            t.copy_(tmp)
        return t

    def all_to_all_v(self, out: torch.Tensor, t: torch.Tensor, send_counts, recv_counts) -> torch.Tensor:
        """Variable all-to-all through the equal-split two-hop path: chunks are padded to the global maximum
        (one scalar max-all-reduce), exchanged, and unpadded.  Correct for any split; bandwidth-optimal only
        for balanced ones (the EP case)."""
        W = self.world_size
        mx = torch.tensor([max(list(send_counts) + [0])], dtype=torch.int64, device=t.device)
        self.all_reduce(mx, "max")
        m = int(mx.item())
        flat = t.reshape(-1)
        pad_in = torch.zeros(W * m, dtype=t.dtype, device=t.device)
        off = 0
        for d, c in enumerate(send_counts):
            pad_in[d * m: d * m + c].copy_(flat[off: off + c])
            off += c
        pad_out = torch.empty_like(pad_in)
        self.all_to_all(pad_out, pad_in)
        oflat = out.reshape(-1)
        off = 0
        for s_, c in enumerate(recv_counts):
            oflat[off: off + c].copy_(pad_out[s_ * m: s_ * m + c])
            off += c
        return out

    def _route(self, peer: int):
        node, lrank = divmod(peer, self.local_size)
        if node == self.node_rank:
            return "local", lrank
        if lrank == self.local_rank:
            return "rail", node
        raise NotImplementedError("uccl_b200: point-to-point between different rails of different nodes is not routed; "
                                  "send to the peer's rail-mate on your node first")

    def batch_send_recv(self, ops) -> None:
        """Grouped point-to-point like :meth:`Communicator.batch_send_recv` with GLOBAL peer ranks: box-mates go to
        the native grouped kernel, rail-mates to the datagram transport (receives are posted first), all concurrently."""
        local_ops, works, staged = [], [], []
        for kind, t, peer in ops:
            route, r = self._route(peer)
            if route == "local":
                local_ops.append((kind, t, r))
            elif kind == "recv":
                h = t.view(-1) if not t.is_cuda else torch.empty(t.numel(), dtype=t.dtype, pin_memory=True)
                works.append(self.net.irecv(h, r))
                if t.is_cuda:
                    staged.append((t, h))
        for kind, t, peer in ops:
            route, r = self._route(peer)
            if route == "rail" and kind == "send":
                h = t.contiguous().view(-1) if not t.is_cuda else t.contiguous().view(-1).to("cpu", non_blocking=False)
                works.append(self.net.isend(h, r))
        if local_ops:
            self.local.batch_send_recv(local_ops)
        for w in works:
            w.wait(self.net.timeout_ms)
        for t, h in staged:
            t.view(-1).copy_(h, non_blocking=True)
        self._sync_local()

    def send(self, t: torch.Tensor, dst: int) -> None:
        kind, r = self._route(dst)
        if kind == "local":
            self.local.send(t, r)
        else:
            self.net.send(self._down(t.contiguous().view(-1)), r)

    def recv(self, t: torch.Tensor, src: int) -> None:
        kind, r = self._route(src)
        if kind == "local":
            self.local.recv(t, r)
        else:
            h = t.view(-1) if not t.is_cuda else self._host(t, t.numel(), slot=2)
            self.net.recv(h, r)
            self._up(t, h)

    def close(self) -> None:
        self.net.close()


class NativeMultiNodeCommunicator:
    """The same hierarchy executed entirely in C++ (`csrc/coll/multi_comm.cc`, the object behind the NCCL drop-in):
    one call per collective, block pipeline on a helper thread, pinned staging owned by the runtime.  Bootstraps
    from a 128-byte unique id like :class:`Communicator` (rank 0 creates it, everybody gets it out of band);
    ranks ``[k*local_size, (k+1)*local_size)`` form box ``k``.  Set ``UCCL_B200_BOOTSTRAP_IP`` on rank 0 to an
    address the other boxes can reach before creating the id."""

    def __init__(self, native):
        from .comm import dtype_code, op_code

        self._m = native
        self._dt, self._op = dtype_code, op_code
        self.rank, self.world_size = native.rank, native.nranks
        self.local_rank, self.local_size = native.local_rank, native.local_size
        self.node_rank, self.num_nodes = native.node, native.nnodes
        self.is_host = native.is_host
        self.device = torch.device("cpu") if native.is_host else torch.device("cuda", native.device)

    @classmethod
    def init(cls, uid: bytes, rank: int, world_size: int, local_size: int, device: Optional[int] = None,
             heap_bytes: int = 1 << 30, stage_bytes: int = 64 << 20, host: Optional[bool] = None,
             timeout_ms: int = -1) -> "NativeMultiNodeCommunicator":
        from .. import _native

        if host is None:
            host = not torch.cuda.is_available()
        if device is None:
            device = -1 if host else torch.cuda.current_device()
        if not host:
            torch.cuda.set_device(device)
            torch.cuda.init()
        return cls(_native.C().MultiComm.create(uid, rank, world_size, local_size, device, heap_bytes, stage_bytes, host,
                                                timeout_ms))

    @classmethod
    def from_torch_dist(cls, local_size: int, group=None, **kw) -> "NativeMultiNodeCommunicator":
        import torch.distributed as dist

        rank, world = dist.get_rank(group), dist.get_world_size(group)
        box = [Communicator.create_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        return cls.init(box[0], rank, world, local_size, **kw)

    def _stream(self, stream=None) -> int:
        if self.is_host:
            return 0
        s = stream or torch.cuda.current_stream(self.device)
        return s.cuda_stream

    @staticmethod
    def _c(t: torch.Tensor) -> torch.Tensor:
        if not t.is_contiguous():
            raise ValueError("uccl_b200: tensors must be contiguous")
        return t

    def all_reduce(self, t: torch.Tensor, op: str = "sum", out: Optional[torch.Tensor] = None, scale: float = 1.0, stream=None):
        out = t if out is None else out
        if out.dtype != t.dtype:
            tmp = torch.empty_like(t)
            self.all_reduce(t, op, out=tmp, scale=scale, stream=stream)
            out.copy_(tmp)
            return out
        self._m.allreduce(self._c(t).data_ptr(), self._c(out).data_ptr(), t.numel(), self._dt(t.dtype), self._op(op),
                          self._stream(stream), float(scale))
        return out

    def all_gather(self, out: torch.Tensor, t: torch.Tensor, stream=None):
        self._m.allgather(self._c(t).data_ptr(), self._c(out).data_ptr(), t.numel(), self._dt(t.dtype), self._stream(stream))
        return out

    def reduce_scatter(self, out: torch.Tensor, t: torch.Tensor, op: str = "sum", stream=None):
        self._m.reduce_scatter(self._c(t).data_ptr(), self._c(out).data_ptr(), out.numel(), self._dt(t.dtype), self._op(op),
                               self._stream(stream))
        return out

    def broadcast(self, t: torch.Tensor, root: int = 0, out: Optional[torch.Tensor] = None, stream=None):
        out = t if out is None else out
        self._m.broadcast(self._c(t).data_ptr(), self._c(out).data_ptr(), t.numel(), self._dt(t.dtype), root, self._stream(stream))
        return out

    def reduce(self, t: torch.Tensor, root: int = 0, op: str = "sum", out: Optional[torch.Tensor] = None, stream=None):
        out = t if out is None else out
        self._m.reduce(self._c(t).data_ptr(), self._c(out).data_ptr(), t.numel(), self._dt(t.dtype), self._op(op), root,
                       self._stream(stream))
        return out

    def all_to_all(self, out: torch.Tensor, t: torch.Tensor, stream=None):
        self._m.alltoall(self._c(t).data_ptr(), self._c(out).data_ptr(), t.numel() // self.world_size, self._dt(t.dtype),
                         self._stream(stream))
        return out

    def all_to_all_v(self, out: torch.Tensor, t: torch.Tensor, send_counts, recv_counts, stream=None):
        sc, rc = [int(c) for c in send_counts], [int(c) for c in recv_counts]
        sd = [sum(sc[:i]) for i in range(len(sc))]
        rd = [sum(rc[:i]) for i in range(len(rc))]
        self._m.alltoallv(self._c(t).data_ptr(), sc, sd, self._c(out).data_ptr(), rc, rd, self._dt(t.dtype), self._stream(stream))
        return out

    def batch_send_recv(self, ops, stream=None) -> None:
        self._m.group_p2p([(kind == "send", self._c(t).data_ptr(), t.numel() * t.element_size(), int(peer))
                           for kind, t, peer in ops], self._stream(stream))

    def send(self, t: torch.Tensor, dst: int, stream=None) -> None:
        self.batch_send_recv([("send", t, dst)], stream)

    def recv(self, t: torch.Tensor, src: int, stream=None) -> None:
        self.batch_send_recv([("recv", t, src)], stream)

    def barrier(self, stream=None) -> None:
        self._m.barrier(self._stream(stream))

    def describe(self) -> str:
        return self._m.describe()


class MultiNodeWork:
    """Handle of a collective queued with :meth:`AsyncMultiNode.all_reduce_async` (c10d ``Work``-like)."""

    def __init__(self):
        self._done = threading.Event()
        self._err: Optional[BaseException] = None
        self._ev_out = None
        self.result: Optional[torch.Tensor] = None

    def is_completed(self) -> bool:
        return self._done.is_set()

    def wait(self, timeout: Optional[float] = None) -> torch.Tensor:
        if not self._done.wait(timeout):
            raise TimeoutError("uccl_b200: multi-box collective did not finish in time")
        if self._err is not None:
            raise self._err
        if self._ev_out is not None:  # order the caller's stream after the side stream's last device op
            torch.cuda.current_stream().wait_event(self._ev_out)
        return self.result


class AsyncMultiNode:
    """Runs a communicator's collectives on a helper thread (and, on GPUs, a side stream), in submission order, so
    that the network phase of gradient bucket k overlaps the backward pass that produces bucket k+1 -- what NCCL's
    proxy thread gives DDP for free.  Works with :class:`MultiNodeCommunicator` and
    :class:`NativeMultiNodeCommunicator`; every rank must submit the same sequence of operations."""

    def __init__(self, comm):
        self.comm = comm
        self._q: "queue.Queue" = queue.Queue()
        self._cuda = comm.device.type == "cuda"
        self._side = torch.cuda.Stream(device=comm.device) if self._cuda else None
        self._th = threading.Thread(target=self._loop, daemon=True, name="uccl-mn-async")
        self._th.start()

    def _loop(self):
        if self._cuda:
            torch.cuda.set_device(self.comm.device)
        while True:
            item = self._q.get()
            if item is None:
                return
            fn, work, ev_in = item
            try:
                if self._cuda:
                    with torch.cuda.stream(self._side):
                        self._side.wait_event(ev_in)
                        work.result = fn()
                        work._ev_out = torch.cuda.Event()
                        work._ev_out.record(self._side)
                else:
                    work.result = fn()
            except BaseException as e:  # noqa: BLE001 - surfaced by wait()
                work._err = e
            work._done.set()

    def submit(self, fn) -> MultiNodeWork:
        w = MultiNodeWork()
        ev = None
        if self._cuda:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self.comm.device))
        self._q.put((fn, w, ev))
        return w

    def all_reduce_async(self, t: torch.Tensor, op: str = "sum", **kw) -> MultiNodeWork:
        return self.submit(lambda: self.comm.all_reduce(t, op, **kw))

    def ddp_hook(self, op: str = "avg"):
        """``model.register_comm_hook(None, async_mn.ddp_hook())``: bucketed gradient all-reduce across boxes that
        overlaps the rest of the backward pass."""

        def hook(state, bucket):
            buf = bucket.buffer()
            fut: torch.futures.Future = torch.futures.Future()
            w = self.all_reduce_async(buf, op)

            def finish():
                try:
                    w.wait()
                    if w._ev_out is not None:
                        w._ev_out.synchronize()
                    fut.set_result(buf)
                except BaseException as e:  # noqa: BLE001
                    fut.set_exception(e)

            threading.Thread(target=finish, daemon=True).start()
            return fut

        return hook

    def close(self) -> None:
        self._q.put(None)
        self._th.join(timeout=30)
