"""Torch-facing communicator over the native symmetric-heap fabric.

One :class:`Communicator` per rank.  Three ways to get one:

* :meth:`Communicator.from_torch_dist` -- one process per GPU (the production layout);
  ``torch.distributed`` (any backend, e.g. gloo or nccl) is used once to ship the
  128-byte unique id, everything after that is our own fabric.
* :meth:`Communicator.init` -- explicit ``(uid, rank, world)`` like ``ncclCommInitRank``.
* :meth:`Communicator.local_world` -- all ranks inside this process (``ncclCommInitAll``
  style; with ``devices=[0]*n`` it gives *virtual ranks* on one GPU, which is what the
  single-GPU test-suite uses to exercise the cross-rank kernels).

API parity notes (reference): the NCCL-style collective entry points mirror
``experimental/lite/nccl/nccl.cu:1838-2102`` (AllReduce/ReduceScatter/AllGather/Broadcast/
Reduce/AllToAll); `empty()` is the ``ncclMemAlloc`` analogue (`nccl.cu:2384-2430`) -- buffers
from it are zero-copy for every collective (peer-mapped and multicast-bound).
"""
from __future__ import annotations

import ctypes
import os
import warnings
from typing import Iterable, List, Optional, Sequence

import torch

from .. import _native

_DTYPE = {
    torch.int8: 0,
    torch.uint8: 1,
    torch.int32: 2,
    torch.int64: 4,
    torch.float16: 6,
    torch.float32: 7,
    torch.float64: 8,
    torch.bfloat16: 9,
}
for _name, _code in (("uint32", 3), ("uint64", 5), ("float8_e4m3fn", 10), ("float8_e5m2", 11)):
    if hasattr(torch, _name):
        _DTYPE[getattr(torch, _name)] = _code
_DTYPE[torch.bool] = 1

_OPS = {"sum": 0, "prod": 1, "product": 1, "max": 2, "min": 3, "avg": 4, "mean": 4}

ALGOS = {
    "auto": 0,
    "oneshot_ll": 1,
    "oneshot_mc": 2,
    "twoshot_p2p": 3,
    "twoshot_nvls": 4,
    "staged_p2p": 5,
    "staged_nvls": 6,
    "staged_pipe": 7,
}


def dtype_code(dt: torch.dtype) -> int:
    try:
        return _DTYPE[dt]
    except KeyError as e:  # pragma: no cover
        raise TypeError(f"uccl_b200: unsupported dtype {dt}") from e


def op_code(op) -> int:
    if isinstance(op, int):
        return op
    name = str(op).lower().split(".")[-1]
    try:
        return _OPS[name]
    except KeyError as e:
        raise ValueError(f"uccl_b200: unsupported reduce op {op!r}") from e


class _HeapBlock:
    """Owns one symmetric-heap allocation; exposes it to torch without copying."""

    def __init__(self, comm: "Communicator", nbytes: int):
        self._comm = comm
        self.nbytes = int(nbytes)
        self.ptr = comm._c.alloc(max(self.nbytes, 1), 256)
        self.__cuda_array_interface__ = {
            "shape": (max(self.nbytes, 1),),
            "typestr": "|u1",
            "data": (self.ptr, False),
            "version": 3,
            "strides": None,
        }

    def __del__(self):
        try:
            self._comm._c.free(self.ptr)
        except Exception:
            pass


class Communicator:
    def __init__(self, c, group=None):
        self._c = c
        self.group = group
        self.rank: int = c.rank
        self.world_size: int = c.nranks
        self.device_index: int = c.device
        self.is_host: bool = c.is_host
        self.device = torch.device("cpu") if self.is_host else torch.device("cuda", c.device)
        # measured (algorithm, CTAs) per size: UCCL_B200_TUNE_FILE, else the table shipped for this world size
        from ..utils.tuner import load_tuning_from_env

        try:
            load_tuning_from_env(self)
        except Exception as e:  # noqa: BLE001 - a bad table must not prevent communication
            import warnings

            warnings.warn(f"uccl_b200: tuning table ignored ({e})")

    # ------------------------------------------------------------------ construction
    @staticmethod
    def create_unique_id() -> bytes:
        return _native.C().create_unique_id()

    @classmethod
    def init(cls, uid: bytes, rank: int, world_size: int, device: Optional[int] = None,
             heap_bytes: int = 1 << 30, stage_bytes: int = 64 << 20, host: Optional[bool] = None,
             timeout_ms: int = -1, max_ctas: int = -1) -> "Communicator":
        C = _native.C()
        if host is None:
            host = not torch.cuda.is_available()
        if device is None:
            device = -1 if host else torch.cuda.current_device()
        if not host:
            torch.cuda.set_device(device)
            torch.cuda.init()
        c = C.Comm.create(uid, rank, world_size, device, heap_bytes, stage_bytes, host, timeout_ms, max_ctas)
        return cls(c)

    @classmethod
    def from_torch_dist(cls, group=None, device: Optional[int] = None, **kw) -> "Communicator":
        import torch.distributed as dist

        rank = dist.get_rank(group)
        world = dist.get_world_size(group)
        box = [cls.create_unique_id() if rank == 0 else None]
        src = dist.get_global_rank(group, 0) if group is not None else 0
        dist.broadcast_object_list(box, src=src, group=group)
        comm = cls.init(box[0], rank, world, device=device, **kw)
        comm.group = group
        return comm

    @classmethod
    def local_world(cls, world_size: Optional[int] = None, devices: Optional[Sequence[int]] = None,
                    heap_bytes: int = 1 << 30, stage_bytes: int = 64 << 20, host: Optional[bool] = None,
                    timeout_ms: int = -1, max_ctas: int = -1) -> List["Communicator"]:
        """Communicators of every rank of a world inside this process, one per entry of `devices`.

        A device listed more than once hosts *virtual ranks*: their kernels wait for each other inside one CUDA
        context.  Under CUDA's lazy module loading the first launch of any kernel may synchronise that context, and
        one issued while a virtual rank's kernel waits for its peer never returns.  Processes that use virtual
        ranks must start with ``CUDA_MODULE_LOADING=EAGER`` (set before CUDA initialises); a warning says so."""
        C = _native.C()
        if host is None:
            host = not torch.cuda.is_available()
        if devices is None:
            n = world_size or (1 if host else torch.cuda.device_count())
            devices = [-1] * n if host else [i % torch.cuda.device_count() for i in range(n)]
        if not host:
            if len(set(devices)) < len(devices) and os.environ.get("CUDA_MODULE_LOADING", "").upper() != "EAGER":
                warnings.warn("uccl_b200: virtual ranks (a device listed twice) can deadlock under lazy CUDA module "
                              "loading; start the process with CUDA_MODULE_LOADING=EAGER", RuntimeWarning, stacklevel=2)
            torch.cuda.init()
        cs = C.Comm.create_local(list(devices), heap_bytes, stage_bytes, host, timeout_ms, max_ctas)
        return [cls(c) for c in cs]

    # ------------------------------------------------------------------------- memory
    def empty(self, *shape, dtype: torch.dtype = torch.float32) -> torch.Tensor:
        """A tensor living in the symmetric heap (same offset on every rank when all ranks
        allocate in the same order).  Zero-copy for every collective / EP / P2P op."""
        if len(shape) == 1 and isinstance(shape[0], (tuple, list, torch.Size)):
            shape = tuple(shape[0])
        numel = 1
        for s in shape:
            numel *= int(s)
        nbytes = numel * torch.empty((), dtype=dtype).element_size()
        blk = _HeapBlock(self, nbytes)
        if self.is_host:
            buf = (ctypes.c_ubyte * max(nbytes, 1)).from_address(blk.ptr)
            flat = torch.frombuffer(buf, dtype=torch.uint8)
            flat._uccl_block = blk  # keep alive
        else:
            flat = torch.as_tensor(blk, device=self.device)
        t = flat[:nbytes].view(dtype).reshape(shape)
        t._uccl_block = blk
        return t

    def zeros(self, *shape, dtype: torch.dtype = torch.float32) -> torch.Tensor:
        t = self.empty(*shape, dtype=dtype)
        t.zero_()
        return t

    def is_symmetric(self, t: torch.Tensor) -> bool:
        return bool(self._c.in_heap(t.data_ptr(), t.numel() * t.element_size()))

    def peer_ptr(self, t: torch.Tensor, peer: int) -> int:
        return self._c.peer_ptr(t.data_ptr(), peer)

    @property
    def has_multicast(self) -> bool:
        return bool(self._c.has_multicast)

    @property
    def native(self):
        return self._c

    def describe(self) -> str:
        return self._c.describe()

    # ------------------------------------------------------------------------ helpers
    def _stream(self, stream=None) -> int:
        if self.is_host:
            return 0
        if stream is None:
            stream = torch.cuda.current_stream(self.device)
        return stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream)

    @staticmethod
    def _check(t: torch.Tensor, name: str):
        if not t.is_contiguous():
            raise ValueError(f"uccl_b200: {name} must be contiguous")

    # -------------------------------------------------------------------- collectives
    def all_reduce(self, tensor: torch.Tensor, op="sum", out: Optional[torch.Tensor] = None, *,
                   scale: float = 1.0, algo="auto", max_ctas: int = -1, stream=None) -> torch.Tensor:
        """out = scale * reduce_over_ranks(tensor); in place when ``out`` is None.  If ``out``
        has a different float dtype the cast is fused into the kernel epilogue."""
        self._check(tensor, "tensor")
        if out is None:
            out = tensor
        self._check(out, "out")
        if out.numel() != tensor.numel():
            raise ValueError("uccl_b200: all_reduce out/in element count mismatch")
        out_dt = -1 if out.dtype == tensor.dtype else dtype_code(out.dtype)
        a = ALGOS[algo] if isinstance(algo, str) else int(algo)
        self._c.allreduce(tensor.data_ptr(), out.data_ptr(), tensor.numel(), dtype_code(tensor.dtype), op_code(op),
                          self._stream(stream), a, float(scale), out_dt, max_ctas)
        return out

    def all_gather(self, out: torch.Tensor, tensor: torch.Tensor, stream=None) -> torch.Tensor:
        self._check(tensor, "tensor")
        self._check(out, "out")
        if out.numel() != tensor.numel() * self.world_size:
            raise ValueError("uccl_b200: all_gather out must hold world_size * tensor.numel() elements")
        self._c.allgather(tensor.data_ptr(), out.data_ptr(), tensor.numel(), dtype_code(tensor.dtype),
                          self._stream(stream))
        return out

    def reduce_scatter(self, out: torch.Tensor, tensor: torch.Tensor, op="sum", stream=None) -> torch.Tensor:
        self._check(tensor, "tensor")
        self._check(out, "out")
        if tensor.numel() != out.numel() * self.world_size:
            raise ValueError("uccl_b200: reduce_scatter input must hold world_size * out.numel() elements")
        self._c.reduce_scatter(tensor.data_ptr(), out.data_ptr(), out.numel(), dtype_code(tensor.dtype), op_code(op),
                               self._stream(stream))
        return out

    def broadcast(self, tensor: torch.Tensor, root: int = 0, out: Optional[torch.Tensor] = None,
                  stream=None) -> torch.Tensor:
        self._check(tensor, "tensor")
        if out is None:
            out = tensor
        self._c.broadcast(tensor.data_ptr(), out.data_ptr(), tensor.numel(), dtype_code(tensor.dtype), root,
                          self._stream(stream))
        return out

    def reduce(self, tensor: torch.Tensor, root: int = 0, op="sum", out: Optional[torch.Tensor] = None,
               stream=None) -> torch.Tensor:
        self._check(tensor, "tensor")
        if out is None:
            out = tensor
        self._c.reduce(tensor.data_ptr(), out.data_ptr(), tensor.numel(), dtype_code(tensor.dtype), op_code(op), root,
                       self._stream(stream))
        return out

    def all_to_all(self, out: torch.Tensor, tensor: torch.Tensor, stream=None) -> torch.Tensor:
        self._check(tensor, "tensor")
        self._check(out, "out")
        if tensor.numel() % self.world_size or out.numel() != tensor.numel():
            raise ValueError("uccl_b200: all_to_all needs equal splits (numel divisible by world size)")
        self._c.alltoall(tensor.data_ptr(), out.data_ptr(), tensor.numel() // self.world_size,
                         dtype_code(tensor.dtype), self._stream(stream))
        return out

    def all_to_all_v(self, out: torch.Tensor, tensor: torch.Tensor, send_counts: Iterable[int],
                     recv_counts: Iterable[int], send_displs: Optional[Iterable[int]] = None,
                     recv_displs: Optional[Iterable[int]] = None, stream=None) -> torch.Tensor:
        sc, rc = [int(x) for x in send_counts], [int(x) for x in recv_counts]

        def _excl(v):
            o, acc = [], 0
            for x in v:
                o.append(acc)
                acc += x
            return o

        sd = [int(x) for x in send_displs] if send_displs is not None else _excl(sc)
        rd = [int(x) for x in recv_displs] if recv_displs is not None else _excl(rc)
        self._c.alltoallv(tensor.data_ptr(), sc, sd, out.data_ptr(), rc, rd, dtype_code(tensor.dtype),
                          self._stream(stream))
        return out

    def barrier(self, stream=None) -> None:
        self._c.barrier(self._stream(stream))

    # ---------------------------------------------------------------- point-to-point
    def batch_send_recv(self, ops, stream=None) -> None:
        """Grouped point-to-point (``ncclGroupStart .. ncclSend/ncclRecv .. ncclGroupEnd``):
        ``ops = [("send", tensor, peer) | ("recv", tensor, peer), ...]``.  Operations towards one peer
        match the peer's operations in posting order; a rank may send to and receive from the same peer
        in one group (ring steps, all-to-all patterns)."""
        raw = []
        for kind, t, peer in ops:
            self._check(t, kind)
            raw.append((kind == "send", t.data_ptr(), t.numel() * t.element_size(), int(peer)))
        self._c.group_p2p(raw, self._stream(stream))

    def send(self, tensor: torch.Tensor, dst: int, stream=None) -> None:
        self.batch_send_recv([("send", tensor, dst)], stream)

    def recv(self, tensor: torch.Tensor, src: int, stream=None) -> None:
        self.batch_send_recv([("recv", tensor, src)], stream)

    # ---------------------------------------------------------------------- tracing
    _TRACE_CODES = {1: "kernel_begin", 2: "kernel_end", 3: "barrier_enter", 4: "barrier_exit", 5: "phase"}

    def enable_trace(self, max_events: int = 1 << 16) -> None:
        """Record a device-side timeline ({globaltimer ns, event, block, aux}) of every kernel of
        this communicator (NPKit analogue; barrier wait time per block falls out directly)."""
        self._c.enable_trace(int(max_events))

    def disable_trace(self) -> None:
        self._c.disable_trace()

    def dump_trace(self, reset: bool = True):
        return [dict(t_ns=t, event=self._TRACE_CODES.get(c, str(c)), block=b, aux=a)
                for t, c, b, a in self._c.dump_trace(reset)]

    def trace_to_chrome(self, path: str, reset: bool = True) -> int:
        """Write the trace as a chrome://tracing JSON (barrier waits as duration events per block)."""
        import json

        ev, open_b = [], {}
        for e in self.dump_trace(reset):
            key = e["block"]
            if e["event"] == "barrier_enter":
                open_b[key] = e
            elif e["event"] == "barrier_exit" and key in open_b:
                s = open_b.pop(key)
                ev.append({"name": f"barrier e{e['aux']}", "ph": "X", "pid": self.rank, "tid": key,
                           "ts": s["t_ns"] / 1e3, "dur": (e["t_ns"] - s["t_ns"]) / 1e3})
            else:
                ev.append({"name": e["event"], "ph": "i", "pid": self.rank, "tid": key, "ts": e["t_ns"] / 1e3, "s": "t"})
        with open(path, "w") as f:
            json.dump({"traceEvents": ev}, f)
        return len(ev)

    # ----------------------------------------------------------------------- tuning
    def select_allreduce(self, nbytes: int, symmetric: bool, dtype: torch.dtype = torch.float32, op="sum"):
        algo, ctas = self._c.select_allreduce(int(nbytes), bool(symmetric), dtype_code(dtype), op_code(op))
        return _native.C().algo_name(algo), ctas

    def set_tuning(self, symmetric: bool, table):
        """table: iterable of (max_bytes, algo_name_or_id, ctas)"""
        C = _native.C()
        ents = []
        for mb, algo, ctas in table:
            a = ALGOS[algo] if isinstance(algo, str) else int(algo)
            ents.append(C.TuneEntry(int(mb), a, int(ctas)))
        self._c.set_tuning(bool(symmetric), ents)


    # ------------------------------------------------------------------ torch memory pool
    def mem_pool(self):
        """A ``torch.cuda.MemPool`` whose blocks live in this communicator's symmetric heap::

            pool = comm.mem_pool()
            with torch.cuda.use_mem_pool(pool):
                grads = torch.empty(n, device="cuda")      # peer-mapped + multicast-bound
            comm.all_reduce(grads)                          # zero-copy two-shot / NVLS path

        (the torch-side analogue of ``ncclMemAlloc``).  When the heap is exhausted the pool falls back
        to ``cudaMalloc`` for that block, which then simply takes the staged paths."""
        if self.is_host:
            raise RuntimeError("uccl_b200: mem_pool needs a CUDA communicator")
        if getattr(self, "_pool", None) is None:
            from torch.cuda.memory import CUDAPluggableAllocator

            C = _native.C()
            C.pool_install(self._c)
            self._pool_alloc = CUDAPluggableAllocator(_native.module_path(), "uccl_b200_pool_malloc",
                                                      "uccl_b200_pool_free")
            self._pool = torch.cuda.MemPool(self._pool_alloc.allocator())
        return self._pool

    def use_mem_pool(self):
        """Context manager: route this thread's CUDA allocations into the symmetric heap."""
        import contextlib

        pool = self.mem_pool()
        C = _native.C()
        comm = self

        @contextlib.contextmanager
        def ctx():
            C.pool_set_thread_comm(comm._c)  # several communicators may share one device (virtual ranks)
            try:
                with torch.cuda.use_mem_pool(pool, device=comm.device):
                    yield pool
            finally:
                C.pool_clear_thread_comm()

        return ctx()

    def set_rs_push(self, on: bool):
        """Staged (plain-buffer) reduce_scatter: push pieces into the peers' stages (True) instead of
        copy-in + pull (False).  Collective setting: use the same value on every rank."""
        self._c.set_rs_push(bool(on))

    def set_xchg_ll_max(self, nbytes: int):
        """Per-rank piece size up to which all_gather / all_to_all / reduce_scatter use the barrier-free
        LL-packet kernels (0: built-in default per world size, negative: never)."""
        self._c.set_xchg_ll_max(int(nbytes))


def launch_count(comms: Iterable[Communicator]) -> int:
    return sum(int(c._c.launches) for c in comms)
