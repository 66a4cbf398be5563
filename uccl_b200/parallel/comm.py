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


def _overlaps(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Do the storage byte ranges of two contiguous tensors intersect?"""
    a0, b0 = a.data_ptr(), b.data_ptr()
    a1, b1 = a0 + a.numel() * a.element_size(), b0 + b.numel() * b.element_size()
    return a.device == b.device and a0 < b1 and b0 < a1


def _rmsnorm_tail_args(op, rows, H, dtype, device, residual, weight, residual_out, out, quant, reads=(), writes=()):
    """Checks and defaults of the fused residual add + RMSNorm layer tails, once ``op`` has checked its own inputs.

    ``residual``, ``residual_out`` (default: ``residual``) and ``out`` (default: a fresh tensor) are contiguous
    ``[rows, H]``, ``weight`` is ``[H]``, all of ``dtype`` except an e4m3 ``out`` with ``quant="fp8"``.  A tensor the op
    writes (``residual_out``, ``out`` and ``writes``) must not overlap another operand (those, ``residual`` and
    ``reads``); only ``residual_out`` may be ``residual`` itself.  ``weight`` is read-only and never conflicts.
    Returns ``(residual_out, out, scales)``; ``scales`` is fp32 ``[rows, H / 128]`` with fp8, else None."""
    if quant not in (None, "fp8"):
        raise ValueError(f"uccl_b200: {op}: unsupported quant {quant!r} (None or 'fp8')")
    fp8 = quant == "fp8"
    out_dtype = torch.float8_e4m3fn if fp8 else dtype
    if residual_out is None:
        residual_out = residual
    if out is None:
        out = torch.empty((rows, H), dtype=out_dtype, device=device)
    for t, name, shape, dt in ((residual, "residual", (rows, H), dtype), (weight, "weight", (H,), dtype),
                               (residual_out, "residual_out", (rows, H), dtype), (out, "out", (rows, H), out_dtype)):
        if t.dtype != dt or t.shape != shape or not t.is_contiguous():
            raise ValueError(f"uccl_b200: {op} {name} must be contiguous {dt} {list(shape)} "
                             f"(got {t.dtype} {list(t.shape)})")
    written = [residual_out, out, *writes]
    operands = written + [residual, *reads]
    for i, w in enumerate(written):
        for j in range(i + 1, len(operands)):
            o = operands[j]
            if i == 0 and j == len(written) and w.data_ptr() == o.data_ptr():
                continue  # residual_out is residual itself
            if _overlaps(w, o):
                raise ValueError(f"uccl_b200: {op} outputs must not overlap each other or an input "
                                 "(residual_out may be residual itself)")
    scales = torch.empty((rows, H // 128), dtype=torch.float32, device=device) if fp8 else None
    return residual_out, out, scales


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

    def all_reduce_rmsnorm(self, x: torch.Tensor, residual: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6, *,
                           residual_out: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                           quant: Optional[str] = None, algo="auto", max_ctas: int = -1, stream=None):
        """Sum all-reduce of ``x`` [T, H] in place, then ``residual_out = x + residual`` (over ``residual`` unless
        given) and ``out = rmsnorm(residual_out, eps) * weight``; returns ``out``, or ``(out_e4m3, scales)`` with
        ``quant="fp8"``.

        The tail of every row-parallel layer of a tensor-parallel transformer in one call.  bf16 or fp16,
        ``H % 8 == 0`` and ``H <= 16384`` (``H % 128 == 0`` for fp8).  Where the plain all-reduce would run one-shot
        (small decode batches) everything is one kernel; larger ones run the selected all-reduce and then one
        epilogue kernel.  Both paths give bitwise identical results on every rank.  The fp8 output is the
        ``(x, scales)`` format of ``ep.utils.per_token_cast_to_fp8`` and ``ep.Buffer.dispatch``."""
        self._check(x, "x")
        if x.dim() != 2:
            raise ValueError("uccl_b200: all_reduce_rmsnorm x must be [tokens, hidden]")
        T, H = x.shape
        residual_out, out, scales = _rmsnorm_tail_args("all_reduce_rmsnorm", T, H, x.dtype, x.device, residual, weight,
                                                       residual_out, out, quant, writes=(x,))
        fp8 = scales is not None
        a = ALGOS[algo] if isinstance(algo, str) else int(algo)
        self._c.allreduce_rmsnorm(x.data_ptr(), residual.data_ptr(), residual_out.data_ptr(), weight.data_ptr(),
                                  out.data_ptr(), scales.data_ptr() if fp8 else 0, T, H, dtype_code(x.dtype),
                                  float(eps), int(fp8), self._stream(stream), a, max_ctas)
        return (out, scales) if fp8 else out

    def reduce_scatter_rmsnorm(self, x: torch.Tensor, residual: torch.Tensor, weight: torch.Tensor,
                               eps: float = 1e-6, *, residual_out: Optional[torch.Tensor] = None,
                               out: Optional[torch.Tensor] = None, quant: Optional[str] = None, stream=None):
        """Sequence-parallel layer tail: reduce-scatter ``x`` [T, H] over tokens, then add + RMSNorm this rank's rows.

        The tail of a row-parallel layer with sequence parallelism in one call.  Returns ``out`` [T/n, H], or
        ``(out_e4m3, scales)`` with ``quant="fp8"``.

        With ``n`` ranks, rank ``r`` and ``Tl = T / n`` (``T % n == 0``): ``x[r*Tl:(r+1)*Tl]`` becomes this rank's
        rows of the sum over ranks, in place as NCCL's in-place reduce-scatter (the rest of ``x`` is unchanged);
        ``residual`` [Tl, H] is this rank's shard, rows ``r*Tl .. (r+1)*Tl`` of the full residual;
        ``residual_out = x[r*Tl:(r+1)*Tl] + residual`` (over ``residual`` unless given) and
        ``out = rmsnorm(residual_out, eps) * weight``.  bf16 or fp16, ``H % 8 == 0`` and ``H <= 16384``
        (``H % 128 == 0`` for fp8).  Where the plain reduce-scatter of one rank's rows would run the LL kernel
        everything is one kernel; larger ones run the reduce-scatter and then one epilogue kernel.  Both paths, and
        the ranks' shards concatenated in rank order, give bitwise what :meth:`all_reduce_rmsnorm` gives on the same
        ``x`` and the full residual.  The fp8 output is the ``(x, scales)`` format of
        ``ep.utils.per_token_cast_to_fp8``; the full ``[T, H]`` pair for the next column-parallel layer is two plain
        :meth:`all_gather` calls, one of ``out_e4m3`` and one of ``scales``."""
        self._check(x, "x")
        if x.dim() != 2:
            raise ValueError("uccl_b200: reduce_scatter_rmsnorm x must be [tokens, hidden]")
        T, H = x.shape
        n = self.world_size
        if T % n:
            raise ValueError(f"uccl_b200: reduce_scatter_rmsnorm needs tokens ({T}) divisible by the world size ({n})")
        residual_out, out, scales = _rmsnorm_tail_args("reduce_scatter_rmsnorm", T // n, H, x.dtype, x.device, residual,
                                                       weight, residual_out, out, quant, writes=(x,))
        fp8 = scales is not None
        self._c.reduce_scatter_rmsnorm(x.data_ptr(), residual.data_ptr(), residual_out.data_ptr(), weight.data_ptr(),
                                       out.data_ptr(), scales.data_ptr() if fp8 else 0, T, H, dtype_code(x.dtype),
                                       float(eps), int(fp8), self._stream(stream))
        return (out, scales) if fp8 else out

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

    def reduce_scatter_ll_max(self) -> int:
        """Per-rank piece size (bytes) up to which reduce_scatter runs the LL-packet kernel, and
        reduce_scatter_rmsnorm its fused kernel (0: never, e.g. on one rank)."""
        return int(self._c.rs_ll_max_bytes())


def launch_count(comms: Iterable[Communicator]) -> int:
    return sum(int(c._c.launches) for c in comms)
