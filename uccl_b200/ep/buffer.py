"""DeepEP-compatible expert-parallel ``Buffer`` on top of the native sm_90a kernels.

API surface follows the reference's ``ep/bench/buffer.py`` (ctor :58-69, get_dispatch_layout
:736, dispatch :837, combine :1190, low_latency_* :263-566, configs :680-733) so code written
against ``deep_ep.Buffer`` / ``uccl.ep`` switches over unchanged.  Differences that matter:

* results (``recv_x`` ...) are by default zero-copy *views* of a ring of receive arenas inside the
  symmetric heap -- valid until ``num_slots`` further dispatches (default 2).  ``Buffer(owned_results=True)``
  (or ``dispatch(..., copy_out=True)``, or the ``deep_ep`` compatibility package) returns freshly allocated
  tensors like the reference does (ep/bench/buffer.py:1068-1106) at the price of one extra pass;
* handles are :class:`EpHandle` tuples in the reference's field order (ep/bench/buffer.py:1147-1158);
* ``dispatch(..., use_fp8=True)`` fuses the per-128-channel amax/scale/e4m3 cast into the
  send (the reference casts with separate torch kernels beforehand, ep/bench/utils.py:666-675);
* ``get_combine_buffer`` hands out the symmetric arena the expert MLP should write into so
  that ``combine`` is a single zero-copy pull-reduce (any other tensor is copied in first).
"""
from __future__ import annotations

from typing import List, Optional, Tuple, Union

import torch

from .. import _native
from ..parallel.comm import Communicator, _rmsnorm_tail_args
from .utils import EpHandle, EventHandle, EventOverlap

RMS_MAX_HIDDEN = 16384  # kRmsMaxH: one 512-thread block holds a row in registers
LL_MAX_HIDDEN = 8192  # limit of the low-latency kernels
LL_MAX_TOPK = 32


def _check_bf16_rows(name, what, ts, T, H):
    for t in ts:
        if t.dtype != torch.bfloat16 or t.shape != (T, H) or not t.is_contiguous():
            raise ValueError(f"uccl_b200.ep: {name} {what} must be contiguous bf16 [{T}, {H}]")


def _combine_rmsnorm_args(x, T, residual, weight, bias, residual_out, out, quant, device):
    """Checks of ``combine_rmsnorm`` shared by the CUDA and the host backend.  Returns
    ``(b0, b1, residual_out, out, scales)`` with the defaults filled in (``scales`` is None without fp8)."""
    if x.dtype != torch.bfloat16 or x.dim() != 2 or not x.is_contiguous():
        raise ValueError("uccl_b200.ep: combine_rmsnorm x must be contiguous bf16 [num_recv, hidden]")
    H = x.size(1)
    if H % 8 or not 8 <= H <= RMS_MAX_HIDDEN:
        raise ValueError(f"uccl_b200.ep: combine_rmsnorm hidden size {H} must be a multiple of 8 in [8, {RMS_MAX_HIDDEN}]")
    if quant == "fp8" and H % 128:
        raise ValueError(f"uccl_b200.ep: combine_rmsnorm fp8 output needs hidden size % 128 == 0 (got {H})")
    b0, b1 = bias if isinstance(bias, tuple) else (bias, None)
    biases = [b for b in (b0, b1) if b is not None]
    _check_bf16_rows("combine_rmsnorm", "bias", biases, T, H)
    # peers read x while the kernel runs, and a row's residual and biases are read before its outputs are stored
    return (b0, b1) + _rmsnorm_tail_args("combine_rmsnorm", T, H, torch.bfloat16, device, residual, weight,
                                         residual_out, out, quant, reads=[x] + biases)


def _ll_combine_rmsnorm_args(x, topk_idx, topk_weights, R, M, H, E, residual, weight, shared, residual_out, out, quant,
                             device):
    """Checks of ``low_latency_combine_rmsnorm`` shared by the CUDA and the host backend (``R`` ranks; ``M``, ``H``
    and ``E`` from the dispatch handle).  Returns ``(T, K, residual_out, out, scales)`` with the defaults filled in."""
    name = "low_latency_combine_rmsnorm"
    if topk_weights.dtype != torch.float32 or topk_weights.dim() != 2 or not topk_weights.is_contiguous():
        raise ValueError(f"uccl_b200.ep: {name} topk_weights must be contiguous float32 [num_tokens, num_topk]")
    T, K = topk_weights.shape
    if not 0 < K <= LL_MAX_TOPK:
        raise ValueError(f"uccl_b200.ep: {name} num_topk {K} must be in [1, {LL_MAX_TOPK}]")
    if topk_idx.dtype != torch.int64 or topk_idx.shape != (T, K):
        raise ValueError(f"uccl_b200.ep: {name} topk_idx must be int64 [{T}, {K}] like topk_weights")
    if H % 128 or not 128 <= H <= LL_MAX_HIDDEN:
        raise ValueError(f"uccl_b200.ep: {name} hidden size {H} must be a multiple of 128 in [128, {LL_MAX_HIDDEN}]")
    if x.dtype != torch.bfloat16 or x.shape != (E // R, R * M, H) or not x.is_contiguous():
        raise ValueError(f"uccl_b200.ep: {name} x must be contiguous bf16 [{E // R}, {R * M}, {H}] "
                         f"(got {x.dtype} {tuple(x.shape)})")
    extra = [shared] if shared is not None else []
    _check_bf16_rows(name, "shared", extra, T, H)
    return (T, K) + _rmsnorm_tail_args(name, T, H, torch.bfloat16, device, residual, weight, residual_out, out, quant,
                                       reads=[x] + extra)


class Config:
    """Performance knobs (reference: ``Config(num_sms, nvl_send, nvl_recv, rdma_send, rdma_recv)``,
    ep/src/uccl_ep.cc:1641-1646).  Only ``num_sms`` matters here: there are no chunked ring
    buffers to size, the other fields are accepted and ignored."""

    def __init__(self, num_sms: int = 24, num_max_nvl_chunked_send_tokens: int = 6,
                 num_max_nvl_chunked_recv_tokens: int = 256, num_max_rdma_chunked_send_tokens: int = 6,
                 num_max_rdma_chunked_recv_tokens: int = 256):
        self.num_sms = num_sms
        self.num_max_nvl_chunked_send_tokens = num_max_nvl_chunked_send_tokens
        self.num_max_nvl_chunked_recv_tokens = num_max_nvl_chunked_recv_tokens
        self.num_max_rdma_chunked_send_tokens = num_max_rdma_chunked_send_tokens
        self.num_max_rdma_chunked_recv_tokens = num_max_rdma_chunked_recv_tokens

    def get_nvl_buffer_size_hint(self, hidden_bytes: int, num_ranks: int, num_max_tokens_per_rank: int = 4096,
                                 num_topk: int = 8, num_slots: int = 2) -> int:
        """Bytes for worst-case routing (every token of every rank lands here)."""
        cap = num_ranks * num_max_tokens_per_rank
        per_tok = hidden_bytes + (hidden_bytes // 128) * 4 + num_topk * 12 + 4
        return int((num_slots + 1) * (cap * per_tok + 8 * 256) + (1 << 20))

    def get_rdma_buffer_size_hint(self, hidden_bytes: int, num_ranks: int) -> int:
        """Bytes of RDMA buffer the normal (high-throughput) kernels need -- the second half of upstream's sizing
        snippet (``max(config.get_rdma_buffer_size_hint(hidden_bytes, group.size()), num_rdma_bytes)``).  Like the
        reference (ep/include/ep_config.hpp:94-97) this is 0 inside one NVLink domain; a group that spans boxes runs
        the host two-hop path, which stages through the communicator and needs no buffer of its own either."""
        return 0


class Buffer:
    num_sms: int = 24

    @staticmethod
    def _spans_boxes(group) -> int:
        """Ranks per box if ``group`` (the default process group) has more members than one box holds, else 0."""
        try:
            import os

            import torch.distributed as dist

            if not dist.is_initialized() or (group is not None and group is not dist.group.WORLD):
                return 0
            world = dist.get_world_size()
            local = int(os.environ.get("UCCL_B200_LOCAL_SIZE", os.environ.get("LOCAL_WORLD_SIZE", str(world))))
            return local if 0 < local < world and world % local == 0 else 0
        except Exception:  # noqa: BLE001
            return 0

    def __new__(cls, group=None, *args, comm: Optional[Communicator] = None, **kwargs):
        if comm is None and group is not None:
            local = cls._spans_boxes(group)
            if local:
                # DeepEP-style construction from a process group that spans boxes (more ranks than LOCAL_WORLD_SIZE):
                # build the hierarchical communicator and take the portable path (docs/multinode.md)
                import torch

                from ..parallel.multinode import MultiNodeCommunicator

                host = not torch.cuda.is_available()
                kw = dict(host=True, heap_bytes=256 << 20, stage_bytes=4 << 20) if host else dict(heap_bytes=1 << 30, stage_bytes=64 << 20)
                comm = MultiNodeCommunicator.from_torch_dist(local, **kw)
        if comm is not None and (comm.is_host or type(comm).__name__ in ("MultiNodeCommunicator", "NativeMultiNodeCommunicator")):
            # CPU reference backend with the same API (GPU-less CI) -- also the portable path for groups that span
            # boxes (MultiNodeCommunicator: two-hop all-to-all, NVLink + datagram rails): see host_ep.HostBuffer
            from .host_ep import HostBuffer

            return HostBuffer(comm, **{k: v for k, v in kwargs.items() if k in ("num_nvl_bytes", "num_rdma_bytes",
                                                                                 "low_latency_mode")})
        return super().__new__(cls)

    def __init__(self, group=None, num_nvl_bytes: int = 0, num_rdma_bytes: int = 0, low_latency_mode: bool = False,
                 num_qps_per_rank: int = 24, allow_nvlink_for_low_latency_mode: bool = True,
                 allow_mnnvl: bool = False, explicitly_destroy: bool = False, is_intranode: Optional[bool] = None,
                 comm: Optional[Communicator] = None, num_slots: int = 2, owned_results: Optional[bool] = None):
        """Either pass a ``torch.distributed`` group (one process per GPU; a private
        Communicator sized for ``num_nvl_bytes + num_rdma_bytes`` is created) or an existing
        ``comm`` (e.g. one rank of ``Communicator.local_world``)."""
        self.group = group
        if owned_results is None:
            import os

            owned_results = os.environ.get("UCCL_B200_EP_OWNED_RESULTS", "0") == "1"
        self.owned_results = bool(owned_results)
        self.low_latency_mode = low_latency_mode
        self.explicitly_destroy = explicitly_destroy
        self.num_nvl_bytes = int(num_nvl_bytes)
        self.num_rdma_bytes = int(num_rdma_bytes)
        total = self.num_nvl_bytes + self.num_rdma_bytes
        self._private_comm = comm is None
        if comm is None:
            assert group is not None, "Buffer needs a process group or a Communicator"
            heap = total + (256 << 20)
            comm = Communicator.from_torch_dist(group, heap_bytes=heap, stage_bytes=16 << 20)
        self.comm = comm
        self.rank = comm.rank
        self.group_size = comm.world_size
        self.device = comm.device
        C = _native.C()
        self._C = C
        self.runtime = C.EpBuffer(comm.native, max(self.num_nvl_bytes, 1 << 20), num_slots)
        self._check_symmetric_placement()
        self._ll = None
        if self.num_rdma_bytes > 0 or low_latency_mode:
            from .low_latency import LowLatencyRuntime

            self._ll = LowLatencyRuntime(self, self.num_rdma_bytes)
        with torch.cuda.device(self.device):
            self.comm_stream = torch.cuda.Stream(device=self.device, priority=-1)
        self._sm_partition = None
        self._layout_cache = None
        self._destroyed = False

    def use_sm_partition(self, partition) -> None:
        """Run this buffer's dispatch / combine kernels on the SMs of `partition`
        (:class:`uccl_b200.utils.SmPartition`, a CUDA green context) instead of wherever the scheduler finds room: the
        communication stream becomes the partition's stream and the SM budget of every launch is capped at the
        partition's size (the kernels synchronise their CTAs with each other, so all of them must be resident).  Give
        the rest of the device to the compute streams (``with rest: ...``) to keep GEMMs off these SMs.  ``None``
        restores an ordinary stream.  The low-latency kernels run on the caller's current stream (DeepEP's contract):
        enter the partition (``with partition:``) around those calls instead; while a partition is set they, too, bring at
        most its SM count of CTAs, so that doing so can never leave part of a launch waiting for an SM."""
        if partition is None:
            with torch.cuda.device(self.device):
                self.comm_stream = torch.cuda.Stream(device=self.device, priority=-1)
            self._sm_partition = None
            return
        if int(partition.device) != int(self.device.index):
            raise ValueError(f"uccl_b200.ep.Buffer: the partition lives on GPU {partition.device}, the buffer on {self.device}")
        if self.comm.native.single_process and self.group_size > 1:
            raise ValueError("uccl_b200.ep.Buffer: a single-process world shares one GPU between its ranks; "
                             "SM partitions are for one process per GPU")
        torch.cuda.current_stream(self.device).synchronize()
        self.comm_stream.synchronize()
        self.comm_stream = partition.stream(-1)  # high priority, like the ordinary communication stream
        self._sm_partition = partition

    def _check_symmetric_placement(self):
        """The kernels address a peer's arenas as `peer_heap + my_offset`, so the EP block must sit at the
        same heap offset on every rank (true when the Buffer is created right after the communicator, or
        after the same sequence of symmetric allocations everywhere).  Verified when a process group is
        available; a mismatch would otherwise corrupt memory silently."""
        if self._private_comm:
            return  # a fresh private communicator: the EP block is its first allocation on every rank
        grp = self.group if self.group is not None else getattr(self.comm, "group", None)
        try:
            import torch.distributed as dist

            if grp is None or not dist.is_initialized() or dist.get_world_size(grp) != self.group_size:
                return
            offs = [None] * self.group_size
            dist.all_gather_object(offs, int(self.runtime.base_offset), group=grp)
        except Exception:  # pragma: no cover - the check is best effort
            return
        if len(set(offs)) != 1:
            raise RuntimeError(f"uccl_b200.ep.Buffer: the EP block landed at different symmetric-heap offsets {offs}; "
                               "create the Buffer before other (rank-dependent) heap allocations")

    # ------------------------------------------------------------------ misc parity API
    def destroy(self):
        self._destroyed = True
        self.runtime = None
        self._ll = None

    @staticmethod
    def is_sm90_compiled() -> bool:
        return True  # sm_90a build: every sm_90+ feature (fp8, TMA, clusters) is available

    @staticmethod
    def set_num_sms(new_num_sms: int) -> None:
        assert new_num_sms % 2 == 0, "The SM count must be even"
        Buffer.num_sms = new_num_sms

    @staticmethod
    def capture() -> EventOverlap:
        """An event on the current stream (DeepEP: `Buffer.capture`); an empty overlap object on a machine without
        CUDA, where the host backend has nothing to order."""
        if not torch.cuda.is_available():
            return EventOverlap()
        return EventOverlap(EventHandle())

    def get_comm_stream(self) -> torch.cuda.Stream:
        return self.comm_stream

    @staticmethod
    def get_dispatch_config(num_ranks: int) -> Config:
        return Config(Buffer.num_sms)

    @staticmethod
    def get_combine_config(num_ranks: int) -> Config:
        return Config(Buffer.num_sms)

    @staticmethod
    def get_low_latency_rdma_size_hint(num_max_dispatch_tokens_per_rank: int, hidden: int, num_ranks: int,
                                       num_experts: int) -> int:
        from .low_latency import ll_size_hint

        return ll_size_hint(num_max_dispatch_tokens_per_rank, hidden, num_ranks, num_experts)

    def _sms(self, config: "Config") -> int:
        """SMs (CTAs) for one kernel.  All ranks of a single-process world that share a GPU must
        be co-resident (their kernels wait for each other), so the budget is split between them."""
        n = int(config.num_sms)
        if self.comm.native.single_process and self.group_size > 1:
            # conservative: assume every rank of the single-process world sits on this GPU
            share = torch.cuda.get_device_properties(self.device).multi_processor_count
            n = max(1, min(n, share // self.group_size))
        if self._sm_partition is not None:
            n = max(1, min(n, int(self._sm_partition.sm_count)))
        return n

    # ------------------------------------------------------------------ stream choreography
    def _enter(self, previous_event, allocate_on_comm_stream):
        compute = torch.cuda.current_stream(self.device)
        if previous_event is not None and previous_event.event is not None:
            self.comm_stream.wait_event(previous_event.event.event)
        else:
            self.comm_stream.wait_stream(compute)
        return compute

    def _exit(self, compute, async_finish, tensors) -> EventOverlap:
        if async_finish:
            ev = EventHandle(self.comm_stream)
            for t in tensors:
                if isinstance(t, torch.Tensor) and t.is_cuda:
                    t.record_stream(self.comm_stream)
                    t.record_stream(compute)
            return EventOverlap(ev, tuple(tensors))
        compute.wait_stream(self.comm_stream)
        return EventOverlap()

    # ------------------------------------------------------------------------- layout
    def get_dispatch_layout(self, topk_idx: torch.Tensor, num_experts: int,
                            previous_event: Optional[EventOverlap] = None, async_finish: bool = False,
                            allocate_on_comm_stream: bool = False):
        assert topk_idx.dtype == torch.int64 and topk_idx.dim() == 2 and topk_idx.is_contiguous()
        T, K = topk_idx.shape
        R = self.group_size
        dev = self.device
        compute = self._enter(previous_event, allocate_on_comm_stream)
        if T == 0:  # a rank without tokens in this step: nothing to scan
            with torch.cuda.stream(self.comm_stream):
                num_tokens_per_rank = torch.zeros(R, dtype=torch.int32, device=dev)
                num_tokens_per_expert = torch.zeros(num_experts, dtype=torch.int32, device=dev)
                is_token_in_rank = torch.zeros((1, R), dtype=torch.bool, device=dev)[:0]
                token_pos = torch.zeros((1, R), dtype=torch.int32, device=dev)[:0]
            self._layout_cache = (is_token_in_rank.data_ptr(), 0, token_pos)
            ev = self._exit(compute, async_finish, (num_tokens_per_rank, num_tokens_per_expert))
            return num_tokens_per_rank, None, num_tokens_per_expert, is_token_in_rank, ev
        with torch.cuda.stream(self.comm_stream):
            num_tokens_per_rank = torch.empty(R, dtype=torch.int32, device=dev)
            num_tokens_per_expert = torch.empty(num_experts, dtype=torch.int32, device=dev)
            is_token_in_rank = torch.empty((T, R), dtype=torch.bool, device=dev)
            token_pos = torch.empty((T, R), dtype=torch.int32, device=dev)
            self.runtime.layout(topk_idx.data_ptr(), T, K, num_experts, num_tokens_per_rank.data_ptr(),
                                num_tokens_per_expert.data_ptr(), is_token_in_rank.data_ptr(), token_pos.data_ptr(),
                                self.comm_stream.cuda_stream)
        # positions ride along with is_token_in_rank so dispatch() does not need to rescan
        self._layout_cache = (is_token_in_rank.data_ptr(), T, token_pos)
        ev = self._exit(compute, async_finish, (topk_idx, num_tokens_per_rank, num_tokens_per_expert,
                                                is_token_in_rank, token_pos))
        return num_tokens_per_rank, None, num_tokens_per_expert, is_token_in_rank, ev

    # ----------------------------------------------------------------------- dispatch
    def dispatch(self, x: Union[torch.Tensor, Tuple[torch.Tensor, torch.Tensor]], handle: Optional[Tuple] = None,
                 num_tokens_per_rank: Optional[torch.Tensor] = None,
                 num_tokens_per_rdma_rank: Optional[torch.Tensor] = None,
                 is_token_in_rank: Optional[torch.Tensor] = None,
                 num_tokens_per_expert: Optional[torch.Tensor] = None, topk_idx: Optional[torch.Tensor] = None,
                 topk_weights: Optional[torch.Tensor] = None, expert_alignment: int = 1, num_worst_tokens: int = 0,
                 config: Optional[Config] = None, previous_event: Optional[EventOverlap] = None,
                 async_finish: bool = False, allocate_on_comm_stream: bool = False, use_fp8: bool = False,
                 round_scale: bool = False, copy_out: Optional[bool] = None):
        C = self._C
        copy_out = self.owned_results if copy_out is None else bool(copy_out)
        config = config or self.get_dispatch_config(self.group_size)
        R = self.group_size
        dev = self.device
        if isinstance(x, tuple):
            x_data, x_scales = x
            assert x_data.dtype == torch.float8_e4m3fn and x_scales.dtype == torch.float32
            assert x_scales.is_contiguous() and x_scales.shape == (x_data.size(0), x_data.size(1) // 128)
            mode = C.EP_X_FP8_SCALED
            assert not use_fp8
        else:
            x_data, x_scales = x, None
            assert x_data.dtype == torch.bfloat16
            mode = C.EP_X_FUSED_FP8 if use_fp8 else C.EP_X_BF16
        assert x_data.dim() == 2 and x_data.is_contiguous()
        T, H = x_data.shape
        out_fp8 = mode != C.EP_X_BF16
        compute = self._enter(previous_event, allocate_on_comm_stream)

        if handle is not None:
            # cached mode: only the payload moves (reference: buffer.py:1013-1023)
            rank_prefix, num_recv, recv_src_idx, h_is_in_rank, send_slot = (handle.rank_prefix, handle.num_recv,
                                                                            handle.recv_src_idx, handle.is_token_in_rank,
                                                                            handle.send_slot)
            h_K = handle.num_topk
            assert send_slot.shape == (T, R)
            with torch.cuda.stream(self.comm_stream):
                o = self.runtime.dispatch(x_data.data_ptr(), x_scales.data_ptr() if x_scales is not None else 0, 0, 0,
                                          0, send_slot.data_ptr(), 0, 0, T, H, h_K, 0, mode, True, -1, 0, 1, 0,
                                          round_scale, self._sms(config), self.comm_stream.cuda_stream)
            recv_x = self._view_x(o, num_recv, H, out_fp8)
            if copy_out:
                with torch.cuda.stream(self.comm_stream):
                    recv_x = tuple(t.clone() for t in recv_x) if isinstance(recv_x, tuple) else recv_x.clone()
            ev = self._exit(compute, async_finish, (x_data, x_scales, send_slot))
            return recv_x, None, None, None, None, ev

        assert num_tokens_per_rank is not None and is_token_in_rank is not None and num_tokens_per_expert is not None
        K = 0
        if topk_idx is not None:
            assert topk_idx.dtype == torch.int64 and topk_idx.is_contiguous() and topk_idx.size(0) == T
            K = topk_idx.size(1)
            if topk_weights is not None:
                assert topk_weights.dtype == torch.float32 and topk_weights.is_contiguous()
        E = num_tokens_per_expert.numel()
        E_local = E // R
        with torch.cuda.stream(self.comm_stream):
            cache = self._layout_cache
            if cache is not None and cache[0] == is_token_in_rank.data_ptr() and cache[1] == T:
                token_pos = cache[2]
            else:
                token_pos = torch.empty((max(T, 1), R), dtype=torch.int32, device=dev)[:T]
                if T > 0:
                    self.runtime.layout(0, T, 0, 0, 0, 0, is_token_in_rank.data_ptr(), token_pos.data_ptr(),
                                        self.comm_stream.cuda_stream)
            send_slot = torch.empty((max(T, 1), R), dtype=torch.int32, device=dev)[:T]  # non-null even for T == 0
            rank_prefix = torch.empty((R, R), dtype=torch.int32, device=dev)
            o = self.runtime.dispatch(
                x_data.data_ptr(), x_scales.data_ptr() if x_scales is not None else 0,
                topk_idx.data_ptr() if topk_idx is not None else 0,
                topk_weights.data_ptr() if topk_weights is not None else 0, token_pos.data_ptr(),
                send_slot.data_ptr(), num_tokens_per_rank.data_ptr(), num_tokens_per_expert.data_ptr(), T, H, K, E,
                mode, False, -1, rank_prefix.data_ptr(), expert_alignment, num_worst_tokens, round_scale,
                self._sms(config), self.comm_stream.cuda_stream)
        if num_worst_tokens > 0:
            num_recv = num_worst_tokens
            per_expert: List[int] = []
        else:
            num_recv, per_expert = self.runtime.wait_counts(E_local, 0.0)
        recv_x = self._view_x(o, num_recv, H, out_fp8)
        recv_topk_idx = recv_topk_weights = None
        if topk_idx is not None:
            recv_topk_idx = self._view(o.recv_topk_idx, (num_recv, K), torch.int64)
            if topk_weights is not None:
                recv_topk_weights = self._view(o.recv_topk_w, (num_recv, K), torch.float32)
        recv_src_idx = self._view(o.recv_src_idx, (num_recv,), torch.int32)
        if copy_out:  # owned tensors (DeepEP semantics): survive any number of later dispatches
            with torch.cuda.stream(self.comm_stream):
                recv_x = tuple(t.clone() for t in recv_x) if isinstance(recv_x, tuple) else recv_x.clone()
                recv_topk_idx = recv_topk_idx.clone() if recv_topk_idx is not None else None
                recv_topk_weights = recv_topk_weights.clone() if recv_topk_weights is not None else None
                recv_src_idx = recv_src_idx.clone()
        handle = EpHandle(rank_prefix, num_recv, recv_src_idx, is_token_in_rank, send_slot, slot=o.slot, num_topk=K)
        ev = self._exit(compute, async_finish, (x_data, x_scales, topk_idx, topk_weights, send_slot, rank_prefix,
                                                token_pos, num_tokens_per_rank, num_tokens_per_expert))
        return recv_x, recv_topk_idx, recv_topk_weights, per_expert, handle, ev

    def _view(self, ptr: int, shape, dtype) -> torch.Tensor:
        numel = 1
        for s in shape:
            numel *= int(s)
        nbytes = max(numel * torch.empty((), dtype=dtype).element_size(), 1)
        holder = _RawView(ptr, nbytes, self)
        flat = torch.as_tensor(holder, device=self.device)
        nb = numel * torch.empty((), dtype=dtype).element_size()
        return flat[:nb].view(dtype).reshape(shape)

    def _view_x(self, o, num_recv, H, out_fp8):
        if out_fp8:
            x = self._view(o.recv_x, (num_recv, H), torch.float8_e4m3fn)
            s = self._view(o.recv_scales, (num_recv, H // 128), torch.float32)
            return (x, s)
        return self._view(o.recv_x, (num_recv, H), torch.bfloat16)

    # ------------------------------------------------------------------------ combine
    def get_combine_buffer(self, num_tokens: int, hidden: int, num_topk: int = 0) -> torch.Tensor:
        """[num_tokens, hidden] bf16 view of the symmetric combine arena: write the expert
        outputs here and pass it to :meth:`combine` for a zero-copy pull-reduce."""
        ptr = self.runtime.combine_input_ptr(num_tokens, hidden, num_topk)
        return self._view(ptr, (num_tokens, hidden), torch.bfloat16)

    def combine(self, x: torch.Tensor, handle: Tuple, topk_weights: Optional[torch.Tensor] = None,
                bias: Union[torch.Tensor, Tuple[torch.Tensor, torch.Tensor], None] = None,
                config: Optional[Config] = None, previous_event: Optional[EventOverlap] = None,
                async_finish: bool = False, allocate_on_comm_stream: bool = False):
        config = config or self.get_combine_config(self.group_size)
        send_slot, num_recv = handle.send_slot, handle.num_recv
        assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.is_contiguous()
        assert x.size(0) >= num_recv or x.size(0) == num_recv
        H = x.size(1)
        T = send_slot.size(0)
        b0 = b1 = None
        if bias is not None:
            if isinstance(bias, tuple):
                b0, b1 = bias
            else:
                b0 = bias
        compute = self._enter(previous_event, allocate_on_comm_stream)
        with torch.cuda.stream(self.comm_stream):
            out = torch.empty((T, H), dtype=torch.bfloat16, device=self.device)
            out_w = None
            if topk_weights is not None:
                assert topk_weights.dtype == torch.float32 and topk_weights.is_contiguous()
                Kw = topk_weights.size(1)
                out_w = torch.empty((T, Kw), dtype=torch.float32, device=self.device)
            else:
                Kw = 0
            self.runtime.combine(x.data_ptr(), x.size(0), topk_weights.data_ptr() if topk_weights is not None else 0,
                                 send_slot.data_ptr(), b0.data_ptr() if b0 is not None else 0,
                                 b1.data_ptr() if b1 is not None else 0, out.data_ptr(),
                                 out_w.data_ptr() if out_w is not None else 0, T, H, Kw, self._sms(config),
                                 self.comm_stream.cuda_stream)
        ev = self._exit(compute, async_finish, (x, topk_weights, b0, b1, out, out_w, send_slot))
        return out, out_w, ev

    def combine_rmsnorm(self, x: torch.Tensor, handle: Tuple, residual: torch.Tensor, weight: torch.Tensor,
                        eps: float = 1e-6, *, bias: Union[torch.Tensor, Tuple[torch.Tensor, torch.Tensor], None] = None,
                        residual_out: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                        quant: Optional[str] = None, config: Optional[Config] = None,
                        previous_event: Optional[EventOverlap] = None, async_finish: bool = False,
                        allocate_on_comm_stream: bool = False):
        """The tail of an MoE layer in one kernel: :meth:`combine`, the residual add and RMSNorm.

        ``combined = combine(x, handle, bias=bias)`` (bitwise what :meth:`combine` returns) is not stored anywhere;
        ``residual_out = bf16(combined + residual)``, written over ``residual`` unless given, and
        ``out = rmsnorm(residual_out, eps) * weight``.  ``residual``, ``residual_out`` and ``out`` are this rank's
        ``[T, H]`` tokens (``T = handle.send_slot.size(0)``), ``weight`` is ``[H]``, all bf16; ``H % 8 == 0`` and
        ``H <= 16384``.  With ``quant="fp8"`` (``H % 128 == 0``) ``out`` is ``(e4m3 [T, H], fp32 scales [T, H/128])``,
        bit-identical to ``per_token_cast_to_fp8`` of the bf16 ``out``: the input format of :meth:`dispatch`.
        Returns ``(out, event)``.  Streams, events and ``config.num_sms`` behave as in :meth:`combine`, so the call
        can be captured in a CUDA graph."""
        config = config or self.get_combine_config(self.group_size)
        send_slot, num_recv = handle.send_slot, handle.num_recv
        T = send_slot.size(0)
        b0, b1, residual_out, out, scales = _combine_rmsnorm_args(x, T, residual, weight, bias, residual_out, out,
                                                                  quant, self.device)
        if x.size(0) < num_recv:
            raise ValueError(f"uccl_b200.ep: combine_rmsnorm x has {x.size(0)} rows, the handle {num_recv}")
        H = x.size(1)
        compute = self._enter(previous_event, allocate_on_comm_stream)
        with torch.cuda.stream(self.comm_stream):
            self.runtime.combine_rmsnorm(x.data_ptr(), x.size(0), send_slot.data_ptr(),
                                         b0.data_ptr() if b0 is not None else 0, b1.data_ptr() if b1 is not None else 0,
                                         residual.data_ptr(), residual_out.data_ptr(), weight.data_ptr(), out.data_ptr(),
                                         scales.data_ptr() if scales is not None else 0, T, H, float(eps),
                                         self._sms(config), self.comm_stream.cuda_stream)
        ev = self._exit(compute, async_finish, (x, b0, b1, residual, residual_out, weight, out, scales, send_slot))
        return ((out, scales) if scales is not None else out), ev

    # ------------------------------------------------------------------ internode entry points
    # The reference routes to RDMA+NVLink two-hop kernels when the group spans several nodes
    # (ep/bench/buffer.py:1333-1552 -> ep/src/internode.cu).  Inside one NVLink domain every rank is
    # a single load/store hop away, so the same call signatures run the direct-placement kernels;
    # `num_tokens_per_rdma_rank` (the per-node histogram of the two-hop scheme) is accepted and
    # ignored.  Callers written against the internode API therefore work unchanged on an NVSwitch
    # node; a group that is not fully peer-mapped cannot be constructed in the first place.
    def internode_dispatch(self, x, handle: Optional[Tuple] = None, num_tokens_per_rank: Optional[torch.Tensor] = None,
                           num_tokens_per_rdma_rank: Optional[torch.Tensor] = None,
                           is_token_in_rank: Optional[torch.Tensor] = None,
                           num_tokens_per_expert: Optional[torch.Tensor] = None,
                           topk_idx: Optional[torch.Tensor] = None, topk_weights: Optional[torch.Tensor] = None,
                           expert_alignment: int = 1, num_worst_tokens: int = 0, config: Optional[Config] = None,
                           previous_event: Optional[EventOverlap] = None, async_finish: bool = False,
                           allocate_on_comm_stream: bool = False, **kw):
        if num_tokens_per_rdma_rank is not None and num_tokens_per_rdma_rank.numel() != self.get_num_rdma_ranks():
            # a layout computed for several RDMA groups does not describe this (single NVLink domain) group
            raise ValueError(f"internode_dispatch: num_tokens_per_rdma_rank has {num_tokens_per_rdma_rank.numel()} entries, "
                             f"this group is {self.get_num_rdma_ranks()} NVLink domain")
        return self.dispatch(x, handle=handle, num_tokens_per_rank=num_tokens_per_rank,
                             num_tokens_per_rdma_rank=None, is_token_in_rank=is_token_in_rank,
                             num_tokens_per_expert=num_tokens_per_expert, topk_idx=topk_idx,
                             topk_weights=topk_weights, expert_alignment=expert_alignment,
                             num_worst_tokens=num_worst_tokens, config=config, previous_event=previous_event,
                             async_finish=async_finish, allocate_on_comm_stream=allocate_on_comm_stream, **kw)

    def internode_combine(self, x: torch.Tensor, handle: Tuple, topk_weights: Optional[torch.Tensor] = None,
                          bias=None, config: Optional[Config] = None, previous_event: Optional[EventOverlap] = None,
                          async_finish: bool = False, allocate_on_comm_stream: bool = False):
        return self.combine(x, handle, topk_weights=topk_weights, bias=bias, config=config,
                            previous_event=previous_event, async_finish=async_finish,
                            allocate_on_comm_stream=allocate_on_comm_stream)

    def get_local_buffer_tensor(self, dtype: torch.dtype, size: Optional[torch.Size] = None, offset: int = 0,
                                use_rdma_buffer: bool = False) -> torch.Tensor:
        """Raw view (slice supported) of this rank's communication memory as a tensor, like the reference's
        (ep/bench/buffer.py:606-647): the NVLink arenas of the EP block, or with ``use_rdma_buffer=True`` the
        low-latency block.  `offset` and `size` count elements of `dtype`.  The control words (barrier flags,
        count tables) are not part of the view."""
        if use_rdma_buffer:
            self._need_ll()
            ptr, nbytes = int(self.runtime.ll_ptr), int(self.runtime.ll_nbytes)
            if nbytes == 0:
                raise RuntimeError("uccl_b200.ep: the low-latency block is allocated by the first low_latency_dispatch")
        else:
            ptr, nbytes = int(self.runtime.arena_area_ptr), int(self.runtime.arena_area_bytes)
        es = torch.empty((), dtype=dtype).element_size()
        total = nbytes // es
        if not 0 <= offset <= total:
            raise ValueError(f"get_local_buffer_tensor: offset {offset} outside the buffer ({total} elements)")
        t = self._view(ptr + offset * es, (total - offset,), dtype)
        if size is None:
            return t
        n = 1
        for d in size:
            n *= int(d)
        if n > t.numel():
            raise ValueError(f"get_local_buffer_tensor: {n} elements requested, {t.numel()} available")
        return t[:n].view(size)

    def reset_rdma_buffer(self) -> None:
        """Reference: zeroes the RDMA buffer for a fresh run (ep/bench/buffer.py:213-218).  Signalling here is epoch
        based, so nothing NEEDS zeroing; the call completes a pending receive hook and clears the low-latency block
        on the current stream so that stale rows cannot be mistaken for results.  Like the reference's it is a LOCAL
        memset: peers write into this block, so call it with the group quiescent (a barrier on both sides)."""
        ll = self._need_ll()
        ll._finish_pending()
        if int(self.runtime.ll_nbytes) > 0:
            self.get_local_buffer_tensor(torch.uint8, use_rdma_buffer=True).zero_()

    def connect_atomic_buffer(self, proxy) -> None:
        """Reference: hands the proxy the buffer its emulated RDMA atomics land in (ep/bench/buffer.py:220-221).
        A :class:`uccl_b200.ep.Proxy` addresses any location of any peer's heap directly (ordered release-add on the
        copy stream), so there is nothing to connect; the call only checks the argument."""
        from .proxy import Proxy

        if not isinstance(proxy, Proxy):
            raise TypeError("connect_atomic_buffer expects a uccl_b200.ep.Proxy")

    def get_num_rdma_ranks(self) -> int:
        """Number of RDMA (inter-node) hops groups: always 1 -- the whole group is one NVLink domain."""
        return 1

    # ------------------------------------------------------------------ low latency
    def _need_ll(self):
        assert self._ll is not None, "construct Buffer with low_latency_mode=True / num_rdma_bytes > 0"
        return self._ll

    def clean_low_latency_buffer(self, num_max_dispatch_tokens_per_rank: int, hidden: int, num_experts: int):
        self._need_ll().clean(num_max_dispatch_tokens_per_rank, hidden, num_experts)

    def low_latency_dispatch(self, x, topk_idx, num_max_dispatch_tokens_per_rank: int, num_experts: int, **kw):
        return self._need_ll().dispatch(x, topk_idx, num_max_dispatch_tokens_per_rank, num_experts, **kw)

    def low_latency_combine(self, x, topk_idx, topk_weights, handle, **kw):
        return self._need_ll().combine(x, topk_idx, topk_weights, handle, **kw)

    def low_latency_combine_rmsnorm(self, x: torch.Tensor, topk_idx: torch.Tensor, topk_weights: torch.Tensor, handle,
                                    residual: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6, *,
                                    shared: Optional[torch.Tensor] = None, residual_out: Optional[torch.Tensor] = None,
                                    out: Optional[torch.Tensor] = None, quant: Optional[str] = None,
                                    use_logfmt: bool = False, zero_copy: bool = False, async_finish: bool = False,
                                    return_recv_hook: bool = False,
                                    combine_wait_recv_cost_stats: Optional[torch.Tensor] = None):
        """The tail of a decode MoE layer in one kernel: :meth:`low_latency_combine`, the shared-expert add, the residual
        add and RMSNorm.

        ``routed = low_latency_combine(x, topk_idx, topk_weights, handle, use_logfmt=...)`` (bitwise what that call
        returns) is not stored anywhere; ``combined = routed``, or ``bf16(routed + shared)`` with a shared-expert output
        (exactly torch's bf16 ``routed + shared``: unlike :meth:`combine_rmsnorm`'s ``bias``, which is added in fp32
        before the single rounding, ``shared`` is added after ``routed`` is rounded, as unfused decode code does);
        ``residual_out = bf16(combined + residual)``, written over ``residual`` unless given, and
        ``out = rmsnorm(residual_out, eps) * weight``.  ``residual``, ``residual_out``, ``shared`` and ``out`` are this
        rank's ``[T, H]`` tokens (``T = topk_weights.size(0)``), ``weight`` is ``[H]``, all bf16; the LL limits hold
        (``H % 128 == 0``, ``H <= 8192``, ``K <= 32``).  With ``quant="fp8"`` ``out`` is
        ``(e4m3 [T, H], fp32 scales [T, H/128])``, bit-identical to ``per_token_cast_to_fp8`` of the bf16 ``out``.
        Returns ``(out, event, hook)`` like :meth:`low_latency_combine`; with ``return_recv_hook=True`` the send half
        runs now and the fused receive half when ``hook()`` is called (or by the next low-latency call)."""
        return self._need_ll().combine_rmsnorm(
            x, topk_idx, topk_weights, handle, residual, weight, eps, shared=shared, residual_out=residual_out, out=out,
            quant=quant, use_logfmt=use_logfmt, zero_copy=zero_copy, async_finish=async_finish,
            return_recv_hook=return_recv_hook, combine_wait_recv_cost_stats=combine_wait_recv_cost_stats)

    def get_next_low_latency_combine_buffer(self, handle):
        return self._need_ll().next_combine_buffer(handle)


class _RawView:
    """Exposes raw heap memory to torch through ``__cuda_array_interface__`` (no ownership)."""

    def __init__(self, ptr: int, nbytes: int, keepalive):
        self._keep = keepalive
        self.__cuda_array_interface__ = {
            "shape": (int(nbytes),),
            "typestr": "|u1",
            "data": (int(ptr), False),
            "version": 3,
            "strides": None,
        }
