"""CPU reference backend of the DeepEP ``Buffer`` API (host-fake communicators).

``Buffer(comm=<host Communicator>)`` returns a :class:`HostBuffer`: the same method signatures and the
same semantics as the CUDA kernels -- receive order (source-rank major, token order minor), top-k ids
remapped to local experts / -1, weights zeroed for foreign experts, cached handles, ``expert_alignment``,
``num_worst_tokens``, unweighted combine (+ bias), low-latency dispatch into per-expert buffers and
weighted low-latency combine -- executed with torch CPU ops, the payload exchanged through the host
communicator's ``all_to_all_v``.  It exists so that code written against the EP API (MoE layers, routing
logic, tests) runs in GPU-less CI, the role ukernel's MockBackend plays for the reference
(experimental/ukernel/src/ccl/test/common/backend_test_utils.h:211).  Contracts: SURVEY Appendix C.
"""
from __future__ import annotations

from typing import List, Optional, Tuple, Union

import torch

from ..parallel.comm import Communicator, dtype_code
from .buffer import _combine_rmsnorm_args, _ll_combine_rmsnorm_args
from .utils import EpHandle, EventOverlap, per_token_cast_to_fp8


def _a2av(comm: Communicator, send: torch.Tensor, send_rows: List[int], recv_rows: List[int]) -> torch.Tensor:
    """all_to_all_v of whole rows of a 2-D (or 1-D) tensor; rows are ordered by destination rank."""
    width = torch.Size(send.shape[1:]).numel()  # 1 for 1-D tensors
    flat = send.contiguous().view(torch.uint8).reshape(-1)
    rb = send.element_size() * width
    out = torch.empty(sum(recv_rows) * rb, dtype=torch.uint8)
    comm.all_to_all_v(out, flat, [r * rb for r in send_rows], [r * rb for r in recv_rows])
    return out.view(send.dtype).reshape((sum(recv_rows),) + tuple(send.shape[1:]))


class _DeviceCommAdapter:
    """Lets the CPU reference algorithm run over a communicator whose collectives want device tensors
    (a :class:`MultiNodeCommunicator` built on GPU communicators): operands hop to the device for the call."""

    def __init__(self, comm):
        self._c, self.rank, self.world_size, self._dev = comm, comm.rank, comm.world_size, comm.device

    def _call(self, fn, out, t, *a):
        o, d = out.to(self._dev), t.to(self._dev)
        fn(o, d, *a)
        torch.cuda.current_stream(self._dev).synchronize()
        out.copy_(o)
        return out

    def all_gather(self, out, t):
        return self._call(self._c.all_gather, out, t)

    def all_to_all_v(self, out, t, send_counts, recv_counts):
        return self._call(self._c.all_to_all_v, out, t, send_counts, recv_counts)


def _portable(fn):
    """Public-method wrapper: tensors (also inside tuples / handles) are brought to the CPU for the reference
    algorithm and results go back to the caller's device.  A no-op for host tensors."""
    import functools

    def to_cpu(v, seen):
        if isinstance(v, torch.Tensor):
            if v.is_cuda:
                seen.append(v.device)
                return v.cpu()
            return v
        if isinstance(v, EpHandle):
            return EpHandle(to_cpu(v.rank_prefix, seen), v.num_recv, to_cpu(v.recv_src_idx, seen),
                            to_cpu(v.is_token_in_rank, seen), to_cpu(v.send_slot, seen), slot=v.slot, num_topk=v.num_topk)
        if isinstance(v, tuple):
            return tuple(to_cpu(e, seen) for e in v)
        if isinstance(v, list):
            return [to_cpu(e, seen) for e in v]
        return v

    def to_dev(v, dev):
        if isinstance(v, torch.Tensor):
            return v.to(dev)
        if isinstance(v, EpHandle):
            return EpHandle(to_dev(v.rank_prefix, dev), v.num_recv, to_dev(v.recv_src_idx, dev),
                            to_dev(v.is_token_in_rank, dev), to_dev(v.send_slot, dev), slot=v.slot, num_topk=v.num_topk)
        if isinstance(v, tuple):
            return tuple(to_dev(e, dev) for e in v)
        return v

    @functools.wraps(fn)
    def wrapper(self, *args, **kw):
        seen = []
        stats = kw.get("cumulative_local_expert_recv_stats")
        a = [to_cpu(v, seen) for v in args]
        k = {n: to_cpu(v, seen) for n, v in kw.items()}
        res = fn(self, *a, **k)
        if not seen:
            return res
        if isinstance(stats, torch.Tensor) and stats.is_cuda:  # in-place output argument
            stats.copy_(k["cumulative_local_expert_recv_stats"])
        return to_dev(res, seen[0])

    return wrapper


def _host_add_rmsnorm(combined, residual, residual_out, weight, out, scales, eps):
    """The C++ epilogue of the fused layer tails (the one behind ``Communicator.all_reduce_rmsnorm`` on the host
    backend) on already combined [T, H] bf16 rows.  It runs on host memory; device tensors (the portable multi-box
    path) hop and are written back."""
    from .. import _native

    T, H = combined.shape
    combined = combined.cpu().contiguous()
    res = residual.cpu()
    ro = res if residual_out is residual else residual_out.cpu()
    o, sc = out.cpu(), scales.cpu() if scales is not None else None
    w = weight.cpu()
    _native.C().host_add_rmsnorm(combined.data_ptr(), res.data_ptr(), ro.data_ptr(), w.data_ptr(), o.data_ptr(),
                                 sc.data_ptr() if sc is not None else 0, T, H, dtype_code(torch.bfloat16), float(eps))
    for dst, src in ((residual_out, ro), (out, o), (scales, sc)):
        if dst is not None and dst is not src:
            dst.copy_(src)


class HostBuffer:
    """DeepEP ``Buffer`` API on the CPU -- and the *portable* path for groups that span boxes: with a
    :class:`uccl_b200.parallel.MultiNodeCommunicator` the token exchange rides its two-hop all-to-all (NVLink
    inside a box, one datagram rail per NIC between boxes), which is the shape of the reference's internode
    dispatch; GPU tensors are accepted (the permutation itself then runs on the host -- functional, not fast)."""

    num_sms: int = 24

    def __init__(self, comm: Communicator, num_nvl_bytes: int = 0, num_rdma_bytes: int = 0,
                 low_latency_mode: bool = False, **_):
        self._raw_comm = comm
        self.comm = comm if comm.is_host else _DeviceCommAdapter(comm)
        self.group = getattr(comm, "group", None)
        self.rank = comm.rank
        self.group_size = comm.world_size
        self.device = torch.device("cpu")
        self.low_latency_mode = low_latency_mode
        self.num_nvl_bytes, self.num_rdma_bytes = int(num_nvl_bytes), int(num_rdma_bytes)
        self._ll_parity = 0

    # ------------------------------------------------------------------ parity helpers
    def destroy(self):
        pass

    @staticmethod
    def is_sm90_compiled() -> bool:
        return False

    @staticmethod
    def set_num_sms(new_num_sms: int) -> None:
        HostBuffer.num_sms = int(new_num_sms)

    @staticmethod
    def capture() -> EventOverlap:
        return EventOverlap()

    def get_num_rdma_ranks(self) -> int:
        return int(getattr(self._raw_comm, "num_nodes", 1))  # boxes the group spans

    def get_local_buffer_tensor(self, dtype: torch.dtype, size=None, offset: int = 0, use_rdma_buffer: bool = False):
        """Same contract as the CUDA Buffer: a raw view of this rank's communication memory -- here a host scratch
        block of `num_nvl_bytes` / `num_rdma_bytes` that exists for API compatibility (the host path exchanges
        tensors through the communicator, not through these blocks)."""
        key = "_scratch_rdma" if use_rdma_buffer else "_scratch_nvl"
        nbytes = self.num_rdma_bytes if use_rdma_buffer else self.num_nvl_bytes
        buf = getattr(self, key, None)
        if buf is None:
            buf = torch.zeros(max(nbytes, 8) // 8 * 8, dtype=torch.uint8)
            setattr(self, key, buf)
        t = buf.view(dtype)
        if not 0 <= offset <= t.numel():
            raise ValueError(f"get_local_buffer_tensor: offset {offset} outside the buffer ({t.numel()} elements)")
        t = t[offset:]
        if size is None:
            return t
        n = 1
        for d in size:
            n *= int(d)
        if n > t.numel():
            raise ValueError(f"get_local_buffer_tensor: {n} elements requested, {t.numel()} available")
        return t[:n].view(size)

    def reset_rdma_buffer(self) -> None:
        if getattr(self, "_scratch_rdma", None) is not None:
            self._scratch_rdma.zero_()

    def connect_atomic_buffer(self, proxy) -> None:
        if proxy is None:
            raise TypeError("connect_atomic_buffer expects a proxy")

    # ------------------------------------------------------------------ layout
    @_portable
    def get_dispatch_layout(self, topk_idx: torch.Tensor, num_experts: int, previous_event=None, async_finish=False,
                            allocate_on_comm_stream=False):
        assert topk_idx.dtype == torch.int64 and topk_idx.dim() == 2
        R = self.group_size
        e_per = num_experts // R
        T = topk_idx.size(0)
        valid = topk_idx >= 0
        rk = torch.where(valid, topk_idx // e_per, torch.zeros_like(topk_idx))
        is_in = torch.zeros(T, R, dtype=torch.bool)
        for k in range(topk_idx.size(1)):  # OR over the top-k slots (scatter_ would keep only the last write)
            m = valid[:, k]
            is_in[m.nonzero().flatten(), rk[m, k]] = True
        tokens_per_rank = is_in.sum(0).to(torch.int32)
        tokens_per_expert = torch.bincount(topk_idx[valid], minlength=num_experts).to(torch.int32)
        return tokens_per_rank, None, tokens_per_expert, is_in, EventOverlap()

    # ------------------------------------------------------------------ dispatch
    def _exchange_counts(self, send_counts: torch.Tensor) -> torch.Tensor:
        """R x R matrix cnt[s][d] = tokens rank s sends to rank d."""
        R = self.group_size
        mat = torch.empty(R * R, dtype=torch.int64)
        self.comm.all_gather(mat, send_counts.to(torch.int64).contiguous())
        return mat.view(R, R)

    @_portable
    def dispatch(self, x: Union[torch.Tensor, Tuple[torch.Tensor, torch.Tensor]], handle: Optional[Tuple] = None,
                 num_tokens_per_rank=None, num_tokens_per_rdma_rank=None, is_token_in_rank=None,
                 num_tokens_per_expert=None, topk_idx=None, topk_weights=None, expert_alignment: int = 1,
                 num_worst_tokens: int = 0, config=None, previous_event=None, async_finish: bool = False,
                 allocate_on_comm_stream: bool = False, use_fp8: bool = False, round_scale: bool = False):
        R, me = self.group_size, self.rank
        if isinstance(x, tuple):
            x_data, x_scales = x
            assert not use_fp8
        else:
            x_data, x_scales = x, None
            if use_fp8:
                x_data, x_scales = per_token_cast_to_fp8(x, round_scale=round_scale)
        T, H = x_data.shape
        cached = handle is not None
        if cached:
            rank_prefix, send_slot, recv_src_idx, is_token_in_rank, num_recv, K = (
                handle.rank_prefix, handle.send_slot, handle.recv_src_idx, handle.is_token_in_rank, handle.num_recv, handle.num_topk)
        else:
            assert is_token_in_rank is not None and num_tokens_per_expert is not None
            rank_prefix = self._exchange_counts(is_token_in_rank.sum(0))
        send_counts = [int(v) for v in rank_prefix[me]]
        recv_counts = [int(v) for v in rank_prefix[:, me]]
        order = [is_token_in_rank[:, d].nonzero().flatten() for d in range(R)]  # token order per destination
        sel = torch.cat(order) if T else torch.empty(0, dtype=torch.int64)

        def ship(t):
            return _a2av(self.comm, t[sel], send_counts, recv_counts)

        total = sum(recv_counts)
        pad = max(num_worst_tokens - total, 0) if num_worst_tokens > 0 else 0

        def padded(t, fill=0):
            if not pad:
                return t
            return torch.cat([t, torch.full((pad,) + tuple(t.shape[1:]), fill, dtype=t.dtype)])

        is_fp8 = x_data.dtype == torch.float8_e4m3fn
        rx = padded(ship(x_data.view(torch.uint8) if is_fp8 else x_data))  # fp8 travels as raw bytes
        if is_fp8:
            rx = rx.view(torch.float8_e4m3fn)
        rs = padded(ship(x_scales)) if x_scales is not None else None
        recv_x = (rx, rs) if rs is not None else rx
        if cached:
            return recv_x, None, None, None, None, EventOverlap()
        K = 0
        recv_idx = recv_w = None
        E = num_tokens_per_expert.numel()
        e_per = E // R
        if topk_idx is not None:
            K = topk_idx.size(1)
            ri = ship(topk_idx)
            mine = (ri >= me * e_per) & (ri < (me + 1) * e_per)
            recv_idx = torch.where(mine, ri - me * e_per, torch.full_like(ri, -1))
            if topk_weights is not None:
                rw = ship(topk_weights)
                recv_w = torch.where(mine, rw, torch.zeros_like(rw))
            recv_idx = padded(recv_idx, -1)
            if recv_w is not None:
                recv_w = padded(recv_w, 0)
        recv_src_idx = ship(torch.arange(T, dtype=torch.int32))
        # where does token t land in destination d's receive buffer?  (prefix over lower source ranks)
        send_slot = torch.full((T, R), -1, dtype=torch.int32)
        for d in range(R):
            base = int(rank_prefix[:me, d].sum())
            send_slot[order[d], d] = torch.arange(base, base + order[d].numel(), dtype=torch.int32)
        if num_worst_tokens > 0:
            per_expert: List[int] = []
            num_recv = num_worst_tokens
        else:
            cnt = torch.bincount(recv_idx[recv_idx >= 0], minlength=e_per) if recv_idx is not None else torch.zeros(e_per, dtype=torch.int64)
            per_expert = [int((int(c) + expert_alignment - 1) // expert_alignment * expert_alignment) for c in cnt]
            num_recv = total
        handle = EpHandle(rank_prefix, num_recv, recv_src_idx, is_token_in_rank, send_slot, slot=0, num_topk=K)
        return recv_x, recv_idx, recv_w, per_expert, handle, EventOverlap()

    # ------------------------------------------------------------------ combine
    def get_combine_buffer(self, num_tokens: int, hidden: int, num_topk: int = 0) -> torch.Tensor:
        return torch.empty(num_tokens, hidden, dtype=torch.bfloat16)

    @_portable
    def combine(self, x: torch.Tensor, handle: Tuple, topk_weights: Optional[torch.Tensor] = None, bias=None,
                config=None, previous_event=None, async_finish: bool = False, allocate_on_comm_stream: bool = False):
        R, me = self.group_size, self.rank
        rank_prefix, send_slot, recv_src_idx, is_token_in_rank, num_recv, K = (
            handle.rank_prefix, handle.send_slot, handle.recv_src_idx, handle.is_token_in_rank, handle.num_recv, handle.num_topk)
        T = send_slot.size(0)
        H = x.size(1)
        back_send = [int(v) for v in rank_prefix[:, me]]   # what I received, grouped by source, goes back
        back_recv = [int(v) for v in rank_prefix[me]]
        total = sum(back_send)
        rows = _a2av(self.comm, x[:total].contiguous(), back_send, back_recv)
        order = torch.cat([is_token_in_rank[:, d].nonzero().flatten() for d in range(R)]) if T else torch.empty(0, dtype=torch.int64)
        out = torch.zeros(T, H, dtype=torch.float32)
        out.index_add_(0, order, rows.float())
        if bias is not None:
            for b in (bias if isinstance(bias, tuple) else (bias,)):
                if b is not None:
                    out += b.float()
        out_w = None
        if topk_weights is not None:
            wr = _a2av(self.comm, topk_weights[:total].contiguous(), back_send, back_recv)
            out_w = torch.zeros(T, topk_weights.size(1), dtype=torch.float32)
            out_w.index_add_(0, order, wr)
        return out.to(torch.bfloat16), out_w, EventOverlap()

    def combine_rmsnorm(self, x: torch.Tensor, handle: Tuple, residual: torch.Tensor, weight: torch.Tensor,
                        eps: float = 1e-6, *, bias=None, residual_out: Optional[torch.Tensor] = None,
                        out: Optional[torch.Tensor] = None, quant: Optional[str] = None, config=None,
                        previous_event=None, async_finish: bool = False, allocate_on_comm_stream: bool = False):
        """:meth:`combine`, then the C++ epilogue of the fused layer tails (the one behind
        ``Communicator.all_reduce_rmsnorm`` on the host backend).  Same contract as the CUDA ``combine_rmsnorm``."""
        T = handle.send_slot.size(0)
        _, _, residual_out, out, scales = _combine_rmsnorm_args(x, T, residual, weight, bias, residual_out, out, quant,
                                                                residual.device)
        combined = self.combine(x, handle, bias=bias)[0]
        _host_add_rmsnorm(combined, residual, residual_out, weight, out, scales, eps)
        return ((out, scales) if scales is not None else out), EventOverlap()

    internode_dispatch = dispatch
    internode_combine = combine

    # ------------------------------------------------------------------ low latency
    @staticmethod
    def get_low_latency_rdma_size_hint(num_max_dispatch_tokens_per_rank: int, hidden: int, num_ranks: int,
                                       num_experts: int) -> int:
        return 0

    def clean_low_latency_buffer(self, *a, **kw):
        pass

    @_portable
    def low_latency_dispatch(self, x: torch.Tensor, topk_idx: torch.Tensor, num_max_dispatch_tokens_per_rank: int,
                             num_experts: int, cumulative_local_expert_recv_stats=None,
                             dispatch_wait_recv_cost_stats=None, use_fp8: bool = True, round_scale: bool = False,
                             use_ue8m0: bool = False, async_finish: bool = False, return_recv_hook: bool = False,
                             scales_row_major: bool = False, use_nvfp4: bool = False, x_global_scale=None):
        if use_nvfp4 or x_global_scale is not None:
            raise NotImplementedError("uccl_b200.ep: NVFP4 low-latency dispatch (use_nvfp4 / x_global_scale) is not "
                                      "supported; use use_fp8=True (e4m3 + per-128 scales) or bf16")
        R, me = self.group_size, self.rank
        T, H = x.shape
        K = topk_idx.size(1)
        M, E = int(num_max_dispatch_tokens_per_rank), int(num_experts)
        e_per = E // R
        assert T <= M
        tk = topk_idx.reshape(-1)
        tok = torch.arange(T).repeat_interleave(K)
        valid = tk >= 0
        ev, tv = tk[valid], tok[valid]
        key = ev * (T + 1) + tv  # sort by (expert, token): experts are rank-major, so this is destination-major
        o = torch.argsort(key, stable=True)
        ev, tv = ev[o], tv[o]
        per_expert = torch.bincount(ev, minlength=E)
        allc = torch.empty(R * E, dtype=torch.int64)
        self.comm.all_gather(allc, per_expert.contiguous())
        allc = allc.view(R, E)  # allc[s][e]: tokens rank s sends to global expert e
        send_rows = [int(per_expert[d * e_per:(d + 1) * e_per].sum()) for d in range(R)]
        recv_rows = [int(allc[s, me * e_per:(me + 1) * e_per].sum()) for s in range(R)]
        payload = x[tv]
        if use_fp8:
            q, s = per_token_cast_to_fp8(payload.contiguous(), round_scale=round_scale)
            rq = _a2av(self.comm, q.view(torch.uint8), send_rows, recv_rows).view(torch.float8_e4m3fn)
            rsc = _a2av(self.comm, s.contiguous(), send_rows, recv_rows)
        else:
            rq = _a2av(self.comm, payload.contiguous(), send_rows, recv_rows)
            rsc = None
        r_src = _a2av(self.comm, tv.to(torch.int32), send_rows, recv_rows)
        # unpack: data from source s arrives ordered by local expert; place it at [e, begin(e, s) + i]
        rows = R * M
        recv_x = torch.zeros(e_per, rows, H, dtype=rq.dtype if not use_fp8 else torch.uint8)
        recv_sc = torch.zeros(e_per, rows, H // 128, dtype=torch.float32) if use_fp8 else None
        src_info = torch.zeros(e_per, rows, dtype=torch.int32)
        layout_range = torch.zeros(e_per, R, dtype=torch.int64)
        mine = allc[:, me * e_per:(me + 1) * e_per]  # [R, e_per]
        begin = torch.cumsum(mine, 0) - mine         # begin(e, s) = sum over lower sources
        pos = 0
        for s in range(R):
            for e in range(e_per):
                c = int(mine[s, e])
                b = int(begin[s, e])
                layout_range[e, s] = (b << 32) | c  # begin in the high word, count in the low one (internode_ll.cu:573)
                if c:
                    seg = slice(pos, pos + c)
                    recv_x[e, b:b + c] = rq[seg].view(torch.uint8) if use_fp8 else rq[seg]
                    if use_fp8:
                        recv_sc[e, b:b + c] = rsc[seg]
                    src_info[e, b:b + c] = r_src[seg]
                    pos += c
        recv_count = mine.sum(0).to(torch.int32)
        if cumulative_local_expert_recv_stats is not None:
            cumulative_local_expert_recv_stats.add_(recv_count)
        if use_fp8:
            scales = recv_sc
            if use_ue8m0:
                from .utils import pack_ue8m0

                assert round_scale and H % 512 == 0
                scales = pack_ue8m0(torch.where(scales > 0, scales, torch.ones_like(scales)))
            elif not scales_row_major:
                # same strides as the CUDA path / DeepEP: column-major in the last two dims
                scales = scales.transpose(1, 2).contiguous().transpose(1, 2)
            out_x = (recv_x.view(torch.float8_e4m3fn), scales)
        else:
            out_x = recv_x
        # my send position of (t, k) inside the destination expert's buffer: begin(e, me) + index among my tokens
        send_pos = torch.full((T, K), -1, dtype=torch.int64)
        gb = torch.cumsum(allc, 0) - allc  # gb[s][e]
        seen = {}
        for e_, t_ in zip(ev.tolist(), tv.tolist()):
            i = seen.get(e_, 0)
            seen[e_] = i + 1
            k_ = int((topk_idx[t_] == e_).nonzero()[0])
            send_pos[t_, k_] = int(gb[me, e_]) + i
        self._ll_parity ^= 1
        handle = (src_info, layout_range, M, H, E, self._ll_parity, send_pos, allc)
        hook = (lambda: None) if return_recv_hook else None
        return out_x, recv_count, handle, EventOverlap(), hook

    def get_next_low_latency_combine_buffer(self, handle):
        src_info, layout_range, M, H, E = handle[:5]
        return torch.zeros(E // self.group_size, self.group_size * M, H, dtype=torch.bfloat16)

    @_portable
    def low_latency_combine(self, x: torch.Tensor, topk_idx: torch.Tensor, topk_weights: torch.Tensor, handle,
                            use_logfmt: bool = False, zero_copy: bool = False, async_finish: bool = False,
                            return_recv_hook: bool = False, out: Optional[torch.Tensor] = None,
                            combine_wait_recv_cost_stats=None):
        if use_logfmt:
            if zero_copy:
                raise ValueError("uccl_b200.ep: zero_copy and use_logfmt are mutually exclusive (as in the reference)")
            from .utils import logfmt10_simulate

            x = logfmt10_simulate(x)  # the reference's simulated cast: payload stays bf16, numerics change
        R, me = self.group_size, self.rank
        src_info, layout_range, M, H, E, _, send_pos, allc = handle
        e_per = E // R
        mine = allc[:, me * e_per:(me + 1) * e_per]
        begin = torch.cumsum(mine, 0) - mine
        # send every source its rows back, grouped by source, ordered by local expert (= its own send order)
        chunks, back_send = [], []
        for s in range(R):
            parts = [x[e, int(begin[s, e]):int(begin[s, e]) + int(mine[s, e])] for e in range(e_per)]
            seg = torch.cat(parts) if parts else x.new_zeros(0, H)
            chunks.append(seg)
            back_send.append(seg.size(0))
        T, K = topk_idx.shape
        back_recv = [int(allc[me, d * e_per:(d + 1) * e_per].sum()) for d in range(R)]
        rows = _a2av(self.comm, torch.cat(chunks).contiguous(), back_send, back_recv)
        # rows arrive destination-major, expert-ascending, token-ascending: the order low_latency_dispatch sent them in
        tk = topk_idx.reshape(-1)
        tok = torch.arange(T).repeat_interleave(K)
        kk = torch.arange(K).repeat(T)
        valid = tk >= 0
        ev, tv, kv = tk[valid], tok[valid], kk[valid]
        o = torch.argsort(ev * (T + 1) + tv, stable=True)
        tv, kv = tv[o], kv[o]
        res = torch.zeros(T, H, dtype=torch.float32)
        res.index_add_(0, tv, rows.float() * topk_weights[tv, kv].unsqueeze(1))
        res = res.to(torch.bfloat16)
        if out is not None:
            out.copy_(res)
            res = out
        hook = (lambda: None) if return_recv_hook else None
        return res, EventOverlap(), hook

    def low_latency_combine_rmsnorm(self, x: torch.Tensor, topk_idx: torch.Tensor, topk_weights: torch.Tensor, handle,
                                    residual: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6, *,
                                    shared: Optional[torch.Tensor] = None, residual_out: Optional[torch.Tensor] = None,
                                    out: Optional[torch.Tensor] = None, quant: Optional[str] = None,
                                    use_logfmt: bool = False, zero_copy: bool = False, async_finish: bool = False,
                                    return_recv_hook: bool = False, combine_wait_recv_cost_stats=None):
        """:meth:`low_latency_combine`, torch's bf16 ``+ shared``, then the C++ epilogue of the fused layer tails (as
        in :meth:`combine_rmsnorm`).  Same contract as the CUDA ``low_latency_combine_rmsnorm``."""
        M, H, E = handle[2:5]
        _, _, residual_out, out, scales = _ll_combine_rmsnorm_args(x, topk_idx, topk_weights, self.group_size, M, H, E,
                                                                   residual, weight, shared, residual_out, out, quant,
                                                                   residual.device)
        combined = self.low_latency_combine(x, topk_idx, topk_weights, handle, use_logfmt=use_logfmt,
                                            zero_copy=zero_copy)[0].cpu()
        if shared is not None:
            combined = combined + shared.cpu()  # bf16 + bf16, rounded once: what unfused decode code computes
        _host_add_rmsnorm(combined, residual, residual_out, weight, out, scales, eps)
        hook = (lambda: None) if return_recv_hook else None
        return ((out, scales) if scales is not None else out), EventOverlap(), hook
