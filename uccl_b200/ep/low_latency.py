"""Low-latency (decode) dispatch / combine -- DeepEP ``low_latency_*`` API.

Reference: ep/bench/buffer.py:263-566 (python), ep/src/internode_ll.cu (kernels).
Return conventions follow DeepEP:
  dispatch -> (recv_x | (recv_x_fp8, scales), recv_count, handle, event, hook)
     recv_x  [E_local, R*M, H]; tokens of expert e are rows [0, recv_count[e]) (packed)
     scales  [E_local, R*M, H/128] float32, column-major in the last two dims like DeepEP's transposed view
             (ep/src/internode_ll.cu:608-636); ``use_ue8m0`` -> [E_local, R*M, H/512] int32 (4 exponent bytes
             per word), packed by the kernel; ``scales_row_major=True`` keeps plain row-major fp32
     handle  (src_info, layout_range, M, H, E, buffer_idx, send_pos)
  combine  -> (combined_x [T, H] bf16, event, hook)
``return_recv_hook=True`` splits each call into a SEND kernel (launched now; it returns as soon as everything is
on the wire) and a RECV kernel launched by ``hook()`` -- between the two no SM is held, which is what lets two
micro-batches overlap (ep/src/uccl_ep.cc:1269-1283).  Outputs are valid after ``hook()``.
Kernels run on the CURRENT stream (as in DeepEP's low-latency path): no stream hop on the decode critical path.
Only two LL buffers exist (as in DeepEP): at most two dispatch results may be alive.
"""
from __future__ import annotations

from typing import Optional

import torch

from .utils import EventHandle, EventOverlap


def ll_size_hint(num_max_dispatch_tokens_per_rank: int, hidden: int, num_ranks: int, num_experts: int) -> int:
    from .. import _native

    return int(_native.C().EpBuffer.ll_size_hint(num_max_dispatch_tokens_per_rank, hidden, num_ranks, num_experts))


class LowLatencyRuntime:
    def __init__(self, buf, num_bytes: int):
        self.buf = buf
        self.rt = buf.runtime
        self.num_bytes = int(num_bytes)
        if self.num_bytes > 0:
            self.rt.ll_init(self.num_bytes)
        self._state = {}
        self._pending = None  # receive hook of a SEND-phase call that has not run yet

    def _ensure(self, M, H, E):
        need = ll_size_hint(M, H, self.buf.group_size, E)
        if self.num_bytes == 0:
            self.num_bytes = need
            self.rt.ll_init(need)
        assert need <= self.num_bytes, f"low-latency buffer too small: need {need} bytes, have {self.num_bytes}"

    def clean(self, M, H, E):
        # signalling is epoch based: nothing to zero (reference needs clean_low_latency_buffer, buffer.py:1797)
        self._ensure(M, H, E)

    def _sms(self, combine: bool = False):
        from .buffer import Config

        # one CTA per token in both directions (a decode batch has about as many tokens as the GPU has SMs)
        return self.buf._sms(Config(128))

    def _finish_pending(self):
        """A hook that was never called would leave the next kernel waiting on a stale epoch: run it now."""
        h = self._pending
        if h is not None:
            h()  # clears self._pending itself

    def dispatch(self, x: torch.Tensor, topk_idx: torch.Tensor, num_max_dispatch_tokens_per_rank: int,
                 num_experts: int, cumulative_local_expert_recv_stats: Optional[torch.Tensor] = None,
                 dispatch_wait_recv_cost_stats: Optional[torch.Tensor] = None, use_fp8: bool = True,
                 round_scale: bool = False, use_ue8m0: bool = False, async_finish: bool = False,
                 return_recv_hook: bool = False, scales_row_major: bool = False, use_nvfp4: bool = False,
                 x_global_scale: Optional[torch.Tensor] = None):
        if use_nvfp4 or x_global_scale is not None:
            # newer DeepEP builds can dispatch NVFP4 (e2m1 + a global scale): vLLM passes these only for NVFP4-quantised
            # models.  Not provided here -- fail with a message instead of a TypeError on an unknown keyword.
            raise NotImplementedError("uccl_b200.ep: NVFP4 low-latency dispatch (use_nvfp4 / x_global_scale) is not "
                                      "supported; use use_fp8=True (e4m3 + per-128 scales) or bf16")
        if use_ue8m0:
            assert use_fp8 and round_scale, "use_ue8m0 needs use_fp8=True and round_scale=True (power-of-two scales)"
            assert x.size(1) % 512 == 0, "use_ue8m0 packs four per-128-channel scales per word: hidden % 512 == 0"
        assert x.dtype == torch.bfloat16 and x.dim() == 2 and x.is_contiguous()
        assert topk_idx.dtype == torch.int64 and topk_idx.is_contiguous()
        assert not (async_finish and return_recv_hook), "async_finish and return_recv_hook are mutually exclusive"
        self._finish_pending()
        b = self.buf
        C = b._C
        R = b.group_size
        T, H = x.shape
        K = topk_idx.size(1)
        M, E = int(num_max_dispatch_tokens_per_rank), int(num_experts)
        E_local = E // R
        self._ensure(M, H, E)
        dev = b.device
        st = torch.cuda.current_stream(dev)
        if dispatch_wait_recv_cost_stats is not None:
            assert dispatch_wait_recv_cost_stats.dtype == torch.int64 and dispatch_wait_recv_cost_stats.numel() >= R
        stats_ptr = dispatch_wait_recv_cost_stats.data_ptr() if dispatch_wait_recv_cost_stats is not None else 0
        layout = C.EP_LL_SCALES_ROW_MAJOR
        if use_fp8 and not scales_row_major:
            layout = C.EP_LL_SCALES_COL_UE8M0 if use_ue8m0 else C.EP_LL_SCALES_COL_MAJOR
        recv_count = torch.empty(E_local, dtype=torch.int32, device=dev)
        layout_range = torch.empty((E_local, R), dtype=torch.int64, device=dev)
        send_pos = torch.empty((T, K), dtype=torch.int64, device=dev)
        sms = self._sms()
        rx, rs, rsrc, cx, idx = self.rt.ll_dispatch(
            x.data_ptr(), topk_idx.data_ptr(), T, H, K, E, M, use_fp8, round_scale, recv_count.data_ptr(),
            layout_range.data_ptr(), send_pos.data_ptr(), sms, st.cuda_stream,
            phase=C.EP_LL_SEND if return_recv_hook else C.EP_LL_FULL, scale_layout=layout, wait_stats=stats_ptr)
        rows = R * M
        if use_fp8:
            if layout == C.EP_LL_SCALES_ROW_MAJOR:
                scales = b._view(rs, (E_local, rows, H // 128), torch.float32)
                if use_ue8m0:
                    from .utils import pack_ue8m0

                    scales = pack_ue8m0(scales)  # torch post-pass (row-major request only)
            elif layout == C.EP_LL_SCALES_COL_MAJOR:
                scales = b._view(rs, (E_local, H // 128, rows), torch.float32).transpose(1, 2)
            else:
                scales = b._view(rs, (E_local, H // 512, rows), torch.int32).transpose(1, 2)
            recv_x = (b._view(rx, (E_local, rows, H), torch.float8_e4m3fn), scales)
        else:
            recv_x = b._view(rx, (E_local, rows, H), torch.bfloat16)
        src_info = b._view(rsrc, (E_local, rows), torch.int32)
        handle = (src_info, layout_range, M, H, E, idx, send_pos)

        def finish():
            if cumulative_local_expert_recv_stats is not None:
                cumulative_local_expert_recv_stats.add_(recv_count)

        hook = None
        if return_recv_hook:
            hook = self._recv_hook(st, lambda s: self.rt.ll_dispatch_recv(sms, stats_ptr, s),
                                   (x, topk_idx, recv_count, layout_range, send_pos, dispatch_wait_recv_cost_stats,
                                    cumulative_local_expert_recv_stats), finish)
        else:
            finish()
        ev = EventOverlap(EventHandle(st)) if async_finish else EventOverlap()
        return recv_x, recv_count, handle, ev, hook

    def _recv_hook(self, st, recv, keep, finish=None):
        """The hook of a SEND-phase call made on stream ``st``: ``recv(stream)`` launches the receive half on the stream
        current when the hook runs, then ``finish()`` runs.  Everything the receive half touches (``keep``) stays alive
        until it has run; the next low-latency call runs a hook that was never called."""
        dev = self.buf.device
        sent = torch.cuda.Event()
        sent.record(st)

        def hook():
            if self._pending is hook:
                self._pending = None
                with torch.cuda.device(dev):
                    cur = torch.cuda.current_stream(dev)
                    cur.wait_event(sent)  # the receive half reads the epoch the send half stored: order them even
                    recv(cur.cuda_stream)  # when the hook runs on another stream
                    if finish is not None:
                        finish()

        hook._keep = keep
        self._pending = hook
        return hook

    def _combine(self, launch, args, layout_range, stats, use_logfmt, async_finish, return_recv_hook, keep):
        """Runs ``launch`` (``rt.ll_combine`` or ``rt.ll_combine_rmsnorm``) on ``args`` on the current stream: the whole
        kernel, or with ``return_recv_hook`` the SEND half now and the RECV half from the returned hook.  Returns
        ``(event, hook)``."""
        assert not (async_finish and return_recv_hook), "async_finish and return_recv_hook are mutually exclusive"
        b = self.buf
        C = b._C
        if stats is not None:
            assert stats.dtype == torch.int64 and stats.numel() >= b.group_size
        self._finish_pending()
        st = torch.cuda.current_stream(b.device)
        args = args + (self._sms(combine=True),)
        kw = dict(layout_range=layout_range.data_ptr(), wait_stats=stats.data_ptr() if stats is not None else 0)
        hook = None
        if return_recv_hook:
            # SEND half: (pack the expert outputs into the symmetric buffer and) announce that they are in place
            launch(*args, st.cuda_stream, phase=C.EP_LL_SEND, use_logfmt=bool(use_logfmt), **kw)
            hook = self._recv_hook(st, lambda s: launch(*args, s, phase=C.EP_LL_RECV, **kw),
                                   keep + (layout_range, stats))
        else:
            launch(*args, st.cuda_stream, phase=C.EP_LL_FULL, use_logfmt=bool(use_logfmt), **kw)
        return (EventOverlap(EventHandle(st)) if async_finish else EventOverlap()), hook

    def next_combine_buffer(self, handle):
        src_info, layout_range, M, H, E, idx, send_pos = handle
        b = self.buf
        ptr = self.rt.ll_combine_buffer(idx, H, E, M)
        return b._view(ptr, (E // b.group_size, b.group_size * M, H), torch.bfloat16)

    def combine(self, x: torch.Tensor, topk_idx: torch.Tensor, topk_weights: torch.Tensor, handle,
                use_logfmt: bool = False, zero_copy: bool = False, async_finish: bool = False,
                return_recv_hook: bool = False, out: Optional[torch.Tensor] = None,
                combine_wait_recv_cost_stats: Optional[torch.Tensor] = None):
        if use_logfmt:
            # the reference's LogFMT-10 is a *simulated* cast (ep/src/internode_ll.cu:934-995): rows are snapped to the
            # logarithmic grid and still travel as bf16.  Here the pass that brings the expert outputs into the
            # symmetric buffer applies it (in place when x already is that buffer).
            if zero_copy:
                raise ValueError("uccl_b200.ep: zero_copy and use_logfmt are mutually exclusive (as in the reference)")
            if x.shape[-1] % 128 != 0:
                raise ValueError("uccl_b200.ep: use_logfmt needs hidden % 128 == 0")
        src_info, layout_range, M, H, E, idx, send_pos = handle
        assert x.dtype == torch.bfloat16 and x.is_contiguous() and x.shape[-1] == H
        assert topk_weights.dtype == torch.float32 and topk_weights.is_contiguous()
        T, K = topk_weights.shape
        if out is None:
            out = torch.empty((T, H), dtype=torch.bfloat16, device=self.buf.device)
        args = (x.data_ptr(), idx, topk_weights.data_ptr(), send_pos.data_ptr(), out.data_ptr(), T, H, K, E, M)
        ev, hook = self._combine(self.rt.ll_combine, args, layout_range, combine_wait_recv_cost_stats, use_logfmt,
                                 async_finish, return_recv_hook, (x, topk_weights, send_pos, out))
        return out, ev, hook

    def combine_rmsnorm(self, x: torch.Tensor, topk_idx: torch.Tensor, topk_weights: torch.Tensor, handle,
                        residual: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6, *,
                        shared: Optional[torch.Tensor] = None, residual_out: Optional[torch.Tensor] = None,
                        out: Optional[torch.Tensor] = None, quant: Optional[str] = None, use_logfmt: bool = False,
                        zero_copy: bool = False, async_finish: bool = False, return_recv_hook: bool = False,
                        combine_wait_recv_cost_stats: Optional[torch.Tensor] = None):
        """``Buffer.low_latency_combine_rmsnorm``: :meth:`combine` with the shared-expert add, residual add and RMSNorm
        fused into its receive half.  The send half (copy-in or LogFMT pass, then the announcement) is combine's."""
        from .buffer import _ll_combine_rmsnorm_args

        if use_logfmt and zero_copy:
            raise ValueError("uccl_b200.ep: zero_copy and use_logfmt are mutually exclusive (as in the reference)")
        src_info, layout_range, M, H, E, idx, send_pos = handle
        T, K, residual_out, out, scales = _ll_combine_rmsnorm_args(
            x, topk_idx, topk_weights, self.buf.group_size, M, H, E, residual, weight, shared, residual_out, out, quant,
            self.buf.device)
        if T > send_pos.size(0) or K != send_pos.size(1):
            raise ValueError(f"uccl_b200.ep: low_latency_combine_rmsnorm got topk_weights [{T}, {K}] for a dispatch of "
                             f"{tuple(send_pos.shape)}")
        args = (x.data_ptr(), idx, topk_weights.data_ptr(), send_pos.data_ptr(),
                shared.data_ptr() if shared is not None else 0, residual.data_ptr(), residual_out.data_ptr(),
                weight.data_ptr(), out.data_ptr(), scales.data_ptr() if scales is not None else 0, T, H, K, E, M,
                float(eps))
        ev, hook = self._combine(self.rt.ll_combine_rmsnorm, args, layout_range, combine_wait_recv_cost_stats,
                                 use_logfmt, async_finish, return_recv_hook,
                                 (x, topk_weights, send_pos, shared, residual, residual_out, weight, out, scales))
        return ((out, scales) if scales is not None else out), ev, hook
