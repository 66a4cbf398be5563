"""GPU tests of ep.Buffer.combine_rmsnorm (EP combine + residual add + RMSNorm [+ fp8 cast], the tail of an MoE layer)
on virtual ranks: bitwise against combine() (register and TMA kernels) followed by the one-rank all_reduce_rmsnorm
epilogue, the fp8 output against per_token_cast_to_fp8, bias forms, arena and copied-in x, a rank without tokens and
tokens routed to no rank, the launch count, interleaving with dispatch / combine on one stream, CUDA-graph replay."""
import pytest
import torch

from rmsnorm_ref import assert_fp8_cast_of, one_rank_epilogue
from test_gpu_ep import get_buffers, make_inputs, run_threads
from uccl_b200.ep.utils import EpHandle

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

EPS = 1e-6
K = 4

# (bias, x, separate residual_out, quant): every input form appears with and without fp8
CASES = [("none", "arena", False, None), ("one", "plain", True, "fp8"), ("tuple", "arena", True, None),
         ("tuple", "plain", False, "fp8"), ("one", "arena", False, "fp8"), ("none", "plain", True, None)]


def _inputs(n, T, H, seed):
    E = n * 4
    xs, idxs, _ = make_inputs(n, T, H, K, E, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for r in range(n):
        idxs[r][3] = -1  # tokens routed to no rank: combined = bias (or 0)
        idxs[r][T // 2] = -1
    residuals = [torch.randn(x.size(0), H, generator=g).to(torch.bfloat16) for x in xs]
    biases = [(torch.randn(x.size(0), H, generator=g).to(torch.bfloat16),
               torch.randn(x.size(0), H, generator=g).to(torch.bfloat16)) for x in xs]
    weight = (torch.rand(H, generator=g) + 0.5).to(torch.bfloat16)
    return E, xs, idxs, residuals, biases, weight


def _bias(mode, pair, dev):
    if mode == "none":
        return None
    if mode == "one":
        return pair[0].to(dev)
    return tuple(b.to(dev) for b in pair)


def _without_tokens(h):
    """The handle of a rank that has no tokens this step.  (dispatch itself needs at least one token per rank, so the
    rank dispatches as usual and only its combine_rmsnorm sees T == 0; its kernel must still join both barriers.)"""
    return EpHandle(h.rank_prefix, h.num_recv, h.recv_src_idx, h.is_token_in_rank, h.send_slot[:0], slot=h.slot,
                    num_topk=h.num_topk)


def _dispatch(b, x, idx, E):
    tpr, _, tpe, in_rank, _ = b.get_dispatch_layout(idx, E)
    recv_x, _, _, _, handle, _ = b.dispatch(x, num_tokens_per_rank=tpr, is_token_in_rank=in_rank,
                                            num_tokens_per_expert=tpe, topk_idx=idx)
    return recv_x, handle


def _check(got_ro, got_y, combined, residual, weight, quant, what):
    if combined.size(0) == 0:  # a rank without tokens: nothing to compare, but it joined every call
        assert got_ro.shape == combined.shape, what
        assert (got_y[0] if quant == "fp8" else got_y).shape == combined.shape, what
        return
    ro, y, q = one_rank_epilogue(combined, residual, weight, EPS, quant)  # combine(), then the unfused epilogue
    assert torch.equal(got_ro, ro), what
    if quant == "fp8":
        gq, gs = got_y
        assert gq.dtype == torch.float8_e4m3fn and gs.dtype == torch.float32, what
        assert gs.shape == (y.size(0), y.size(1) // 128), what
        assert_fp8_cast_of(gq, gs, y, what)
    else:
        assert torch.equal(got_y, y), what


@pytest.mark.parametrize("n,H", [(n, H) for n in (1, 2, 4, 8) for H in (512, 2560, 7168)] + [(2, 16384)])
def test_combine_rmsnorm_bitwise(n, H):
    T = 96
    bufs = get_buffers(n)
    E, xs, idxs, residuals, biases, weight = _inputs(n, T, H, seed=10 * n + H % 97)

    def fn(b):
        r, dev = b.rank, b.device
        # every host -> device copy comes first: a copy from pageable memory can wait for another rank's stream, which
        # may be blocked in a kernel that waits for this rank
        x, idx, res0, w = xs[r].to(dev), idxs[r].to(dev), residuals[r].to(dev), weight.to(dev)
        dev_biases = {m: _bias(m, biases[r], dev) for m in ("none", "one", "tuple")}
        recv_x, handle = _dispatch(b, x, idx, E)
        num_recv = recv_x.size(0)
        cb = b.get_combine_buffer(num_recv, H)
        cb.copy_((recv_x.float() * (r + 1)).to(torch.bfloat16))
        plain = cb.clone()
        zero = n > 1 and r == n - 1  # the last rank combines no tokens
        rows = 0 if zero else T
        h_rms = _without_tokens(handle) if zero else handle
        res0 = res0[:rows]
        out = []
        for impl in (1, 2):
            b.runtime.impl = impl
            for bias_mode, x_mode, separate, quant in CASES:
                xin = cb if x_mode == "arena" else plain
                bias = dev_biases[bias_mode]
                combined, _, _ = b.combine(xin, handle, bias=bias)
                combined = combined[:rows]
                if zero and bias is not None:
                    bias = tuple(t[:0] for t in bias) if isinstance(bias, tuple) else bias[:0]
                res = res0.clone()
                ro = torch.empty_like(res) if separate else None
                l0 = b.runtime.launches
                y, _ = b.combine_rmsnorm(xin, h_rms, res, w, EPS, bias=bias, residual_out=ro, quant=quant)
                launches = b.runtime.launches - l0
                torch.cuda.current_stream().synchronize()
                if separate:
                    assert torch.equal(res, res0)  # residual itself untouched
                y = tuple(t.cpu() for t in y) if isinstance(y, tuple) else y.cpu()
                out.append(((impl, bias_mode, x_mode, separate, quant), combined.cpu(), (ro if separate else res).cpu(),
                            y, launches, b.runtime.last_combine_impl))
        b.runtime.impl = 0
        return out

    outs = run_threads(bufs, fn)
    for r in range(n):
        for case, combined, ro, y, launches, used_impl in outs[r]:
            what = (r, case)
            assert used_impl == case[0], what  # the reference ran the register (1) or the TMA (2) combine
            if case[2] == "arena":
                assert launches == 1, what  # one kernel, no copy-in
            _check(ro, y, combined, residuals[r], weight, case[4], what)


@pytest.mark.parametrize("n", [2, 4])
def test_combine_rmsnorm_interleaved_with_dispatch_and_combine(n):
    """dispatch -> combine_rmsnorm -> dispatch -> combine -> combine_rmsnorm on one stream, no host sync in between."""
    T, H = 80, 2048
    bufs = get_buffers(n)
    E, xs, idxs, residuals, biases, weight = _inputs(n, T, H, seed=77 + n)
    g = torch.Generator().manual_seed(5)
    xs2 = [torch.randn(x.shape, generator=g).to(torch.bfloat16) for x in xs]

    def fn(b):
        r, dev = b.rank, b.device
        # all host -> device copies before the first collective (see test_combine_rmsnorm_bitwise)
        x, idx, x2, w = xs[r].to(dev), idxs[r].to(dev), xs2[r].to(dev), weight.to(dev)
        res1, res3 = residuals[r].to(dev), residuals[r].to(dev)
        recv_x, handle = _dispatch(b, x, idx, E)
        num_recv = recv_x.size(0)
        y1_in = (recv_x.float() * (r + 1)).to(torch.bfloat16)
        cb = b.get_combine_buffer(num_recv, H)
        cb.copy_(y1_in)
        y1, _ = b.combine_rmsnorm(cb, handle, res1, w, EPS)
        recv2, *_ = b.dispatch(x2, handle=handle)
        y2_in = (recv2.float() * (r + 2)).to(torch.bfloat16)
        cb.copy_(y2_in)
        c2, _, _ = b.combine(cb, handle)
        y3, _ = b.combine_rmsnorm(cb, handle, res3, w, EPS, quant="fp8")
        torch.cuda.current_stream().synchronize()
        # the combine of the first expert outputs, for the reference of y1
        cb.copy_(y1_in)
        c1, _, _ = b.combine(cb, handle)
        torch.cuda.current_stream().synchronize()
        return c1.cpu(), res1.cpu(), y1.cpu(), c2.cpu(), res3.cpu(), tuple(t.cpu() for t in y3)

    outs = run_threads(bufs, fn)
    for r, (c1, ro1, y1, c2, ro3, y3) in enumerate(outs):
        _check(ro1, y1, c1, residuals[r], weight, None, (r, 1))
        _check(ro3, y3, c2, residuals[r], weight, "fp8", (r, 3))


def test_combine_rmsnorm_cuda_graph_replay():
    """A graph of cached dispatch + copy into the combine arena + combine_rmsnorm, replayed with new inputs, gives the
    eager results."""
    n, T, H = 2, 64, 4096
    bufs = get_buffers(n)
    E, xs, idxs, residuals, biases, weight = _inputs(n, T, H, seed=900)
    dev = bufs[0].device
    statics = []
    for b in bufs:
        r = b.rank
        statics.append(dict(x=xs[r].to(dev), res=torch.zeros(xs[r].size(0), H, dtype=torch.bfloat16, device=dev),
                            ro=torch.empty(xs[r].size(0), H, dtype=torch.bfloat16, device=dev),
                            out=torch.empty(xs[r].size(0), H, dtype=torch.bfloat16, device=dev), w=weight.to(dev),
                            bias=biases[r][0].to(dev)))

    def step(b, s, handle, cb):
        recv, *_ = b.dispatch(s["x"], handle=handle)
        cb.copy_((recv.float() * (b.rank + 1)).to(torch.bfloat16))
        b.combine_rmsnorm(cb, handle, s["res"], s["w"], EPS, bias=s["bias"], residual_out=s["ro"], out=s["out"])

    def warm(b):
        recv_x, handle = _dispatch(b, xs[b.rank].to(b.device), idxs[b.rank].to(b.device), E)
        cb = b.get_combine_buffer(recv_x.size(0), H)
        step(b, statics[b.rank], handle, cb)  # eager warm-up of every kernel the graph captures
        return handle, cb

    hc = run_threads(bufs, warm)
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(device=dev) for _ in bufs]
    graphs = []
    for b, st, s, (handle, cb) in zip(bufs, streams, statics, hc):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            step(b, s, handle, cb)
        graphs.append(g)
    g = torch.Generator().manual_seed(901)
    for rep in range(3):
        new = [(torch.randn(s["x"].shape, generator=g).to(torch.bfloat16),
                torch.randn(s["res"].shape, generator=g).to(torch.bfloat16)) for s in statics]
        for s, (x, res) in zip(statics, new):
            s["x"].copy_(x)
            s["res"].copy_(res)
        torch.cuda.synchronize()
        for st, gr in zip(streams, graphs):
            with torch.cuda.stream(st):
                gr.replay()
        for st in streams:
            st.synchronize()
        replayed = [(s["ro"].cpu(), s["out"].cpu()) for s in statics]

        def eager(b):
            s = statics[b.rank]
            handle, cb = hc[b.rank]
            step(b, s, handle, cb)
            torch.cuda.current_stream().synchronize()
            return s["ro"].cpu(), s["out"].cpu()

        for (ro_g, y_g), (ro_e, y_e) in zip(replayed, run_threads(bufs, eager)):
            assert torch.equal(ro_g, ro_e), rep
            assert torch.equal(y_g, y_e), rep
