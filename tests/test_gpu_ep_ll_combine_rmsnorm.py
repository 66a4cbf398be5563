"""GPU tests of ep.Buffer.low_latency_combine_rmsnorm (LL combine + shared-expert add + residual add + RMSNorm [+ fp8
cast], the tail of a decode MoE layer) on virtual ranks: bitwise against low_latency_combine(), torch's bf16 + shared and
the one-rank all_reduce_rmsnorm epilogue, the fp8 output against per_token_cast_to_fp8, shared / residual_out / x forms,
use_logfmt, K > 9, tokens routed nowhere, a rank without tokens, launch counts, receive hooks (called, or completed by
the next dispatch), interleaving with LL dispatch and combine on one stream, CUDA-graph replay."""
import pytest
import torch

from helpers import get_world
from rmsnorm_ref import assert_fp8_cast_of, one_rank_epilogue
from test_gpu_ep import run_threads
from uccl_b200.ep import Buffer

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

EPS = 1e-6
E = 16  # every world size divides it, and K = 11 finds 11 distinct experts
M = 32  # num_max_dispatch_tokens_per_rank
H_MAX = 7168

_BUFFERS = {}


def get_ll_buffers(n):
    """Buffers of their own world, with the LL block sized for the largest shape here: EpBuffer fixes the LL block
    size on first use, so the buffers other test files cache (sized for smaller shapes) cannot be reused."""
    if n not in _BUFFERS:
        comms = get_world(n, heap_mb=320, stage_mb=8, max_ctas=4)
        ll = Buffer.get_low_latency_rdma_size_hint(M, H_MAX, n, E)
        bufs = []
        for c in comms:
            with torch.cuda.device(c.device):
                bufs.append(Buffer(comm=c, num_nvl_bytes=1 << 20, num_rdma_bytes=ll, low_latency_mode=True))
        torch.cuda.synchronize()
        _BUFFERS[n] = bufs
    return _BUFFERS[n]


def _inputs(n, T, H, K, seed):
    g = torch.Generator().manual_seed(seed)
    xs, idxs, ws, residuals, shareds = [], [], [], [], []
    for _ in range(n):
        xs.append((torch.randn(T, H, generator=g) * 2).to(torch.bfloat16))
        idx = torch.rand(T, E, generator=g).topk(K, dim=1).indices.to(torch.int64)
        idx = idx.masked_fill(torch.rand(T, K, generator=g) < 0.05, -1)
        idx[3] = -1  # tokens routed to no expert: routed = 0
        idx[T // 2] = -1
        idxs.append(idx.contiguous())
        ws.append(torch.rand(T, K, generator=g).float())
        residuals.append(torch.randn(T, H, generator=g).to(torch.bfloat16))
        shareds.append(torch.randn(T, H, generator=g).to(torch.bfloat16))
    weight = (torch.rand(H, generator=g) + 0.5).to(torch.bfloat16)
    return xs, idxs, ws, residuals, shareds, weight


def _experts(rx, r):
    """The "expert" multiplies every row by its global expert id + 1.  Rows past recv_count are never read.  No host
    sync: a blocking device -> host copy while this rank's dispatch still waits for a peer can hold up that peer's
    host -> device copies, and with them the peer's own dispatch."""
    e_local = rx.size(0)
    f = torch.arange(r * e_local + 1, (r + 1) * e_local + 1, dtype=torch.float32, device=rx.device).view(-1, 1, 1)
    return (rx.float() * f).to(torch.bfloat16)


def _check(got_ro, got_y, routed, shared, residual, weight, quant, what):
    T = got_ro.size(0)
    if T == 0:  # a rank without tokens: nothing to compare, but it joined every call
        assert (got_y[0] if quant == "fp8" else got_y).size(0) == 0, what
        return
    # torch's bf16 routed + shared, then the unfused epilogue
    x = routed[:T].cuda() if shared is None else routed[:T].cuda() + shared.cuda()
    ro, y, q = one_rank_epilogue(x, residual[:T], weight, EPS, quant)
    assert torch.equal(got_ro, ro), what
    if quant == "fp8":
        gq, gs = got_y
        assert gq.dtype == torch.float8_e4m3fn and gs.dtype == torch.float32, what
        assert gs.shape == (T, y.size(1) // 128), what
        assert_fp8_cast_of(gq, gs, y, what)
    else:
        assert torch.equal(got_y, y), what


def _cpu(y):
    return tuple(t.cpu() for t in y) if isinstance(y, tuple) else y.cpu()


# (shared, x, separate residual_out, quant, use_logfmt); LogFMT works in place on the combine buffer, so it runs with
# an ordinary x
CASES = [(False, "buffer", False, None, False), (True, "plain", True, "fp8", False), (True, "buffer", True, None, False),
         (False, "plain", False, "fp8", False), (True, "buffer", False, "fp8", False), (True, "plain", False, None, True),
         (False, "plain", True, "fp8", True)]


@pytest.mark.parametrize("n,H,K", [(n, H, 4) for n in (1, 2, 4, 8) for H in (1024, 2560, 7168)]
                         + [(2, 7168, 8), (4, 2560, 8), (2, 2560, 11), (2, 7168, 11)])
def test_ll_combine_rmsnorm_bitwise(n, H, K):
    T = 24
    bufs = get_ll_buffers(n)
    xs, idxs, ws, residuals, shareds, weight = _inputs(n, T, H, K, seed=10 * n + H % 97 + K)

    def fn(b):
        r, dev = b.rank, b.device
        # every host -> device copy comes first: a copy from pageable memory can wait for another rank's stream, which
        # may be blocked in a kernel that waits for this rank
        x, idx, w, w8 = xs[r].to(dev), idxs[r].to(dev), ws[r].to(dev), weight.to(dev)
        res0, sh = residuals[r].to(dev), shareds[r].to(dev)
        rx, _, handle, _, _ = b.low_latency_dispatch(x, idx, M, E, use_fp8=False)
        cb = b.get_next_low_latency_combine_buffer(handle)
        cb.copy_(_experts(rx, r))
        plain = cb.clone()
        zero = n > 1 and r == n - 1  # the last rank combines no tokens (its kernel still joins the barriers)
        rows = 0 if zero else T
        out = []
        for with_shared, x_mode, separate, quant, logfmt in CASES:
            xin = cb if x_mode == "buffer" else plain
            routed, _, _ = b.low_latency_combine(xin, idx, w, handle, use_logfmt=logfmt)
            res = res0[:rows].clone()
            ro = torch.empty_like(res) if separate else None
            l0 = b.runtime.launches
            y, _, hook = b.low_latency_combine_rmsnorm(xin, idx[:rows], w[:rows], handle, res, w8, EPS,
                                                       shared=sh[:rows] if with_shared else None, residual_out=ro,
                                                       quant=quant, use_logfmt=logfmt)
            launches = b.runtime.launches - l0
            assert hook is None
            torch.cuda.current_stream().synchronize()
            if separate:
                assert torch.equal(res, res0[:rows])  # residual itself untouched
            out.append(((with_shared, x_mode, separate, quant, logfmt), routed.cpu(), (ro if separate else res).cpu(),
                        _cpu(y), launches))
        return out

    outs = run_threads(bufs, fn)
    for r in range(n):
        for case, routed, ro, y, launches in outs[r]:
            what = (r, case)
            assert launches == (1 if case[1] == "buffer" and not case[4] else 2), what  # + the copy-in otherwise
            _check(ro, y, routed, shareds[r] if case[0] else None, residuals[r], weight, case[3], what)


@pytest.mark.parametrize("n", [2, 4])
def test_ll_combine_rmsnorm_hooks(n):
    """return_recv_hook: SEND + RECV launches, bitwise the no-hook result, whether the hook is called or a pending hook
    is completed by the next low_latency_dispatch."""
    T, H, K = 20, 2560, 4
    bufs = get_ll_buffers(n)
    xs, idxs, ws, residuals, shareds, weight = _inputs(n, T, H, K, seed=40 + n)

    def fn(b):
        r, dev = b.rank, b.device
        x, idx, w, w8 = xs[r].to(dev), idxs[r].to(dev), ws[r].to(dev), weight.to(dev)
        res0, sh = residuals[r].to(dev), shareds[r].to(dev)
        rx, _, handle, _, _ = b.low_latency_dispatch(x, idx, M, E, use_fp8=False)
        cb = b.get_next_low_latency_combine_buffer(handle)
        cb.copy_(_experts(rx, r))
        plain = cb.clone()
        results = []
        for use_hook, pending in ((False, False), (True, False), (True, True)):
            for x_mode in ("buffer", "plain"):
                ro = torch.empty_like(res0)
                l0 = b.runtime.launches
                y, _, hook = b.low_latency_combine_rmsnorm(cb if x_mode == "buffer" else plain, idx, w, handle, res0,
                                                           w8, EPS, shared=sh, residual_out=ro, quant="fp8",
                                                           return_recv_hook=use_hook)
                assert (hook is not None) == use_hook
                if use_hook and not pending:
                    hook()
                elif pending:
                    # the next LL call completes the pending receive half first (its dispatch result is not used)
                    b.low_latency_dispatch(x, idx, M, E, use_fp8=False)
                launches = b.runtime.launches - l0 - (1 if pending else 0)
                torch.cuda.current_stream().synchronize()
                results.append(((use_hook, pending, x_mode), launches, ro.cpu(), _cpu(y)))
        return results

    outs = run_threads(bufs, fn)
    for r in range(n):
        base = outs[r][0]
        for (case, launches, ro, y) in outs[r]:
            # buffer x: one kernel, or SEND + RECV with a hook; plain x adds the copy-in
            assert launches == (2 if case[0] else 1) + (case[2] == "plain"), (r, case, launches)
            assert torch.equal(ro, base[2]), (r, case)
            assert all(torch.equal(p.view(torch.uint8), q.view(torch.uint8)) for p, q in zip(y, base[3])), (r, case)


@pytest.mark.parametrize("n", [2, 4])
def test_ll_combine_rmsnorm_interleaved(n):
    """LL dispatch -> fused -> LL dispatch -> LL combine -> fused on one stream, no host sync, both LL buffers."""
    T, H, K = 28, 4096, 6
    bufs = get_ll_buffers(n)
    xs, idxs, ws, residuals, shareds, weight = _inputs(n, T, H, K, seed=77 + n)
    g = torch.Generator().manual_seed(5)
    xs2 = [torch.randn(x.shape, generator=g).to(torch.bfloat16) for x in xs]

    def scaled(rx, r, k):
        return (rx.float() * (r + k)).to(torch.bfloat16)  # rows past recv_count are not read

    def fn(b):
        r, dev = b.rank, b.device
        x, idx, w, x2, w8 = xs[r].to(dev), idxs[r].to(dev), ws[r].to(dev), xs2[r].to(dev), weight.to(dev)
        res1, res3, sh = residuals[r].to(dev), residuals[r].to(dev), shareds[r].to(dev)
        rx1, _, h1, _, _ = b.low_latency_dispatch(x, idx, M, E, use_fp8=False)
        cb1 = b.get_next_low_latency_combine_buffer(h1)
        cb1.copy_(scaled(rx1, r, 1))
        y1, _, _ = b.low_latency_combine_rmsnorm(cb1, idx, w, h1, res1, w8, EPS, shared=sh)
        rx2, _, h2, _, _ = b.low_latency_dispatch(x2, idx, M, E, use_fp8=False)
        assert h2[5] != h1[5]  # the second LL buffer
        cb2 = b.get_next_low_latency_combine_buffer(h2)
        cb2.copy_(scaled(rx2, r, 2))
        c2, _, _ = b.low_latency_combine(cb2, idx, w, h2)
        y3, _, _ = b.low_latency_combine_rmsnorm(cb2, idx, w, h2, res3, w8, EPS, quant="fp8")
        torch.cuda.current_stream().synchronize()
        c1, _, _ = b.low_latency_combine(cb1, idx, w, h1)  # the reference of y1: buffer 1 still holds its inputs
        torch.cuda.current_stream().synchronize()
        return c1.cpu(), res1.cpu(), y1.cpu(), c2.cpu(), res3.cpu(), _cpu(y3)

    outs = run_threads(bufs, fn)
    for r, (c1, ro1, y1, c2, ro3, y3) in enumerate(outs):
        _check(ro1, y1, c1, shareds[r], residuals[r], weight, None, (r, 1))
        _check(ro3, y3, c2, None, residuals[r], weight, "fp8", (r, 3))


def test_ll_combine_rmsnorm_cuda_graph_replay():
    """A graph of the copy of new expert outputs into the LL combine buffer + the fused call, replayed with new inputs,
    gives the eager results."""
    n, T, H, K = 2, 16, 7168, 8
    bufs = get_ll_buffers(n)
    xs, idxs, ws, residuals, shareds, weight = _inputs(n, T, H, K, seed=900)
    dev = bufs[0].device

    def setup(b):
        r = b.rank
        # all host -> device copies before the first collective (see test_ll_combine_rmsnorm_bitwise)
        x, idx, w, sh, w8 = xs[r].to(dev), idxs[r].to(dev), ws[r].to(dev), shareds[r].to(dev), weight.to(dev)
        rx, _, handle, _, _ = b.low_latency_dispatch(x, idx, M, E, use_fp8=False)
        cb = b.get_next_low_latency_combine_buffer(handle)
        s = dict(idx=idx, w=w, handle=handle, cb=cb, eo=rx.clone(), res=torch.zeros(T, H, dtype=torch.bfloat16, device=dev),
                 sh=sh, ro=torch.empty(T, H, dtype=torch.bfloat16, device=dev),
                 out=torch.empty(T, H, dtype=torch.bfloat16, device=dev), w8=w8)
        step(b, s)  # eager warm-up of every kernel the graph captures
        return s

    def step(b, s):
        s["cb"].copy_(s["eo"])
        b.low_latency_combine_rmsnorm(s["cb"], s["idx"], s["w"], s["handle"], s["res"], s["w8"], EPS, shared=s["sh"],
                                      residual_out=s["ro"], out=s["out"])

    statics = run_threads(bufs, setup)
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(device=dev) for _ in bufs]
    graphs = []
    for b, st, s in zip(bufs, streams, statics):
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=st):
            step(b, s)
        graphs.append(gr)
    g = torch.Generator().manual_seed(901)
    for rep in range(3):
        for s in statics:
            s["eo"].copy_(torch.randn(s["eo"].shape, generator=g).to(torch.bfloat16))
            s["res"].copy_(torch.randn(s["res"].shape, generator=g).to(torch.bfloat16))
            s["sh"].copy_(torch.randn(s["sh"].shape, generator=g).to(torch.bfloat16))
        torch.cuda.synchronize()
        for st, gr in zip(streams, graphs):
            with torch.cuda.stream(st):
                gr.replay()
        for st in streams:
            st.synchronize()
        replayed = [(s["ro"].cpu(), s["out"].cpu()) for s in statics]

        def eager(b):
            s = statics[b.rank]
            step(b, s)
            torch.cuda.current_stream().synchronize()
            return s["ro"].cpu(), s["out"].cpu()

        for (ro_g, y_g), (ro_e, y_e) in zip(replayed, run_threads(bufs, eager)):
            assert torch.equal(ro_g, ro_e), rep
            assert torch.equal(y_g, y_e), rep
