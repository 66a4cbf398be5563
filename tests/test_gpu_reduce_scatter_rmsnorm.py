"""GPU tests of reduce_scatter_rmsnorm (reduce-scatter + residual add + RMSNorm [+ fp8 cast] on each rank's rows, the
sequence-parallel tail of a row-parallel layer) on virtual ranks: x's own rows against the plain reduce_scatter,
residual_out / out against an fp64 reference, the ranks' shards against all_reduce_rmsnorm (SP followed by an
all-gather is TP, bit for bit), the fused LL kernel against the unfused composition, the fp8 output against
per_token_cast_to_fp8, the LL epoch shared with the other LL collectives, and CUDA-graph replay."""
import pytest
import torch

from helpers import get_world, run_ranks
from rmsnorm_ref import assert_fp8_cast_of, rmsnorm_ref
from uccl_b200.parallel.comm import launch_count

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

EPS = 1e-6


def _inputs(n, T, H, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(T, H, generator=g).to(dtype) for _ in range(n)]
    residual = (torch.randn(T, H, generator=g) * 2).to(dtype)  # the full residual; rank r holds rows r*Tl .. (r+1)*Tl
    weight = (torch.rand(H, generator=g) + 0.5).to(dtype)
    return xs, residual, weight


def _tol(dtype):
    return dict(rtol=2e-2, atol=6e-2) if dtype == torch.bfloat16 else dict(rtol=4e-3, atol=1e-2)


def _rank_order_sum(xs):
    """The sum the kernels compute: fp32 in rank order, rounded once."""
    acc = xs[0].float()
    for x in xs[1:]:
        acc = acc + x.float()
    return acc.to(xs[0].dtype)


def _place(c, t, sym):
    if sym:
        x = c.empty(t.shape, dtype=t.dtype)
        x.copy_(t)
        return x
    return t.to(c.device)


def _cpu(y):
    return tuple(t.cpu() for t in y) if isinstance(y, tuple) else y.cpu()


def _sp(comms, xs, residual, weight, sym, separate, **kw):
    """One reduce_scatter_rmsnorm per rank; returns per rank (x, residual_out, out) on the CPU."""
    Tl = residual.size(0) // len(comms)

    def prepare(c):
        res = residual[c.rank * Tl:(c.rank + 1) * Tl].to(c.device)
        return dict(x=_place(c, xs[c.rank], sym), res=res, ro=torch.empty_like(res) if separate else res,
                    w=weight.to(c.device))

    def launch(c, s):
        s["y"] = c.reduce_scatter_rmsnorm(s["x"], s["res"], s["w"], EPS, residual_out=s["ro"] if separate else None,
                                          **kw)

    return [(s["x"].cpu(), s["ro"].cpu(), _cpu(s["y"])) for s in run_ranks(comms, prepare, launch)]


def _tp(comms, xs, residual, weight, sym, **kw):
    """all_reduce_rmsnorm of the same x with the full residual; returns rank 0's (residual_out, out)."""

    def prepare(c):
        return dict(x=_place(c, xs[c.rank], sym), res=residual.to(c.device), w=weight.to(c.device))

    def launch(c, s):
        s["y"] = c.all_reduce_rmsnorm(s["x"], s["res"], s["w"], EPS, **kw)

    s = run_ranks(comms, prepare, launch)[0]
    return s["res"].cpu(), _cpu(s["y"])


def _plain_reduce_scatter(comms, xs, sym):
    Tl, H = xs[0].size(0) // len(comms), xs[0].size(1)

    def prepare(c):
        return dict(x=_place(c, xs[c.rank], sym), out=torch.empty(Tl, H, dtype=xs[0].dtype, device=c.device))

    return [s["out"].cpu() for s in run_ranks(comms, prepare, lambda c, s: c.reduce_scatter(s["out"], s["x"]))]


def _set_knobs(comms, ll_max, push):
    for c in comms:
        c.set_xchg_ll_max(ll_max)
        c.set_rs_push(push)


# (rows per rank, H): one row per rank; 8 and 16 rows (16 x 5120 is past the 8-rank LL limit); 64 x 8192 is past every
# LL limit, so AUTO runs reduce_scatter + the epilogue kernel; the largest hidden size once
SHAPES = [(1, 4096), (8, 7168), (16, 5120), (64, 8192), (2, 16384)]


@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("Tl,H", SHAPES)
@pytest.mark.parametrize("sym", [False, True])
def test_reduce_scatter_rmsnorm(n, dtype, Tl, H, sym):
    comms = get_world(n)
    T = Tl * n
    # residual_out is a separate tensor for plain x and the residual itself for symmetric x
    separate = not sym
    fused = Tl * H * dtype.itemsize <= comms[0].reduce_scatter_ll_max()
    if Tl == 64:
        assert not fused  # AUTO takes the unfused path here
    xs, residual, weight = _inputs(n, T, H, dtype, seed=n * 1000 + Tl)
    before = launch_count(comms)
    res = _sp(comms, xs, residual, weight, sym, separate)
    # the fused path is one kernel per rank; the unfused one is the reduce-scatter, then the epilogue kernel
    assert launch_count(comms) - before == n * (1 if fused else 2)
    ref_x = _plain_reduce_scatter(comms, xs, sym)
    for r, (x, ro, y) in enumerate(res):
        lo, hi = r * Tl, (r + 1) * Tl
        # 1. my rows of x are exactly what the out-of-place reduce_scatter returns; the other rows are untouched
        assert torch.equal(x[lo:hi], ref_x[r])
        assert torch.equal(x[:lo], xs[r][:lo]) and torch.equal(x[hi:], xs[r][hi:])
        # 2. residual_out and out against fp64
        assert ro.shape == (Tl, H) and y.shape == (Tl, H)
        assert torch.allclose(ro.double(), x[lo:hi].double() + residual[lo:hi].double(), **_tol(dtype))
        assert torch.allclose(y.double(), rmsnorm_ref(ro, weight, EPS), **_tol(dtype))

    # 3. SP == TP: the shards in rank order are what all_reduce_rmsnorm gives on the same x with the full residual
    ro_tp, y_tp = _tp(comms, xs, residual, weight, sym)
    assert torch.equal(torch.cat([ro for _, ro, _ in res]), ro_tp)
    assert torch.equal(torch.cat([y for _, _, y in res]), y_tp)

    # 5. fp8: per_token_cast_to_fp8 of the 16-bit out; SP == TP holds for the e4m3 bytes and the scales too
    q8 = _sp(comms, xs, residual, weight, sym, separate, quant="fp8")
    for (x, ro, y), (x8, ro8, (q, sc)) in zip(res, q8):
        assert torch.equal(x, x8) and torch.equal(ro, ro8)
        assert_fp8_cast_of(q, sc, y)
        assert q.dtype == torch.float8_e4m3fn and sc.dtype == torch.float32
        assert sc.is_contiguous() and sc.shape == (Tl, H // 128)
    _, (q_tp, sc_tp) = _tp(comms, xs, residual, weight, sym, quant="fp8")
    assert torch.equal(torch.cat([q for _, _, (q, _) in q8]).view(torch.uint8), q_tp.view(torch.uint8))
    assert torch.equal(torch.cat([sc for _, _, (_, sc) in q8]), sc_tp)

    # 4. the fused kernel and the unfused composition (push and pull reduce-scatter) agree bitwise
    try:
        for push in (True, False):
            _set_knobs(comms, -1, push)
            for base, kw in ((res, {}), (q8, dict(quant="fp8"))):
                other = _sp(comms, xs, residual, weight, sym, separate, **kw)
                for (x, ro, y), (x2, ro2, y2) in zip(base, other):
                    assert torch.equal(x, x2) and torch.equal(ro, ro2), (push, kw)
                    if isinstance(y, tuple):
                        assert torch.equal(y[0].view(torch.uint8), y2[0].view(torch.uint8)), (push, kw)
                        assert torch.equal(y[1], y2[1]), (push, kw)
                    else:
                        assert torch.equal(y, y2), (push, kw)
    finally:
        _set_knobs(comms, 0, True)


@pytest.mark.parametrize("n", [2, 8])
def test_reduce_scatter_rmsnorm_interleaved_with_ll_collectives(n):
    """The fused kernel shares the LL epoch word and packet parity with every LL collective: mix them on a stream."""
    comms = get_world(n)
    Tl, H, dtype = 4, 2048, torch.bfloat16
    T, m = Tl * n, 1024
    for c in comms:
        assert Tl * H * dtype.itemsize <= c.reduce_scatter_ll_max() and m * 4 <= c.reduce_scatter_ll_max()
    for rnd in range(3):
        xs, residual, weight = _inputs(n, T, H, dtype, seed=300 + rnd)
        xs2, residual2, _ = _inputs(n, T, H, dtype, seed=400 + rnd)
        g = torch.Generator().manual_seed(500 + rnd)
        rs_in = [torch.randn(n * m, generator=g) for _ in range(n)]
        ag_in = [torch.randn(m, generator=g) for _ in range(n)]
        ar_in = [torch.randn(3000, generator=g) for _ in range(n)]

        def prepare(c):
            d, sl = c.device, slice(c.rank * Tl, (c.rank + 1) * Tl)
            return dict(rs_in=rs_in[c.rank].to(d), rs_out=torch.empty(m, device=d), x=xs[c.rank].to(d),
                        res=residual[sl].to(d), ag_in=ag_in[c.rank].to(d), ag_out=torch.empty(n * m, device=d),
                        ar=ar_in[c.rank].to(d), tx=xs[c.rank].to(d), tres=residual.to(d), x2=xs2[c.rank].to(d),
                        res2=residual2[sl].to(d), w=weight.to(d))

        def launch(c, s):
            c.reduce_scatter(s["rs_out"], s["rs_in"])
            s["y"] = c.reduce_scatter_rmsnorm(s["x"], s["res"], s["w"], EPS)
            c.all_gather(s["ag_out"], s["ag_in"])
            c.all_reduce(s["ar"], "sum", algo="oneshot_ll")
            s["ty"] = c.all_reduce_rmsnorm(s["tx"], s["tres"], s["w"], EPS, algo="oneshot_ll")
            s["y2"] = c.reduce_scatter_rmsnorm(s["x2"], s["res2"], s["w"], EPS)

        states = run_ranks(comms, prepare, launch)
        exp_rs = torch.stack(rs_in).double().sum(0)
        exp_ar = torch.stack(ar_in).double().sum(0)
        for r, s in enumerate(states):
            sl = slice(r * Tl, (r + 1) * Tl)
            assert torch.allclose(s["rs_out"].cpu().double(), exp_rs[r * m:(r + 1) * m], rtol=1e-5, atol=1e-5), rnd
            assert torch.equal(s["ag_out"].cpu(), torch.cat(ag_in)), rnd
            assert torch.allclose(s["ar"].cpu().double(), exp_ar, rtol=1e-5, atol=1e-5), rnd
            for xk, rk, yk, x_in, res_in in (("x", "res", "y", xs, residual), ("x2", "res2", "y2", xs2, residual2)):
                xr = _rank_order_sum(x_in)[sl]
                assert torch.equal(s[xk].cpu()[sl], xr), (rnd, xk)
                assert torch.equal(s[rk].cpu(), (xr.float() + res_in[sl].float()).to(dtype)), (rnd, xk)
                assert torch.allclose(s[yk].cpu().double(), rmsnorm_ref(s[rk].cpu(), weight, EPS), **_tol(dtype)), rnd
        # the interleaved TP call agrees with the SP calls around it
        assert torch.equal(torch.cat([s["y"].cpu() for s in states]), states[0]["ty"].cpu()), rnd


def test_reduce_scatter_rmsnorm_cuda_graph_replay():
    """One fused call per rank captured in a CUDA graph, replayed three times with new inputs."""
    n = 2
    comms = get_world(n)
    Tl, H, dtype = 8, 4096, torch.bfloat16
    T = Tl * n
    assert Tl * H * dtype.itemsize <= comms[0].reduce_scatter_ll_max()  # the fused kernel is what gets captured
    xs = [c.empty(T, H, dtype=dtype) for c in comms]
    rs = [torch.empty(Tl, H, dtype=dtype, device=c.device) for c in comms]
    ws = [torch.empty(H, dtype=dtype, device=c.device) for c in comms]
    ys = [torch.empty(Tl, H, dtype=dtype, device=c.device) for c in comms]
    for t in xs + rs + ws + ys:
        t.zero_()
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(device=c.device) for c in comms]
    graphs = []
    for c, st, x, r, w, y in zip(comms, streams, xs, rs, ws, ys):
        with torch.cuda.device(c.device):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=st):
                c.reduce_scatter_rmsnorm(x, r, w, EPS, out=y)
            graphs.append(g)
    for rep in range(3):
        ins, residual, weight = _inputs(n, T, H, dtype, seed=600 + rep)
        for k, (x, r, w, xi) in enumerate(zip(xs, rs, ws, ins)):
            x.copy_(xi)
            r.copy_(residual[k * Tl:(k + 1) * Tl])
            w.copy_(weight)
        torch.cuda.synchronize()
        for c, st, g in zip(comms, streams, graphs):
            with torch.cuda.device(c.device), torch.cuda.stream(st):
                g.replay()
        for st in streams:
            st.synchronize()
        exp_x = _rank_order_sum(ins)
        for k, (x, r, y) in enumerate(zip(xs, rs, ys)):
            lo, hi = k * Tl, (k + 1) * Tl
            sl = slice(lo, hi)
            xc = x.cpu()
            assert torch.equal(xc[sl], exp_x[sl]), rep
            assert torch.equal(xc[:lo], ins[k][:lo]) and torch.equal(xc[hi:], ins[k][hi:]), rep
            assert torch.equal(r.cpu(), (exp_x[sl].float() + residual[sl].float()).to(dtype)), rep
            assert torch.allclose(y.cpu().double(), rmsnorm_ref(r.cpu(), weight, EPS), **_tol(dtype)), rep
