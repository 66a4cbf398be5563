"""GPU tests of all_reduce_rmsnorm (all-reduce + residual add + RMSNorm [+ fp8 cast]) on virtual ranks: the reduced x
against the plain all-reduce, residual_out / out against an fp64 reference, bitwise agreement between ranks and
between the fused one-shot kernel and the unfused composition, the fp8 output against per_token_cast_to_fp8, the LL
epoch shared with the plain one-shot all-reduce, and CUDA-graph replay."""
import pytest
import torch

from helpers import get_world, run_ranks
from rmsnorm_ref import assert_fp8_cast_of, rmsnorm_ref

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

EPS = 1e-6
LL_MAX = 1 << 20


def _inputs(n, T, H, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(T, H, generator=g).to(dtype) for _ in range(n)]
    residual = (torch.randn(T, H, generator=g) * 2).to(dtype)  # replicated on every rank, as in a TP layer
    weight = (torch.rand(H, generator=g) + 0.5).to(dtype)
    return xs, residual, weight


def _tol(dtype):
    return dict(rtol=2e-2, atol=6e-2) if dtype == torch.bfloat16 else dict(rtol=4e-3, atol=1e-2)


def _run(comms, xs, residual, weight, sym, separate, **kw):
    """One all_reduce_rmsnorm per rank; returns per rank (x, residual_out, out) on the CPU."""

    def prepare(c):
        if sym:
            x = c.empty(xs[c.rank].shape, dtype=xs[c.rank].dtype)
            x.copy_(xs[c.rank])
        else:
            x = xs[c.rank].to(c.device)
        res = residual.to(c.device)
        return dict(x=x, res=res, ro=torch.empty_like(res) if separate else res, w=weight.to(c.device))

    def launch(c, s):
        s["y"] = c.all_reduce_rmsnorm(s["x"], s["res"], s["w"], EPS, residual_out=s["ro"] if separate else None, **kw)

    states = run_ranks(comms, prepare, launch)
    out = []
    for s in states:
        y = s["y"]
        y = tuple(t.cpu() for t in y) if isinstance(y, tuple) else y.cpu()
        out.append((s["x"].cpu(), s["ro"].cpu(), y))
    return out


def _plain_allreduce(comms, xs, sym):
    def prepare(c):
        if sym:
            x = c.empty(xs[c.rank].shape, dtype=xs[c.rank].dtype)
            x.copy_(xs[c.rank])
            return x
        return xs[c.rank].to(c.device)

    return [x.cpu() for x in run_ranks(comms, prepare, lambda c, x: c.all_reduce(x, "sum"))]


@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("T,H", [(1, 4096), (7, 5120), (64, 8192), (128, 7168)])
@pytest.mark.parametrize("sym", [False, True])
@pytest.mark.parametrize("separate", [False, True])
def test_allreduce_rmsnorm(n, dtype, T, H, sym, separate):
    comms = get_world(n)
    xs, residual, weight = _inputs(n, T, H, dtype, seed=n * 1000 + T)
    res = _run(comms, xs, residual, weight, sym, separate)
    ref_x = _plain_allreduce(comms, xs, sym)
    for r, (x, ro, y) in enumerate(res):
        # 1. x is exactly what the plain all-reduce leaves
        assert torch.equal(x, ref_x[r])
        # 2. residual_out and out against fp64
        assert torch.allclose(ro.double(), x.double() + residual.double(), **_tol(dtype))
        assert torch.allclose(y.double(), rmsnorm_ref(ro, weight, EPS), **_tol(dtype))
        # 3. bitwise identical on every rank
        assert torch.equal(x, res[0][0]) and torch.equal(ro, res[0][1]) and torch.equal(y, res[0][2])

    # 4. the fused kernel and the unfused composition agree bitwise
    forced = ["twoshot_p2p" if sym else "staged_p2p"]
    if T * H * dtype.itemsize <= LL_MAX:
        forced.append("oneshot_ll")
    for algo in forced:
        other = _run(comms, xs, residual, weight, sym, separate, algo=algo)
        for (x, ro, y), (x2, ro2, y2) in zip(res, other):
            assert torch.equal(x, x2) and torch.equal(ro, ro2) and torch.equal(y, y2), algo

    # 5. fp8: per_token_cast_to_fp8 of the 16-bit out, in the (x, scales) format of ep.Buffer.dispatch
    q8 = _run(comms, xs, residual, weight, sym, separate, quant="fp8")
    for (x, ro, y), (x8, ro8, (q, sc)) in zip(res, q8):
        assert torch.equal(x, x8) and torch.equal(ro, ro8)
        assert_fp8_cast_of(q, sc, y)
        assert q.dtype == torch.float8_e4m3fn and sc.dtype == torch.float32
        assert sc.is_contiguous() and sc.shape == (q.size(0), q.size(1) // 128)


@pytest.mark.parametrize("n", [2, 8])
def test_allreduce_rmsnorm_interleaved_with_oneshot_allreduce(n):
    """Fused calls and plain one-shot all-reduces share the LL epoch and packet parity: alternate them."""
    comms = get_world(n)
    T, H, dtype = 4, 2048, torch.bfloat16
    for rnd in range(3):
        xs, residual, weight = _inputs(n, T, H, dtype, seed=100 + rnd)
        plain_in = [torch.randn(3000, generator=torch.Generator().manual_seed(rnd * 10 + r)) for r in range(n)]

        def prepare(c):
            return dict(x=xs[c.rank].to(c.device), res=residual.to(c.device), w=weight.to(c.device),
                        p=plain_in[c.rank].to(c.device), p2=plain_in[c.rank].to(c.device))

        def launch(c, s):
            c.all_reduce(s["p"], "sum", algo="oneshot_ll")
            s["y"] = c.all_reduce_rmsnorm(s["x"], s["res"], s["w"], EPS, algo="oneshot_ll")
            c.all_reduce(s["p2"], "sum", algo="oneshot_ll")

        states = run_ranks(comms, prepare, launch)
        exp_p = torch.stack(plain_in).double().sum(0)
        exp_x = torch.stack([x.float() for x in xs]).sum(0).to(dtype)
        for s in states:
            assert torch.allclose(s["p"].cpu().double(), exp_p, rtol=1e-5, atol=1e-5), rnd
            assert torch.equal(s["p"].cpu(), s["p2"].cpu()), rnd
            assert torch.allclose(s["x"].cpu().double(), exp_x.double(), **_tol(dtype)), rnd
            assert torch.allclose(s["y"].cpu().double(), rmsnorm_ref(s["res"].cpu(), weight, EPS), **_tol(dtype)), rnd


def test_allreduce_rmsnorm_cuda_graph_replay():
    """One fused call per rank captured in a CUDA graph, replayed three times with new inputs."""
    n = 2
    comms = get_world(n)
    T, H, dtype = 8, 4096, torch.bfloat16
    xs = [c.empty(T, H, dtype=dtype) for c in comms]
    rs = [torch.empty(T, H, dtype=dtype, device=c.device) for c in comms]
    ws = [torch.empty(H, dtype=dtype, device=c.device) for c in comms]
    ys = [torch.empty(T, H, dtype=dtype, device=c.device) for c in comms]
    for t in xs + rs + ws + ys:
        t.zero_()
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(device=c.device) for c in comms]
    graphs = []
    for c, st, x, r, w, y in zip(comms, streams, xs, rs, ws, ys):
        with torch.cuda.device(c.device):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=st):
                c.all_reduce_rmsnorm(x, r, w, EPS, out=y, algo="oneshot_ll")
            graphs.append(g)
    for rep in range(3):
        ins, residual, weight = _inputs(n, T, H, dtype, seed=500 + rep)
        for x, r, w, xi in zip(xs, rs, ws, ins):
            x.copy_(xi)
            r.copy_(residual)
            w.copy_(weight)
        torch.cuda.synchronize()
        for c, st, g in zip(comms, streams, graphs):
            with torch.cuda.device(c.device), torch.cuda.stream(st):
                g.replay()
        for st in streams:
            st.synchronize()
        exp_x = torch.stack([x.float() for x in ins]).sum(0).to(dtype)
        for x, r, y in zip(xs, rs, ys):
            assert torch.equal(x.cpu(), exp_x), rep
            assert torch.equal(r.cpu(), (exp_x.float() + residual.float()).to(dtype)), rep
            assert torch.allclose(y.cpu().double(), rmsnorm_ref(r.cpu(), weight, EPS), **_tol(dtype)), rep
