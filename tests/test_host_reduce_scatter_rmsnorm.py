"""CPU tests of reduce_scatter_rmsnorm (reduce-scatter + residual add + RMSNorm [+ fp8 cast] on this rank's rows)
through the host backend: semantics against an fp64 torch reference, the in-place reduce-scatter of x against the
plain reduce_scatter, fp8 output against per_token_cast_to_fp8, argument checks."""
import pytest
import torch

from helpers import run_host_ranks
from rmsnorm_ref import assert_fp8_cast_of, rmsnorm_ref
from uccl_b200 import Communicator

N = 4
EPS = 1e-6


@pytest.fixture(scope="module")
def world4():
    return Communicator.local_world(N, host=True, heap_bytes=96 << 20, stage_bytes=1 << 20, timeout_ms=20000)


def _inputs(T, H, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(T, H, generator=g).to(dtype) for _ in range(N)]
    residual = (torch.randn(T, H, generator=g) * 2).to(dtype)  # full residual; rank r gets rows r*Tl .. (r+1)*Tl
    weight = (torch.rand(H, generator=g) + 0.5).to(dtype)
    return xs, residual, weight


def _tol(dtype):
    return dict(rtol=2e-2, atol=3e-2) if dtype == torch.bfloat16 else dict(rtol=4e-3, atol=4e-3)


def _run(comms, xs, residual, weight, separate, quant=None):
    """One reduce_scatter_rmsnorm per rank; returns per rank (x, residual shard, residual_out, out)."""
    Tl = residual.size(0) // N

    def fn(c):
        x, res = xs[c.rank].clone(), residual[c.rank * Tl:(c.rank + 1) * Tl].clone()
        ro = torch.empty_like(res) if separate else None
        y = c.reduce_scatter_rmsnorm(x, res, weight, EPS, residual_out=ro, quant=quant)
        return x, res, (ro if separate else res), y

    return run_host_ranks(comms, fn)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("separate", [False, True])
@pytest.mark.parametrize("T,H", [(4, 256), (20, 4096), (12, 1032)])
def test_host_reduce_scatter_rmsnorm_matches_fp64_reference(world4, dtype, separate, T, H):
    xs, residual, weight = _inputs(T, H, dtype)
    outs = _run(world4, xs, residual, weight, separate)
    Tl = T // N
    s = torch.stack([x.double() for x in xs]).sum(0)
    # the plain reduce_scatter of the same inputs, out of place
    plain = run_host_ranks(world4, lambda c: c.reduce_scatter(torch.empty(Tl, H, dtype=dtype), xs[c.rank].clone()))
    for r, (x, res, ro, y) in enumerate(outs):
        lo, hi = r * Tl, (r + 1) * Tl
        xr = x[lo:hi]
        assert torch.equal(xr, plain[r])  # in-place reduce-scatter: my rows of x hold my rows of the sum
        assert torch.equal(x[:lo], xs[r][:lo]) and torch.equal(x[hi:], xs[r][hi:])  # the rest of x is untouched
        assert torch.allclose(xr.double(), s[lo:hi], **_tol(dtype))
        assert torch.allclose(ro.double(), xr.double() + residual[lo:hi].double(), **_tol(dtype))
        if separate:
            assert torch.equal(res, residual[lo:hi])  # the residual shard itself is untouched
        assert torch.allclose(y.double(), rmsnorm_ref(ro, weight, EPS), **_tol(dtype))
        assert y.shape == (Tl, H)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_host_reduce_scatter_rmsnorm_equals_all_reduce_rmsnorm(world4, dtype):
    """The ranks' shards concatenated in rank order are what all_reduce_rmsnorm gives with the full residual."""
    T, H = 8, 1024
    xs, residual, weight = _inputs(T, H, dtype, seed=2)
    sp = _run(world4, xs, residual, weight, separate=True)

    def tp(c):
        x, res = xs[c.rank].clone(), residual.clone()
        return res, c.all_reduce_rmsnorm(x, res, weight, EPS)

    ro_tp, y_tp = run_host_ranks(world4, tp)[0]
    assert torch.equal(torch.cat([ro for _, _, ro, _ in sp]), ro_tp)
    assert torch.equal(torch.cat([y for _, _, _, y in sp]), y_tp)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("separate", [False, True])
def test_host_reduce_scatter_rmsnorm_fp8_is_per_token_cast_of_out(world4, dtype, separate):
    T, H = 24, 1024
    xs, residual, weight = _inputs(T, H, dtype, seed=1)
    plain = _run(world4, xs, residual, weight, separate)
    quant = _run(world4, xs, residual, weight, separate, quant="fp8")
    for (x0, _, ro0, y0), (x1, _, ro1, (q, sc)) in zip(plain, quant):
        assert torch.equal(x0, x1) and torch.equal(ro0, ro1)
        assert q.dtype == torch.float8_e4m3fn and q.shape == (T // N, H)
        assert sc.dtype == torch.float32 and sc.shape == (T // N, H // 128) and sc.is_contiguous()
        assert_fp8_cast_of(q, sc, y0)


def test_host_reduce_scatter_rmsnorm_argument_checks(world4):
    c = world4[0]
    T, H = 8, 256
    x = torch.zeros(T, H, dtype=torch.bfloat16)
    res = torch.zeros(T // N, H, dtype=torch.bfloat16)
    w = torch.ones(H, dtype=torch.bfloat16)
    # tokens must split evenly over the ranks
    with pytest.raises(ValueError, match="divisible"):
        c.reduce_scatter_rmsnorm(torch.zeros(6, H, dtype=torch.bfloat16), res, w)
    # the residual is this rank's shard [T / n, H], not the full [T, H]
    with pytest.raises(ValueError):
        c.reduce_scatter_rmsnorm(x, torch.zeros_like(x), w)
    # aliasing: out must not overlap x or residual
    with pytest.raises(ValueError):
        c.reduce_scatter_rmsnorm(x, res, w, out=x[:T // N])
    with pytest.raises(ValueError):
        c.reduce_scatter_rmsnorm(x, res, w, out=res)
    # residual and residual_out must not overlap x
    with pytest.raises(ValueError):
        c.reduce_scatter_rmsnorm(x, x[:T // N], w)
    with pytest.raises(ValueError):
        c.reduce_scatter_rmsnorm(x, res, w, residual_out=x[T // N:2 * T // N])
    # residual_out may be residual itself, but must not overlap anything else
    big = torch.zeros(T // N + 1, H, dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        c.reduce_scatter_rmsnorm(x, big[:T // N], w, residual_out=big[1:])
    y = torch.empty(T // N, H, dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        c.reduce_scatter_rmsnorm(x, res, w, residual_out=y, out=y)
    # shapes, dtypes, quant mode
    with pytest.raises(ValueError):
        c.reduce_scatter_rmsnorm(x, res, w.float())
    with pytest.raises(ValueError):
        c.reduce_scatter_rmsnorm(x, res, w, quant="int8")
    with pytest.raises(ValueError):
        c.reduce_scatter_rmsnorm(x.view(-1), res.view(-1), w)
    # native checks: dtype, hidden size range, fp8 group size
    xf = torch.zeros(T, H)
    with pytest.raises(RuntimeError, match="bf16 or fp16"):
        c.reduce_scatter_rmsnorm(xf, torch.zeros(T // N, H), torch.ones(H))
    for Hb in (12, 16384 + 8):
        xh = torch.zeros(N, Hb, dtype=torch.float16)
        with pytest.raises(RuntimeError, match="multiple of 8"):
            c.reduce_scatter_rmsnorm(xh, torch.zeros(1, Hb, dtype=torch.float16), torch.ones(Hb, dtype=torch.float16))
    x8 = torch.zeros(N, 192, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="128"):
        c.reduce_scatter_rmsnorm(x8, torch.zeros(1, 192, dtype=torch.bfloat16), torch.ones(192, dtype=torch.bfloat16),
                                 quant="fp8")


def test_host_reduce_scatter_rmsnorm_zero_tokens_is_noop(world4):
    x = torch.zeros(0, 512, dtype=torch.bfloat16)
    res = torch.zeros_like(x)
    y = world4[0].reduce_scatter_rmsnorm(x, res, torch.ones(512, dtype=torch.bfloat16))
    assert y.shape == (0, 512)
    q, sc = world4[0].reduce_scatter_rmsnorm(x, res, torch.ones(512, dtype=torch.bfloat16), quant="fp8")
    assert q.shape == (0, 512) and sc.shape == (0, 4)
