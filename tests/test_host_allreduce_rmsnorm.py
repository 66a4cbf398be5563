"""CPU tests of all_reduce_rmsnorm (all-reduce + residual add + RMSNorm [+ fp8 cast]) through the host backend:
semantics against an fp64 torch reference, fp8 output against per_token_cast_to_fp8, argument checks."""
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
    residual = (torch.randn(T, H, generator=g) * 2).to(dtype)
    weight = (torch.rand(H, generator=g) + 0.5).to(dtype)
    return xs, residual, weight


def _tol(dtype):
    return dict(rtol=2e-2, atol=3e-2) if dtype == torch.bfloat16 else dict(rtol=4e-3, atol=4e-3)


def _run(comms, xs, residual, weight, separate, quant=None):
    def fn(c):
        x, res = xs[c.rank].clone(), residual.clone()
        ro = torch.empty_like(res) if separate else None
        y = c.all_reduce_rmsnorm(x, res, weight, EPS, residual_out=ro, quant=quant)
        return x, res, (ro if separate else res), y

    return run_host_ranks(comms, fn)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("separate", [False, True])
@pytest.mark.parametrize("T,H", [(1, 256), (5, 4096), (3, 1032)])
def test_host_allreduce_rmsnorm_matches_fp64_reference(world4, dtype, separate, T, H):
    xs, residual, weight = _inputs(T, H, dtype)
    outs = _run(world4, xs, residual, weight, separate)
    s = torch.stack([x.double() for x in xs]).sum(0)
    for x, res, ro, y in outs:
        assert torch.allclose(x.double(), s, **_tol(dtype))
        ref_ro = x.double() + residual.double()
        assert torch.allclose(ro.double(), ref_ro, **_tol(dtype))
        if separate:
            assert torch.equal(res, residual)  # residual itself untouched
        assert torch.allclose(y.double(), rmsnorm_ref(ro, weight, EPS), **_tol(dtype))
    for x, _, ro, y in outs[1:]:  # every rank holds the same bits
        assert torch.equal(x, outs[0][0]) and torch.equal(ro, outs[0][2]) and torch.equal(y, outs[0][3])


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("separate", [False, True])
def test_host_allreduce_rmsnorm_fp8_is_per_token_cast_of_out(world4, dtype, separate):
    T, H = 6, 1024
    xs, residual, weight = _inputs(T, H, dtype, seed=1)
    plain = _run(world4, xs, residual, weight, separate)
    quant = _run(world4, xs, residual, weight, separate, quant="fp8")
    for (x0, _, ro0, y0), (x1, _, ro1, (q, sc)) in zip(plain, quant):
        assert torch.equal(x0, x1) and torch.equal(ro0, ro1)
        assert q.dtype == torch.float8_e4m3fn and q.shape == (T, H)
        assert sc.dtype == torch.float32 and sc.shape == (T, H // 128)
        assert_fp8_cast_of(q, sc, y0)


def test_host_allreduce_rmsnorm_argument_checks(world4):
    c = world4[0]
    x = torch.zeros(2, 256, dtype=torch.bfloat16)
    res = torch.zeros_like(x)
    w = torch.ones(256, dtype=torch.bfloat16)
    # output aliasing
    with pytest.raises(ValueError):
        c.all_reduce_rmsnorm(x, res, w, out=x)
    with pytest.raises(ValueError):
        c.all_reduce_rmsnorm(x, res, w, out=res)
    with pytest.raises(ValueError):
        c.all_reduce_rmsnorm(x, x, w)
    # shapes, dtypes, quant mode
    with pytest.raises(ValueError):
        c.all_reduce_rmsnorm(x, res[:1].contiguous(), w)
    with pytest.raises(ValueError):
        c.all_reduce_rmsnorm(x, res, w.float())
    with pytest.raises(ValueError):
        c.all_reduce_rmsnorm(x, res, w, quant="int8")
    with pytest.raises(ValueError):
        c.all_reduce_rmsnorm(x.view(-1), res.view(-1), w)
    # native checks: dtype, hidden size range and alignment, fp8 group size
    xf = torch.zeros(2, 256)
    with pytest.raises(RuntimeError, match="bf16 or fp16"):
        c.all_reduce_rmsnorm(xf, torch.zeros_like(xf), torch.ones(256))
    for H in (12, 16384 + 8):
        xh = torch.zeros(1, H, dtype=torch.float16)
        with pytest.raises(RuntimeError, match="multiple of 8"):
            c.all_reduce_rmsnorm(xh, torch.zeros_like(xh), torch.ones(H, dtype=torch.float16))
    x8 = torch.zeros(1, 192, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="128"):
        c.all_reduce_rmsnorm(x8, torch.zeros_like(x8), torch.ones(192, dtype=torch.bfloat16), quant="fp8")


def test_host_allreduce_rmsnorm_zero_tokens_is_noop(world4):
    x = torch.zeros(0, 512, dtype=torch.bfloat16)
    res = torch.zeros_like(x)
    y = world4[0].all_reduce_rmsnorm(x, res, torch.ones(512, dtype=torch.bfloat16))
    assert y.shape == (0, 512)
    q, sc = world4[0].all_reduce_rmsnorm(x, res, torch.ones(512, dtype=torch.bfloat16), quant="fp8")
    assert q.shape == (0, 512) and sc.shape == (0, 4)
