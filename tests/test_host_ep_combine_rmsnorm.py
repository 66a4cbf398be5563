"""CPU tests of ep.Buffer.combine_rmsnorm (EP combine + residual add + RMSNorm [+ fp8 cast]) through the host backend:
semantics against an fp64 torch reference and against combine() followed by the residual add, fp8 output against
per_token_cast_to_fp8, bias forms, a rank without tokens, argument and aliasing checks."""
import pytest
import torch

from helpers import run_host_ranks
from rmsnorm_ref import assert_fp8_cast_of, rmsnorm_ref
from uccl_b200 import Communicator
from uccl_b200.ep import Buffer

N = 4
EPS = 1e-6
E = 8


@pytest.fixture(scope="module")
def world4():
    return Communicator.local_world(N, host=True, heap_bytes=96 << 20, stage_bytes=1 << 20, timeout_ms=20000)


def _inputs(Ts, H, K=3, seed=0):
    g = torch.Generator().manual_seed(seed)
    xs, idxs, residuals, biases = [], [], [], []
    for T in Ts:
        xs.append((torch.randn(T, H, generator=g) * 2).to(torch.bfloat16))
        idx = torch.rand(T, E, generator=g).topk(K, dim=1).indices
        idx = idx.masked_fill(torch.rand(T, K, generator=g) < 0.1, -1)
        if T > 2:
            idx[1] = -1  # a token routed to no rank: combined = bias (or 0)
        idxs.append(idx.contiguous())
        residuals.append(torch.randn(T, H, generator=g).to(torch.bfloat16))
        biases.append((torch.randn(T, H, generator=g).to(torch.bfloat16), torch.randn(T, H, generator=g).to(torch.bfloat16)))
    weight = (torch.rand(H, generator=g) + 0.5).to(torch.bfloat16)
    return xs, idxs, residuals, biases, weight


def _bias_arg(bias_mode, pair):
    return {"none": None, "one": pair[0], "tuple": pair}[bias_mode]


def _run(comms, xs, idxs, residuals, biases, weight, bias_mode="none", separate=False, quant=None):
    """Per rank: dispatch, identity-times-(rank + 1) experts, then combine() and combine_rmsnorm() of the same rows.
    Returns (combined, residual_out, out, residual after the call, in-rank mask)."""

    def fn(c):
        r = c.rank
        b = Buffer(comm=c, num_nvl_bytes=1 << 20)
        tpr, _, tpe, inr, _ = b.get_dispatch_layout(idxs[r], E)
        rx, _, _, _, h, _ = b.dispatch(xs[r], num_tokens_per_rank=tpr, is_token_in_rank=inr,
                                       num_tokens_per_expert=tpe, topk_idx=idxs[r])
        y = (rx.float() * (r + 1)).to(torch.bfloat16)
        bias = _bias_arg(bias_mode, biases[r])
        combined, _, _ = b.combine(y, h, bias=bias)
        res = residuals[r].clone()
        ro = torch.empty_like(res) if separate else None
        o, _ = b.combine_rmsnorm(y, h, res, weight, EPS, bias=bias, residual_out=ro, quant=quant)
        return combined, (ro if separate else res), o, res, inr

    return run_host_ranks(comms, fn)


@pytest.mark.parametrize("bias_mode", ["none", "one", "tuple"])
@pytest.mark.parametrize("separate", [False, True])
@pytest.mark.parametrize("H", [256, 1032])
def test_host_combine_rmsnorm_matches_fp64_reference(world4, bias_mode, separate, H):
    Ts = [21, 9, 16, 5]
    xs, idxs, residuals, biases, weight = _inputs(Ts, H)
    outs = _run(world4, xs, idxs, residuals, biases, weight, bias_mode, separate)
    tol = dict(rtol=2e-2, atol=3e-2)
    for r, (combined, ro, y, res, inr) in enumerate(outs):
        # fp64 formula: every destination rank d returns the token times (d + 1)
        fan = (inr.double() * torch.arange(1, N + 1, dtype=torch.float64)).sum(1, keepdim=True)
        ref_c = xs[r].double() * fan
        bias = _bias_arg(bias_mode, biases[r])
        for bb in (bias if isinstance(bias, tuple) else (bias,)):
            if bb is not None:
                ref_c = ref_c + bb.double()
        ref_ro = ref_c + residuals[r].double()
        ref_y = rmsnorm_ref(ref_ro, weight, EPS)
        assert torch.allclose(ro.double(), ref_ro, **tol)
        assert torch.allclose(y.double(), ref_y, **tol)
        # residual_out is bf16(combine() + residual) exactly
        assert torch.equal(ro, (combined.float() + residuals[r].float()).to(torch.bfloat16))
        if separate:
            assert torch.equal(res, residuals[r])  # the residual itself is untouched
        assert y.shape == (Ts[r], H) and y.dtype == torch.bfloat16


@pytest.mark.parametrize("separate", [False, True])
def test_host_combine_rmsnorm_fp8_is_per_token_cast_of_out(world4, separate):
    Ts, H = [12, 7, 0, 30], 1024
    xs, idxs, residuals, biases, weight = _inputs(Ts, H, seed=1)
    plain = _run(world4, xs, idxs, residuals, biases, weight, "one", separate)
    quant = _run(world4, xs, idxs, residuals, biases, weight, "one", separate, quant="fp8")
    for r, ((_, ro0, y0, _, _), (_, ro1, (q, sc), _, _)) in enumerate(zip(plain, quant)):
        assert torch.equal(ro0, ro1)
        assert q.dtype == torch.float8_e4m3fn and q.shape == (Ts[r], H)
        assert sc.dtype == torch.float32 and sc.shape == (Ts[r], H // 128) and sc.is_contiguous()
        if Ts[r]:
            assert_fp8_cast_of(q, sc, y0)


def test_host_combine_rmsnorm_rank_without_tokens(world4):
    Ts, H = [10, 0, 6, 3], 512
    xs, idxs, residuals, biases, weight = _inputs(Ts, H, seed=2)
    outs = _run(world4, xs, idxs, residuals, biases, weight, "tuple")
    combined, ro, y, _, _ = outs[1]
    assert combined.shape == ro.shape == y.shape == (0, H)
    for r in (0, 2, 3):
        combined, ro, y, _, _ = outs[r]
        assert torch.equal(ro, (combined.float() + residuals[r].float()).to(torch.bfloat16))


def test_host_combine_rmsnorm_argument_checks(world4):
    H, T = 256, 6
    xs, idxs, residuals, biases, weight = _inputs([T] * N, H, seed=3)

    def fn(c):
        r = c.rank
        b = Buffer(comm=c, num_nvl_bytes=1 << 20)
        tpr, _, tpe, inr, _ = b.get_dispatch_layout(idxs[r], E)
        rx, _, _, _, h, _ = b.dispatch(xs[r], num_tokens_per_rank=tpr, is_token_in_rank=inr,
                                       num_tokens_per_expert=tpe, topk_idx=idxs[r])
        x = rx.clone()
        res, w = residuals[r].clone(), weight

        def expect(**kw):
            # every check fires before any communication, so one rank can run them alone
            if r != 0:
                return
            args = dict(x=x, residual=res, weight=w)
            args.update(kw)
            with pytest.raises(ValueError):
                b.combine_rmsnorm(args.pop("x"), h, args.pop("residual"), args.pop("weight"), EPS, **args)

        # shapes and dtypes
        expect(residual=torch.zeros(T + 1, H, dtype=torch.bfloat16))
        expect(residual=res.float())
        expect(weight=torch.ones(H + 8, dtype=torch.bfloat16))
        expect(weight=w.half())
        expect(x=x.float())
        expect(bias=torch.zeros(T, H + 8, dtype=torch.bfloat16))
        expect(out=torch.empty(T, H, dtype=torch.float16))
        expect(out=torch.empty(T, H, dtype=torch.bfloat16), quant="fp8")
        expect(quant="int8")
        x12 = torch.zeros(x.size(0), 12, dtype=torch.bfloat16)
        expect(x=x12, residual=torch.zeros(T, 12, dtype=torch.bfloat16), weight=torch.ones(12, dtype=torch.bfloat16))
        x192 = torch.zeros(x.size(0), 192, dtype=torch.bfloat16)
        expect(x=x192, residual=torch.zeros(T, 192, dtype=torch.bfloat16), weight=torch.ones(192, dtype=torch.bfloat16),
               quant="fp8")
        # aliasing: out must not overlap x, residual or residual_out
        big = torch.zeros(max(x.size(0), T) + 1, H, dtype=torch.bfloat16)
        expect(x=big[:x.size(0)], out=big[1:T + 1])
        expect(out=res)
        ro = torch.empty(T, H, dtype=torch.bfloat16)
        expect(residual_out=ro, out=ro)
        # residual_out must not overlap x, and overlaps residual only by being residual itself
        expect(x=big[:x.size(0)], residual_out=big[1:T + 1])
        pair = torch.zeros(T + 1, H, dtype=torch.bfloat16)
        expect(residual=pair[:T], residual_out=pair[1:])
        # residual_out may be residual itself (the default), explicitly too
        y, _ = b.combine_rmsnorm(x, h, res, w, EPS, residual_out=res)
        return y.shape

    assert run_host_ranks(world4, fn) == [(T, H)] * N
