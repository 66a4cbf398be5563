"""CPU tests of ep.Buffer.low_latency_combine_rmsnorm (LL combine + shared-expert add + residual add + RMSNorm [+ fp8
cast], the tail of a decode MoE layer) through the host backend: semantics against an fp64 torch reference and against
low_latency_combine() -> + shared -> host_add_rmsnorm, fp8 output against per_token_cast_to_fp8, shared and
residual_out forms, use_logfmt, the receive hook, argument and aliasing checks."""
import pytest
import torch

from helpers import run_host_ranks
from rmsnorm_ref import assert_fp8_cast_of, rmsnorm_ref
from uccl_b200 import Communicator, _native
from uccl_b200.ep import Buffer
from uccl_b200.parallel.comm import dtype_code

N = 4
EPS = 1e-6
E = 8
E_LOCAL = E // N
K = 3
M = 32


@pytest.fixture(scope="module")
def world4():
    return Communicator.local_world(N, host=True, heap_bytes=96 << 20, stage_bytes=1 << 20, timeout_ms=20000)


def _inputs(Ts, H, seed=0):
    g = torch.Generator().manual_seed(seed)
    xs, idxs, ws, residuals, shareds = [], [], [], [], []
    for T in Ts:
        xs.append((torch.randn(T, H, generator=g) * 2).to(torch.bfloat16))
        idx = torch.rand(T, E, generator=g).topk(K, dim=1).indices
        idx = idx.masked_fill(torch.rand(T, K, generator=g) < 0.1, -1)
        if T > 2:
            idx[1] = -1  # a token routed to no expert: routed = 0
        idxs.append(idx.contiguous())
        ws.append(torch.rand(T, K, generator=g).float())
        residuals.append(torch.randn(T, H, generator=g).to(torch.bfloat16))
        shareds.append(torch.randn(T, H, generator=g).to(torch.bfloat16))
    weight = (torch.rand(H, generator=g) + 0.5).to(torch.bfloat16)
    return xs, idxs, ws, residuals, shareds, weight


def _expert_outputs(b, rx, cnt, handle, r):
    """The "expert" multiplies every row by its global expert id + 1."""
    y = b.get_next_low_latency_combine_buffer(handle)
    for el in range(E_LOCAL):
        c = int(cnt[el])
        y[el, :c] = (rx[el, :c].float() * (r * E_LOCAL + el + 1)).to(torch.bfloat16)
    return y


def _unfused(routed, shared, residual, weight, fp8):
    """low_latency_combine() -> torch's bf16 + shared -> the C++ epilogue (host_add_rmsnorm)."""
    combined = (routed + shared) if shared is not None else routed.clone()
    T, H = combined.shape
    ro = residual.clone()
    y = torch.empty(T, H, dtype=torch.float8_e4m3fn if fp8 else torch.bfloat16)
    sc = torch.empty(T, H // 128, dtype=torch.float32) if fp8 else None
    _native.C().host_add_rmsnorm(combined.data_ptr(), ro.data_ptr(), ro.data_ptr(), weight.data_ptr(), y.data_ptr(),
                                 sc.data_ptr() if fp8 else 0, T, H, dtype_code(torch.bfloat16), EPS)
    return ro, ((y, sc) if fp8 else y)


def _run(comms, xs, idxs, ws, residuals, shareds, weight, with_shared=False, separate=False, quant=None,
         use_logfmt=False, hook=False):
    """Per rank: LL dispatch, the experts, then low_latency_combine() and low_latency_combine_rmsnorm() of the same
    rows.  Returns (routed, residual_out, out, residual after the call)."""

    def fn(c):
        r = c.rank
        b = Buffer(comm=c, num_nvl_bytes=1 << 20, low_latency_mode=True)
        rx, cnt, handle, _, _ = b.low_latency_dispatch(xs[r], idxs[r], M, E, use_fp8=False)
        y = _expert_outputs(b, rx, cnt, handle, r)
        routed, _, _ = b.low_latency_combine(y, idxs[r], ws[r], handle, use_logfmt=use_logfmt)
        res = residuals[r].clone()
        ro = torch.empty_like(res) if separate else None
        o, _, h = b.low_latency_combine_rmsnorm(y, idxs[r], ws[r], handle, res, weight, EPS,
                                                shared=shareds[r] if with_shared else None, residual_out=ro,
                                                quant=quant, use_logfmt=use_logfmt, return_recv_hook=hook)
        assert (h is not None) == hook
        if hook:
            h()
        return routed, (ro if separate else res), o, res

    return run_host_ranks(comms, fn)


@pytest.mark.parametrize("with_shared", [False, True])
@pytest.mark.parametrize("separate", [False, True])
@pytest.mark.parametrize("use_logfmt", [False, True])
def test_host_ll_combine_rmsnorm_matches_unfused_and_fp64(world4, with_shared, separate, use_logfmt):
    Ts, H = [21, 9, 16, 5], 256
    xs, idxs, ws, residuals, shareds, weight = _inputs(Ts, H)
    outs = _run(world4, xs, idxs, ws, residuals, shareds, weight, with_shared, separate, use_logfmt=use_logfmt)
    for r, (routed, ro, y, res) in enumerate(outs):
        shared = shareds[r] if with_shared else None
        ro_u, y_u = _unfused(routed, shared, residuals[r], weight, False)
        assert torch.equal(ro, ro_u) and torch.equal(y, y_u)
        if separate:
            assert torch.equal(res, residuals[r])  # the residual itself is untouched
        assert y.shape == (Ts[r], H) and y.dtype == torch.bfloat16
        if use_logfmt:
            continue  # the simulated LogFMT cast changes the numerics of routed on purpose
        # fp64 formula: sum_k w[t,k] * (e_k + 1) * x[t]
        coef = torch.where(idxs[r] >= 0, ws[r].double() * (idxs[r] + 1).double(), torch.zeros((), dtype=torch.float64))
        ref = xs[r].double() * coef.sum(1, keepdim=True)
        if with_shared:
            ref = ref + shared.double()
        ref_ro = ref + residuals[r].double()
        ref_y = rmsnorm_ref(ref_ro, weight, EPS)
        assert torch.allclose(ro.double(), ref_ro, rtol=2e-2, atol=5e-2)
        assert torch.allclose(y.double(), ref_y, rtol=2e-2, atol=5e-2)


@pytest.mark.parametrize("with_shared", [False, True])
def test_host_ll_combine_rmsnorm_fp8_is_per_token_cast_of_out(world4, with_shared):
    Ts, H = [12, 7, 3, 30], 384
    xs, idxs, ws, residuals, shareds, weight = _inputs(Ts, H, seed=1)
    plain = _run(world4, xs, idxs, ws, residuals, shareds, weight, with_shared, separate=True)
    quant = _run(world4, xs, idxs, ws, residuals, shareds, weight, with_shared, separate=True, quant="fp8")
    for r, ((_, ro0, y0, _), (routed, ro1, (q, sc), _)) in enumerate(zip(plain, quant)):
        assert torch.equal(ro0, ro1)
        assert q.dtype == torch.float8_e4m3fn and q.shape == (Ts[r], H)
        assert sc.dtype == torch.float32 and sc.shape == (Ts[r], H // 128) and sc.is_contiguous()
        assert_fp8_cast_of(q, sc, y0)
        _, (q_u, sc_u) = _unfused(routed, shareds[r] if with_shared else None, residuals[r], weight, True)
        assert torch.equal(q.view(torch.uint8), q_u.view(torch.uint8)) and torch.equal(sc, sc_u)


def test_host_ll_combine_rmsnorm_hook(world4):
    Ts, H = [10, 4, 6, 3], 128
    xs, idxs, ws, residuals, shareds, weight = _inputs(Ts, H, seed=2)
    plain = _run(world4, xs, idxs, ws, residuals, shareds, weight, True, True)
    hooked = _run(world4, xs, idxs, ws, residuals, shareds, weight, True, True, hook=True)
    for (_, ro0, y0, _), (_, ro1, y1, _) in zip(plain, hooked):
        assert torch.equal(ro0, ro1) and torch.equal(y0, y1)


def test_host_ll_combine_rmsnorm_argument_checks(world4):
    H, T = 256, 6
    xs, idxs, ws, residuals, shareds, weight = _inputs([T] * N, H, seed=3)

    def fn(c):
        r = c.rank
        b = Buffer(comm=c, num_nvl_bytes=1 << 20, low_latency_mode=True)
        rx, cnt, handle, _, _ = b.low_latency_dispatch(xs[r], idxs[r], M, E, use_fp8=False)
        y = _expert_outputs(b, rx, cnt, handle, r)
        res, w, sh = residuals[r].clone(), weight, shareds[r]

        def expect(**kw):
            # every check fires before any communication, so one rank can run them alone
            if r != 0:
                return
            args = dict(x=y, topk_idx=idxs[r], topk_weights=ws[r], residual=res, weight=w)
            args.update(kw)
            with pytest.raises(ValueError):
                b.low_latency_combine_rmsnorm(args.pop("x"), args.pop("topk_idx"), args.pop("topk_weights"), handle,
                                              args.pop("residual"), args.pop("weight"), EPS, **args)

        # shapes and dtypes
        expect(residual=torch.zeros(T + 1, H, dtype=torch.bfloat16))
        expect(residual=res.float())
        expect(weight=torch.ones(H + 128, dtype=torch.bfloat16))
        expect(weight=w.half())
        expect(x=y.float())
        expect(x=y[:, :M])
        expect(x=y.reshape(-1, H))
        expect(topk_weights=ws[r].double())
        expect(topk_idx=idxs[r].int())
        expect(topk_idx=idxs[r][:, :2])
        expect(shared=torch.zeros(T, H + 128, dtype=torch.bfloat16))
        expect(shared=sh.float())
        expect(out=torch.empty(T, H, dtype=torch.float16))
        expect(out=torch.empty(T, H, dtype=torch.bfloat16), quant="fp8")
        expect(quant="int8")
        expect(topk_idx=torch.zeros(T, 33, dtype=torch.int64), topk_weights=torch.zeros(T, 33))
        # aliasing: out must not overlap x, residual, residual_out or shared
        expect(out=y.view(-1)[:T * H].view(T, H))
        expect(out=res)
        expect(shared=sh, out=sh)
        ro = torch.empty(T, H, dtype=torch.bfloat16)
        expect(residual_out=ro, out=ro)
        # residual_out must not overlap x or shared, and overlaps residual only by being residual itself
        expect(residual_out=y.view(-1)[H:(T + 1) * H].view(T, H))
        expect(shared=sh, residual_out=sh)
        pair = torch.zeros(T + 1, H, dtype=torch.bfloat16)
        expect(residual=pair[:T], residual_out=pair[1:])
        # residual_out may be residual itself (the default), explicitly too
        o, _, _ = b.low_latency_combine_rmsnorm(y, idxs[r], ws[r], handle, res, w, EPS, residual_out=res)
        return o.shape

    assert run_host_ranks(world4, fn) == [(T, H)] * N


def test_host_ll_combine_rmsnorm_hidden_limits(world4):
    """The LL limits: hidden % 128 == 0 and hidden <= 8192 (checked from the handle, before any communication)."""
    b = Buffer(comm=world4[0], num_nvl_bytes=1 << 20, low_latency_mode=True)
    T = 2
    for H in (192, 8320):
        handle = (None, None, M, H, E, 0, None, None)
        x = torch.zeros(E_LOCAL, N * M, H, dtype=torch.bfloat16)
        with pytest.raises(ValueError):
            b.low_latency_combine_rmsnorm(x, torch.zeros(T, K, dtype=torch.int64), torch.zeros(T, K), handle,
                                          torch.zeros(T, H, dtype=torch.bfloat16), torch.ones(H, dtype=torch.bfloat16))
