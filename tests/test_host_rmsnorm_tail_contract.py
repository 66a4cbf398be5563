"""The argument contract shared by the four fused residual add + RMSNorm layer tails (all_reduce_rmsnorm,
reduce_scatter_rmsnorm, combine_rmsnorm, low_latency_combine_rmsnorm), pinned on a one-rank host world: which
operand overlaps each op accepts, and which exception type each bad argument raises.

The overlap rule: no tensor the op writes (residual_out, out, and x for the all-reduce and reduce-scatter tails, which
reduce x in place) may overlap another operand (x, residual, residual_out, out, the EP biases, the LL shared-expert
output) except weight; only residual_out may be residual itself."""
import pytest
import torch

from uccl_b200 import Communicator
from uccl_b200.ep import Buffer

T, H, E, K = 8, 256, 4, 2
EPS = 1e-6
OPS = ("tp", "sp", "ep", "ll")
EXTRA = {"ep": "bias", "ll": "shared"}  # the extra input each EP tail reads


@pytest.fixture(scope="module")
def comm():
    return Communicator.local_world(1, host=True, heap_bytes=96 << 20, stage_bytes=1 << 20, timeout_ms=20000)[0]


def _bf16(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(torch.bfloat16)


def _op(comm, op):
    """Returns (x, call): x is the op's input rows, call(x, residual, weight, **kw) runs the op."""
    idx = torch.rand(T, E, generator=torch.Generator().manual_seed(1)).topk(K, dim=1).indices.contiguous()
    if op == "tp":
        return _bf16(T, H, seed=2), lambda x, r, w, **kw: comm.all_reduce_rmsnorm(x, r, w, EPS, **kw)
    if op == "sp":
        return _bf16(T, H, seed=2), lambda x, r, w, **kw: comm.reduce_scatter_rmsnorm(x, r, w, EPS, **kw)
    if op == "ep":
        b = Buffer(comm=comm, num_nvl_bytes=1 << 20)
        tpr, _, tpe, inr, _ = b.get_dispatch_layout(idx, E)
        rx, _, _, _, h, _ = b.dispatch(_bf16(T, H, seed=2), num_tokens_per_rank=tpr, is_token_in_rank=inr,
                                       num_tokens_per_expert=tpe, topk_idx=idx)
        return rx.clone(), lambda x, r, w, **kw: b.combine_rmsnorm(x, h, r, w, EPS, **kw)
    b = Buffer(comm=comm, num_nvl_bytes=1 << 20, low_latency_mode=True)
    rx, _, handle, _, _ = b.low_latency_dispatch(_bf16(T, H, seed=2), idx, T, E, use_fp8=False)
    wts = torch.rand(T, K, generator=torch.Generator().manual_seed(3))
    x = b.get_next_low_latency_combine_buffer(handle)
    x.copy_(rx)
    return x, lambda x, r, w, **kw: b.low_latency_combine_rmsnorm(x, idx, wts, handle, r, w, EPS, **kw)


def _rows(t):
    """[T, H] over the first bytes of t."""
    return t.reshape(-1)[:T * H].view(T, H)


# name -> (keyword arguments built from x and the op's extra-input name, the ops that accept them)
OVERLAP_CASES = {
    "defaults": (lambda x, e: {}, OPS),
    "residual_out_is_residual": (lambda x, e: dict(residual=(r := _bf16(T, H)), residual_out=r), OPS),
    "weight_overlaps_x": (lambda x, e: dict(weight=x.reshape(-1)[:H]), OPS),
    # x is read-only in the EP tails, and reduced in place by the collective ones
    "residual_overlaps_x": (lambda x, e: dict(residual=_rows(x), residual_out=_bf16(T, H)), ("ep", "ll")),
    "residual_overlaps_x_in_place": (lambda x, e: dict(residual=_rows(x)), ()),
    "out_overlaps_x": (lambda x, e: dict(out=_rows(x)), ()),
    "out_is_residual": (lambda x, e: dict(residual=(r := _bf16(T, H)), out=r), ()),
    "out_is_residual_out": (lambda x, e: dict(residual_out=(r := _bf16(T, H)), out=r), ()),
    "residual_out_overlaps_x": (lambda x, e: dict(residual_out=_rows(x)), ()),
    "residual_out_straddles_residual": (
        lambda x, e: dict(residual=(big := _bf16(T + 1, H))[:T], residual_out=big[1:]), ()),
    # the extra inputs of the EP tails are read-only
    "extra_is_residual": (lambda x, e: {e: (r := _bf16(T, H)), "residual": r, "residual_out": _bf16(T, H)},
                          ("ep", "ll")),
    "extra_is_residual_in_place": (lambda x, e: {e: (r := _bf16(T, H)), "residual": r}, ()),
    "extra_is_out": (lambda x, e: {e: (o := torch.empty(T, H, dtype=torch.bfloat16)), "out": o}, ()),
}


@pytest.mark.parametrize("op,case", [(op, case) for op in OPS for case in OVERLAP_CASES
                                     if op in EXTRA or not case.startswith("extra")])
def test_rmsnorm_tail_overlap_rule(comm, op, case):
    build, accepted = OVERLAP_CASES[case]
    x, call = _op(comm, op)
    kw = dict(residual=_bf16(T, H, seed=4), weight=(torch.rand(H) + 0.5).to(torch.bfloat16))
    kw.update(build(x, EXTRA.get(op)))
    r, w = kw.pop("residual"), kw.pop("weight")
    if op in accepted:
        call(x, r, w, **kw)
    else:
        with pytest.raises(ValueError):
            call(x, r, w, **kw)


# name -> (arguments built from x as (x, residual, weight, kw), exception per op)
BAD_ARGUMENTS = {
    "float32": (lambda x: (x.float(), torch.zeros(T, H), torch.ones(H), {}),
                dict(tp=RuntimeError, sp=RuntimeError, ep=ValueError, ll=ValueError)),
    "quant_int8": (lambda x: (x, _bf16(T, H), torch.ones(H, dtype=torch.bfloat16), dict(quant="int8")),
                   dict.fromkeys(OPS, ValueError)),
    "residual_shape": (lambda x: (x, _bf16(T + 1, H), torch.ones(H, dtype=torch.bfloat16), {}),
                       dict.fromkeys(OPS, ValueError)),
    "weight_dtype": (lambda x: (x, _bf16(T, H), torch.ones(H, dtype=torch.float16), {}),
                     dict.fromkeys(OPS, ValueError)),
    "out_dtype": (lambda x: (x, _bf16(T, H), torch.ones(H, dtype=torch.bfloat16),
                             dict(out=torch.empty(T, H, dtype=torch.bfloat16), quant="fp8")),
                  dict.fromkeys(OPS, ValueError)),
    "residual_out_not_contiguous": (lambda x: (x, _bf16(T, H), torch.ones(H, dtype=torch.bfloat16),
                                               dict(residual_out=_bf16(H, T).t())),
                                    dict.fromkeys(OPS, ValueError)),
}


@pytest.mark.parametrize("case", list(BAD_ARGUMENTS))
@pytest.mark.parametrize("op", OPS)
def test_rmsnorm_tail_bad_arguments(comm, op, case):
    build, raises = BAD_ARGUMENTS[case]
    x, call = _op(comm, op)
    x, r, w, kw = build(x)
    with pytest.raises(raises[op], match="bf16 or fp16" if raises[op] is RuntimeError else None):
        call(x, r, w, **kw)
