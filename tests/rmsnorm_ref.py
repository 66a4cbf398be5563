"""References shared by the tests of the fused residual add + RMSNorm layer tails."""
import torch

from uccl_b200.ep.utils import per_token_cast_to_fp8


def rmsnorm_ref(ro, weight, eps):
    """fp64 ``rmsnorm(ro, eps) * weight``."""
    rr = ro.double()
    return rr * torch.rsqrt(rr.pow(2).mean(1, keepdim=True) + eps) * weight.double()


def assert_fp8_cast_of(q, sc, y, what=None):
    """The fp8 pair ``(q, sc)`` is bitwise ``per_token_cast_to_fp8`` of the 16-bit ``y``."""
    q_ref, sc_ref = per_token_cast_to_fp8(y)
    assert torch.equal(q.view(torch.uint8), q_ref.view(torch.uint8)), what
    assert torch.equal(sc, sc_ref), what


def one_rank_epilogue(x, residual, weight, eps, quant):
    """The unfused tail on the GPU: the epilogue kernel of a one-rank ``all_reduce_rmsnorm`` (add_rmsnorm_kernel) on
    already combined rows ``x``.  Returns ``(residual_out, out, fp8 pair or None)`` on the CPU."""
    from helpers import get_world

    c1 = get_world(1)[0]
    dev = c1.device
    ro = residual.to(dev).clone()
    y = c1.all_reduce_rmsnorm(x.to(dev), ro, weight.to(dev), eps).cpu()
    # on the host, like the other fp8 tests: torch's CUDA division by a scalar multiplies by its reciprocal instead
    q = per_token_cast_to_fp8(y) if quant == "fp8" else None
    return ro.cpu(), y, q
