#!/usr/bin/env python
"""Same-box anchor: the UPSTREAM DeepEP intranode kernels vendored by the reference
(thirdparty/DeepEP of the reference, unmodified sources, its own setup.py with the DISABLE_NVSHMEM branch,
built for sm_90a into oracle/_ref/deepep by oracle/build_deepep.sh) on the headline config.

The reference's own `uccl.ep` cannot be built offline (nanobind + libibverbs headers are absent), but its
intranode dispatch/combine kernels are DeepEP's re-hosted (SURVEY.md section 0, fact 5; ep/src/intranode.cu),
so this is the closest thing to "the reference's kernels re-measured on the box".  It is a DIAGNOSTIC, not the
driver's reference arm: bench.py --impl reference attaches it under "diagnostic".

Measured exactly like the reference measures itself (ep/bench/test_intranode.py:457-539, thirdparty/DeepEP/
tests/test_intranode.py:175-226): cached-handle dispatch of a pre-cast (e4m3, scales) tuple and of bf16,
bf16 combine, `num_sms` = 24, best over a sweep of NVL chunk sizes; CUDA events, 256 MiB L2 flush before
every timed call, max over ranks.  The bf16 -> fp8 cast the reference runs as separate torch kernels before the
dispatch (ep/bench/utils.py:666-675) is timed separately.

  torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 benchmarks/deepep_baseline.py [--out f.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEEPEP_DIR = os.path.join(ROOT, "oracle", "_ref", "deepep")


def available() -> str | None:
    """None if the vendored DeepEP build is importable, else the reason."""
    if not os.path.isdir(os.path.join(DEEPEP_DIR, "deep_ep")):
        return "oracle/_ref/deepep not built (oracle/build_deepep.sh)"
    return None


def per_token_cast_to_fp8(x):
    """The reference's pre-dispatch cast (ep/bench/utils.py:666-675): separate elementwise torch kernels."""
    import torch

    m, n = x.shape
    xv = x.view(m, -1, 128)
    amax = xv.abs().float().amax(dim=2).view(m, -1).clamp(1e-4)
    return (xv * (448.0 / amax.unsqueeze(2))).to(torch.float8_e4m3fn).view(m, n), (amax / 448.0).view(m, -1)


def run(tokens=4096, hidden=7168, topk=8, experts=256, num_sms=24, iters=20, warmup=5,
        dispatch_chunks=(0, 8, 12, 16, 20, 24, 28, 32), combine_chunks=(0, 2, 4, 6, 8, 10, 12, 16), quiet=False):
    """Must be called on every rank of an initialised NCCL process group (one process per GPU)."""
    import torch
    import torch.distributed as dist

    if DEEPEP_DIR not in sys.path:
        sys.path.insert(0, DEEPEP_DIR)
    import deep_ep  # noqa: E402  (the vendored upstream build)

    rank, n = dist.get_rank(), dist.get_world_size()
    dev = torch.device("cuda", torch.cuda.current_device())
    group = dist.group.WORLD
    buffer = deep_ep.Buffer(group, int(2e9), 0, low_latency_mode=False, num_qps_per_rank=1, explicitly_destroy=True)
    T, H, K, E = tokens, hidden, topk, experts
    g = torch.Generator(device="cpu").manual_seed(1234 + rank)
    x = torch.randn(T, H, generator=g).to(torch.bfloat16).to(dev)
    scores = torch.randn(T, E, generator=g).abs() + 1
    topk_idx = scores.topk(K, dim=-1, largest=True, sorted=False).indices.to(torch.int64).contiguous().to(dev)
    topk_w = torch.rand(T, K, generator=g).float().to(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def mx(v: float) -> float:
        t = torch.tensor([v], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def timed(fn):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        dist.barrier()
        evs = []
        for _ in range(iters):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            evs.append((s, e))
        torch.cuda.synchronize()
        v = [a.elapsed_time(b) for a, b in evs]
        return mx(sum(v) / len(v)) * 1e3  # us, max over ranks of the per-rank mean

    cast_us = timed(lambda: per_token_cast_to_fp8(x))
    x_e4m3 = per_token_cast_to_fp8(x)
    x_e4m3 = (x_e4m3[0], x_e4m3[1].T.contiguous().T)  # the layout DeepEP's test feeds (test_intranode.py:29)

    tpr, _, tpe, in_rank, _ = buffer.get_dispatch_layout(topk_idx, E)
    layout_us = timed(lambda: buffer.get_dispatch_layout(topk_idx, E))
    nvl_buffer_size = 256
    cfg0 = deep_ep.Config(num_sms, 8, nvl_buffer_size)
    recv_x, recv_idx, recv_w, per_expert, handle, _ = buffer.dispatch(
        x=x, num_tokens_per_rank=tpr, is_token_in_rank=in_rank, num_tokens_per_expert=tpe, topk_idx=topk_idx,
        topk_weights=topk_w, config=cfg0)
    num_recv = int(recv_x.size(0))

    def config_for(chunk, which):
        if chunk > 0:
            return deep_ep.Config(num_sms, chunk, nvl_buffer_size)
        deep_ep.Buffer.set_num_sms(num_sms)
        return deep_ep.Buffer.get_dispatch_config(n) if which == "d" else deep_ep.Buffer.get_combine_config(n)

    rows = {"dispatch_fp8": {}, "dispatch_bf16": {}, "combine_bf16": {}}
    for name, cur in (("dispatch_fp8", x_e4m3), ("dispatch_bf16", x)):
        for ch in dispatch_chunks:
            cfg = config_for(ch, "d")
            rows[name][str(ch) if ch else "default"] = timed(lambda: buffer.dispatch(x=cur, handle=handle, config=cfg))
    for ch in combine_chunks:
        cfg = config_for(ch, "c")
        rows["combine_bf16"][str(ch) if ch else "default"] = timed(lambda: buffer.combine(x=recv_x, handle=handle, config=cfg))
    best = {k: min(v.values()) for k, v in rows.items()}
    out = {
        "what": "upstream DeepEP (reference/thirdparty/DeepEP, unmodified, DISABLE_NVSHMEM, sm_90a) intranode kernels",
        "n_gpus": n, "tokens": T, "hidden": H, "topk": K, "experts": E, "num_sms": num_sms,
        "num_recv_tokens": num_recv, "iters": iters, "timing": "CUDA events, 256 MiB L2 flush per call, max over ranks",
        "fp8_cast_torch_us": cast_us, "layout_us": layout_us,
        "best_us": best,
        "dispatch_fp8_incl_cast_us": best["dispatch_fp8"] + cast_us,
        "step_us_fp8_dispatch_plus_bf16_combine": best["dispatch_fp8"] + best["combine_bf16"],
        "step_us_incl_cast": best["dispatch_fp8"] + cast_us + best["combine_bf16"],
        "by_nvl_chunk_us": rows,
    }
    if rank == 0 and not quiet:
        print(json.dumps(out), flush=True)
    buffer.destroy()
    return out


def main():
    import torch
    import torch.distributed as dist

    p = argparse.ArgumentParser()
    p.add_argument("--tokens", type=int, default=4096)
    p.add_argument("--hidden", type=int, default=7168)
    p.add_argument("--topk", type=int, default=8)
    p.add_argument("--experts", type=int, default=256)
    p.add_argument("--num-sms", type=int, default=24)
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--out", default=None)
    a = p.parse_args()
    why = available()
    rank = int(os.environ.get("RANK", 0))
    if why:
        if rank == 0:
            print(json.dumps({"unavailable": why}))
        return 0
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    try:
        out = run(a.tokens, a.hidden, a.topk, a.experts, a.num_sms, a.iters)
    except Exception as e:  # noqa: BLE001 - a diagnostic must never take the caller down
        out = {"unavailable": f"{type(e).__name__}: {e}"[:400]}
        if rank == 0:
            print(json.dumps(out), flush=True)
    if rank == 0 and a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    dist.barrier()
    dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
