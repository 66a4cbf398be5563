#!/usr/bin/env python
"""EP dispatch/combine timing sweep over the SM budget (the reference tunes NVL chunk sizes at a
fixed 24 SMs, ep/bench/test_intranode.py:457-539; here the only knob is the number of CTAs).

  torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 benchmarks/ep_sweep.py [--out f.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

from uccl_b200 import Communicator
from uccl_b200.ep import Buffer, Config


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--tokens", type=int, default=4096)
    p.add_argument("--hidden", type=int, default=7168)
    p.add_argument("--topk", type=int, default=8)
    p.add_argument("--experts", type=int, default=256)
    p.add_argument("--sms", default="16,24,32,48,64,96,128,132")
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--impls", default="reg,tma", help="kernel implementations to sweep: reg (register path), tma (TMA pipelines)")
    p.add_argument("--modes", default="fp8_fused,bf16")
    p.add_argument("--stages", default="0", help="TMA pipeline depths to try (0 = fill shared memory), e.g. 0,4,6")
    p.add_argument("--ll", action="store_true", help="also time the low-latency path (128 tokens)")
    p.add_argument("--out", default=None)
    args = p.parse_args()
    rank, n, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if n > 1:
        dist.init_process_group("cpu:gloo,cuda:nccl", device_id=dev)
    T, H, K, E = args.tokens, args.hidden, args.topk, args.experts
    arena = n * T * (H * 2 + K * 4) + (1 << 20)
    nvl = 3 * arena + (2 << 20)
    ll_bytes = Buffer.get_low_latency_rdma_size_hint(128, H, n, E) if args.ll else 0
    heap = nvl + ll_bytes + (1 << 30)
    comm = Communicator.from_torch_dist(None, heap_bytes=heap, stage_bytes=64 << 20) if n > 1 else \
        Communicator.local_world(1, devices=[local], heap_bytes=heap)[0]
    buf = Buffer(comm=comm, num_nvl_bytes=nvl, num_rdma_bytes=ll_bytes, low_latency_mode=args.ll)
    g = torch.Generator(device="cpu").manual_seed(1234 + rank)
    x = torch.randn(T, H, generator=g).to(torch.bfloat16).to(dev)
    scores = torch.randn(T, E, generator=g).abs() + 1
    idx = scores.topk(K, dim=-1).indices.to(torch.int64).contiguous().to(dev)
    w = torch.rand(T, K, generator=g).float().to(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def mx(v):
        if n == 1:
            return v
        t = torch.tensor([v], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return t.item()

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        if n > 1:
            dist.barrier()
        evs = []
        for _ in range(args.iters):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            evs.append((s, e))
        torch.cuda.synchronize()
        v = sorted(a.elapsed_time(b) for a, b in evs)
        return mx(sum(v) / len(v)) * 1e3, mx(v[0]) * 1e3

    rows = []
    C = buf._C
    impl_ids = {"reg": C.EP_IMPL_REG, "tma": C.EP_IMPL_TMA, "auto": C.EP_IMPL_AUTO}
    mode_kw = {"fp8_fused": dict(use_fp8=True), "bf16": dict()}
    combos = []
    for impl in args.impls.split(","):
        for stg in ([int(s) for s in args.stages.split(",")] if impl == "tma" else [0]):
            for sms in [int(s) for s in args.sms.split(",")]:
                combos.append((impl, stg, sms))
    for impl, stg, sms in combos:
        cfg = Config(sms)
        buf.runtime.impl = impl_ids[impl]
        buf.runtime.set_stages(stg, stg, stg)
        tpr, _, tpe, in_rank, _ = buf.get_dispatch_layout(idx, E)
        for mode in args.modes.split(","):
            kw = mode_kw[mode]
            rx, ri, rw, pe, handle, _ = buf.dispatch(x, num_tokens_per_rank=tpr, is_token_in_rank=in_rank,
                                                     num_tokens_per_expert=tpe, topk_idx=idx, topk_weights=w,
                                                     config=cfg, **kw)
            nrecv = handle.num_recv
            d_avg, d_min = timed(lambda: buf.dispatch(x, handle=handle, config=cfg, **kw))
            row = {"impl": impl, "stages": stg, "sms": sms, "mode": mode, "num_recv": nrecv, "dispatch_us": d_avg, "dispatch_min_us": d_min,
                   "dispatch_GBps": nrecv * (H if mode != "bf16" else 2 * H) / (d_avg * 1e-6) / 1e9}
            if mode == "bf16":
                cin = buf.get_combine_buffer(nrecv, H, K)
                c_avg, c_min = timed(lambda: buf.combine(cin, handle, config=cfg))
                row.update({"combine_us": c_avg, "combine_min_us": c_min,
                            "combine_GBps": nrecv * 2 * H / (c_avg * 1e-6) / 1e9})
            rows.append(row)
            if rank == 0:
                print(json.dumps(row), flush=True)
    if args.ll:
        M = 128
        xl, il, wl = x[:M].contiguous(), idx[:M].contiguous(), w[:M].contiguous()
        for use_fp8 in (True, False):
            rx, rc, handle, _, _ = buf.low_latency_dispatch(xl, il, M, E, use_fp8=use_fp8)
            d_avg, d_min = timed(lambda: buf.low_latency_dispatch(xl, il, M, E, use_fp8=use_fp8))
            cb = buf.get_next_low_latency_combine_buffer(handle)
            c_avg, c_min = timed(lambda: buf.low_latency_combine(cb, il, wl, handle))
            # back-to-back pairs without the L2 flush and without host gaps between the ranks (how the reference times
            # its low-latency kernels: kineto kernel time over many iterations, ep/bench/test_low_latency.py)
            def pair():
                _, _, h2, _, _ = buf.low_latency_dispatch(xl, il, M, E, use_fp8=use_fp8)
                buf.low_latency_combine(buf.get_next_low_latency_combine_buffer(h2), il, wl, h2)

            for _ in range(5):
                pair()
            torch.cuda.synchronize()
            if n > 1:
                dist.barrier()
            s0, e0 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            for _ in range(50):
                pair()
            e0.record()
            torch.cuda.synchronize()
            pair_us = mx(s0.elapsed_time(e0) / 50) * 1e3
            row = {"ll": True, "use_fp8": use_fp8, "tokens": M, "dispatch_us": d_avg, "dispatch_min_us": d_min,
                   "combine_us": c_avg, "combine_min_us": c_min, "pair_back_to_back_us": pair_us}
            rows.append(row)
            if rank == 0:
                print(json.dumps(row), flush=True)
    if rank == 0 and args.out:
        with open(args.out, "w") as f:
            json.dump({"n_gpus": n, "tokens": T, "hidden": H, "topk": K, "experts": E, "rows": rows}, f, indent=1)
    if n > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
