#!/usr/bin/env python
"""all_reduce_rmsnorm (all-reduce + residual add + RMSNorm [+ fp8 cast]) at decode shapes of a tensor-parallel layer.

Arms, each timed with CUDA events around one replay of a CUDA graph of --iters calls (after --warmup eager calls),
max over ranks:
  fused    Communicator.all_reduce_rmsnorm (one kernel where the all-reduce runs one-shot)
  unfused  our all_reduce, then x + residual, torch.nn.functional.rms_norm [, per_token_cast_to_fp8]
  nccl     torch.distributed.all_reduce (NCCL), then the same torch tail

  torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 benchmarks/allreduce_rmsnorm_bench.py [--out f.json]

Run without torchrun it uses one GPU: there is no communication, so it times the epilogue kernel
(add_rmsnorm_kernel) against the torch tail and reports its achieved HBM bandwidth next to the H100 SXM data-sheet
3.35 TB/s.  Virtual ranks on one GPU are not timed here: their kernels share one GPU's SMs and HBM.

--mode sp times the sequence-parallel tail, reduce_scatter_rmsnorm, at prefill sizes (--tokens is the global T, a
multiple of the world size; every rank normalises T / n rows):
  fused    Communicator.reduce_scatter_rmsnorm (one kernel where the reduce-scatter runs the LL kernel)
  unfused  our reduce_scatter, then x + residual, torch.nn.functional.rms_norm [, per_token_cast_to_fp8]
  nccl     torch.distributed.reduce_scatter_tensor (NCCL), then the same torch tail
Each row records which path the fused arm took ("path": fused / unfused, from the LL limit).  It needs torchrun with
at least 2 ranks: on one GPU there is no communication to time, and --mode tp already times the epilogue kernel.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

from uccl_b200 import Communicator
from uccl_b200.ep.utils import per_token_cast_to_fp8

HBM_PEAK_GBPS = 3350.0  # H100 SXM data sheet


def card():
    name = torch.cuda.get_device_name()
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return {"gpu": name, "power_limit": power}


def epilogue_bytes(T, H, fp8):
    """HBM traffic of the epilogue: read x, residual, weight; write residual_out and out (+ scales)."""
    out = T * H + T * (H // 128) * 4 if fp8 else T * H * 2
    return 3 * T * H * 2 + H * 2 + out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--mode", choices=("tp", "sp"), default="tp",
                   help="tp: all_reduce_rmsnorm at decode shapes; sp: reduce_scatter_rmsnorm at prefill shapes")
    p.add_argument("--tokens", default=None, help="default 1,4,16,64,256 (tp) or 128,512,2048,8192 (sp, global T)")
    p.add_argument("--hidden", default="4096,7168,8192")
    p.add_argument("--iters", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--eps", type=float, default=1e-6)
    p.add_argument("--out", default=None)
    a = p.parse_args()
    if a.tokens is None:
        a.tokens = "128,512,2048,8192" if a.mode == "sp" else "1,4,16,64,256"
    if a.mode == "sp" and int(os.environ.get("WORLD_SIZE", "1")) < 2:
        sys.exit("--mode sp needs torchrun with at least 2 ranks: on one GPU there is no reduce-scatter to time")

    dist = None
    if "RANK" in os.environ:
        import torch.distributed as dist

        rank, n, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
        torch.cuda.set_device(local)
        dev = torch.device("cuda", local)
        dist.init_process_group("cpu:gloo,cuda:nccl", device_id=dev)
        comm = Communicator.from_torch_dist(None, heap_bytes=512 << 20, stage_bytes=64 << 20)
    else:
        rank, n = 0, 1
        torch.cuda.set_device(0)
        dev = torch.device("cuda", 0)
        comm = Communicator.local_world(1, devices=[0], heap_bytes=512 << 20, stage_bytes=64 << 20)[0]
    info = card()

    def mx(v):
        if dist is None:
            return v
        t = torch.tensor([v], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def timed(fn):
        # --iters calls captured in one CUDA graph: at these sizes enqueuing a call from Python takes longer than
        # the GPU takes to run it, and eager timing would measure the host
        for _ in range(a.warmup):
            fn()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(a.iters):
                fn()
        graph.replay()
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        graph.replay()
        e.record()
        torch.cuda.synchronize()
        return mx(s.elapsed_time(e) / a.iters) * 1e3

    rows = []
    g = torch.Generator(device="cpu").manual_seed(rank)

    def tail(x, res, w, H, fp8):
        r = x + res
        y = F.rms_norm(r, (H,), w, a.eps)
        return per_token_cast_to_fp8(y) if fp8 else y

    for H in [int(v) for v in a.hidden.split(",")]:
        w = (torch.rand(H, generator=g) + 0.5).to(torch.bfloat16).to(dev)
        if a.mode == "sp":
            for T in [int(v) for v in a.tokens.split(",")]:
                if T % n:
                    raise SystemExit(f"--tokens: {T} is not a multiple of the world size {n}")
                Tl = T // n
                x0 = torch.randn(T, H, generator=g).to(torch.bfloat16).to(dev) * 0.01
                res0 = torch.randn(Tl, H, generator=g).to(torch.bfloat16).to(dev)
                x, res = x0.clone(), res0.clone()
                xs = torch.empty(Tl, H, dtype=torch.bfloat16, device=dev)  # reduce-scatter output of the torch arms
                for fp8 in (False, True):
                    quant = "fp8" if fp8 else None
                    nbytes = Tl * H * 2  # one rank's piece
                    row = {"mode": "sp", "T": T, "rows_per_rank": Tl, "H": H, "fp8": fp8, "bytes_per_rank": nbytes,
                           "n_gpus": n, "path": "fused" if nbytes <= comm.reduce_scatter_ll_max() else "unfused"}
                    # x and residual are updated in place by every timed call; no arm's time depends on their values
                    row["fused_us"] = timed(lambda: comm.reduce_scatter_rmsnorm(x, res, w, a.eps, quant=quant))
                    row["unfused_us"] = timed(lambda: tail(comm.reduce_scatter(xs, x), res, w, H, fp8))
                    x.copy_(x0)
                    row["nccl_us"] = timed(lambda: (dist.reduce_scatter_tensor(xs, x), tail(xs, res, w, H, fp8)))
                    x.copy_(x0)
                    res.copy_(res0)
                    rows.append(row)
                    if rank == 0:
                        print(json.dumps(row), flush=True)
            continue
        for T in [int(v) for v in a.tokens.split(",")]:
            x0 = torch.randn(T, H, generator=g).to(torch.bfloat16).to(dev) * 0.01
            res0 = torch.randn(T, H, generator=g).to(torch.bfloat16).to(dev)
            x, res = x0.clone(), res0.clone()
            for fp8 in (False, True):
                quant = "fp8" if fp8 else None
                nbytes = T * H * 2
                row = {"T": T, "H": H, "fp8": fp8, "bytes": nbytes, "n_gpus": n}
                if n > 1:
                    row["fused_path"] = comm.select_allreduce(nbytes, comm.is_symmetric(x), torch.bfloat16)[0]

                # x and residual are updated in place by every timed call; no arm's time depends on their values
                row["fused_us"] = timed(lambda: comm.all_reduce_rmsnorm(x, res, w, a.eps, quant=quant))
                if n > 1:
                    row["unfused_us"] = timed(lambda: tail(comm.all_reduce(x, "sum"), res, w, H, fp8))
                    x.copy_(x0)
                    row["nccl_us"] = timed(lambda: (dist.all_reduce(x), tail(x, res, w, H, fp8)))
                else:
                    row["torch_tail_us"] = timed(lambda: tail(x, res, w, H, fp8))
                    row["epilogue_GBps"] = epilogue_bytes(T, H, fp8) / (row["fused_us"] * 1e-6) / 1e9
                    row["epilogue_share_of_hbm_peak"] = row["epilogue_GBps"] / HBM_PEAK_GBPS
                x.copy_(x0)
                res.copy_(res0)
                rows.append(row)
                if rank == 0:
                    print(json.dumps(row), flush=True)
    result = {"mode": a.mode, "n_gpus": n, "dtype": "bf16", "iters": a.iters, **info, "rows": rows}
    if rank == 0:
        print(json.dumps({"mode": a.mode, "n_gpus": n, **info, "shapes": len(rows)}), flush=True)
        if a.out:
            with open(a.out, "w") as f:
                json.dump(result, f, indent=1)
    if dist is not None:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
