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

--mode ep times the tail of an expert-parallel MoE layer, ep.Buffer.combine_rmsnorm, with the routing of bench.py (top-8
of 256 experts, --tokens per rank, default 128,512,4096 at H = 7168), bf16 and fp8 out, and config.num_sms of 24 and of
every SM:
  fused    Buffer.combine_rmsnorm (one kernel)
  unfused  Buffer.combine, then add_rmsnorm_kernel (all_reduce_rmsnorm of a one-rank communicator)
  torch    Buffer.combine, then x + residual, torch.nn.functional.rms_norm [, per_token_cast_to_fp8]
Fused and unfused outputs are checked bitwise equal first.  The arms' graphs are replayed alternately --rounds times;
each row reports the median, min and max per call, the bytes moved (from shapes) and the achieved rate next to the
3.35 TB/s data sheet.  It runs on one GPU without torchrun (no NVLink traffic, HBM-bound) and under torchrun for n >= 2.

--mode ll times the tail of a decode MoE layer, ep.Buffer.low_latency_combine_rmsnorm, after a bf16 low_latency_dispatch
(top-8 of 256 experts, --tokens per rank, default 1,8,32,128, num_max_dispatch_tokens_per_rank 128, H = 7168) with a
shared-expert output, bf16 and fp8 out:
  fused    Buffer.low_latency_combine_rmsnorm (one kernel)
  unfused  Buffer.low_latency_combine, + shared, then add_rmsnorm_kernel (all_reduce_rmsnorm of a one-rank communicator)
  torch    Buffer.low_latency_combine, + shared + residual, torch.nn.functional.rms_norm [, per_token_cast_to_fp8]
Fused and unfused outputs are checked bitwise equal first; the graphs are replayed alternately as in --mode ep.  It runs
on one GPU without torchrun and under torchrun for n >= 2.
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


def combine_bytes(T, num_recv, H):
    """HBM traffic of Buffer.combine without bias: read the expert rows, write the combined rows."""
    return num_recv * H * 2 + T * H * 2


def ep_fused_bytes(T, num_recv, H, fp8):
    """combine_rmsnorm: read the expert rows, residual and weight; write residual_out and out (+ scales)."""
    return combine_bytes(T, num_recv, H) + epilogue_bytes(T, H, fp8) - 2 * T * H * 2


def run_ep(a, rank, n, dev, dist, info):
    """--mode ep: see the module docstring."""
    from uccl_b200.ep import Buffer, Config

    H, K, E = [int(v) for v in a.hidden.split(",")][0], 8, 256
    tokens = [int(v) for v in a.tokens.split(",")]
    T_max = max(tokens)
    nvl = Config().get_nvl_buffer_size_hint(H * 2, n, T_max, K)
    if dist is not None:
        comm = Communicator.from_torch_dist(None, heap_bytes=nvl + (256 << 20), stage_bytes=16 << 20)
    else:
        comm = Communicator.local_world(1, devices=[dev.index], heap_bytes=nvl + (256 << 20), stage_bytes=16 << 20)[0]
    buf = Buffer(comm=comm, num_nvl_bytes=nvl)
    one = Communicator.local_world(1, devices=[dev.index], heap_bytes=256 << 20, stage_bytes=8 << 20)[0]
    all_sms = torch.cuda.get_device_properties(dev).multi_processor_count
    g = torch.Generator(device="cpu").manual_seed(rank)
    w = (torch.rand(H, generator=g) + 0.5).to(torch.bfloat16).to(dev)
    rows = []

    for T in tokens:
        x = torch.randn(T, H, generator=g).to(torch.bfloat16).to(dev)
        idx = torch.rand(T, E, generator=g).topk(K, dim=1).indices.to(torch.int64).to(dev)
        tpr, _, tpe, in_rank, _ = buf.get_dispatch_layout(idx, E)
        recv_x, _, _, _, handle, _ = buf.dispatch(x, num_tokens_per_rank=tpr, is_token_in_rank=in_rank,
                                                  num_tokens_per_expert=tpe, topk_idx=idx)
        num_recv = recv_x.size(0)
        cb = buf.get_combine_buffer(num_recv, H)
        cb.copy_(recv_x)
        res = torch.randn(T, H, generator=g).to(torch.bfloat16).to(dev)
        torch.cuda.synchronize()
        for sms in (24, all_sms):
            cfg = Config(sms)
            for fp8 in (False, True):
                quant = "fp8" if fp8 else None
                ro_f, ro_u = torch.empty_like(res), torch.empty_like(res)  # residual stays the input of every call

                def fused():
                    return buf.combine_rmsnorm(cb, handle, res, w, a.eps, residual_out=ro_f, quant=quant, config=cfg)[0]

                def unfused():
                    c = buf.combine(cb, handle, config=cfg)[0]
                    return one.all_reduce_rmsnorm(c, res, w, a.eps, residual_out=ro_u, quant=quant)

                def torch_tail():
                    c = buf.combine(cb, handle, config=cfg)[0]
                    y = F.rms_norm(c + res, (H,), w, a.eps)
                    return per_token_cast_to_fp8(y) if fp8 else y

                yf, yu = fused(), unfused()
                torch.cuda.synchronize()
                same = torch.equal(ro_f, ro_u) and all(
                    torch.equal(p.view(torch.uint8), q.view(torch.uint8))
                    for p, q in zip(yf if fp8 else (yf,), yu if fp8 else (yu,)))
                if not same:
                    raise SystemExit(f"--mode ep: fused and unfused outputs differ (T={T}, num_sms={sms}, fp8={fp8})")
                graphs = {k: graph_of(fn, a) for k, fn in (("fused", fused), ("unfused", unfused), ("torch", torch_tail))}
                times = {k: [] for k in graphs}
                for _ in range(a.rounds):  # alternate the arms so drift and neighbours hit them alike
                    for k, gr in graphs.items():
                        times[k].append(replay_us(gr, a, dist, dev))
                del graphs
                row = {"mode": "ep", "T": T, "num_recv": num_recv, "H": H, "topk": K, "experts": E, "fp8": fp8,
                       "num_sms": sms, "n_gpus": n, "bitwise_fused_eq_unfused": same}
                for k, v in times.items():
                    v = sorted(v)
                    row[f"{k}_us"] = v[len(v) // 2]
                    row[f"{k}_us_min"], row[f"{k}_us_max"] = v[0], v[-1]
                row["fused_bytes"] = ep_fused_bytes(T, num_recv, H, fp8)
                row["unfused_bytes"] = combine_bytes(T, num_recv, H) + epilogue_bytes(T, H, fp8)
                for k in ("fused", "unfused"):
                    row[f"{k}_GBps"] = row[f"{k}_bytes"] / (row[f"{k}_us"] * 1e-6) / 1e9
                    row[f"{k}_share_of_hbm_peak"] = row[f"{k}_GBps"] / HBM_PEAK_GBPS
                row["speedup_vs_unfused"] = row["unfused_us"] / row["fused_us"]
                rows.append(row)
                if rank == 0:
                    print(json.dumps(row), flush=True)
    return rows


def ll_fused_bytes(T, routed_rows, H, fp8):
    """low_latency_combine_rmsnorm: read the routed expert rows, residual, shared and weight; write residual_out and
    out (+ scales)."""
    out = T * H + T * (H // 128) * 4 if fp8 else T * H * 2
    return routed_rows * H * 2 + 2 * T * H * 2 + H * 2 + T * H * 2 + out


def ll_unfused_bytes(T, routed_rows, H, fp8):
    """low_latency_combine (read the routed rows, write [T, H]), + shared (read 2, write 1), then the epilogue."""
    return routed_rows * H * 2 + T * H * 2 + 3 * T * H * 2 + epilogue_bytes(T, H, fp8)


def run_ll(a, rank, n, dev, dist, info):
    """--mode ll: see the module docstring."""
    from uccl_b200.ep import Buffer

    H, K, E, M = [int(v) for v in a.hidden.split(",")][0], 8, 256, 128
    tokens = [int(v) for v in a.tokens.split(",")]
    if max(tokens) > M:
        raise SystemExit(f"--mode ll: --tokens must be <= num_max_dispatch_tokens_per_rank {M}")
    ll = Buffer.get_low_latency_rdma_size_hint(M, H, n, E)
    if dist is not None:
        comm = Communicator.from_torch_dist(None, heap_bytes=ll + (256 << 20), stage_bytes=16 << 20)
    else:
        comm = Communicator.local_world(1, devices=[dev.index], heap_bytes=ll + (256 << 20), stage_bytes=16 << 20)[0]
    buf = Buffer(comm=comm, num_nvl_bytes=1 << 20, num_rdma_bytes=ll, low_latency_mode=True)
    one = Communicator.local_world(1, devices=[dev.index], heap_bytes=256 << 20, stage_bytes=8 << 20)[0]
    g = torch.Generator(device="cpu").manual_seed(rank)
    w = (torch.rand(H, generator=g) + 0.5).to(torch.bfloat16).to(dev)
    rows = []

    for T in tokens:
        x = torch.randn(T, H, generator=g).to(torch.bfloat16).to(dev)
        idx = torch.rand(T, E, generator=g).topk(K, dim=1).indices.to(torch.int64).to(dev)
        tw = torch.rand(T, K, generator=g).float().to(dev)
        rx, _, handle, _, _ = buf.low_latency_dispatch(x, idx, M, E, use_fp8=False)
        cb = buf.get_next_low_latency_combine_buffer(handle)
        cb.copy_(rx)
        res = torch.randn(T, H, generator=g).to(torch.bfloat16).to(dev)
        shared = torch.randn(T, H, generator=g).to(torch.bfloat16).to(dev)
        routed_rows = int((idx >= 0).sum())
        torch.cuda.synchronize()
        for fp8 in (False, True):
            quant = "fp8" if fp8 else None
            ro_f, ro_u = torch.empty_like(res), torch.empty_like(res)  # residual stays the input of every call

            def fused():
                return buf.low_latency_combine_rmsnorm(cb, idx, tw, handle, res, w, a.eps, shared=shared,
                                                       residual_out=ro_f, quant=quant)[0]

            def unfused():
                c = buf.low_latency_combine(cb, idx, tw, handle)[0]
                return one.all_reduce_rmsnorm(c + shared, res, w, a.eps, residual_out=ro_u, quant=quant)

            def torch_tail():
                c = buf.low_latency_combine(cb, idx, tw, handle)[0]
                y = F.rms_norm(c + shared + res, (H,), w, a.eps)
                return per_token_cast_to_fp8(y) if fp8 else y

            yf, yu = fused(), unfused()
            torch.cuda.synchronize()
            same = torch.equal(ro_f, ro_u) and all(
                torch.equal(p.view(torch.uint8), q.view(torch.uint8))
                for p, q in zip(yf if fp8 else (yf,), yu if fp8 else (yu,)))
            if not same:
                raise SystemExit(f"--mode ll: fused and unfused outputs differ (T={T}, fp8={fp8})")
            graphs = {k: graph_of(fn, a) for k, fn in (("fused", fused), ("unfused", unfused), ("torch", torch_tail))}
            times = {k: [] for k in graphs}
            for _ in range(a.rounds):  # alternate the arms so drift and neighbours hit them alike
                for k, gr in graphs.items():
                    times[k].append(replay_us(gr, a, dist, dev))
            del graphs
            row = {"mode": "ll", "T": T, "routed_rows": routed_rows, "H": H, "topk": K, "experts": E, "M": M,
                   "fp8": fp8, "n_gpus": n, "bitwise_fused_eq_unfused": same, **info}
            for k, v in times.items():
                v = sorted(v)
                row[f"{k}_us"] = v[len(v) // 2]
                row[f"{k}_us_min"], row[f"{k}_us_max"] = v[0], v[-1]
            row["fused_bytes"] = ll_fused_bytes(T, routed_rows, H, fp8)
            row["unfused_bytes"] = ll_unfused_bytes(T, routed_rows, H, fp8)
            row["speedup_vs_unfused"] = row["unfused_us"] / row["fused_us"]
            row["speedup_vs_torch"] = row["torch_us"] / row["fused_us"]
            rows.append(row)
            if rank == 0:
                print(json.dumps(row), flush=True)
    return rows


def mx(v, dist, dev):
    if dist is None:
        return v
    t = torch.tensor([v], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def graph_of(fn, a):
    """--iters calls of fn captured in one CUDA graph, after --warmup eager calls and one replay: at these sizes
    enqueuing a call from Python takes longer than the GPU takes to run it, and eager timing would measure the host."""
    for _ in range(a.warmup):
        fn()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(a.iters):
            fn()
    graph.replay()
    torch.cuda.synchronize()
    return graph


def replay_us(graph, a, dist, dev):
    """Microseconds per call of one replay of graph_of's graph, the slowest rank's."""
    if dist is not None:
        dist.barrier()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    graph.replay()
    e.record()
    torch.cuda.synchronize()
    return mx(s.elapsed_time(e) / a.iters * 1e3, dist, dev)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--mode", choices=("tp", "sp", "ep", "ll"), default="tp",
                   help="tp: all_reduce_rmsnorm at decode shapes; sp: reduce_scatter_rmsnorm at prefill shapes; "
                        "ep: ep.Buffer.combine_rmsnorm at bench.py's MoE routing; "
                        "ll: ep.Buffer.low_latency_combine_rmsnorm at decode shapes")
    p.add_argument("--tokens", default=None,
                   help="default 1,4,16,64,256 (tp), 128,512,2048,8192 (sp, global T), 128,512,4096 (ep, per rank) "
                        "or 1,8,32,128 (ll, per rank)")
    p.add_argument("--hidden", default=None, help="default 4096,7168,8192 (tp, sp) or 7168 (ep, ll: first value used)")
    p.add_argument("--rounds", type=int, default=5, help="ep, ll: alternating replays of each arm's graph")
    p.add_argument("--iters", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--eps", type=float, default=1e-6)
    p.add_argument("--out", default=None)
    a = p.parse_args()
    if a.tokens is None:
        a.tokens = {"sp": "128,512,2048,8192", "ep": "128,512,4096", "ll": "1,8,32,128"}.get(a.mode, "1,4,16,64,256")
    if a.hidden is None:
        a.hidden = "7168" if a.mode in ("ep", "ll") else "4096,7168,8192"
    if a.mode == "sp" and int(os.environ.get("WORLD_SIZE", "1")) < 2:
        sys.exit("--mode sp needs torchrun with at least 2 ranks: on one GPU there is no reduce-scatter to time")

    dist = None
    if "RANK" in os.environ:
        import torch.distributed as dist

        rank, n, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
        torch.cuda.set_device(local)
        dev = torch.device("cuda", local)
        dist.init_process_group("cpu:gloo,cuda:nccl", device_id=dev)
    else:
        rank, n = 0, 1
        torch.cuda.set_device(0)
        dev = torch.device("cuda", 0)
    info = card()
    if a.mode in ("ep", "ll"):
        rows = (run_ep if a.mode == "ep" else run_ll)(a, rank, n, dev, dist, info)
        if rank == 0:
            print(json.dumps({"mode": a.mode, "n_gpus": n, **info, "shapes": len(rows)}), flush=True)
            if a.out:
                with open(a.out, "w") as f:
                    json.dump({"mode": a.mode, "n_gpus": n, "dtype": "bf16", "iters": a.iters, "rounds": a.rounds,
                               **info, "rows": rows}, f, indent=1)
        if dist is not None:
            dist.barrier()
            dist.destroy_process_group()
        return
    if dist is not None:
        comm = Communicator.from_torch_dist(None, heap_bytes=512 << 20, stage_bytes=64 << 20)
    else:
        comm = Communicator.local_world(1, devices=[0], heap_bytes=512 << 20, stage_bytes=64 << 20)[0]

    def timed(fn):
        return replay_us(graph_of(fn, a), a, dist, dev)

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
