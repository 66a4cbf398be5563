#!/usr/bin/env python
"""nccl-tests-style sweep (all_reduce_perf / all_gather_perf / reduce_scatter_perf): 1 KB - 1 GB,
device-timed, max over ranks, our kernels (every applicable algorithm) next to NCCL on the same box.

  torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 benchmarks/allreduce_perf.py [--coll allreduce]

Reference scripts: collective/rdma/run_nccl_test.sh:95-98 (-b 1K -e 1G -f 2), experimental/lite/
scripts/run-nccl-tests.sh.  Output: a table on stdout + JSON rows in --out.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

from uccl_b200 import Communicator


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--coll", default="allreduce", choices=["allreduce", "allgather", "reduce_scatter", "alltoall", "broadcast"])
    # (--min-bytes / --max-bytes: torchrun's own parser swallows an unambiguous-prefix-less "--max" as --max-restarts)
    p.add_argument("--min", "--min-bytes", dest="min", type=int, default=1 << 10)
    p.add_argument("--max", "--max-bytes", dest="max", type=int, default=1 << 30)
    p.add_argument("--factor", type=int, default=4)
    p.add_argument("--dtype", default="bf16")
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--ctas", default="", help="comma list of CTA counts to sweep (allreduce)")
    p.add_argument("--out", default=None)
    args = p.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("cpu:gloo,cuda:nccl", device_id=dev)
    dt = {"bf16": torch.bfloat16, "fp32": torch.float32, "fp16": torch.float16}[args.dtype]
    es = torch.empty((), dtype=dt).element_size()
    comm = Communicator.from_torch_dist(heap_bytes=(6 << 30), stage_bytes=256 << 20, max_ctas=132)
    n = world
    big_in = comm.empty(args.max // es, dtype=dt)
    big_out = comm.empty(args.max // es, dtype=dt)
    plain_in = torch.ones(args.max // es, dtype=dt, device=dev)
    plain_out = torch.ones(args.max // es, dtype=dt, device=dev)
    big_in.fill_(1)

    def timeit(fn, iters):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        dist.barrier()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        t = torch.tensor([s.elapsed_time(e) / iters], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return t.item()

    def ll_variants(row, fn, per, tot, f, iters):
        """the same call with the LL-packet exchange forced off / forced on (threshold tuning data)"""
        if per * es > (1 << 20) or (per * es) % 16:
            return
        for name, v in (("plain_noll", -1), ("plain_ll", 1 << 20)):
            comm.set_xchg_ll_max(v)
            ms = timeit(fn, iters)
            row[name] = {"us": ms * 1e3, "busbw": tot / (ms * 1e-3) * f / 1e9}
        comm.set_xchg_ll_max(0)

    rows = []
    size = args.min
    cta_list = [int(c) for c in args.ctas.split(",") if c] or [-1]
    while size <= args.max:
        cnt = size // es
        iters = args.iters if size <= (16 << 20) else max(3, args.iters // 4)
        row = {"bytes": size}
        if args.coll == "allreduce":
            f = 2 * (n - 1) / n
            variants = []
            if size <= (256 << 10):
                variants += [("oneshot_ll", True)] + ([("oneshot_mc", True)] if comm.has_multicast else [])
            variants += [("twoshot_p2p", True)] + ([("twoshot_nvls", True)] if comm.has_multicast else [])
            variants += [("staged_p2p", False)] + ([("staged_nvls", False)] if comm.has_multicast else [])
            if comm.has_multicast and n > 2 and size >= (32 << 20) and size % 16 == 0:
                variants += [("staged_pipe", False)]
            for algo, sym in variants:
                for ctas in cta_list:
                    src = big_in if sym else plain_in
                    dst = big_out if sym else plain_out
                    if algo.startswith("oneshot"):
                        fn = lambda: comm.all_reduce(src[:cnt], "sum", out=dst[:cnt], algo=algo, max_ctas=ctas)
                    else:
                        if size % 16:
                            continue
                        fn = lambda: comm.all_reduce(src[:cnt], "sum", out=dst[:cnt], algo=algo, max_ctas=ctas)
                    ms = timeit(fn, iters)
                    key = algo if ctas < 0 else f"{algo}@{ctas}"
                    row[key] = {"us": ms * 1e3, "busbw": size / (ms * 1e-3) * f / 1e9}
            ms = timeit(lambda: comm.all_reduce(big_in[:cnt], "sum", out=big_out[:cnt]), iters)
            row["auto_sym"] = {"us": ms * 1e3, "busbw": size / (ms * 1e-3) * f / 1e9,
                               "algo": comm.select_allreduce(size, True, dt)[0]}
            ms = timeit(lambda: dist.all_reduce(plain_in[:cnt]), iters)
            row["nccl"] = {"us": ms * 1e3, "busbw": size / (ms * 1e-3) * f / 1e9}
        elif args.coll == "allgather":
            per = max(cnt // n, 1)
            f = (n - 1) / n
            tot = per * n * es
            for name, i_, o_ in (("sym_out", plain_in, big_out), ("sym_in", big_in, plain_out), ("plain", plain_in, plain_out)):
                ms = timeit(lambda: comm.all_gather(o_[:per * n], i_[:per]), iters)
                row[name] = {"us": ms * 1e3, "busbw": tot / (ms * 1e-3) * f / 1e9}
            ll_variants(row, lambda: comm.all_gather(plain_out[:per * n], plain_in[:per]), per, tot, f, iters)
            ms = timeit(lambda: dist.all_gather_into_tensor(plain_out[:per * n], plain_in[:per]), iters)
            row["nccl"] = {"us": ms * 1e3, "busbw": tot / (ms * 1e-3) * f / 1e9}
        elif args.coll == "reduce_scatter":
            per = max(cnt // n, 1)
            f = (n - 1) / n
            tot = per * n * es
            for name, i_ in (("sym_in", big_in), ("plain", plain_in)):
                ms = timeit(lambda: comm.reduce_scatter(plain_out[:per], i_[:per * n], "sum"), iters)
                row[name] = {"us": ms * 1e3, "busbw": tot / (ms * 1e-3) * f / 1e9}
            ll_variants(row, lambda: comm.reduce_scatter(plain_out[:per], plain_in[:per * n], "sum"), per, tot, f, iters)
            ms = timeit(lambda: dist.reduce_scatter_tensor(plain_out[:per], plain_in[:per * n]), iters)
            row["nccl"] = {"us": ms * 1e3, "busbw": tot / (ms * 1e-3) * f / 1e9}
        elif args.coll == "alltoall":
            per = max(cnt // n, 1)
            f = (n - 1) / n
            tot = per * n * es
            for name, i_, o_ in (("sym_out", plain_in, big_out), ("sym_in", big_in, plain_out), ("plain", plain_in, plain_out)):
                ms = timeit(lambda: comm.all_to_all(o_[:per * n], i_[:per * n]), iters)
                row[name] = {"us": ms * 1e3, "busbw": tot / (ms * 1e-3) * f / 1e9}
            ll_variants(row, lambda: comm.all_to_all(plain_out[:per * n], plain_in[:per * n]), per, tot, f, iters)
            ms = timeit(lambda: dist.all_to_all_single(plain_out[:per * n], plain_in[:per * n]), iters)
            row["nccl"] = {"us": ms * 1e3, "busbw": tot / (ms * 1e-3) * f / 1e9}
        else:
            f = 1.0
            for name, t_ in (("sym", big_out), ("plain", plain_out)):
                ms = timeit(lambda: comm.broadcast(t_[:cnt], root=0), iters)
                row[name] = {"us": ms * 1e3, "busbw": size / (ms * 1e-3) * f / 1e9}
            ms = timeit(lambda: dist.broadcast(plain_out[:cnt], src=0), iters)
            row["nccl"] = {"us": ms * 1e3, "busbw": size / (ms * 1e-3) * f / 1e9}
        rows.append(row)
        if rank == 0:
            cols = " | ".join(f"{k}: {v['us']:9.1f}us {v['busbw']:7.1f}GB/s" for k, v in row.items() if isinstance(v, dict))
            print(f"{size:>11d} B | {cols}", flush=True)
        size *= args.factor
    if rank == 0 and args.out:
        with open(args.out, "w") as fjson:
            json.dump({"coll": args.coll, "n_gpus": n, "dtype": args.dtype, "nvls": comm.has_multicast, "rows": rows}, fjson, indent=1)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
