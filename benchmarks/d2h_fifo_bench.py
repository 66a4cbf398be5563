"""GPU -> CPU command queue microbenchmark (role of the reference's ep/bench/fifo + ep/tests/*_bench.cu):
throughput with many producer threads and single-command round-trip latency.

    python benchmarks/d2h_fifo_bench.py [--capacity 4096]
"""
import argparse
import json

import torch

from uccl_b200 import Communicator
from uccl_b200.ep import Proxy


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--capacity", type=int, default=4096)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    comm = Communicator.local_world(1, devices=[0], heap_bytes=256 << 20, stage_bytes=8 << 20)[0]
    p = Proxy(comm, capacity=a.capacity)
    res = {"capacity": a.capacity, "throughput": [], "latency_us": None}
    with torch.cuda.device(comm.device):
        for blocks, threads in ((1, 32), (1, 256), (8, 256), (32, 256), (132, 256)):
            p.bench_throughput(blocks, threads, 16)  # warm-up
            r = p.bench_throughput(blocks, threads, 64)
            res["throughput"].append({"blocks": blocks, "threads": threads, "mcmd_per_s": r / 1e6})
            print(f"{blocks:4d} x {threads:3d} threads: {r / 1e6:8.2f} Mcmd/s")
        p.bench_latency(100)
        res["latency_us"] = p.bench_latency(2000)
        print(f"round trip: {res['latency_us']:.2f} us")
    res["proxy"] = p.stats()
    p.stop()
    if a.out:
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
