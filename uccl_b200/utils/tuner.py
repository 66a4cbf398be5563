"""Measured algorithm selection for AllReduce.

The reference hard-codes its thresholds (experimental/lite/collective/algorithm_selector.cc:
71-101, "TODO: automatically tune" in ep/bench/buffer.py:691-703).  Here the table is measured:
`autotune_allreduce` times every applicable (algorithm, CTA count) per message size on the live
communicator -- device-timed, max over ranks -- installs the winners with
`Communicator.set_tuning`, and can persist them as JSON (`save_tuning` / `load_tuning`).
"""
from __future__ import annotations

import json
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import torch

DEFAULT_SIZES = [1 << s for s in range(10, 31, 2)]


def _timeit(fn, iters: int, sync) -> float:
    for _ in range(2):
        fn()
    sync()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def autotune_allreduce(comm, sizes: Sequence[int] = DEFAULT_SIZES, dtype: torch.dtype = torch.bfloat16,
                       cta_options: Iterable[int] = (16, 32, 64, 128), group=None, symmetric: bool = True,
                       install: bool = True) -> List[Tuple[int, str, int, float]]:
    """Returns [(max_bytes, algo, ctas, ms)] (one row per size) and installs it on `comm`.
    Must be called by every rank of the communicator (it runs collectives)."""
    import torch.distributed as dist

    use_dist = dist.is_available() and dist.is_initialized() and comm.world_size > 1

    def sync():
        torch.cuda.synchronize()
        if use_dist:
            dist.barrier(group=group)

    def max_over_ranks(v: float) -> float:
        if not use_dist:
            return v
        t = torch.tensor([v], dtype=torch.float64, device=comm.device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
        return float(t.item())

    es = torch.empty((), dtype=dtype).element_size()
    maxn = max(sizes) // es
    buf_in = comm.empty(maxn, dtype=dtype) if symmetric else torch.empty(maxn, dtype=dtype, device=comm.device)
    buf_out = comm.empty(maxn, dtype=dtype) if symmetric else torch.empty(maxn, dtype=dtype, device=comm.device)
    buf_in.fill_(1)
    from .. import _native

    ll_max = int(_native.C().LL_MAX_BYTES)
    table = []
    for size in sorted(sizes):
        n = size // es
        algos = []
        if size <= ll_max:
            algos += ["oneshot_ll"] + (["oneshot_mc"] if comm.has_multicast else [])
        if size % 16 == 0:
            if symmetric:
                algos += ["twoshot_p2p"] + (["twoshot_nvls"] if comm.has_multicast else [])
            else:
                algos += ["staged_p2p"] + (["staged_nvls"] if comm.has_multicast else [])
        best: Optional[Tuple[float, str, int]] = None
        iters = 20 if size <= (8 << 20) else 5
        for algo in algos:
            for ctas in cta_options:
                try:
                    ms = _timeit(lambda: comm.all_reduce(buf_in[:n], "sum", out=buf_out[:n], algo=algo, max_ctas=ctas),
                                 iters, sync)
                except RuntimeError:
                    continue
                ms = max_over_ranks(ms)
                if best is None or ms < best[0]:
                    best = (ms, algo, ctas)
                if algo.startswith("oneshot"):
                    break  # CTA count is derived from the size for the packet path
        if best is not None:
            table.append((size, best[1], best[2], best[0]))
    if install and table:
        comm.set_tuning(symmetric, [(mb, a, c) for mb, a, c, _ in table])
    return table


def save_tuning(path: str, tables: Dict[str, List[Tuple[int, str, int, float]]], meta: Optional[dict] = None) -> None:
    with open(path, "w") as f:
        json.dump({"meta": meta or {}, "tables": {k: [list(r) for r in v] for k, v in tables.items()}}, f, indent=1)


def load_tuning(comm, path: str) -> None:
    with open(path) as f:
        d = json.load(f)
    for key, rows in d.get("tables", {}).items():
        comm.set_tuning(key == "symmetric", [(int(r[0]), r[1], int(r[2])) for r in rows])


def tuning_from_sweep(sweep: dict) -> Dict[str, List[Tuple[int, str, int, float]]]:
    """Tables from the JSON that ``benchmarks/allreduce_perf.py`` writes (one row per message size with
    the device-timed latency of every algorithm, optionally ``algo@ctas`` columns): the fastest symmetric
    algorithm and the fastest plain-buffer algorithm per size.  CTA count -1 keeps the built-in choice."""
    sym_algos = ("oneshot_ll", "oneshot_mc", "twoshot_p2p", "twoshot_nvls")
    plain_algos = ("oneshot_ll", "oneshot_mc", "staged_p2p", "staged_nvls", "staged_pipe")
    out: Dict[str, List[Tuple[int, str, int, float]]] = {"symmetric": [], "plain": []}
    for row in sweep["rows"]:
        for key, cands in (("symmetric", sym_algos), ("plain", plain_algos)):
            best = None
            for col, v in row.items():
                if not isinstance(v, dict) or "us" not in v:
                    continue
                algo, _, ctas = col.partition("@")
                if algo not in cands:
                    continue
                if best is None or v["us"] < best[3]:
                    best = (int(row["bytes"]), algo, int(ctas) if ctas else -1, float(v["us"]))
            if best is not None:
                out[key].append(best)
    return out


def packaged_tuning_path(world_size: int) -> str:
    """Measured table shipped with the package for an N x H100 NVSwitch box (uccl_b200/tuning/)."""
    import os

    return os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tuning", f"tuning_{world_size}xH100.json")


def load_tuning_from_env(comm) -> bool:
    """Install the table named by ``UCCL_B200_TUNE_FILE`` (written by :func:`save_tuning`); without the variable the
    table measured on this box type for this world size (uccl_b200/tuning/tuning_<N>xH100.json) is used if it is
    shipped.  ``UCCL_B200_TUNE_FILE=none`` keeps the built-in thresholds of ``Comm::select_allreduce``."""
    import os

    path = os.environ.get("UCCL_B200_TUNE_FILE", "")
    if path.lower() in ("none", "off", "0"):
        return False
    if not path:
        path = packaged_tuning_path(comm.world_size)
        if comm.is_host or not os.path.exists(path):
            return False
    load_tuning(comm, path)
    return True
