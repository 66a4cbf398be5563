#!/usr/bin/env python
"""profiles/allreduce_<N>.json (benchmarks/allreduce_perf.py --coll allreduce --out ...) -> uccl_b200/tuning/tuning_<N>xH100.json,
the table Communicator loads by default for that world size.  Only rows where the measured winner beats the
built-in choice by > 3 % are worth keeping, but the whole table is stored (it documents the sweep)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from uccl_b200.utils.tuner import save_tuning, tuning_from_sweep  # noqa: E402

for path in sys.argv[1:]:
    d = json.load(open(path))
    n = d["n_gpus"]
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "uccl_b200", "tuning", f"tuning_{n}xH100.json")
    save_tuning(out, tuning_from_sweep(d), {"source": os.path.basename(path), "n_gpus": n, "dtype": d.get("dtype"), "nvls": d.get("nvls")})
    print("wrote", out)
