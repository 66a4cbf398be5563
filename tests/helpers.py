"""Shared helpers for the tests: virtual ranks on one device (or real devices when the box has enough of
them), and the stored call signatures of the reference project."""
import functools
import json
import os
import threading

import torch

from uccl_b200 import Communicator

_WORLDS = {}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@functools.lru_cache(maxsize=None)
def reference_signatures():
    """Parameter names of the reference project's public Python / binding API (oracle/extract_signatures.py)."""
    with open(os.path.join(GOLDEN, "reference_signatures.json")) as f:
        return json.load(f)


def devices_for(n):
    ng = torch.cuda.device_count()
    return list(range(n)) if ng >= n else [0] * n


def get_world(n, heap_mb=256, stage_mb=8, max_ctas=4):
    """Cached local world of n ranks (heap creation is the slow part)."""
    key = (n, heap_mb, stage_mb, max_ctas)
    if key not in _WORLDS:
        _WORLDS[key] = Communicator.local_world(
            n, devices=devices_for(n), heap_bytes=heap_mb << 20, stage_bytes=stage_mb << 20, timeout_ms=5000,
            max_ctas=max_ctas)
    return _WORLDS[key]


def run_ranks(comms, prepare, launch):
    """prepare(c) -> state for every rank (may allocate / sync), then launch(c, state) for every
    rank on its own stream without any host synchronisation in between, then sync all."""
    states = []
    for c in comms:
        with torch.cuda.device(c.device):
            states.append(prepare(c))
    for c in comms:
        torch.cuda.synchronize(c.device)
    streams = [torch.cuda.Stream(device=c.device) for c in comms]
    for c, s, st in zip(comms, streams, states):
        with torch.cuda.device(c.device), torch.cuda.stream(s):
            launch(c, st)
    for s in streams:
        s.synchronize()
    return states


def run_host_ranks(comms, fn):
    out = [None] * len(comms)
    errs = []

    def w(c):
        try:
            out[c.rank] = fn(c)
        except Exception as e:  # pragma: no cover
            errs.append(e)

    ts = [threading.Thread(target=w, args=(c,)) for c in comms]
    [t.start() for t in ts]
    [t.join() for t in ts]
    if errs:
        raise errs[0]
    return out
