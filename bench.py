#!/usr/bin/env python
"""Headline benchmark (BASELINE.json): EP dispatch+combine at EP=N on N H100s of one node, the
reference's DeepEP-intranode config (4096 tokens/rank, hidden 7168, top-8 of 256 experts,
bf16 -> fp8 dispatch, bf16 combine), plus an AllReduce bus-bandwidth sweep next to NCCL.

Usage:  python bench.py --gpus N --steps K --warmup W [--dump-outputs DIR]   (torchrun for N > 1)
prints ONE JSON line on rank 0.  `value` = whole-job tokens/s through dispatch+combine
(weak scaling: 4096 tokens per GPU), device-timed with CUDA events, max over ranks.

A "step" = one dispatch (payload + fused fp8 cast + metadata, cached layout handle -- the same
thing the reference times, ep/bench/test_intranode.py:457-539) followed by one combine.
The e2e number runs the whole public API per step: pinned-host -> device copy of the inputs,
get_dispatch_layout, non-cached dispatch (incl. the count exchange and its CPU sync), combine,
and a device -> host read of the result checksum.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import threading

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

BASELINE_DISPATCH_US = 500.0  # the reference's ep/README.md, intranode (8xH200, EP=8, FP8 dispatch)
BASELINE_COMBINE_US = 973.0   # the reference's ep/README.md, intranode (8xH200, EP=8, BF16 combine)
DUMP_BYTES = 60 << 20         # cap of what --dump-outputs writes (a seeded sample of rows when the outputs are larger)


def parse_args():
    p = argparse.ArgumentParser()
    p.add_argument("--gpus", type=int, default=1)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--impl", default="ours", choices=["ours", "reference"])
    p.add_argument("--metric", default="ep", choices=["ep", "allreduce"])
    p.add_argument("--no-graph", action="store_true", help="launch the timed steps eagerly instead of replaying CUDA graphs")
    p.add_argument("--tokens", type=int, default=4096)
    p.add_argument("--hidden", type=int, default=7168)
    p.add_argument("--topk", type=int, default=8)
    p.add_argument("--experts", type=int, default=256)
    p.add_argument("--num-sms", type=int, default=int(os.environ.get("UCCL_B200_EP_SMS", "0")),
                   help="CTAs per EP kernel of the headline (0: every SM at 1 GPU, else 24 = the reference's budget)")
    p.add_argument("--no-allreduce-sweep", action="store_true")
    p.add_argument("--no-sm-sweep", action="store_true", help="only time the headline SM budget")
    p.add_argument("--out", default=None, help="also write the JSON line to this file")
    p.add_argument("--dump-outputs", default=None, metavar="DIR",
                   help="write the arrays the last timed step returned (rank 0) as DIR/<name>.npy")
    return p.parse_args()


# ------------------------------------------------------------------------------ clocks
class ClockSampler:
    """Samples SM clock + throttle reasons of this rank's GPU during the timed region (NVML)."""

    def __init__(self, index: int):
        self.index = index
        self.samples = []
        self.reasons = set()
        self.max_mhz = None
        self._stop = threading.Event()
        self._t = None
        self._ok = False
        try:
            import pynvml

            pynvml.nvmlInit()
            self._nv = pynvml
            self._h = pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = pynvml.nvmlDeviceGetMaxClockInfo(self._h, pynvml.NVML_CLOCK_SM)
            self._ok = True
        except Exception:
            self._ok = False

    def _run(self):
        nv = self._nv
        names = {
            "hw_slowdown": getattr(nv, "nvmlClocksThrottleReasonHwSlowdown", 0x8),
            "hw_thermal_slowdown": getattr(nv, "nvmlClocksThrottleReasonHwThermalSlowdown", 0x40),
            "sw_thermal_slowdown": getattr(nv, "nvmlClocksThrottleReasonSwThermalSlowdown", 0x20),
            "sw_power_cap": getattr(nv, "nvmlClocksThrottleReasonSwPowerCap", 0x4),
            "hw_power_brake": getattr(nv, "nvmlClocksThrottleReasonHwPowerBrakeSlowdown", 0x80),
        }
        while not self._stop.is_set():
            try:
                self.samples.append(nv.nvmlDeviceGetClockInfo(self._h, nv.NVML_CLOCK_SM))
                try:
                    r = nv.nvmlDeviceGetCurrentClocksEventReasons(self._h)
                except Exception:
                    r = nv.nvmlDeviceGetCurrentClocksThrottleReasons(self._h)
                for k, bit in names.items():
                    if r & bit:
                        self.reasons.add(k)
            except Exception:
                pass
            self._stop.wait(0.05)

    def start(self):
        if self._ok:
            self._t = threading.Thread(target=self._run, daemon=True)
            self._t.start()

    def stop(self):
        self._stop.set()
        if self._t:
            self._t.join(1.0)
        if not self._ok or not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": self.max_mhz, "reasons": ["unavailable"]}
        return {"sm_mhz": statistics.median(self.samples), "sm_max_mhz": self.max_mhz,
                "reasons": sorted(self.reasons)}


# --------------------------------------------------------------------------- reference
def run_reference(args):
    """The unmodified reference from oracle/_ref through its own public API.  For the EP
    metric that is `uccl.ep.Buffer`, a native module the offline install cannot build (needs
    nanobind + libibverbs headers + its docker toolchain) -- see DESIGN.md."""
    ref = os.path.join(os.path.dirname(os.path.abspath(__file__)), "oracle", "_ref")
    rank = int(os.environ.get("RANK", "0"))
    if args.metric == "ep":
        why = None
        if not os.path.isdir(os.path.join(ref, "uccl")):
            why = "oracle/_ref/uccl not installed"
        else:
            sys.path.insert(0, ref)
            try:
                import uccl  # noqa: F401
                from uccl import ep as ref_ep  # noqa: F401
            except Exception as e:  # ImportError: native ep module absent
                why = ("reference installs offline only as a pure-python stub: uccl.ep native module missing "
                       f"(needs nanobind/libibverbs to build): {type(e).__name__}: {e}")
        if why is None:
            # the native module imported: run the reference's own DeepEP-style Buffer (ep/bench/buffer.py)
            try:
                return run_reference_ep(args, ref)
            except Exception as e:  # noqa: BLE001
                why = f"uccl.ep imported but its intranode bench failed: {type(e).__name__}: {e}"
        out = {"impl": "reference", "unavailable": why[:300]}
        # labelled DIAGNOSTIC (not the reference arm): the upstream DeepEP kernels the reference vendors and
        # re-hosts as its intranode path, built from oracle/_ref/deepep, same config, num_sms = 24
        diag = None
        if args.gpus >= 2:
            # watchdog: a diagnostic must never hang the reference arm (the JSON line above is what the driver needs)
            import signal

            def _give_up(signum, frame):
                if rank == 0:
                    out["diagnostic"] = {"vendored_upstream_deepep_intranode": {"unavailable": "timed out after 300 s"}}
                    emit(out)
                os._exit(0)

            signal.signal(signal.SIGALRM, _give_up)
            signal.alarm(300)
            try:
                sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "benchmarks"))
                import deepep_baseline

                if deepep_baseline.available() is None:
                    import torch
                    import torch.distributed as dist

                    local = int(os.environ.get("LOCAL_RANK", "0"))
                    torch.cuda.set_device(local)
                    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
                    diag = deepep_baseline.run(args.tokens, args.hidden, args.topk, args.experts, 24,
                                               iters=max(5, min(args.steps, 20)), quiet=True)
                    dist.barrier()
                    dist.destroy_process_group()
                else:
                    diag = {"unavailable": deepep_baseline.available()}
            except Exception as e:  # noqa: BLE001
                diag = {"unavailable": f"{type(e).__name__}: {e}"[:300]}
        if args.gpus >= 2:
            signal.alarm(0)
        if diag is not None:
            out["diagnostic"] = {"vendored_upstream_deepep_intranode": diag}
        if rank == 0:
            emit(out)
        return 0
    # allreduce: the reference's collective product is stock NCCL + its net plugin
    # (README.md:109-119); on one NVSwitch node no byte reaches the plugin, so this arm is NCCL
    # launched the way the reference documents (NCCL_NET_PLUGIN from uccl.nccl_plugin_path()).
    import torch
    import torch.distributed as dist

    sys.path.insert(0, ref)
    try:
        import uccl

        plugin = uccl.nccl_plugin_path()
        if os.path.exists(plugin):
            os.environ["NCCL_NET_PLUGIN"] = plugin
    except Exception:
        pass
    n = args.gpus
    if n == 1:
        if rank == 0:
            emit({"impl": "reference", "unavailable": "allreduce bus bandwidth is undefined at 1 GPU"})
        return 0
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    size = 1 << 30
    x = torch.ones(size // 2, dtype=torch.bfloat16, device="cuda")
    for _ in range(max(args.warmup, 3)):
        dist.all_reduce(x)
    torch.cuda.synchronize()
    dist.barrier()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(args.steps):
        dist.all_reduce(x)
    e.record()
    torch.cuda.synchronize()
    ms = torch.tensor([s.elapsed_time(e) / args.steps], device="cuda")
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    busbw = size / (ms.item() * 1e-3) * 2 * (n - 1) / n / 1e9
    if rank == 0:
        emit({"impl": "reference", "metric": "allreduce_busbw_1GiB_bf16", "value": busbw, "unit": "GB/s",
              "n_gpus": n, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms.item(),
              "higher_is_better": True, "dtype": "bf16", "data": "synthetic"})
    dist.destroy_process_group()
    return 0


def run_reference_ep(args, ref):
    """The reference's own EP path (only reachable where `uccl.ep` builds: nanobind + libibverbs): its
    DeepEP-compatible Buffer from ep/bench/buffer.py, cached-handle fp8 dispatch + bf16 combine at its
    default SM budget, timed like our arm."""
    import torch
    import torch.distributed as dist

    sys.path.insert(0, os.path.join(ref, "uccl", "ep_bench"))
    from buffer import Buffer as RefBuffer  # type: ignore
    from utils import per_token_cast_to_fp8 as ref_cast  # type: ignore

    n = args.gpus
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    T, H, K, E = args.tokens, args.hidden, args.topk, args.experts
    buf = RefBuffer(dist.group.WORLD, int(2e9), 0)
    g = torch.Generator(device="cpu").manual_seed(1234 + rank)
    x = torch.randn(T, H, generator=g).to(torch.bfloat16).to(dev)
    scores = torch.randn(T, E, generator=g).abs() + 1
    idx = scores.topk(K, dim=-1, largest=True, sorted=False).indices.to(torch.int64).contiguous().to(dev)
    w = torch.rand(T, K, generator=g).float().to(dev)
    tpr, _, tpe, in_rank, _ = buf.get_dispatch_layout(idx, E)
    x8 = ref_cast(x)
    rx, _, _, _, handle, _ = buf.dispatch(x, num_tokens_per_rank=tpr, is_token_in_rank=in_rank,
                                          num_tokens_per_expert=tpe, topk_idx=idx, topk_weights=w)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def step():
        buf.dispatch(x8, handle=handle)
        buf.combine(rx, handle)

    for _ in range(max(args.warmup, 3)):
        step()
    torch.cuda.synchronize()
    dist.barrier()
    evs = []
    for _ in range(args.steps):
        flush.zero_()
        s0, e0 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s0.record()
        step()
        e0.record()
        evs.append((s0, e0))
    torch.cuda.synchronize()
    ms = torch.tensor([sum(a.elapsed_time(b) for a, b in evs) / len(evs)], device=dev)
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    if rank == 0:
        emit({"impl": "reference", "metric": "ep_dispatch_combine_tokens_per_s", "value": n * T / (ms.item() * 1e-3),
              "unit": "tokens/s", "n_gpus": n, "steps": args.steps, "warmup": max(args.warmup, 3),
              "ms_per_step": ms.item(), "higher_is_better": True, "scaling": "weak", "dtype": "bf16",
              "data": "synthetic"})
    dist.barrier()
    dist.destroy_process_group()
    return 0


# ------------------------------------------------------------------------------- ours
_RESULT_OUT = None


def _claim_stdout():
    """Keep stdout for the ONE JSON result line: libraries (e.g. the "NCCL version ..." banner) print to
    fd 1 too, so fd 1 is pointed at stderr for the rest of the run and the result goes to a saved copy."""
    global _RESULT_OUT
    if _RESULT_OUT is None:
        sys.stdout.flush()
        _RESULT_OUT = os.fdopen(os.dup(1), "w")
        os.dup2(2, 1)
    return _RESULT_OUT


def emit(obj) -> None:
    out = _claim_stdout()
    out.write((obj if isinstance(obj, str) else json.dumps(obj)) + "\n")
    out.flush()


def main():
    args = parse_args()
    _claim_stdout()
    if args.impl == "reference":
        return run_reference(args)

    import torch

    from uccl_b200 import Communicator
    from uccl_b200.ep import Buffer

    n = args.gpus
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    assert torch.cuda.is_available(), "bench.py needs a GPU"
    dist = None
    if n > 1:
        assert world == n, f"launch with torchrun --nproc-per-node {n} (WORLD_SIZE={world})"
        import torch.distributed as dist  # type: ignore

        torch.cuda.set_device(local)
        dist.init_process_group("cpu:gloo,cuda:nccl", device_id=torch.device("cuda", local))
    else:
        torch.cuda.set_device(0)
    dev = torch.device("cuda", torch.cuda.current_device())

    T, H, K, E = args.tokens, args.hidden, args.topk, args.experts
    assert E % n == 0
    # worst case: every token of every rank lands on one rank
    cap_tokens = n * T
    arena = cap_tokens * (H * 2 + K * 4) + (1 << 20)
    nvl_bytes = 3 * arena + (2 << 20)
    heap = nvl_bytes + (1 << 30) + (2 << 30 if n > 1 else 0)
    if n > 1:
        comm = Communicator.from_torch_dist(None, heap_bytes=heap, stage_bytes=256 << 20)
    else:
        comm = Communicator.local_world(1, devices=[dev.index], heap_bytes=heap, stage_bytes=64 << 20)[0]
    buf = Buffer(comm=comm, num_nvl_bytes=nvl_bytes)
    from uccl_b200.ep import Config

    # SM budget of the headline: the reference publishes its numbers at 24 SMs (ep/bench/test_intranode.py:571)
    # so that expert GEMMs can run beside the communication kernels -- the same budget is the default here for
    # N > 1 (like for like); other budgets are measured too and reported under "sm_sweep" / "best".  At N = 1
    # nothing crosses NVLink (a pure HBM permutation) and the whole GPU is used: one CTA per SM, because the
    # TMA pipelines fill an SM's shared memory and more CTAs than SMs would run in two waves.
    head_sms = args.num_sms if args.num_sms > 0 else (torch.cuda.get_device_properties(dev).multi_processor_count
                                                      if n == 1 else 24)
    cfg = Config(head_sms)

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()

    def max_over_ranks(v: float) -> float:
        if dist is None:
            return v
        t = torch.tensor([v], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    # synthetic inputs (random-init MoE tokens; routing = top-k of |N(0,1)|+1 scores like the reference test)
    g = torch.Generator(device="cpu").manual_seed(1234 + rank)
    x_host = torch.randn(T, H, generator=g).to(torch.bfloat16).pin_memory()
    scores = torch.randn(T, E, generator=g).abs() + 1
    idx_host = scores.topk(K, dim=-1, largest=True, sorted=False).indices.to(torch.int64).contiguous().pin_memory()
    w_host = torch.rand(T, K, generator=g).float().pin_memory()
    x = x_host.to(dev, non_blocking=True)
    topk_idx = idx_host.to(dev, non_blocking=True)
    topk_w = w_host.to(dev, non_blocking=True)
    torch.cuda.synchronize()

    # one full (non-cached) round to obtain the handle used by the kernel-timed loop
    tpr, _, tpe, in_rank, _ = buf.get_dispatch_layout(topk_idx, E)
    recv_x, recv_idx, recv_w, per_expert, handle, _ = buf.dispatch(
        x, num_tokens_per_rank=tpr, is_token_in_rank=in_rank, num_tokens_per_expert=tpe, topk_idx=topk_idx,
        topk_weights=topk_w, use_fp8=True, config=cfg)
    num_recv = handle.num_recv
    # ---- correctness on THIS world before anything is timed: identity experts through the same kernels must give
    #      back every token multiplied by the number of ranks it was routed to (bit-exact: fp32 sum, one bf16 rounding);
    #      the fused-fp8 dispatch must dequantise to the same rows within e4m3 tolerance
    vx, _, _, _, vh, _ = buf.dispatch(x, num_tokens_per_rank=tpr, is_token_in_rank=in_rank, num_tokens_per_expert=tpe,
                                      topk_idx=topk_idx, topk_weights=topk_w, config=cfg)
    vin = buf.get_combine_buffer(vh.num_recv, H, K)
    vin.copy_(vx)
    vout, _, _ = buf.combine(vin, vh, config=cfg)
    fan = in_rank.sum(dim=1, keepdim=True).to(torch.float32)
    ok_bf16 = bool(torch.equal(vout, (x.float() * fan).to(torch.bfloat16)))  # fp32 sum of f equal values, one rounding
    q8, sc8 = recv_x
    deq = (q8[: min(num_recv, 2048)].float().view(-1, H // 128, 128) * sc8[: min(num_recv, 2048)].unsqueeze(2)).view(-1, H)
    src_rows = vx[: deq.size(0)].float()  # same arena order: bf16 dispatch of the same routing
    ok_fp8 = bool(torch.allclose(deq, src_rows, rtol=0.07, atol=0.05))
    verified = torch.tensor([1 if (ok_bf16 and ok_fp8) else 0], device=dev)
    if dist is not None:
        dist.all_reduce(verified, op=dist.ReduceOp.MIN)
    assert int(verified.item()) == 1, f"EP dispatch/combine verification failed on rank {rank}: bf16 {ok_bf16}, fp8 {ok_fp8}"
    comb_in = buf.get_combine_buffer(num_recv, H, K)
    # stand-in for the expert MLP output (bf16), lives in the symmetric arena; seeded so that every run combines
    # the same values
    comb_in.normal_(generator=torch.Generator(device=dev).manual_seed(4321 + rank))
    barrier()

    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    impl_name = {1: "register", 2: "tma"}

    def launches():
        return int(buf.runtime.launches) + int(comm.native.launches)

    def measure(num_sms: int, steps: int, warm: int, sample_clocks: bool = False):
        """Times `steps` (dispatch + combine) steps at one SM budget: CUDA events around every step on the
        launching stream, 256 MiB L2 flush write between steps (untimed), max over ranks.  Also returns what the
        last step gave back to the caller: (dispatched fp8 rows, their scales, combined rows)."""
        c = Config(num_sms)

        def step_cached():
            buf.dispatch(x, handle=handle, use_fp8=True, config=c)
            buf.combine(comb_in, handle, config=c)

        for _ in range(warm):
            step_cached()
        barrier()
        # ---- the step is launch-bound at small N (two short kernels per step, ~0.5 ms of Python per call):
        # capture dispatch and combine into CUDA graphs so the timed region measures the GPU, not the
        # interpreter (the kernels keep their cross-rank epochs on the device, so replays are safe).
        graphs = None
        outs = None
        per_step_launches = 2
        if not args.no_graph:
            try:
                l_before = launches()
                g_d, g_c = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
                with torch.cuda.graph(g_d):
                    d_out = buf.dispatch(x, handle=handle, use_fp8=True, config=c)
                with torch.cuda.graph(g_c):
                    c_out = buf.combine(comb_in, handle, config=c)
                outs = (d_out, c_out)  # a replay rewrites these tensors in place
                per_step_launches = launches() - l_before
                graphs = (g_d, g_c)
            except Exception as exc:  # pragma: no cover - fall back to eager launches
                if rank == 0:
                    print(f"[bench] CUDA graph capture unavailable ({type(exc).__name__}: {exc}); eager launches",
                          file=sys.stderr)
                graphs = None
                torch.cuda.synchronize()
        use_graph = torch.tensor([1 if graphs is not None else 0], device=dev)
        if dist is not None:
            dist.all_reduce(use_graph, op=dist.ReduceOp.MIN)  # every rank must take the same path
        if int(use_graph.item()) == 0:
            graphs = None
        if graphs is not None:
            for _ in range(3):
                graphs[0].replay()
                graphs[1].replay()
        barrier()
        sampler = ClockSampler(dev.index) if sample_clocks else None
        starts = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
        mids = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
        ends = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
        # Enqueuing a step costs the host more than the GPU needs to run it (flush + dispatch + combine), so a GPU fed
        # step by step would idle inside the timed events waiting for the next launch.  A device-side sleep in front
        # lets the host queue the timed steps ahead of the GPU: the events then time GPU work only.
        torch.cuda._sleep(int(steps * (0.4e-3 if graphs is not None else 2e-3) * 2e9))  # cycles at <= 2 GHz
        # The host-side barrier above releases the ranks up to ~1 ms apart; without re-aligning the GPUs the
        # first timed dispatch would absorb that skew in its cross-rank entry barrier.  A device-side
        # barrier kernel (untimed) lines the GPUs up to within microseconds.
        comm.barrier()
        l0 = launches()
        if sampler:
            sampler.start()
        for i in range(steps):
            flush.zero_()
            starts[i].record()
            if graphs is not None:
                graphs[0].replay()
                mids[i].record()
                graphs[1].replay()
            else:
                d_out = buf.dispatch(x, handle=handle, use_fp8=True, config=c)
                mids[i].record()
                c_out = buf.combine(comb_in, handle, config=c)
                outs = (d_out, c_out)
            ends[i].record()
        barrier()
        wall = starts[0].elapsed_time(ends[-1]) * 1e-3  # first step's start to last step's end, on the device
        clocks = sampler.stop() if sampler else None
        step_ms = [s.elapsed_time(e) for s, e in zip(starts, ends)]
        r = {
            "num_sms": num_sms,
            "ms_per_step": max_over_ranks(sum(step_ms) / len(step_ms)),
            # split of the same timed steps (dispatch = start..mid, combine = mid..end)
            "dispatch_us": max_over_ranks(sum(s.elapsed_time(m) for s, m in zip(starts, mids)) / steps) * 1e3,
            "combine_us": max_over_ranks(sum(m.elapsed_time(e) for m, e in zip(mids, ends)) / steps) * 1e3,
            "kernels": {"dispatch": impl_name.get(int(buf.runtime.last_dispatch_impl), "?"),
                        "combine": impl_name.get(int(buf.runtime.last_combine_impl), "?")},
            "steps": steps,
            "launch": "cuda_graph_replay" if graphs is not None else "eager",
            "gpu_launches": (launches() - l0) if graphs is None else per_step_launches * steps,
            "step_us_min_med_max": [min(step_ms) * 1e3, statistics.median(step_ms) * 1e3, max(step_ms) * 1e3],
            "wall_s": wall, "clocks": clocks,
        }
        r["tokens_per_s"] = n * T / (r["ms_per_step"] * 1e-3)
        (q, sc), *_ = outs[0]
        return r, (q[:num_recv], sc[:num_recv], outs[1][0])

    # ---- timed region of the headline: exactly K steps after W warm-up steps
    head, head_out = measure(head_sms, args.steps, max(args.warmup, 3), sample_clocks=True)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, head_out)  # before the sweep below reuses the arena
    ms_per_step, disp_ms, comb_ms = head["ms_per_step"], head["dispatch_us"] * 1e-3, head["combine_us"] * 1e-3
    tokens_per_s = head["tokens_per_s"]
    clocks, gpu_launches, wall, step_ms_stats = head["clocks"], head["gpu_launches"], head["wall_s"], head["step_us_min_med_max"]
    graphs_used = head["launch"]
    # other SM budgets (shorter runs): the reference's 24 and the budgets between it and most of the GPU
    sweep_rows = [head]
    if not args.no_sm_sweep:
        for sms in ([24, 48, 96] if n > 1 else [24, 64]):
            if sms != head_sms:
                sweep_rows.append(measure(sms, args.steps, 3)[0])
    best = max(sweep_rows, key=lambda r: r["tokens_per_s"])

    disp_bytes = num_recv * (H + H // 128 * 4)   # fp8 payload + scales received per rank
    comb_bytes = num_recv * H * 2                # bf16 rows pulled per rank
    remote_frac = (n - 1) / n
    nvlink_nominal = 450.0  # NVLink 4 of an H100 SXM, one direction (data sheet)

    # ---- end-to-end through the public API, inputs from pinned host memory every step
    # Inputs of step i+1 are copied on a side stream while step i runs (every step still copies its
    # own inputs inside the timed region; the copies are just not serialised with the kernels).
    copy_stream = torch.cuda.Stream(device=dev)

    def prefetch():
        with torch.cuda.stream(copy_stream):
            xd = x_host.to(dev, non_blocking=True)
            idd = idx_host.to(dev, non_blocking=True)
            wd = w_host.to(dev, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(copy_stream)
        return xd, idd, wd, ev

    def step_e2e(inputs):
        xd, idd, wd, ev = inputs
        cur = torch.cuda.current_stream(dev)
        cur.wait_event(ev)
        for t in (xd, idd, wd):
            t.record_stream(cur)
        a, _, b, c, _ = buf.get_dispatch_layout(idd, E)
        rx, ri, rw, pe, h, _ = buf.dispatch(xd, num_tokens_per_rank=a, is_token_in_rank=c, num_tokens_per_expert=b,
                                            topk_idx=idd, topk_weights=wd, use_fp8=True, config=cfg)
        # stand-in for the expert MLP: dequantise the received (e4m3, scale) rows into the combine arena
        # (a real pass over every received token; the expert GEMMs themselves are not part of this metric)
        cin = buf.get_combine_buffer(h.num_recv, H, K)
        torch.mul(rx[0].view(h.num_recv, H // 128, 128).to(torch.bfloat16), rx[1].to(torch.bfloat16).unsqueeze(2),
                  out=cin.view(h.num_recv, H // 128, 128))
        out, _, _ = buf.combine(cin, h, config=cfg)
        return out[:, :8].float().sum(dim=1).cpu()  # D2H read of a per-token checksum

    def run_e2e(steps):
        nxt = prefetch()
        res = None
        for i in range(steps):
            cur_in = nxt
            if i + 1 < steps:
                nxt = prefetch()
            res = step_e2e(cur_in)
        return res

    run_e2e(3)
    barrier()
    e2e_steps = args.steps
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    res = run_e2e(e2e_steps)
    e.record()
    barrier()
    e2e_ms = max_over_ranks(s.elapsed_time(e) / e2e_steps)
    h2d = x_host.numel() * 2 + idx_host.numel() * 8 + w_host.numel() * 4
    d2h = res.numel() * 4

    out = {
        "metric": "ep_dispatch_combine_tokens_per_s",
        "value": tokens_per_s,
        "unit": "tokens/s",
        "n_gpus": n,
        "steps": args.steps,
        "warmup": max(args.warmup, 3),
        "ms_per_step": ms_per_step,
        "higher_is_better": True,
        "scaling": "weak",
        "vs_baseline": (tokens_per_s / (8 * 4096 / ((BASELINE_DISPATCH_US + BASELINE_COMBINE_US) * 1e-6))) if n == 8 else None,
        "dtype": "bf16",
        "data": "synthetic",
        "impl": "ours",
        "config": {
            "model": "DeepEP intranode dispatch+combine (DeepSeek-V3 MoE shape)",
            "global_batch": n * T, "seq_len": T, "tokens_per_rank": T, "hidden": H, "num_topk": K,
            "num_experts": E, "parallelism": f"ep{n}", "dispatch": "bf16 -> fused e4m3 + per-128 scales",
            "combine": "bf16", "num_sms": head_sms, "kernels": head["kernels"],
            "handle": "cached (as the reference times it)", "launch": graphs_used,
            "l2": "256 MiB flush write between timed steps (untimed); per-step working set > 50 MB L2",
        },
        "dispatch_us": disp_ms * 1e3,
        "combine_us": comb_ms * 1e3,
        "dispatch_recv_GBps": disp_bytes / (disp_ms * 1e-3) / 1e9,
        "combine_recv_GBps": comb_bytes / (comb_ms * 1e-3) / 1e9,
        # roofline: bytes that must cross NVLink over the nominal link bandwidth (450 GB/s per direction)
        "roofline": {
            "nvlink_GBps_nominal": nvlink_nominal,
            "dispatch_nvlink_GBps": disp_bytes * remote_frac / (disp_ms * 1e-3) / 1e9 if n > 1 else None,
            "combine_nvlink_GBps": comb_bytes * remote_frac / (comb_ms * 1e-3) / 1e9 if n > 1 else None,
            "dispatch_floor_us": disp_bytes * remote_frac / (nvlink_nominal * 1e9) * 1e6 if n > 1 else None,
            "combine_floor_us": comb_bytes * remote_frac / (nvlink_nominal * 1e9) * 1e6 if n > 1 else None,
            "dispatch_frac_of_nominal": (disp_bytes * remote_frac / (nvlink_nominal * 1e9)) / (disp_ms * 1e-3) if n > 1 else None,
            "combine_frac_of_nominal": (comb_bytes * remote_frac / (nvlink_nominal * 1e9)) / (comb_ms * 1e-3) if n > 1 else None,
            "hbm_GBps_single_gpu": ((T * H * 2 + disp_bytes) / (disp_ms * 1e-3) / 1e9) if n == 1 else None,
        },
        # the same step at other SM budgets (shorter runs); "best" = highest tokens/s of the sweep
        "sm_sweep": [{k: r[k] for k in ("num_sms", "ms_per_step", "dispatch_us", "combine_us", "tokens_per_s", "kernels", "steps")}
                     for r in sweep_rows],
        "best": {k: best[k] for k in ("num_sms", "ms_per_step", "dispatch_us", "combine_us", "tokens_per_s", "kernels")},
        "baseline_us": {"dispatch": BASELINE_DISPATCH_US, "combine": BASELINE_COMBINE_US, "n_gpus": 8},
        "num_recv_tokens": num_recv,
        "verified": "identity-expert round trip exact in bf16, fused fp8 dispatch within e4m3 tolerance, on every rank",
        "clocks": clocks,
        "e2e": {"value": n * T / (e2e_ms * 1e-3), "unit": "tokens/s", "ms_per_step": e2e_ms,
                "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h, "steps": e2e_steps,
                "note": "per step: H2D of x/topk_idx/topk_weights from pinned memory (step i+1 prefetched on a side stream), "
                        "get_dispatch_layout, non-cached fp8 dispatch incl. count exchange + CPU sync, dequantise into the "
                        "combine arena (expert stand-in), combine, D2H checksum"},
        "gpu_launches": gpu_launches,
        "step_us_min_med_max": step_ms_stats,
        "wall_s_timed_region": wall,
        "nvls": bool(comm.has_multicast),
    }

    if n > 1 and not args.no_allreduce_sweep:
        out["allreduce"] = allreduce_sweep(comm, dist, dev, n, max_over_ranks, barrier)

    if rank == 0:
        line = json.dumps(out)
        emit(line)
        if args.out:
            with open(args.out, "w") as f:
                f.write(line + "\n")
    barrier()
    if dist is not None:
        dist.destroy_process_group()
    return 0


def dump_outputs(path, outs):
    """Writes the dispatched e4m3 rows, their per-128-channel scales and the combined bf16 rows as float32 .npy
    files, at most DUMP_BYTES in all: when the full arrays are larger, every array keeps the same seeded sample
    of rows, so that two builds can be compared output for output."""
    import numpy as np
    import torch

    os.makedirs(path, exist_ok=True)
    row_bytes = sum(t[0].numel() * 4 for t in outs)
    keep = max(1, DUMP_BYTES // row_bytes)
    for name, t in zip(("dispatch_x", "dispatch_scales", "combine_x"), outs):
        t = t.float()
        if t.size(0) > keep:
            rows = torch.randperm(t.size(0), generator=torch.Generator().manual_seed(0))[:keep].sort().values
            t = t[rows.to(t.device)]
        np.save(os.path.join(path, name + ".npy"), t.cpu().numpy())


def allreduce_sweep(comm, dist, dev, n, max_over_ranks, barrier):
    """Bus bandwidth (nccl-tests formula) of our allreduce on symmetric buffers vs NCCL, bf16 sum."""
    import torch

    rows = []
    sizes = [1 << 10, 8 << 10, 64 << 10, 512 << 10, 4 << 20, 32 << 20, 256 << 20, 1 << 30]
    big = comm.empty(max(sizes) // 2, dtype=torch.bfloat16)
    big.fill_(1.0)
    plain = torch.ones(max(sizes) // 2, dtype=torch.bfloat16, device=dev)
    for sz in sizes:
        cnt = sz // 2
        iters = 20 if sz <= (4 << 20) else 5

        def timeit(fn):
            for _ in range(3):
                fn()
            barrier()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            barrier()
            return max_over_ranks(s.elapsed_time(e) / iters)

        ours = timeit(lambda: comm.all_reduce(big[:cnt], "sum"))
        ours_plain = timeit(lambda: comm.all_reduce(plain[:cnt], "sum"))
        nccl = timeit(lambda: dist.all_reduce(plain[:cnt]))
        f = 2 * (n - 1) / n
        rows.append({"bytes": sz, "algo": comm.select_allreduce(sz, True, torch.bfloat16)[0],
                     "ours_us": ours * 1e3, "ours_busbw_GBps": sz / (ours * 1e-3) * f / 1e9,
                     "ours_unregistered_us": ours_plain * 1e3,
                     "ours_unregistered_busbw_GBps": sz / (ours_plain * 1e-3) * f / 1e9,
                     "nccl_us": nccl * 1e3, "nccl_busbw_GBps": sz / (nccl * 1e-3) * f / 1e9})
    return rows


if __name__ == "__main__":
    sys.exit(main())
