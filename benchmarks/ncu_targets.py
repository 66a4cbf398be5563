#!/usr/bin/env python
"""One launch of every hot kernel at a realistic size on ONE GPU (one-rank communicator with
UCCL_B200_FORCE_KERNELS=1, so the real kernels run instead of the cudaMemcpy shortcut) -- the target of
`ncu --set full` (scripts/ncu_capture.sh).  ncu serialises kernels, so nothing here may wait for another rank.

  python benchmarks/ncu_targets.py [--tokens 4096] [--mb 64]
"""
import argparse
import os
import sys

os.environ.setdefault("UCCL_B200_FORCE_KERNELS", "1")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from uccl_b200 import Communicator, _native
from uccl_b200.ep import Buffer, Config


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--tokens", type=int, default=4096)
    p.add_argument("--hidden", type=int, default=7168)
    p.add_argument("--mb", type=int, default=64)
    p.add_argument("--reps", type=int, default=2)
    a = p.parse_args()
    torch.cuda.set_device(0)
    C = _native.C()
    T, H, K, E = a.tokens, a.hidden, 8, 256
    arena = T * (H * 2 + K * 4) + (1 << 20)
    ll = Buffer.get_low_latency_rdma_size_hint(128, H, 1, E)
    comm = Communicator.local_world(1, devices=[0], heap_bytes=3 * arena + ll + (1 << 30) + (a.mb << 21),
                                    stage_bytes=64 << 20)[0]
    buf = Buffer(comm=comm, num_nvl_bytes=3 * arena + (2 << 20), num_rdma_bytes=ll, low_latency_mode=True)
    g = torch.Generator(device="cpu").manual_seed(1)
    x = torch.randn(T, H, generator=g).to(torch.bfloat16).cuda()
    idx = (torch.randn(T, E, generator=g).abs() + 1).topk(K, dim=-1).indices.to(torch.int64).contiguous().cuda()
    w = torch.rand(T, K, generator=g).float().cuda()
    for _ in range(a.reps):
        for impl, sms in ((C.EP_IMPL_REG, 132), (C.EP_IMPL_TMA, 132), (C.EP_IMPL_TMA, 24), (C.EP_IMPL_REG, 24)):
            buf.runtime.impl = impl
            cfg = Config(sms)
            tpr, _, tpe, in_rank, _ = buf.get_dispatch_layout(idx, E)
            rx, ri, rw, pe, h, _ = buf.dispatch(x, num_tokens_per_rank=tpr, is_token_in_rank=in_rank, num_tokens_per_expert=tpe,
                                                topk_idx=idx, topk_weights=w, use_fp8=True, config=cfg)
            buf.dispatch(x, handle=h, use_fp8=True, config=cfg)      # cached fused-fp8 dispatch (the headline kernel)
            buf.dispatch(x, handle=h, config=cfg)                    # cached bf16 dispatch
            cin = buf.get_combine_buffer(h.num_recv, H, K)
            buf.combine(cin, h, config=cfg)                          # bf16 combine
        buf.runtime.impl = C.EP_IMPL_AUTO
        M = 128
        xl, il, wl = x[:M].contiguous(), idx[:M].contiguous(), w[:M].contiguous()
        rxl, cnt, hl, _, _ = buf.low_latency_dispatch(xl, il, M, E, use_fp8=True)
        cb = buf.get_next_low_latency_combine_buffer(hl)
        buf.low_latency_combine(cb, il, wl, hl)
        n = (a.mb << 20) // 2
        s = comm.empty(n, dtype=torch.bfloat16)
        s.fill_(1.0)
        for algo in ("oneshot_ll", "twoshot_p2p", "staged_p2p"):
            sz = (1 << 19) if algo == "oneshot_ll" else n
            comm.all_reduce(s[:sz], "sum", algo=algo)
        pl = torch.ones(n, dtype=torch.bfloat16, device="cuda")
        o = torch.empty_like(pl)
        comm.all_reduce(pl, "sum", out=o)
        comm.all_gather(o, pl)
        comm.reduce_scatter(o, pl)
        comm.all_to_all(o, pl)
        comm.broadcast(pl, 0, out=o)
        small = pl[: 1 << 16]
        comm.all_gather(o[: 1 << 16], small)                         # LL-packet exchange kernel
        comm.batch_send_recv([("send", pl, 0), ("recv", o, 0)])      # send/recv kernel (self pair)
        torch.cuda.synchronize()
    # P2P copy engine: GPU0 -> GPU0 through two endpoints (same TMA kernel as a peer copy)
    try:
        from uccl_b200.p2p import Endpoint

        ea, eb = Endpoint(0), Endpoint(0)
        ok, conn = ea.connect(remote_metadata=eb.get_metadata())
        eb.accept(5000)
        src = torch.ones(a.mb << 20, dtype=torch.uint8, device="cuda")
        dst = torch.zeros(a.mb << 20, dtype=torch.uint8, device="cuda")
        la = ea.register_memory([src])
        ra = ea.deserialize_descs(eb.get_serialized_descs(eb.register_memory([dst])))
        for _ in range(a.reps):
            ok, tid = ea.transfer(conn, "write", la, ra)
            ea.wait(tid)
    except Exception as e:  # noqa: BLE001
        print("p2p target skipped:", e)
    torch.cuda.synchronize()
    print("ncu targets done")


if __name__ == "__main__":
    main()
