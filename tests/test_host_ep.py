"""CPU reference backend of the DeepEP Buffer API (`uccl_b200.ep.host_ep.HostBuffer`): the EP contract
of SURVEY Appendix C checked without a GPU -- receive order, local-expert remapping, cached handles,
fp8 payloads, expert_alignment, num_worst_tokens, unweighted combine, low-latency dispatch/combine."""
import threading

import pytest
import torch

from uccl_b200 import Communicator
from uccl_b200.ep import Buffer, per_token_cast_back, per_token_cast_to_fp8
from uccl_b200.ep.host_ep import HostBuffer


def _run(comms, fn):
    res, errs = [None] * len(comms), []

    def body(c):
        try:
            res[c.rank] = fn(c)
        except Exception as e:  # pragma: no cover
            import traceback

            traceback.print_exc()
            errs.append(e)

    ths = [threading.Thread(target=body, args=(c,)) for c in comms]
    [t.start() for t in ths]
    [t.join() for t in ths]
    assert not errs, errs
    return res


def _inputs(n, T, H, K, E, seed=0):
    g = torch.Generator().manual_seed(seed)
    xs = [(torch.randn(T, H, generator=g) * 2).to(torch.bfloat16) for _ in range(n)]
    idxs, ws = [], []
    for _ in range(n):
        idx = torch.rand(T, E, generator=g).topk(K, dim=1).indices
        idxs.append(idx.masked_fill(torch.rand(T, K, generator=g) < 0.1, -1).contiguous())
        ws.append(torch.rand(T, K, generator=g))
    return xs, idxs, ws


@pytest.mark.parametrize("n", [2, 4])
def test_host_ep_dispatch_combine(n):
    T, H, K, E = 37, 256, 3, 8
    e_per = E // n
    comms = Communicator.local_world(n, host=True, heap_bytes=128 << 20, stage_bytes=1 << 20)
    xs, idxs, ws = _inputs(n, T, H, K, E, seed=n)

    def fn(c):
        b = Buffer(comm=c, num_nvl_bytes=1 << 20)
        assert isinstance(b, HostBuffer)
        r = c.rank
        tpr, _, tpe, inr, _ = b.get_dispatch_layout(idxs[r], E)
        rx, ri, rw, pe, h, _ = b.dispatch(xs[r], num_tokens_per_rank=tpr, is_token_in_rank=inr,
                                          num_tokens_per_expert=tpe, topk_idx=idxs[r], topk_weights=ws[r],
                                          expert_alignment=4)
        comb, cw, _ = b.combine(rx, h, topk_weights=rw, bias=torch.ones(T, H, dtype=torch.bfloat16))
        rx_cached, *_ = b.dispatch(xs[r], handle=h)
        (q, s), *_ = b.dispatch(xs[r], handle=h, use_fp8=True)
        pre_q, pre_s = per_token_cast_to_fp8(xs[r])
        (q2, s2), *_ = b.dispatch((pre_q, pre_s), handle=h)
        # CUDA-graph friendly variant: fixed-size outputs, no per-expert list
        wx, wi, ww, wpe, wh, _ = b.dispatch(xs[r], num_tokens_per_rank=tpr, is_token_in_rank=inr,
                                            num_tokens_per_expert=tpe, topk_idx=idxs[r], topk_weights=ws[r],
                                            num_worst_tokens=n * T)
        return dict(rx=rx, ri=ri, rw=rw, pe=pe, h=h, comb=comb, cw=cw, rxc=rx_cached, q=q, s=s, q2=q2, s2=s2, inr=inr,
                    tpr=tpr, tpe=tpe, wx=wx, wi=wi, wpe=wpe)

    res = _run(comms, fn)
    for r, o in enumerate(res):
        rows, eidx, ew, src = [], [], [], []
        for s_ in range(n):
            sel = res[s_]["inr"][:, r].nonzero().flatten()
            rows.append(xs[s_][sel])
            li = idxs[s_][sel]
            mine = (li >= r * e_per) & (li < (r + 1) * e_per)
            eidx.append(torch.where(mine, li - r * e_per, torch.full_like(li, -1)))
            ew.append(torch.where(mine, ws[s_][sel], torch.zeros_like(ws[s_][sel])))
            src.append(sel.to(torch.int32))
        exp_rows = torch.cat(rows)
        assert torch.equal(o["rx"], exp_rows) and torch.equal(o["rxc"], exp_rows)
        assert torch.equal(o["ri"], torch.cat(eidx)) and torch.equal(o["rw"], torch.cat(ew))
        # handle fields sit where the reference puts them (ep/bench/buffer.py:1147-1158)
        assert torch.equal(o["h"][4], torch.cat(src)) and o["h"][3] == exp_rows.size(0) and len(o["h"]) == 7
        assert torch.equal(o["h"].recv_src_idx, o["h"][4]) and o["h"][6].shape == (T, n) and o["h"][0].shape == (n, n)
        assert torch.equal(o["tpr"], o["inr"].sum(0).to(torch.int32))
        assert torch.equal(o["tpe"], torch.bincount(idxs[r][idxs[r] >= 0], minlength=E).to(torch.int32))
        counts = [int(sum((idxs[s_] == r * e_per + e).sum() for s_ in range(n))) for e in range(e_per)]
        assert o["pe"] == [(c + 3) // 4 * 4 for c in counts]
        # fp8 payloads: fused cast == pre-cast input, and both dequantise to the bf16 rows
        assert torch.equal(o["q"].view(torch.uint8), o["q2"].view(torch.uint8)) and torch.equal(o["s"], o["s2"])
        assert torch.allclose(per_token_cast_back(o["q"], o["s"]).float(), exp_rows.float(), rtol=0.07, atol=0.15)
        # unweighted combine (+ bias) returns fan-out * x + 1, weights are summed back
        fan = o["inr"].sum(1).float()
        assert torch.allclose(o["comb"].float(), xs[r].float() * fan[:, None] + 1.0, rtol=2e-2, atol=1e-1)
        assert torch.allclose(o["cw"], torch.where(idxs[r] >= 0, ws[r], torch.zeros_like(ws[r])))
        # worst-case mode pads to the requested size with -1 expert ids
        assert o["wx"].size(0) == n * T and o["wpe"] == []
        assert torch.equal(o["wx"][:exp_rows.size(0)], exp_rows) and bool((o["wi"][exp_rows.size(0):] == -1).all())


def test_host_ep_low_latency():
    n, T, H, K, E, M = 4, 29, 512, 4, 16, 32
    e_per = E // n
    comms = Communicator.local_world(n, host=True, heap_bytes=128 << 20, stage_bytes=1 << 20)
    xs, idxs, ws = _inputs(n, T, H, K, E, seed=11)

    def fn(c):
        b = Buffer(comm=c, num_rdma_bytes=1 << 20, low_latency_mode=True)
        r = c.rank
        stats = torch.zeros(e_per, dtype=torch.int32)
        (qx, qs), cnt, hq, _, hook = b.low_latency_dispatch(xs[r], idxs[r], M, E, use_fp8=True, round_scale=True,
                                                           use_ue8m0=True, cumulative_local_expert_recv_stats=stats,
                                                           return_recv_hook=True)
        hook()
        bx, cntb, hb, _, _ = b.low_latency_dispatch(xs[r], idxs[r], M, E, use_fp8=False)
        with pytest.raises(ValueError):  # as in the reference: the in-place buffer cannot be re-encoded
            b.low_latency_combine(bx, idxs[r], ws[r], hb, use_logfmt=True, zero_copy=True)
        small = (bx.float() * 0.125).to(torch.bfloat16)  # |x| <= 1 almost everywhere: the LogFMT grid applies
        out_l, _, _ = b.low_latency_combine(small, idxs[r], ws[r], hb, use_logfmt=True)
        out, _, _ = b.low_latency_combine(bx, idxs[r], ws[r], hb)
        return dict(qx=qx, qs=qs, cnt=cnt, stats=stats, bx=bx, cntb=cntb, out=out, hb=hb, out_l=out_l)

    res = _run(comms, fn)
    for r, o in enumerate(res):
        counts = [int(sum((idxs[s_] == r * e_per + e).sum() for s_ in range(n))) for e in range(e_per)]
        assert o["cnt"].tolist() == counts == o["cntb"].tolist() == o["stats"].tolist()
        assert o["bx"].shape == (e_per, n * M, H) and o["qx"].dtype == torch.float8_e4m3fn
        assert o["qs"].dtype == torch.int32 and o["qs"].shape == (e_per, n * M, H // 512)
        src_info, layout_range = o["hb"][0], o["hb"][1]
        for e in range(e_per):
            # rows of expert e: source-rank major, token order minor; layout_range packs (begin << 32 | count) like the reference
            exp_rows, exp_src = [], []
            for s_ in range(n):
                toks = (idxs[s_] == r * e_per + e).any(1).nonzero().flatten()
                exp_rows.append(xs[s_][toks])
                exp_src.append(toks.to(torch.int32))
                lr = int(layout_range[e, s_])
                assert (lr & 0xFFFFFFFF) == toks.numel() and lr >> 32 == sum(x.size(0) for x in exp_rows[:-1])
            assert torch.equal(o["bx"][e, :counts[e]], torch.cat(exp_rows))
            assert torch.equal(src_info[e, :counts[e]], torch.cat(exp_src))
        wsum = torch.where(idxs[r] >= 0, ws[r], torch.zeros_like(ws[r])).sum(1)
        assert torch.allclose(o["out"].float(), xs[r].float() * wsum[:, None], rtol=3e-2, atol=1e-1)
        # use_logfmt: every routed copy of token t is the simulated cast of the same row
        from uccl_b200.ep.utils import logfmt10_simulate

        q = logfmt10_simulate((xs[r].float() * 0.125).to(torch.bfloat16)).float()
        assert torch.allclose(o["out_l"].float(), q * wsum[:, None], rtol=3e-2, atol=2e-2)
        assert not torch.equal(q, xs[r].float() * 0.125)  # the grid really changed the values


def test_deep_ep_package_uses_the_same_buffer():
    import deep_ep
    import deep_ep.buffer
    import deep_ep.utils
    import deep_ep_cpp

    assert deep_ep.buffer.Buffer is deep_ep.Buffer and deep_ep.utils.EventOverlap is deep_ep.EventOverlap
    assert deep_ep_cpp.Config is deep_ep.Config and callable(deep_ep.utils.check_nvlink_connections)

    c = Communicator.local_world(1, host=True, heap_bytes=128 << 20, stage_bytes=1 << 20)[0]
    b = deep_ep.Buffer(comm=c)
    assert isinstance(b, HostBuffer)
    x = torch.randn(8, 128).to(torch.bfloat16)
    idx = torch.tensor([[0, 1]] * 8)
    tpr, _, tpe, inr, _ = b.get_dispatch_layout(idx, 2)
    rx, ri, rw, pe, h, _ = b.dispatch(x, num_tokens_per_rank=tpr, is_token_in_rank=inr, num_tokens_per_expert=tpe,
                                      topk_idx=idx, topk_weights=torch.ones(8, 2))
    out, _, _ = b.combine(rx, h)
    assert torch.equal(out, x) and pe == [8, 8]


def test_moe_layer_on_the_cpu_backend():
    """models.ExpertParallelMoE through the host Buffer == dense single-process evaluation of the same experts."""
    import torch.nn.functional as F

    from uccl_b200.models.moe import ExpertParallelMoE

    n, T, H, FFN, E, K = 2, 24, 128, 64, 4, 2
    comms = Communicator.local_world(n, host=True, heap_bytes=128 << 20, stage_bytes=1 << 20)
    torch.manual_seed(5)
    router_w = (torch.randn(E, H) * H ** -0.5).to(torch.bfloat16)
    xs = [torch.randn(T, H).to(torch.bfloat16) for _ in range(n)]
    mods = [None] * n

    def fn(c):
        torch.manual_seed(100 + c.rank)
        m = ExpertParallelMoE(H, FFN, E, K, Buffer(comm=c))
        with torch.no_grad():
            m.router.weight.copy_(router_w)
        mods[c.rank] = m
        return m(xs[c.rank])

    ys = _run(comms, fn)
    e_per = E // n
    for r in range(n):
        x = xs[r]
        w, idx = torch.topk(F.softmax((x @ router_w.T).float(), dim=-1), K, dim=-1)
        ref = torch.zeros(T, H)
        for t in range(T):
            for k in range(K):
                e = int(idx[t, k])
                m = mods[e // e_per]
                h = F.silu(x[t:t + 1] @ m.w1[e % e_per]) @ m.w2[e % e_per]
                ref[t] += (h * w[t, k].to(h.dtype)).float()[0]
        assert torch.allclose(ys[r].float(), ref, rtol=5e-2, atol=5e-2), (ys[r][0, :4], ref[0, :4])


def test_moe_layer_backward_matches_dense_autograd():
    """Training path: gradients through ep_dispatch / ep_combine (each other's adjoint) equal the
    gradients of a dense single-process evaluation of the same MoE."""
    import torch.nn.functional as F

    from uccl_b200.models.moe import ExpertParallelMoE

    n, T, H, FFN, E, K = 2, 16, 128, 64, 4, 2
    e_per = E // n
    comms = Communicator.local_world(n, host=True, heap_bytes=128 << 20, stage_bytes=1 << 20)
    torch.manual_seed(9)
    router_w = (torch.randn(E, H) * H ** -0.5).to(torch.bfloat16)
    xs = [torch.randn(T, H).to(torch.bfloat16) for _ in range(n)]
    gs = [torch.randn(T, H).to(torch.bfloat16) for _ in range(n)]  # dL/dy per rank
    mods = [None] * n

    def fn(c):
        torch.manual_seed(200 + c.rank)
        m = ExpertParallelMoE(H, FFN, E, K, Buffer(comm=c))
        with torch.no_grad():
            m.router.weight.copy_(router_w)
        mods[c.rank] = m
        x = xs[c.rank].clone().requires_grad_(True)
        y = m(x)
        (y.float() * gs[c.rank].float()).sum().backward()
        return y.detach(), x.grad, m.w1.grad, m.w2.grad, m.router.weight.grad

    outs = _run(comms, fn)
    # dense reference with fresh leaf copies of every parameter
    w1 = [m.w1.detach().clone().float().requires_grad_(True) for m in mods]
    w2 = [m.w2.detach().clone().float().requires_grad_(True) for m in mods]
    rw = [router_w.clone().float().requires_grad_(True) for _ in range(n)]
    xr = [x.clone().float().requires_grad_(True) for x in xs]
    loss = 0
    ys = []
    for r in range(n):
        logits = xr[r] @ rw[r].T
        w, idx = torch.topk(F.softmax(logits, dim=-1), K, dim=-1)
        y = torch.zeros(T, H)
        for e in range(E):
            sel = (idx == e)
            rows = sel.any(1).nonzero().flatten()
            if rows.numel() == 0:
                continue
            gate = (w * sel).sum(1)[rows]
            h = F.silu(xr[r][rows] @ w1[e // e_per][e % e_per]) @ w2[e // e_per][e % e_per]
            y = y.index_add(0, rows, h * gate[:, None])
        ys.append(y)
        loss = loss + (y * gs[r].float()).sum()
    loss.backward()

    def close(a, b, tol):
        a, b = a.float(), b.float()
        return (a - b).abs().max().item() <= tol * max(1.0, b.abs().max().item())

    for r in range(n):
        y, gx, gw1, gw2, grw = outs[r]
        assert close(y, ys[r].detach(), 4e-2)
        assert close(gx, xr[r].grad, 6e-2)
        assert close(gw1, w1[r].grad, 6e-2) and close(gw2, w2[r].grad, 6e-2)
        assert close(grw, rw[r].grad, 8e-2)


def _moe_train_worker(rank, world, port, q):
    import os
    import sys

    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import moe_train

    losses = moe_train.run(rank, world, cpu=True, steps=6, tokens=64, hidden=128, ffn=128, verbose=False, lr=1.0,
                           fixed_batch=True)
    q.put((rank, losses))
    dist.destroy_process_group()


def test_moe_training_example_two_processes():
    """examples/moe_train.py on the CPU backend: two processes, shm symmetric heaps, EP forward + backward,
    router gradient all-reduce; the loss goes down and both ranks agree on it."""
    import multiprocessing as mp
    import socket

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_moe_train_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in ps]
    got = dict(q.get(timeout=240) for _ in range(2))
    [p.join(60) for p in ps]
    assert got[0] == pytest.approx(got[1])
    assert all(b < a for a, b in zip(got[0], got[0][1:])), got[0]  # fixed batch: monotonically decreasing


def test_host_buffer_raw_views_and_resets():
    """DeepEP surface that frameworks poke at: get_local_buffer_tensor (slices, dtypes), reset_rdma_buffer,
    connect_atomic_buffer (reference: ep/bench/buffer.py:213-221,606-647)."""
    c = Communicator.local_world(1, host=True, heap_bytes=128 << 20, stage_bytes=1 << 20)[0]
    b = Buffer(comm=c, num_nvl_bytes=1 << 16, num_rdma_bytes=1 << 12, low_latency_mode=True)
    t = b.get_local_buffer_tensor(torch.float32)
    assert t.dtype == torch.float32 and t.numel() == (1 << 16) // 4
    t[5] = 3.0
    v = b.get_local_buffer_tensor(torch.float32, torch.Size([2, 3]), offset=4)
    assert v.shape == (2, 3) and float(v[0, 1]) == 3.0  # same memory
    r = b.get_local_buffer_tensor(torch.int32, use_rdma_buffer=True)
    assert r.numel() == (1 << 12) // 4
    r.fill_(7)
    b.reset_rdma_buffer()
    assert int(b.get_local_buffer_tensor(torch.int32, use_rdma_buffer=True).abs().sum()) == 0
    with pytest.raises(ValueError):
        b.get_local_buffer_tensor(torch.float32, torch.Size([1 << 20]))
    with pytest.raises(TypeError):
        b.connect_atomic_buffer(None)


def test_uccl_ep_module_level_functions():
    """Functions scripts call on the reference's native `uccl.ep` module (ep/src/uccl_ep.cc:1676-1760,2187)."""
    import uccl_b200.ep as ep

    assert ep.get_low_latency_rdma_size_hint(128, 7168, 8, 288) == Buffer.get_low_latency_rdma_size_hint(128, 7168, 8, 288) > 0
    assert ep.get_num_proxy_threads() == 1 and isinstance(ep.get_oob_ip(), str) and isinstance(ep.is_sm90_compiled(), bool)
    assert ep.can_register_rdma_gpu_buffer(0, 1 << 20) and not ep.rdma_buffer_should_use_host_alloc(0)
    t, host = ep.get_rdma_buffer(4096, -1)
    assert t.numel() == 4096 and host is False

    class P:
        stopped = 0

        def stop(self):
            P.stopped += 1

    ep.register_proxies(0, [P(), P()])
    ep.register_proxies(1, [P()])
    ep.stop_all_registered_proxies()
    ep.stop_all_registered_proxies()
    assert P.stopped == 3


def test_ep_bootstrap_helpers():
    import uccl_b200.ep as ep

    hca = ep.detect_ib_hca()
    assert hca is None or isinstance(hca, str)
    assert ep.get_peer_ip(0, 1) == ""
    meta = ep.get_cpu_proxies_meta([object(), object()], 0, 4096, 64, 1)
    assert meta[0]["ptr"] == 4096 and meta[0]["nbytes"] == 64 and meta[0]["listen_ports"] == [0, 0]


def test_buffer_signature_audit_against_the_reference_and_upstream_deepep():
    """Every public method of the reference's `Buffer` (ep/bench/buffer.py) and of the upstream DeepEP it vendors
    (thirdparty/DeepEP/deep_ep/buffer.py) exists here with the same parameter names (frameworks call them by keyword).
    The reference's signatures are stored in tests/golden/reference_signatures.json (oracle/extract_signatures.py)."""
    import inspect

    import deep_ep
    from helpers import reference_signatures
    from uccl_b200.ep.buffer import Buffer as Native
    from uccl_b200.ep.low_latency import LowLatencyRuntime

    files = reference_signatures()["ep_buffer"]
    assert len(files) == 3
    ll = {"low_latency_dispatch": LowLatencyRuntime.dispatch, "low_latency_combine": LowLatencyRuntime.combine}
    internal = {"connect_atomic_buffer"}  # takes the reference's own proxy type; checked by name only
    for path, methods in files.items():
        for name, want in methods.items():
            assert hasattr(deep_ep.Buffer, name) and hasattr(Native, name), f"{path}: Buffer.{name} missing"
            if name in internal:
                continue
            target = ll.get(name, getattr(Native, name))
            have = set(inspect.signature(target).parameters)
            missing = [w for w in want if w not in have]
            assert not missing, f"{path}: Buffer.{name} lacks parameters {missing}"


def test_utils_signature_audit_against_the_reference_helpers():
    """Every public helper of the reference's ep/bench/utils.py (what its tests and benchmarks import) and of
    upstream DeepEP's utils exists under `uccl_b200.ep` with the same parameter names."""
    import inspect

    import uccl_b200.ep as E
    import uccl_b200.ep.utils as U
    from helpers import reference_signatures

    files = reference_signatures()["ep_utils"]
    assert len(files) == 4
    for path, funcs in files.items():
        for name, want in funcs.items():
            target = getattr(U, name, None) or getattr(E, name, None)
            assert target is not None, f"{path}: {name} missing"
            have = set(inspect.signature(target).parameters)
            missing = [w for w in want if w not in have]
            assert not missing, f"{path}: {name} lacks parameters {missing}"


def test_per_token_cast_back_accepts_both_spellings():
    from uccl_b200.ep.utils import per_token_cast_back, per_token_cast_to_fp8

    if not hasattr(torch, "float8_e4m3fn"):
        pytest.skip("no fp8 dtype")
    x = torch.randn(4, 256, dtype=torch.bfloat16)
    q, s = per_token_cast_to_fp8(x)
    a = per_token_cast_back(q, s)
    assert torch.equal(a, per_token_cast_back(x_fp8=q, x_scales=s)) and torch.equal(a, per_token_cast_back(q, scales=s))
    with pytest.raises(TypeError):
        per_token_cast_back(q)


def test_upstream_sizing_snippet_runs():
    """The buffer-sizing loop every DeepEP consumer copies from upstream's README works unchanged."""
    hidden_bytes = 7168 * 2
    num_nvl_bytes = num_rdma_bytes = 0
    for config in (Buffer.get_dispatch_config(8), Buffer.get_combine_config(8)):
        num_nvl_bytes = max(config.get_nvl_buffer_size_hint(hidden_bytes, 8), num_nvl_bytes)
        num_rdma_bytes = max(config.get_rdma_buffer_size_hint(hidden_bytes, 8), num_rdma_bytes)
    assert num_nvl_bytes > (1 << 20) and num_rdma_bytes == 0


def test_vllm_call_shapes_on_the_host_backend():
    """The exact keyword calls vLLM's DeepEP integration makes (vllm/model_executor/layers/fused_moe/prepare_finalize/
    deepep_ht.py:114-170,362-376 and deepep_ll.py:298-314,399-408 in vLLM 0.22) run against the Buffer API."""
    n, T, H, K, E, M = 2, 24, 512, 4, 8, 32
    comms = Communicator.local_world(n, host=True, heap_bytes=128 << 20, stage_bytes=1 << 20)
    xs, idxs, ws = _inputs(n, T, H, K, E, seed=21)

    def fn(c):
        buffer = Buffer(comm=c, num_nvl_bytes=1 << 20, num_rdma_bytes=1 << 20, low_latency_mode=True,
                        num_qps_per_rank=E // n, allow_nvlink_for_low_latency_mode=True, allow_mnnvl=False,
                        explicitly_destroy=True)
        r = c.rank
        previous_event = None
        (num_tokens_per_rank, num_tokens_per_rdma_rank, dispatch_expert_num_tokens, is_token_in_rank, event) = \
            buffer.get_dispatch_layout(topk_idx=idxs[r], num_experts=E, previous_event=previous_event, async_finish=False,
                                       allocate_on_comm_stream=False)
        (token_data, expert_topk_ids, expert_topk_weights, expert_num_tokens_per_expert_list, handle, event) = buffer.dispatch(
            x=xs[r], handle=None, num_tokens_per_rank=num_tokens_per_rank, num_tokens_per_rdma_rank=num_tokens_per_rdma_rank,
            is_token_in_rank=is_token_in_rank, num_tokens_per_expert=dispatch_expert_num_tokens, topk_idx=idxs[r],
            topk_weights=ws[r], expert_alignment=1, config=Buffer.get_dispatch_config(n), previous_event=previous_event,
            async_finish=False, allocate_on_comm_stream=False)
        assert isinstance(expert_num_tokens_per_expert_list, list) and len(expert_num_tokens_per_expert_list) == E // n
        if event.event is not None:
            event.current_stream_wait()
        combined_x, _, event = buffer.combine(x=token_data, handle=handle, topk_weights=None,
                                              config=Buffer.get_combine_config(n), previous_event=previous_event,
                                              async_finish=False, allocate_on_comm_stream=False)
        # low latency, as deepep_ll.py calls it
        expert_x, expert_num_tokens, ll_handle, _, hook = buffer.low_latency_dispatch(
            xs[r], idxs[r], M, E, use_fp8=False, round_scale=False, use_ue8m0=False, async_finish=False,
            return_recv_hook=True)
        hook()
        output = torch.empty(T, H, dtype=torch.bfloat16)
        _, _, recv_hook = buffer.low_latency_combine(expert_x, idxs[r], ws[r], ll_handle, async_finish=False,
                                                    zero_copy=False, return_recv_hook=True, out=output)
        recv_hook()
        with pytest.raises(NotImplementedError):
            buffer.low_latency_dispatch(xs[r], idxs[r], M, E, use_fp8=True, use_nvfp4=True)
        type(buffer).set_num_sms(20)
        buffer.destroy()
        return combined_x, output

    for r, (comb, out) in enumerate(_run(comms, fn)):
        in_rank = torch.stack([((idxs[r] >= d * (E // n)) & (idxs[r] < (d + 1) * (E // n))).any(1) for d in range(n)], 1)
        assert torch.allclose(comb.float(), xs[r].float() * in_rank.sum(1, keepdim=True), rtol=2e-2, atol=1e-2)
        wsum = torch.where(idxs[r] >= 0, ws[r], torch.zeros_like(ws[r])).sum(1)
        assert torch.allclose(out.float(), xs[r].float() * wsum[:, None], rtol=3e-2, atol=1e-1)


def test_megatron_call_shapes_on_the_host_backend():
    """The keyword calls of Megatron-LM's flex dispatcher (megatron/core/transformer/moe/fused_a2a.py: FusedDispatch /
    FusedCombine, forward and backward) against the Buffer API: sizing through the Config hints, dispatch with
    probabilities, combine of the expert outputs, then the backward pair -- combine of the dispatched gradient with
    `topk_weights=` the probability gradient, dispatch of the combined gradient through the cached handle."""
    n, T, H, K, E = 2, 32, 256, 2, 4
    comms = Communicator.local_world(n, host=True, heap_bytes=128 << 20, stage_bytes=1 << 20)
    xs, idxs, ws = _inputs(n, T, H, K, E, seed=33)

    def fn(c):
        r = c.rank
        x, token_indices, token_probs = xs[r], idxs[r], ws[r]
        hidden_bytes = x.size(1) * max(x.element_size(), 2)
        num_nvl_bytes, num_rdma_bytes = 0, 0
        for config in (Buffer.get_dispatch_config(n), Buffer.get_combine_config(n)):
            num_nvl_bytes = max(config.get_nvl_buffer_size_hint(hidden_bytes, n), num_nvl_bytes)
            num_rdma_bytes = max(config.get_rdma_buffer_size_hint(hidden_bytes, n), num_rdma_bytes)
        buffer = Buffer(comm=c, num_nvl_bytes=num_nvl_bytes, num_rdma_bytes=num_rdma_bytes)
        # FusedDispatch.forward
        (num_tokens_per_rank, num_tokens_per_rdma_rank, num_tokens_per_expert, is_token_in_rank, previous_event) = \
            buffer.get_dispatch_layout(token_indices, E, previous_event=None, async_finish=False,
                                       allocate_on_comm_stream=False)
        (recv_x, recv_token_indices, recv_token_probs, num_recv_tokens_per_expert_list, handle, event) = buffer.dispatch(
            x, topk_idx=token_indices, topk_weights=token_probs.float(), num_tokens_per_rank=num_tokens_per_rank,
            num_tokens_per_rdma_rank=num_tokens_per_rdma_rank, is_token_in_rank=is_token_in_rank,
            num_tokens_per_expert=num_tokens_per_expert, previous_event=None, async_finish=False,
            allocate_on_comm_stream=False)
        tokens_per_expert = torch.tensor(num_recv_tokens_per_expert_list)
        assert int(tokens_per_expert.sum()) == int((recv_token_indices >= 0).sum())
        # FusedCombine.forward (experts = identity)
        combined_x, _, event = buffer.combine(recv_x, handle=handle, async_finish=False, previous_event=None,
                                              allocate_on_comm_stream=False)
        # FusedCombine.backward: the gradient of the combined activations is dispatched through the cached handle
        grad_out = torch.ones_like(combined_x)
        grad_x, _, _, _, _, event = buffer.dispatch(grad_out.contiguous(), handle=handle, previous_event=None,
                                                    async_finish=False, allocate_on_comm_stream=False)
        assert grad_x.shape == recv_x.shape
        # FusedDispatch.backward: gradients of the received rows and of their probabilities travel back together
        grad_probs = torch.where(recv_token_indices >= 0, torch.ones_like(recv_token_probs), torch.zeros_like(recv_token_probs))
        gx, gprobs, event = buffer.combine(grad_x.contiguous(), handle, topk_weights=grad_probs.float(),
                                           previous_event=None, async_finish=False, allocate_on_comm_stream=False)
        return combined_x, gx, gprobs

    for r, (comb, gx, gprobs) in enumerate(_run(comms, fn)):
        in_rank = torch.stack([((idxs[r] >= d * (E // n)) & (idxs[r] < (d + 1) * (E // n))).any(1) for d in range(n)], 1)
        fan = in_rank.sum(1, keepdim=True).float()
        assert torch.allclose(comb.float(), xs[r].float() * fan, rtol=2e-2, atol=1e-2)
        assert torch.allclose(gx.float(), torch.ones(T, H) * fan, rtol=2e-2, atol=1e-2)
        assert torch.equal(gprobs, (idxs[r] >= 0).float())


def test_sglang_call_shapes_on_the_host_backend():
    """SGLang's DeepEP dispatcher (sglang/srt/layers/moe/token_dispatcher/deepep.py): normal mode with a captured
    previous event, async_finish and a pre-cast fp8 input; low-latency mode with async_finish (no hook) followed by
    clean_low_latency_buffer; Config built from explicit numbers."""
    from uccl_b200.ep import Config

    n, T, H, K, E, M = 2, 16, 512, 2, 4, 16
    comms = Communicator.local_world(n, host=True, heap_bytes=128 << 20, stage_bytes=1 << 20)
    xs, idxs, ws = _inputs(n, T, H, K, E, seed=44)

    def fn(c):
        r = c.rank
        buffer = Buffer(comm=c, num_nvl_bytes=1 << 20,
                        num_rdma_bytes=Buffer.get_low_latency_rdma_size_hint(M, H, n, E), low_latency_mode=True,
                        num_qps_per_rank=max(E // n, Buffer.num_sms // 2), allow_mnnvl=True)
        cfg = Config(Buffer.num_sms, 6, 256, 6, 128)
        previous_event = Buffer.capture()
        (num_tokens_per_rank, num_tokens_per_rdma_rank, num_tokens_per_expert, is_token_in_rank, previous_event) = \
            buffer.get_dispatch_layout(idxs[r], E, previous_event=previous_event, async_finish=True,
                                       allocate_on_comm_stream=previous_event is not None)
        x8 = per_token_cast_to_fp8(xs[r])
        (recv_x, recv_topk_idx, recv_topk_weights, num_recv_tokens_per_expert_list, handle, event) = buffer.dispatch(
            x8, topk_idx=idxs[r], topk_weights=ws[r], num_tokens_per_rank=num_tokens_per_rank,
            num_tokens_per_rdma_rank=num_tokens_per_rdma_rank, is_token_in_rank=is_token_in_rank,
            num_tokens_per_expert=num_tokens_per_expert, previous_event=previous_event, async_finish=True,
            allocate_on_comm_stream=True, expert_alignment=128, config=cfg)
        event.current_stream_wait()
        assert isinstance(recv_x, tuple) and all(v % 128 == 0 for v in num_recv_tokens_per_expert_list)
        y = per_token_cast_back(*recv_x)
        combined, _, event = buffer.combine(y, handle, async_finish=True, previous_event=Buffer.capture(),
                                            allocate_on_comm_stream=True, config=cfg)
        event.current_stream_wait()
        packed, counts, ll_handle, event, hook = buffer.low_latency_dispatch(
            xs[r], idxs[r], M, E, use_fp8=True, async_finish=True, return_recv_hook=False, round_scale=False,
            use_ue8m0=False)
        assert hook is None
        event.current_stream_wait()
        q, s = packed
        deq = per_token_cast_back(q.view(-1, H), s.reshape(-1, H // 128).contiguous()).view(E // n, n * M, H)
        out, event, hook = buffer.low_latency_combine(deq, idxs[r], ws[r], ll_handle, async_finish=True,
                                                      return_recv_hook=False)
        event.current_stream_wait()
        buffer.clean_low_latency_buffer(M, H, E)
        return combined, out

    for r, (comb, out) in enumerate(_run(comms, fn)):
        in_rank = torch.stack([((idxs[r] >= d * (E // n)) & (idxs[r] < (d + 1) * (E // n))).any(1) for d in range(n)], 1)
        assert torch.allclose(comb.float(), xs[r].float() * in_rank.sum(1, keepdim=True), rtol=0.08, atol=0.3)
        wsum = torch.where(idxs[r] >= 0, ws[r], torch.zeros_like(ws[r])).sum(1)
        assert torch.allclose(out.float(), xs[r].float() * wsum[:, None], rtol=0.08, atol=0.3)


def test_deep_ep_package_exports_what_the_reference_wrapper_exports():
    import deep_ep
    from helpers import reference_signatures

    exported = reference_signatures()["deep_ep_all"]  # __all__ of the reference's ep/deep_ep_wrapper/deep_ep
    assert exported
    missing = [x for x in exported if not hasattr(deep_ep, x)]
    assert not missing, missing
