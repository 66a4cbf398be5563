"""GPU tests of EP layout / dispatch / combine against a plain PyTorch reference
(the oracle style of the reference's ep/bench/test_intranode.py:98-118: layout vs torch counts,
every received row must equal the source row, combine must equal x * num_dst_ranks)."""
import threading

import pytest
import torch

from helpers import get_world
from uccl_b200.ep import Buffer, per_token_cast_back, per_token_cast_to_fp8

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

_BUFFERS = {}


def get_buffers(n, nbytes=192 << 20):
    if n not in _BUFFERS:
        comms = get_world(n, heap_mb=256 + 224, stage_mb=8, max_ctas=4)
        _BUFFERS[n] = [Buffer(comm=c, num_nvl_bytes=nbytes) for c in comms]
        # virtual ranks share one GPU: all n kernels must be co-resident (n * num_sms <= 132 SMs)
        Buffer.set_num_sms(8)
    return _BUFFERS[n]


def run_threads(bufs, fn):
    out = [None] * len(bufs)
    errs = []

    def w(b):
        try:
            torch.cuda.set_device(b.device)
            with torch.cuda.stream(torch.cuda.Stream(device=b.device)):
                out[b.rank] = fn(b)
                torch.cuda.current_stream().synchronize()
        except Exception as e:  # pragma: no cover
            import traceback

            traceback.print_exc()
            errs.append(e)

    ts = [threading.Thread(target=w, args=(b,)) for b in bufs]
    [t.start() for t in ts]
    [t.join() for t in ts]
    if errs:
        raise errs[0]
    return out


def make_inputs(n, T, H, K, E, seed=0):
    g = torch.Generator().manual_seed(seed)
    xs, idxs, ws = [], [], []
    for r in range(n):
        xs.append((torch.randn(T, H, generator=g) * 3).to(torch.bfloat16))
        scores = torch.rand(T, E, generator=g)
        idx = scores.topk(K, dim=1).indices.to(torch.int64)
        # sprinkle some -1 (no selection) entries
        drop = torch.rand(T, K, generator=g) < 0.05
        idx = idx.masked_fill(drop, -1)
        idxs.append(idx.contiguous())
        ws.append(torch.rand(T, K, generator=g).float())
    return xs, idxs, ws


def ref_layout(idx, n, E):
    E_local = E // n
    T = idx.size(0)
    in_rank = torch.zeros(T, n, dtype=torch.bool)
    for r in range(n):
        in_rank[:, r] = ((idx >= r * E_local) & (idx < (r + 1) * E_local)).any(dim=1)
    per_expert = torch.zeros(E, dtype=torch.int32)
    valid = idx[idx >= 0]
    per_expert += torch.bincount(valid, minlength=E).to(torch.int32)
    return in_rank.sum(0).to(torch.int32), per_expert, in_rank


def set_impl(bufs, impl):
    """Force the register-path (1) or the TMA-pipelined (2) dispatch/combine kernels; 0 = auto."""
    for b in bufs:
        b.runtime.impl = impl


@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("mode", ["bf16", "fp8_fused", "fp8_pre"])
@pytest.mark.parametrize("impl", ["reg", "tma"])
def test_dispatch_combine(n, mode, impl):
    T, H, K = 257, 1024, 4
    E = n * 4
    E_local = E // n
    bufs = get_buffers(n)
    set_impl(bufs, 1 if impl == "reg" else 2)
    xs, idxs, ws = make_inputs(n, T, H, K, E, seed=n)
    layouts = [ref_layout(idxs[r], n, E) for r in range(n)]

    def fn(b):
        r = b.rank
        dev = b.device
        x = xs[r].to(dev)
        idx = idxs[r].to(dev)
        w = ws[r].to(dev)
        tpr, _, tpe, in_rank, _ = b.get_dispatch_layout(idx, E)
        assert torch.equal(tpr.cpu(), layouts[r][0])
        assert torch.equal(tpe.cpu(), layouts[r][1])
        assert torch.equal(in_rank.cpu(), layouts[r][2])
        if mode == "fp8_pre":
            xin = per_token_cast_to_fp8(x)
            kw = {}
        else:
            xin = x
            kw = dict(use_fp8=(mode == "fp8_fused"))
        recv_x, recv_idx, recv_w, per_expert, handle, _ = b.dispatch(
            xin, num_tokens_per_rank=tpr, is_token_in_rank=in_rank, num_tokens_per_expert=tpe, topk_idx=idx,
            topk_weights=w, **kw)
        torch.cuda.current_stream().synchronize()
        if isinstance(recv_x, tuple):
            rx = per_token_cast_back(recv_x[0], recv_x[1])
        else:
            rx = recv_x
        num_recv = rx.size(0)
        # combine: identity "experts" -> every token comes back multiplied by its rank fan-out
        cb = b.get_combine_buffer(num_recv, H, K)
        cb.copy_(rx)
        comb, comb_w, _ = b.combine(cb, handle, topk_weights=recv_w)
        # cached dispatch must reproduce the payload
        recv_x2, *_ = b.dispatch(xin, handle=handle, **kw)
        torch.cuda.current_stream().synchronize()
        rx2 = per_token_cast_back(*recv_x2) if isinstance(recv_x2, tuple) else recv_x2
        return dict(rx=rx.cpu(), rx2=rx2.cpu(), idx=recv_idx.cpu(), w=recv_w.cpu(), per_expert=per_expert,
                    src=handle.recv_src_idx.cpu(), comb=comb.cpu(), comb_w=comb_w.cpu(), raw=recv_x)

    outs = run_threads(bufs, fn)
    want = 1 if impl == "reg" else 2
    assert all(b.runtime.last_dispatch_impl == want and b.runtime.last_combine_impl == want for b in bufs)
    set_impl(bufs, 0)
    for r in range(n):
        o = outs[r]
        # expected receive order: source rank major, token order minor
        exp_rows, exp_idx, exp_w, exp_src = [], [], [], []
        for s in range(n):
            sel = layouts[s][2][:, r].nonzero().flatten()
            xsrc = xs[s][sel]
            if mode != "bf16":
                xsrc = per_token_cast_back(*per_token_cast_to_fp8(xsrc))
            exp_rows.append(xsrc)
            li = idxs[s][sel]
            mine = (li >= r * E_local) & (li < (r + 1) * E_local)
            exp_idx.append(torch.where(mine, li - r * E_local, torch.full_like(li, -1)))
            exp_w.append(torch.where(mine, ws[s][sel], torch.zeros_like(ws[s][sel])))
            exp_src.append(sel.to(torch.int32))
        exp_rows = torch.cat(exp_rows)
        assert o["rx"].shape == exp_rows.shape
        if mode == "bf16":
            assert torch.equal(o["rx"], exp_rows)
        else:
            # identical math up to e4m3 rounding ties (the CPU reference computes 448/amax with a
            # reciprocal-multiply, 1 ulp off the IEEE division used on the GPU)
            bad = ~torch.isclose(o["rx"].float(), exp_rows.float(), rtol=0.07, atol=0.05)
            assert bad.float().mean().item() < 5e-3, bad.float().mean().item()
            assert torch.allclose(o["rx"].float(), exp_rows.float(), rtol=0.15, atol=0.1)
        assert torch.equal(o["rx2"], o["rx"])
        assert torch.equal(o["idx"], torch.cat(exp_idx))
        assert torch.equal(o["w"], torch.cat(exp_w))
        assert torch.equal(o["src"], torch.cat(exp_src))
        exp_pe = [int(sum(((idxs[s] == r * E_local + e).sum()) for s in range(n))) for e in range(E_local)]
        assert o["per_expert"] == exp_pe
        # combine
        fan = layouts[r][2].sum(1).float()
        base = xs[r].float() if mode == "bf16" else per_token_cast_back(*per_token_cast_to_fp8(xs[r])).float()
        exp_comb = base * fan[:, None]
        badc = ~torch.isclose(o["comb"].float(), exp_comb, rtol=2e-2, atol=2e-1)
        assert badc.float().mean().item() < (0 if mode == "bf16" else 5e-3) + 1e-9, badc.float().mean().item()
        exp_cw = torch.where(idxs[r] >= 0, ws[r], torch.zeros_like(ws[r]))
        assert torch.allclose(o["comb_w"], exp_cw, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("n,H", [(1, 7168), (2, 7168), (2, 4096), (4, 2560), (8, 512)])
def test_tma_pipeline_matches_register_path(n, H):
    """The TMA-pipelined kernels (ep_tma_kernels.cu) must reproduce the register path bit for bit: same
    quantiser, same fixed summation order, incl. bias, routed weights, cached handles and the
    num_worst_tokens (CUDA-graph) mode, on row sizes that span one / several / partial pipeline slices."""
    T, K = 301, 8
    E = n * 8
    bufs = get_buffers(n)
    xs, idxs, ws = make_inputs(n, T, H, K, E, seed=100 + n)
    g = torch.Generator().manual_seed(5)
    biases = [((torch.randn(T, H, generator=g)).to(torch.bfloat16), (torch.randn(T, H, generator=g)).to(torch.bfloat16))
              for _ in range(n)]

    def run(impl):
        set_impl(bufs, impl)

        def fn(b):
            dev = b.device
            x, idx, w = xs[b.rank].to(dev), idxs[b.rank].to(dev), ws[b.rank].to(dev)
            b0, b1 = (t.to(dev) for t in biases[b.rank])
            res = {}
            tpr, _, tpe, in_rank, _ = b.get_dispatch_layout(idx, E)
            for mode in ("bf16", "fp8_fused", "fp8_pre"):
                xin = per_token_cast_to_fp8(x) if mode == "fp8_pre" else x
                kw = dict(use_fp8=True) if mode == "fp8_fused" else {}
                rx, ridx, rw, pe, handle, _ = b.dispatch(xin, num_tokens_per_rank=tpr, is_token_in_rank=in_rank,
                                                         num_tokens_per_expert=tpe, topk_idx=idx, topk_weights=w, **kw)
                torch.cuda.current_stream().synchronize()
                parts = list(rx) if isinstance(rx, tuple) else [rx]
                res[mode] = [p.clone().view(torch.uint8).cpu() for p in parts] + [ridx.cpu(), rw.cpu(), handle.recv_src_idx.cpu(), pe]
                rx2, *_ = b.dispatch(xin, handle=handle, **kw)
                torch.cuda.current_stream().synchronize()
                parts2 = list(rx2) if isinstance(rx2, tuple) else [rx2]
                res[mode + "_cached"] = [p.clone().view(torch.uint8).cpu() for p in parts2]
                if mode == "bf16":
                    cb = b.get_combine_buffer(rx.size(0), H, K)
                    cb.copy_(rx)
                    out, out_w, _ = b.combine(cb, handle, topk_weights=rw)
                    outb, _, _ = b.combine(cb, handle, bias=(b0, b1))
                    torch.cuda.current_stream().synchronize()
                    res["combine"] = [out.cpu(), out_w.cpu(), outb.cpu()]
            # CUDA-graph friendly mode: no CPU sync, padded tail
            worst = n * T
            rx, ridx, rw, pe, handle, _ = b.dispatch(x, num_tokens_per_rank=tpr, is_token_in_rank=in_rank,
                                                     num_tokens_per_expert=tpe, topk_idx=idx, topk_weights=w,
                                                     num_worst_tokens=worst)
            torch.cuda.current_stream().synchronize()
            res["worst"] = [ridx.cpu()]
            return res

        return run_threads(bufs, fn)

    ref = run(1)
    got = run(2)
    assert all(b.runtime.last_dispatch_impl == 2 for b in bufs)
    set_impl(bufs, 0)
    for r in range(n):
        assert ref[r].keys() == got[r].keys()
        for k in ref[r]:
            for a, b_ in zip(ref[r][k], got[r][k]):
                if isinstance(a, torch.Tensor):
                    assert a.shape == b_.shape and torch.equal(a, b_), (r, k)
                else:
                    assert a == b_, (r, k)
    # and the register path itself is right: combine(identity experts) = x * fan-out (+ biases)
    for r in range(n):
        in_rank = ref_layout(idxs[r], n, E)[2]
        fan = in_rank.sum(1).float()[:, None]
        exp = xs[r].float() * fan
        assert torch.allclose(got[r]["combine"][0].float(), exp, rtol=2e-2, atol=2e-1)
        expb = exp + biases[r][0].float() + biases[r][1].float()
        assert torch.allclose(got[r]["combine"][2].float(), expb, rtol=2e-2, atol=3e-1)


@pytest.mark.parametrize("T", [0, 1, 127, 128, 129, 4096, 9001])
def test_layout_multi_cta(T):
    """Multi-CTA layout (chained per-CTA counts) against a torch reference, incl. the stable positions."""
    n, K = 4, 8
    E = n * 8
    bufs = get_buffers(n)
    b = bufs[0]
    g = torch.Generator().manual_seed(T)
    idx = torch.rand(max(T, 1), E, generator=g).topk(K, dim=1).indices.to(torch.int64)[:T]
    idx = idx.masked_fill(torch.rand(T, K, generator=g) < 0.1, -1).contiguous()
    exp_tpr, exp_tpe, exp_in = ref_layout(idx, n, E) if T else (torch.zeros(n, dtype=torch.int32),
                                                                  torch.zeros(E, dtype=torch.int32),
                                                                  torch.zeros(0, n, dtype=torch.bool))
    with torch.cuda.device(b.device):
        for _ in range(2):  # twice: the device-side call epoch must advance
            tpr, _, tpe, in_rank, _ = b.get_dispatch_layout(idx.to(b.device), E)
            pos = b._layout_cache[2]
            torch.cuda.synchronize()
            assert torch.equal(tpr.cpu(), exp_tpr)
            assert torch.equal(tpe.cpu(), exp_tpe)
            assert torch.equal(in_rank.cpu(), exp_in)
            exp_pos = torch.where(exp_in, exp_in.to(torch.int32).cumsum(0).to(torch.int32) - 1,
                                  torch.full((T, n), -1, dtype=torch.int32))
            assert torch.equal(pos.cpu(), exp_pos)


def test_owned_results_survive_later_dispatches():
    """`copy_out=True` / `Buffer(owned_results=True)` (what the `deep_ep` compatibility package uses) returns
    tensors the caller owns, like the reference (ep/bench/buffer.py:1068-1106): they must survive more
    dispatches than the arena ring has slots, while the default zero-copy views are recycled."""
    n, T, H, K = 2, 130, 512, 4
    E = n * 4
    bufs = get_buffers(n)
    xs, idxs, ws = make_inputs(n, T, H, K, E, seed=55)

    def fn(b):
        dev = b.device
        x, idx, w = xs[b.rank].to(dev), idxs[b.rank].to(dev), ws[b.rank].to(dev)
        tpr, _, tpe, in_rank, _ = b.get_dispatch_layout(idx, E)
        kw = dict(num_tokens_per_rank=tpr, is_token_in_rank=in_rank, num_tokens_per_expert=tpe, topk_idx=idx, topk_weights=w)
        own_x, own_idx, own_w, _, h, _ = b.dispatch(x, copy_out=True, **kw)
        view_x, *_ = b.dispatch(x, **kw)
        torch.cuda.current_stream().synchronize()
        assert len(h) == 7 and h[3] == own_x.size(0) and h[6].shape == (T, n)
        assert torch.equal(own_x, view_x)
        ref = own_x.clone()
        for i in range(b.runtime.num_slots + 1):  # recycle every arena with different payloads
            b.dispatch(x * (i + 2), **kw)
        torch.cuda.current_stream().synchronize()
        assert torch.equal(own_x, ref), "owned result was overwritten"
        assert not torch.equal(view_x, ref), "the zero-copy view is expected to be recycled"
        return True

    assert run_threads(bufs, fn) == [True] * n


def test_internode_api_runs_on_the_fabric():
    """The reference's internode_dispatch / internode_combine signatures (incl. the per-RDMA-rank
    histogram) are accepted and give exactly the intranode results inside one NVLink domain."""
    n, T, H, K = 2, 129, 512, 2
    E = n * 2
    bufs = get_buffers(n)
    xs, idxs, ws = make_inputs(n, T, H, K, E, seed=77)

    def fn(b):
        dev = b.device
        x, idx, w = xs[b.rank].to(dev), idxs[b.rank].to(dev), ws[b.rank].to(dev)
        tpr, tprr, tpe, in_rank, _ = b.get_dispatch_layout(idx, E)
        a = b.dispatch(x, num_tokens_per_rank=tpr, is_token_in_rank=in_rank, num_tokens_per_expert=tpe, topk_idx=idx,
                       topk_weights=w)
        torch.cuda.current_stream().synchronize()
        ref = (a[0].clone(), a[1].clone(), a[2].clone(), list(a[3]))
        c = b.internode_dispatch(x, None, tpr, tprr, in_rank, tpe, idx, w)
        torch.cuda.current_stream().synchronize()
        assert torch.equal(c[0], ref[0]) and torch.equal(c[1], ref[1]) and torch.equal(c[2], ref[2]) and c[3] == ref[3]
        cb = b.get_combine_buffer(c[0].size(0), H, K)
        cb.copy_(c[0])
        comb, _, _ = b.internode_combine(cb, c[4], topk_weights=c[2])
        torch.cuda.current_stream().synchronize()
        assert b.get_num_rdma_ranks() == 1
        return comb.cpu(), in_rank.cpu()

    for r, (comb, in_rank) in enumerate(run_threads(bufs, fn)):
        exp = xs[r].float() * in_rank.sum(1).float()[:, None]
        assert torch.allclose(comb.float(), exp, rtol=2e-2, atol=2e-1)


def test_dispatch_realistic_shape_single_rank():
    """EP=1 with the BASELINE shape (hidden 7168, top-8): pure local permutation + fused cast."""
    n = 1
    T, H, K, E = 512, 7168, 8, 32
    bufs = get_buffers(n, nbytes=128 << 20)
    xs, idxs, ws = make_inputs(n, T, H, K, E, seed=7)

    def fn(b):
        dev = b.device
        x, idx, w = xs[0].to(dev), idxs[0].to(dev), ws[0].to(dev)
        tpr, _, tpe, in_rank, _ = b.get_dispatch_layout(idx, E)
        (rx, rs), ridx, rw, pe, handle, _ = b.dispatch(x, num_tokens_per_rank=tpr, is_token_in_rank=in_rank,
                                                       num_tokens_per_expert=tpe, topk_idx=idx, topk_weights=w,
                                                       use_fp8=True)
        torch.cuda.current_stream().synchronize()
        ref_q, ref_s = per_token_cast_to_fp8(x[in_rank[:, 0]])
        assert torch.allclose(rs, ref_s, rtol=1e-6, atol=0)
        mism = (rx.view(torch.uint8) != ref_q.view(torch.uint8)).float().mean().item()
        assert mism < 1e-3, mism  # identical math up to rare 1-ulp ties
        out, _, _ = b.combine(per_token_cast_back(rx, rs), handle)
        torch.cuda.current_stream().synchronize()
        exp = per_token_cast_back(ref_q, ref_s).float()
        got = out[in_rank[:, 0]].float()
        bad = ~torch.isclose(got, exp, rtol=1e-2, atol=1e-1)  # only the rare fp8 rounding-tie elements may differ
        assert bad.float().mean().item() < 2e-3, bad.float().mean().item()
        return True

    assert run_threads(bufs, fn) == [True]


@pytest.mark.parametrize("n", [2, 4, 8])
@pytest.mark.parametrize("use_fp8", [True, False])
def test_low_latency_dispatch_combine(n, use_fp8):
    """Decode-shaped path: packed per-expert layout + weighted top-k combine
    (reference oracle: ep/bench/test_low_latency.py)."""
    T, H, K, M = 48, 1024, 4, 64
    E = n * 2
    E_local = E // n
    bufs = get_buffers(n)
    xs, idxs, ws = make_inputs(n, T, H, K, E, seed=100 + n)
    # allocate the LL regions up front (device-synchronising calls must not race with kernels of
    # other virtual ranks that are already spinning on this GPU)
    from uccl_b200.ep.low_latency import LowLatencyRuntime, ll_size_hint

    for b in bufs:
        if b._ll is None:
            with torch.cuda.device(b.device):
                b._ll = LowLatencyRuntime(b, ll_size_hint(M, H, n, 16))
    torch.cuda.synchronize()

    def fn(b):
        r, dev = b.rank, b.device
        x, idx, w = xs[r].to(dev), idxs[r].to(dev), ws[r].to(dev)
        recv_x, recv_count, handle, _, _ = b.low_latency_dispatch(x, idx, M, E, use_fp8=use_fp8)
        torch.cuda.current_stream().synchronize()
        if use_fp8:
            assert recv_x[1].shape == (E_local, n * M, H // 128) and recv_x[1].stride(1) == 1  # DeepEP's column-major view
        rx = per_token_cast_back(recv_x[0].view(-1, H), recv_x[1].reshape(-1, H // 128)).view(E_local, n * M, H) if use_fp8 else recv_x
        # "expert" = multiply by (global expert id + 1), written into the zero-copy combine buffer
        cb = b.get_next_low_latency_combine_buffer(handle)
        for el in range(E_local):
            cb[el].copy_((rx[el].float() * (r * E_local + el + 1)).to(torch.bfloat16))
        out, _, _ = b.low_latency_combine(cb, idx, w, handle)
        torch.cuda.current_stream().synchronize()
        return dict(rx=rx.cpu(), cnt=recv_count.cpu(), src=handle[0].cpu(), lr=handle[1].cpu(), out=out.cpu())

    outs = run_threads(bufs, fn)
    for r in range(n):
        o = outs[r]
        for el in range(E_local):
            e = r * E_local + el
            exp_cnt = sum(int((idxs[s] == e).sum()) for s in range(n))
            assert int(o["cnt"][el]) == exp_cnt
            begin = 0
            for s in range(n):
                sel = (idxs[s] == e).any(dim=1).nonzero().flatten()
                cnt = int(o["lr"][el, s] & 0xffffffff)
                beg = int(o["lr"][el, s] >> 32)
                assert cnt == sel.numel() and beg == begin
                got_src = o["src"][el, beg:beg + cnt].long()
                assert sorted(got_src.tolist()) == sorted(sel.tolist())  # slot order inside a (expert, rank) block is free
                want = xs[s][got_src]
                if use_fp8:
                    want = per_token_cast_back(*per_token_cast_to_fp8(want))
                    bad = ~torch.isclose(o["rx"][el, beg:beg + cnt].float(), want.float(), rtol=0.07, atol=0.05)
                    assert bad.float().mean().item() < 5e-3
                else:
                    assert torch.equal(o["rx"][el, beg:beg + cnt], want)
                begin += cnt
        # combine: sum_k w[t,k] * (e_k + 1) * x[t]   (entries with idx == -1 contribute nothing)
        base = xs[r].float() if not use_fp8 else per_token_cast_back(*per_token_cast_to_fp8(xs[r])).float()
        coef = (torch.where(idxs[r] >= 0, ws[r] * (idxs[r] + 1).float(), torch.zeros_like(ws[r]))).sum(1)
        exp_out = base * coef[:, None]
        bad = ~torch.isclose(o["out"].float(), exp_out, rtol=3e-2, atol=3e-1)
        assert bad.float().mean().item() < 5e-3, bad.float().mean().item()


def _ll_setup(n, M, H):
    from uccl_b200.ep.low_latency import LowLatencyRuntime, ll_size_hint

    bufs = get_buffers(n)
    for b in bufs:
        if b._ll is None:
            with torch.cuda.device(b.device):
                b._ll = LowLatencyRuntime(b, ll_size_hint(64, 1024, n, 16))
    torch.cuda.synchronize()
    return bufs


def _unpack_ue8m0(words, H):
    """[.., rows, H/512] int32 (4 exponent bytes per word) -> [.., rows, H/128] float32 power-of-two scales."""
    w = words.contiguous().to(torch.int64) & 0xffffffff
    ex = torch.stack([(w >> (8 * b)) & 0xff for b in range(4)], dim=-1).reshape(*words.shape[:-1], H // 128)
    return torch.pow(2.0, ex.float() - 127.0)


@pytest.mark.parametrize("n", [2, 4])
@pytest.mark.parametrize("variant", ["col_major", "row_major", "ue8m0"])
def test_low_latency_scale_layouts_hooks_and_stats(n, variant):
    """The fp8 scale layouts the kernel emits (DeepEP's column-major view, plain row-major, packed UE8M0), the
    SEND/RECV hook split (results must be bit-identical to the single-kernel path), a combine input that does not
    live in the symmetric buffer (occupied rows are packed in) and the wait-cost / receive-count statistics."""
    T, H, K, M = 40, 1024, 4, 64
    E = n * 2
    E_local = E // n
    bufs = _ll_setup(n, M, H)
    xs, idxs, ws = make_inputs(n, T, H, K, E, seed=300 + n)
    kw = dict(use_fp8=True)
    if variant == "row_major":
        kw["scales_row_major"] = True
    if variant == "ue8m0":
        kw.update(round_scale=True, use_ue8m0=True)

    def run(use_hook):
        def fn(b):
            r, dev = b.rank, b.device
            x, idx, w = xs[r].to(dev), idxs[r].to(dev), ws[r].to(dev)
            cum = torch.zeros(E_local, dtype=torch.int32, device=dev)
            dstat = torch.zeros(n, dtype=torch.int64, device=dev)
            cstat = torch.zeros(n, dtype=torch.int64, device=dev)
            (q, sc), cnt, handle, _, hook = b.low_latency_dispatch(
                x, idx, M, E, cumulative_local_expert_recv_stats=cum, dispatch_wait_recv_cost_stats=dstat,
                return_recv_hook=use_hook, **kw)
            assert (hook is not None) == use_hook
            if use_hook:
                hook()
            torch.cuda.current_stream().synchronize()
            if variant == "ue8m0":
                assert sc.dtype == torch.int32 and sc.shape == (E_local, n * M, H // 512) and sc.stride(1) == 1
                scf = _unpack_ue8m0(sc, H)
            else:
                assert sc.dtype == torch.float32 and sc.shape == (E_local, n * M, H // 128)
                assert sc.stride(1) == (H // 128 if variant == "row_major" else 1)
                scf = sc
            rx = per_token_cast_back(q.view(-1, H), scf.reshape(-1, H // 128).contiguous()).view(E_local, n * M, H)
            # expert outputs in an ORDINARY tensor (not the symmetric combine buffer): combine packs the occupied rows in
            eo = torch.zeros(E_local, n * M, H, dtype=torch.bfloat16, device=dev)
            for el in range(E_local):
                c = int(cnt[el])
                eo[el, :c] = (rx[el, :c].float() * (r * E_local + el + 1)).to(torch.bfloat16)
            out, _, chook = b.low_latency_combine(eo, idx, w, handle, return_recv_hook=use_hook,
                                                  combine_wait_recv_cost_stats=cstat)
            if use_hook:
                chook()
            torch.cuda.current_stream().synchronize()
            return dict(q=q.view(torch.uint8).cpu().clone(), sc=sc.cpu().clone(), cnt=cnt.cpu(), cum=cum.cpu(), out=out.cpu(),
                        src=handle[0].cpu().clone(), lr=handle[1].cpu(), dstat=dstat.cpu(), cstat=cstat.cpu())

        return run_threads(bufs, fn)

    plain = run(False)
    hooked = run(True)
    for r in range(n):
        a, h = plain[r], hooked[r]
        assert torch.equal(a["cnt"], h["cnt"]) and torch.equal(a["cum"], a["cnt"]) and torch.equal(a["lr"], h["lr"])
        assert (a["dstat"] >= 0).all() and (a["cstat"] >= 0).all() and int(a["dstat"][r]) == 0
        # combine: sum_k w[t,k] * (e_k + 1) * dequant(x[t])
        if variant == "ue8m0":
            base = xs[r].float()  # power-of-two scales: compare against the original with the e4m3 tolerance
        else:
            base = per_token_cast_back(*per_token_cast_to_fp8(xs[r])).float()
        coef = (torch.where(idxs[r] >= 0, ws[r] * (idxs[r] + 1).float(), torch.zeros_like(ws[r]))).sum(1)
        exp_out = base * coef[:, None]
        for o in (a, h):
            bad = ~torch.isclose(o["out"].float(), exp_out, rtol=8e-2 if variant == "ue8m0" else 3e-2, atol=3e-1)
            assert bad.float().mean().item() < 1e-2, bad.float().mean().item()
        # hash determinism across the hook / non-hook variants: identical rows per (expert, source rank) block as a
        # multiset (slot order inside a block is claimed atomically), identical combine output bit for bit
        assert torch.equal(a["out"], h["out"])
        for el in range(E_local):
            for s_ in range(n):
                beg, c = int(a["lr"][el, s_] >> 32), int(a["lr"][el, s_] & 0xffffffff)
                ka = sorted(zip(a["src"][el, beg:beg + c].tolist(), [hash(bytes(v.tolist())) for v in a["q"].view(E_local, n * M, H)[el, beg:beg + c]]))
                kh = sorted(zip(h["src"][el, beg:beg + c].tolist(), [hash(bytes(v.tolist())) for v in h["q"].view(E_local, n * M, H)[el, beg:beg + c]]))
                assert ka == kh


def test_low_latency_pressure_loop():
    """Back-to-back decode steps alternating hook / non-hook calls and both LL buffers (reference: the pressure
    mode of ep/bench/test_low_latency.py:619-622): epochs, parities and the pending-hook bookkeeping must hold."""
    n, T, H, K, M = 4, 32, 1024, 4, 64
    E = n * 2
    bufs = _ll_setup(n, M, H)
    xs, idxs, ws = make_inputs(n, T, H, K, E, seed=900)

    def fn(b):
        r, dev = b.rank, b.device
        x, idx, w = xs[r].to(dev), idxs[r].to(dev), ws[r].to(dev)
        first, prev = None, None
        for it in range(24):
            use_hook = it % 3 != 0
            rx, cnt, handle, _, hook = b.low_latency_dispatch(x, idx, M, E, use_fp8=False, return_recv_hook=use_hook)
            if prev is not None:  # a combine hook left pending was run by the dispatch call above
                if first is None:
                    first = prev.clone()
                assert torch.equal(prev, first), it
            if hook is not None:
                hook()
            cb = b.get_next_low_latency_combine_buffer(handle)
            cb.copy_(rx)
            out, _, chook = b.low_latency_combine(cb, idx, w, handle, return_recv_hook=use_hook)
            if chook is not None and it % 2 == 0:
                chook()
            prev = out
        b._ll._finish_pending()
        assert torch.equal(prev, first)
        torch.cuda.current_stream().synchronize()
        return first.cpu()

    outs = run_threads(bufs, fn)
    for r in range(n):
        coef = torch.where(idxs[r] >= 0, ws[r], torch.zeros_like(ws[r])).sum(1)
        assert torch.allclose(outs[r].float(), xs[r].float() * coef[:, None], rtol=3e-2, atol=3e-1)
