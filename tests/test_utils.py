"""CPU unit tests of the host utilities (rings, pool, histogram, seqnos, congestion control) --
the plain-`main` unit tests of the reference (include/util/util_test.cc, collective/*/timely_test.cc)."""
import pytest

from uccl_b200 import _native

U = _native.C().util


def test_spsc_ring_fifo_and_capacity():
    r = U.SpscRing(8)
    assert r.capacity == 8
    for i in range(8):
        assert r.push(i)
    assert not r.push(99)
    assert [r.pop() for _ in range(8)] == list(range(8))
    assert r.pop() is None
    for rnd in range(100):  # wrap-around
        assert r.push(rnd) and r.pop() == rnd


def test_mpmc_ring_concurrent_stress():
    r = U.MpmcRing(256)
    producers, consumers, per = 4, 3, 20000
    s, c = r.stress(producers, consumers, per)
    assert c == producers * per
    assert s == producers * per * (per + 1) // 2
    assert r.pop() is None


def test_shared_pool_recycles():
    p = U.SharedPool(64)
    for i in range(40):
        assert p.release_global(i)
    got = [p.get() for _ in range(40)]
    assert sorted(got) == list(range(40))
    assert p.get() is None
    for v in got:
        p.put(v)
    assert sorted(p.get() for _ in range(40)) == list(range(40))


def test_latency_hist_percentiles():
    h = U.LatencyHist()
    for v in range(1, 10001):
        h.record(v)
    assert h.count() == 10000 and h.min() == 1 and h.max() == 10000
    assert abs(h.mean() - 5000.5) < 1e-6
    for p, exp in ((50, 5000), (90, 9000), (99, 9900)):
        got = h.percentile(p)
        assert exp <= got <= exp * 1.07, (p, got)  # <= 1/16 relative bucket error
    assert "p99" in h.summary()


def test_seqno_wraparound():
    assert U.seqno_less(16, 65530, 5)      # 65530 is "before" 5 after wrap
    assert not U.seqno_less(16, 5, 65530)
    assert U.seqno_less(8, 250, 3)
    assert U.seqno_less(32, 1, 2)


def test_timely_reacts_to_rtt_gradient():
    t = U.Timely()
    r0 = t.rate_gbps()
    rtt = 10.0
    for _ in range(30):  # rising RTT inside [t_low, t_high] -> multiplicative decrease
        rtt += 1.5
        t.on_rtt(rtt)
    assert t.rate_gbps() < 0.5 * r0
    low = t.rate_gbps()
    for _ in range(200):  # RTT back at the floor -> additive (then hyper-active) increase
        t.on_rtt(3.0)
    assert t.rate_gbps() > low
    assert t.pacing_delay_us(1 << 20) > 0


def test_swift_window_tracks_target_delay():
    s = U.Swift()
    c0 = s.cwnd()
    now = 0.0
    for _ in range(50):
        now += 10.0
        s.on_ack(2.0, 1.0, now, 10.0)  # below target -> grow
    assert s.cwnd() > c0
    grown = s.cwnd()
    for _ in range(50):
        now += 10.0
        s.on_ack(500.0, 1.0, now, 10.0)  # far above target -> shrink (at most once per RTT)
    assert s.cwnd() < grown * 0.1
    assert s.target_delay_us() > 8.0  # flow scaling raises the target for tiny windows


def test_eqds_pacer_is_fair_and_rate_limited():
    p = U.EqdsPacer()
    for sender in range(4):
        p.add_demand(sender, 64 << 20)
    t, total = 0.0, 0
    for _ in range(2000):
        t += 1.0  # 1 us ticks; 900 GB/s -> 900 KB per tick ~ 13 credits of 64 KiB
        for sender, nbytes in p.tick(t):
            total += nbytes
            p.on_data(sender, nbytes)
    grants = [p.granted(s) for s in range(4)]
    assert sum(grants) == total
    assert max(grants) - min(grants) <= 2 * 65536   # round-robin fairness
    assert total <= 900e9 * 2000e-6 * 1.02          # never above line rate
    assert total >= min(4 * (64 << 20), 900e9 * 2000e-6 * 0.9)


# ------------------------------------------------------------------ stage-slice invariant
def _slices(C, msg, chunk, parts):
    """[(chunk index, block, lo, hi)] in 16-byte units for every chunk of a `msg`-byte message."""
    out = []
    base, k = 0, 0
    while base < msg:
        cb = min(chunk, msg - base)
        for b in range(parts):
            lo, hi = C.chunk_slice(msg, chunk, cb, parts, b)
            out.append((k, b, lo, hi))
        base += chunk
        k += 1
    return out


def test_chunk_slices_are_stable_across_chunks():
    """The chunked (staged) kernels only synchronise same-index blocks across ranks, so a block must
    own the same range of the staging area in every chunk: ranges of different blocks may never
    overlap across chunks (regression: a short tail chunk used to be re-sliced and a faster peer block of
    another index overwrote stage bytes still being read), and every chunk must be fully covered."""
    from hypothesis import given, settings
    from hypothesis import strategies as st

    from uccl_b200 import _native

    C = _native.C()

    @settings(max_examples=200, deadline=None)
    @given(chunk16=st.integers(1, 1 << 14), nfull=st.integers(0, 6), tail=st.integers(0, (1 << 18) - 1),
           parts=st.integers(1, 132))
    def prop(chunk16, nfull, tail, parts):
        chunk = chunk16 * 16
        msg = nfull * chunk + (tail % chunk)
        if msg == 0:
            msg = 1
        sl = _slices(C, msg, chunk, parts)
        nchunks = max(k for k, *_ in sl) + 1
        own = {}  # block -> union range over chunks
        for k, b, lo, hi in sl:
            assert lo <= hi
            if lo < hi:
                plo, phi = own.get(b, (lo, hi))
                own[b] = (min(plo, lo), max(phi, hi))
        # coverage of every chunk, in order, without gaps
        for k in range(nchunks):
            cb = min(chunk, msg - k * chunk)
            cu = (cb + 15) // 16
            pos = 0
            for kk, b, lo, hi in sl:
                if kk == k and lo < hi:
                    assert lo == pos
                    pos = hi
            assert pos == cu
        # ranges owned by different blocks (over all chunks) are disjoint
        spans = sorted(own.values())
        for (alo, ahi), (blo, bhi) in zip(spans, spans[1:]):
            assert ahi <= blo

    prop()
    # the concrete case that exposed the bug: 8 ranks, 1 MiB stage, 140002-byte pieces, 4 CTAs
    sl = _slices(C, 140002, 131072, 4)
    assert [s for s in sl if s[0] == 1 and s[2] < s[3]] == [(1, 0, 0, 559)]


def test_compression_strategy_selection(monkeypatch):
    from uccl_b200.p2p import compress

    monkeypatch.delenv("UCCL_B200_P2P_COMPRESS", raising=False)
    monkeypatch.delenv("UCCL_P2P_COMPRESS_STRATEGY", raising=False)
    assert compress.default_strategy() == "none"
    monkeypatch.setenv("UCCL_P2P_COMPRESS_STRATEGY", "split")  # the reference's names map onto our codec
    assert compress.default_strategy() == "for"
    monkeypatch.setenv("UCCL_B200_P2P_COMPRESS", "none")      # our own variable wins
    assert compress.default_strategy() == "none"
    monkeypatch.setenv("UCCL_B200_P2P_COMPRESS", "zstd")
    with pytest.raises(ValueError):
        compress.default_strategy()
    c = compress.Compressor("for")
    import torch

    assert not c.wants(torch.zeros(8))  # CPU tensors / small tensors are never compressed
    from uccl_b200 import _native

    C = _native.C()
    assert C.cmp_supported(9) and C.cmp_supported(7) and not C.cmp_supported(2)  # bf16, f32, not int32
    # worst case = header + metadata + raw planes + 8 exponent bits per element
    assert C.cmp_bound(4096, 9) >= 64 + 4096 + 4096 and C.cmp_bound(4096 * 3, 7) >= 3 * 4096 * 4


def test_mem_pool_needs_cuda_communicator():
    from uccl_b200 import Communicator

    c = Communicator.local_world(1, host=True, heap_bytes=128 << 20, stage_bytes=1 << 20)[0]
    with pytest.raises(RuntimeError):
        c.mem_pool()


def test_ue8m0_scale_packing_roundtrip():
    import torch

    from uccl_b200.ep import pack_ue8m0, unpack_ue8m0

    g = torch.Generator().manual_seed(3)
    exps = torch.randint(-40, 40, (3, 17, 56), generator=g)          # [experts, rows, hidden/128] for hidden 7168
    scales = torch.pow(torch.tensor(2.0), exps.float())
    packed = pack_ue8m0(scales)
    assert packed.dtype == torch.int32 and packed.shape == (3, 17, 14)
    assert packed.stride(-2) == 1 and packed.stride(-1) == 17           # column-major last two dimensions
    assert torch.equal(unpack_ue8m0(packed), scales)
    # byte i of word j is the biased exponent of scale 4j+i
    w = int(packed[1, 5, 2].item()) & 0xFFFFFFFF
    for i in range(4):
        assert (w >> (8 * i)) & 0xFF == int(exps[1, 5, 8 + i].item()) + 127


def test_tuning_table_from_sweep_and_env(tmp_path, monkeypatch):
    import torch

    from uccl_b200 import Communicator
    from uccl_b200.utils import tuner

    sweep = {"rows": [
        {"bytes": 4096, "oneshot_ll": {"us": 12.0}, "twoshot_p2p": {"us": 19.0}, "staged_p2p": {"us": 30.0}, "nccl": {"us": 25.0}},
        {"bytes": 1 << 20, "oneshot_ll": {"us": 40.0}, "twoshot_p2p@32": {"us": 22.0}, "twoshot_p2p@64": {"us": 21.0},
         "staged_p2p": {"us": 33.0}},
    ]}
    t = tuner.tuning_from_sweep(sweep)
    assert t["symmetric"] == [(4096, "oneshot_ll", -1, 12.0), (1 << 20, "twoshot_p2p", 64, 21.0)]
    assert t["plain"] == [(4096, "oneshot_ll", -1, 12.0), (1 << 20, "staged_p2p", -1, 33.0)]
    path = tmp_path / "tune.json"
    tuner.save_tuning(str(path), t, meta={"n_gpus": 2})
    c = Communicator.local_world(2, host=True, heap_bytes=128 << 20, stage_bytes=1 << 20)[0]
    monkeypatch.setenv("UCCL_B200_TUNE_FILE", str(path))
    assert tuner.load_tuning_from_env(c)
    assert c.select_allreduce(1 << 20, True, torch.bfloat16) == ("twoshot_p2p", 64)
    assert c.select_allreduce(2048, False, torch.bfloat16)[0] == "oneshot_ll"


def test_prometheus_exporter_renders_runtime_counters():
    import torch

    from uccl_b200 import Communicator
    from uccl_b200.p2p import Endpoint
    from uccl_b200.utils.metrics import MetricsExporter

    c = Communicator.local_world(1, host=True, heap_bytes=128 << 20, stage_bytes=1 << 20)[0]
    a, b = Endpoint(-1), Endpoint(-1)
    ok, conn = a.connect(remote_metadata=b.get_metadata())
    b.accept(5000)
    src, dst = torch.ones(256, dtype=torch.uint8), torch.zeros(256, dtype=torch.uint8)
    ok, rt = b.recv_async(1, 0, dst.data_ptr(), 256)
    assert a.send(conn, 0, src.data_ptr(), 256) and b.wait(rt, 5000)
    exp = MetricsExporter(rank=3)
    exp.watch_communicator(c)
    exp.watch_endpoint(a)
    exp.watch("custom", lambda: {"answer": 42})
    from uccl_b200 import net

    eng = net.Engine(bind_ip="127.0.0.1", paths=2)
    exp.watch_net_engine(eng)
    text = exp.render()
    assert 'uccl_b200_net_tx_pkts{rank="3"}' in text and 'uccl_b200_net_rto_rexmit{rank="3"}' in text
    assert 'uccl_b200_p2p_bytes_sent{rank="3"} 256.0' in text
    assert 'uccl_b200_comm_heap_free_bytes{rank="3"}' in text and 'uccl_b200_custom_answer{rank="3"} 42.0' in text


def test_ep_harness_helpers():
    import torch

    from uccl_b200.ep import utils as U

    a = torch.arange(1000, dtype=torch.float32)
    b = a.clone()
    b[17] = -1
    assert U.hash_tensor(a) == U.hash_tensor(a.clone()) != U.hash_tensor(b)
    assert U.hash_tensor(torch.ones(3, dtype=torch.uint8)) == 0x010101  # sizes that are not multiples of 8
    s = torch.rand(6, 8)
    g = U.create_grouped_scores(s, torch.tensor([[1, 3]] * 6), 4).view(6, 4, 2)
    assert bool((g[:, 0] == 0).all() and (g[:, 2] == 0).all() and (g[:, 1] == s.view(6, 4, 2)[:, 1]).all())
    x = torch.tensor([[3, 3, -1, 5], [0, 0, 0, -1]])
    U.inplace_unique(x, 8)
    assert sorted(v for v in x[0].tolist() if v >= 0) == [3, 5] and [v for v in x[1].tolist() if v >= 0] == [0]
    assert U.detect_group_topology() == (1, 1, 0, True) and U.initialize_uccl() == ([], None)
    with U.suppress_stdout_stderr():
        print("not shown")
    assert abs(U.calc_diff(a, a)) < 1e-9


def test_timing_wheel_never_fires_early_and_keeps_far_deadlines():
    """2000 random deadlines up to 8x the wheel's horizon, clock advanced in random steps: nothing fires before its
    deadline, nothing is lost, lateness is bounded by the step plus one slot."""
    import random

    from uccl_b200._native import C

    w = C().util.TimingWheel(1000, 64, 0)  # 1 us slots, 64 us horizon
    assert w.horizon_ns == 64_000
    rnd = random.Random(1)
    items = {i: rnd.randrange(0, 500_000) for i in range(2000)}
    for i, d in items.items():
        w.insert(d, i)
    fired, now = {}, 0
    while len(w):
        step = rnd.randrange(1, 5000)
        now += step
        for i in w.advance(now):
            assert i not in fired
            fired[i] = now
    assert set(fired) == set(items)
    assert min(fired[i] - items[i] for i in items) >= 0
    assert max(fired[i] - items[i] for i in items) <= 5000 + 1000


def test_ep_handle_has_the_reference_field_order():
    """Handles are 7-tuples in the reference's order (ep/bench/buffer.py:1147-1158) with the extras as attributes."""
    import torch

    from uccl_b200.ep.utils import EpHandle

    rp = torch.zeros(4, 4, dtype=torch.int32)
    src = torch.arange(5, dtype=torch.int32)
    inr = torch.zeros(7, 4, dtype=torch.bool)
    slot = torch.full((7, 4), -1, dtype=torch.int32)
    h = EpHandle(rp, 5, src, inr, slot, slot=1, num_topk=8)
    assert isinstance(h, tuple) and len(h) == 7
    rank_prefix, ch, rch, num_recv, recv_src_idx, is_in, send_head = h  # unpacks like the reference's handle
    assert rank_prefix is rp and num_recv == 5 and recv_src_idx is src and is_in is inr and send_head is slot
    assert ch.shape == (4, 1) and rch.shape == (4, 1)
    assert (h.slot, h.num_topk, h.num_recv) == (1, 8, 5) and h.send_slot is slot


def test_packaged_tuning_is_optional_and_env_can_disable_it(monkeypatch):
    from uccl_b200.utils import tuner

    assert tuner.packaged_tuning_path(8).endswith("tuning/tuning_8xH100.json")

    class FakeComm:
        world_size, is_host = 3, False  # no table is shipped for 3 ranks
        calls = []

        def set_tuning(self, sym, rows):
            self.calls.append((sym, rows))

    c = FakeComm()
    monkeypatch.delenv("UCCL_B200_TUNE_FILE", raising=False)
    assert tuner.load_tuning_from_env(c) is False and not c.calls
    monkeypatch.setenv("UCCL_B200_TUNE_FILE", "none")
    assert tuner.load_tuning_from_env(c) is False


def test_logfmt10_simulated_cast_properties():
    """Definition check of the LogFMT-10 simulated cast (reference: ep/src/internode_ll.cu:934-995)."""
    import torch

    from uccl_b200.ep.utils import logfmt10_simulate

    g = torch.Generator().manual_seed(5)
    x = (torch.randn(64, 512, generator=g) * 0.2).to(torch.bfloat16)
    x[0, :128] *= 40          # a group with |max| > 1 passes through untouched
    x[1, 128:256] = 0         # all-zero group
    x[2, 5] = 0               # a zero inside a live group stays zero
    x[3, 256:384] = 0.25      # a single magnitude: nothing to quantise
    q = logfmt10_simulate(x)
    assert q.dtype == torch.bfloat16 and q.shape == x.shape
    assert torch.equal(q[0, :128], x[0, :128]) and torch.equal(q[1, 128:256], x[1, 128:256])
    assert q[2, 5] == 0 and torch.equal(q[3, 256:384], x[3, 256:384])
    xf, qf = x.float(), q.float()
    assert torch.equal(torch.signbit(qf), torch.signbit(xf))
    live = (xf.reshape(64, 4, 128).abs().amax(-1, keepdim=True) <= 1).expand(64, 4, 128).reshape(64, 512) & (xf != 0)
    # one grid step is at most 32 / 510 octaves -> < 4.5 % relative error (plus bf16 rounding), except where the
    # magnitude falls below the clipped range (2^-32 of the group maximum), which random data never reaches
    rel = ((qf - xf).abs() / xf.abs())[live]
    assert float(rel.max()) < 0.05 and float(rel.mean()) > 1e-4
    # at most 2^9 - 1 magnitudes per group
    for grp in qf.reshape(-1, 128)[:16]:
        assert grp.abs().unique().numel() <= 511
    assert torch.equal(logfmt10_simulate(q), logfmt10_simulate(logfmt10_simulate(q)))  # stable under re-application


def test_region_index_matches_brute_force():
    """Containment lookup of registered regions (reference: interval tree in p2p/utils.py:114-206 and its
    test_util_interval_tree.py): randomized against a linear scan, with nested / overlapping / adjacent regions."""
    import random

    from uccl_b200.utils.regions import RegionIndex

    rng = random.Random(7)
    idx = RegionIndex()
    live = {}
    for step in range(3000):
        op = rng.random()
        if op < 0.45 or not live:
            start, size = rng.randrange(0, 5000), rng.randrange(1, 400)
            if (start, size) in live:
                continue
            live[(start, size)] = step
            idx.add(start, size, step)
        elif op < 0.6:
            (start, size), v = rng.choice(list(live.items()))
            assert idx.remove(start, size) == v
            del live[(start, size)]
        else:
            q, n = rng.randrange(0, 5400), rng.randrange(1, 64)
            cands = [(sz, s, v) for (s, sz), v in live.items() if s <= q and q + n <= s + sz]
            got = idx.find(q, n)
            if not cands:
                assert got is None
            else:
                assert got is not None and got[1] == min(c[0] for c in cands)
                assert (got[0], got[1]) in live and live[(got[0], got[1])] == got[2]
        assert len(idx) == len(live)
    assert idx.remove(10 ** 9) is None and idx.exact(10 ** 9) is None
    with pytest.raises(ValueError):
        idx.add(0, 0, 1)


def test_collective_registration_covers_views():
    """A view into a registered buffer resolves to the covering registration instead of registering again."""
    import torch

    from uccl_b200.collective import CollectiveContext

    class FakeEndpoint:
        def __init__(self):
            self.regs, self.deregs = [], []

        def reg(self, ptr, size, ftype=None):
            self.regs.append((ptr, size))
            return True, len(self.regs)

        def dereg(self, mr):
            self.deregs.append(mr)
            return True

    ctx = CollectiveContext.__new__(CollectiveContext)
    from uccl_b200.utils.regions import RegionIndex

    ctx._registered, ctx.ep = RegionIndex(), FakeEndpoint()
    big = torch.zeros(4096, dtype=torch.float32)
    mr = ctx.register_tensor(big)
    view = big[1024:2048]
    assert ctx.register_tensor(view) == mr and ctx.check_tensor_registered(view) == mr and len(ctx.ep.regs) == 1
    other = torch.zeros(16)
    assert ctx.check_tensor_registered(other) is None
    mr2 = ctx.register_tensor(other)
    assert mr2 != mr and len(ctx.ep.regs) == 2
    assert not ctx.deregister_tensor(view)          # a view does not own the registration
    assert ctx.deregister_tensor(big) and ctx.ep.deregs == [mr]
    assert ctx.check_tensor_registered(view) is None


def test_info_cli_reports_the_installation():
    import json
    import subprocess
    import sys

    import os

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "uccl_b200", "--json"], capture_output=True, text=True, timeout=300, cwd=root)
    assert r.returncode == 0, r.stderr
    d = json.loads(r.stdout)
    assert d["module_built"] and d["nccl_shim_built"] and d["native"]["max_ranks"] == 8
    assert "sm_90a" in d["arch_flags"] and isinstance(d["gpus"], list)


def test_perf_gate_flags_regressions(tmp_path):
    """scripts/perf_gate.py: the committed 1-GPU bench line passes against itself, a 20 % slower dispatch fails."""
    import json
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    base = os.path.join(root, "profiles", "bench1.json")
    gate = os.path.join(root, "scripts", "perf_gate.py")
    ok = subprocess.run([sys.executable, gate, base], capture_output=True, text=True)
    assert ok.returncode == 0 and "passed" in ok.stdout, ok.stdout + ok.stderr
    d = json.loads(open(base).read().strip().splitlines()[-1])
    d["dispatch_us"] *= 1.2
    worse = tmp_path / "worse.json"
    worse.write_text(json.dumps(d))
    bad = subprocess.run([sys.executable, gate, str(worse)], capture_output=True, text=True)
    assert bad.returncode == 1 and "REGRESSION" in bad.stdout
    d["dispatch_us"] /= 1.2 * 1.1  # faster than the baseline is fine
    worse.write_text(json.dumps(d))
    assert subprocess.run([sys.executable, gate, str(worse)], capture_output=True, text=True).returncode == 0


def test_lockfree_rings_and_pool_under_tsan(tmp_path):
    """tests/cpp/ring_pool_stress.cc: SPSC ring, 4x4 MPMC ring and the thread-cached pool under ThreadSanitizer --
    every item exactly once, per-producer order preserved, no token lost or duplicated."""
    import os
    import shutil
    import subprocess

    if shutil.which("g++") is None:
        pytest.skip("no host compiler")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "ring_pool_stress")
    b = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=thread", "-I" + os.path.join(root, "uccl_b200/csrc"),
                        os.path.join(root, "tests/cpp/ring_pool_stress.cc"), "-lpthread", "-o", exe],
                       capture_output=True, text=True, timeout=600)
    assert b.returncode == 0, b.stderr[-2000:]
    r = subprocess.run([exe, "100000"], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, TSAN_OPTIONS="halt_on_error=1 exitcode=66"))
    assert r.returncode == 0 and "ring_pool_stress: OK" in r.stdout, r.stdout[-1000:] + r.stderr[-3000:]


def test_logfmt10_kernel_arithmetic_matches_definition():
    """csrc/ep/ep_logfmt.h -- the lines `ep_ll_pack_logfmt_kernel` compiles (grid parameters, quantiser, bf16 rounding, sign
    packing) -- run on the host through `_C.ep_logfmt10_host` and compared with the PyTorch definition: bit-identical
    up to a handful of values that sit on a grid boundary (libm vs torch log2 / exp2)."""
    import torch

    from uccl_b200.ep.utils import logfmt10_simulate

    C = _native.C()
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(256, 1024, generator=g) * 0.2).to(torch.bfloat16)
    x[0, :128] *= 40
    x[1, 128:256] = 0
    x[2, 5] = 0
    x[3, 256:384] = 0.25
    x[4, :128] = -x[4, :128].abs()
    x[5, :128] *= 1e-6          # tiny magnitudes: the 2^-32 range clip is not reached, the grid still applies
    x[6, 0] = 1.0               # a group whose maximum is exactly the threshold
    ref = logfmt10_simulate(x)
    y = x.clone()
    C.ep_logfmt10_host(y.data_ptr(), y.size(0), y.size(1))
    same = y.view(torch.int16) == ref.view(torch.int16)
    assert float(same.float().mean()) > 0.9999
    if not bool(same.all()):
        rel = ((y.float() - ref.float()).abs() / ref.float().abs().clamp_min(1e-30))[~same]
        assert float(rel.max()) < 0.05  # one grid step
    assert torch.equal(y[0, :128], x[0, :128]) and torch.equal(torch.signbit(y.float()), torch.signbit(x.float()))
    with pytest.raises(RuntimeError):
        C.ep_logfmt10_host(y.data_ptr(), 1, 100)


def test_uccl_alias_package():
    """`uccl_b200.compat.install()`: code written against the reference's package names imports unchanged."""
    import importlib
    import sys

    import uccl_b200
    import uccl_b200.compat as compat

    assert "uccl" not in sys.modules or getattr(sys.modules["uccl"], "__uccl_b200_alias__", False)
    compat.install()
    try:
        import uccl
        from uccl import collective, p2p
        from uccl.ep import Buffer
        from uccl.p2p import Endpoint

        assert p2p is uccl_b200.p2p and collective is uccl_b200.collective and Buffer is uccl_b200.ep.Buffer
        assert Endpoint is uccl_b200.p2p.Endpoint and uccl.nccl_plugin_path() == uccl_b200.nccl_plugin_path()
        assert importlib.import_module("uccl.ep") is uccl_b200.ep
        with pytest.raises(NotImplementedError):
            uccl.rccl_plugin_path()
        assert compat.install() is uccl  # idempotent
    finally:
        compat.uninstall()
    assert "uccl" not in sys.modules and "uccl.p2p" not in sys.modules


def test_sm_partition_reports_unavailable_without_a_gpu():
    """SM partitions (green contexts) need a device: on a CPU box the probe says why and split raises."""
    import torch

    from uccl_b200.utils import SmPartition

    if torch.cuda.is_available():
        pytest.skip("GPU box: covered by tests/test_zzzz_gpu_sm_partition.py")
    ok, why = SmPartition.supported()
    assert not ok and why
    with pytest.raises(RuntimeError, match="unavailable"):
        SmPartition.split(24)
