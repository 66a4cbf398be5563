"""P2P engine in host mode (``Endpoint(-1)``): the TCP control plane, send/recv matching with advertised
receives, one-sided vector write/read against exchanged descriptors, async handles + polling, notifications
and error paths run exactly the production code; only the copy itself is a memcpy.  Mirrors the
reference's p2p/tests/test_engine_{send,read,write,metadata}.py without needing a GPU."""
import threading
import time

import pytest
import torch

from uccl_b200.p2p import Endpoint


def _pair():
    a, b = Endpoint(-1), Endpoint(-1)
    ok, conn = a.connect(remote_metadata=b.get_metadata())
    assert ok
    ok2, ip, gpu, conn_b = b.accept(5000)
    assert ok2 and gpu == -1
    return a, b, conn, conn_b


def test_host_metadata_and_connect():
    a, b, conn, conn_b = _pair()
    ip, port, gpu = Endpoint.parse_metadata(b.get_metadata())
    assert gpu == -1 and port > 0 and ip
    assert conn != 0 and conn_b != 0


@pytest.mark.parametrize("nbytes", [1, 4096, (3 << 20) + 5])
def test_host_send_recv(nbytes):
    a, b, conn, conn_b = _pair()
    src = torch.randint(0, 255, (nbytes,), dtype=torch.uint8)
    dst = torch.zeros(nbytes, dtype=torch.uint8)
    ok, rt = b.recv_async(conn_b, 0, dst.data_ptr(), nbytes)  # receiver advertises first ...
    assert ok
    assert a.send(conn, 0, src.data_ptr(), nbytes)              # ... the sender's engine matches and copies
    assert b.wait(rt, 10000)
    assert torch.equal(dst, src)
    # the other order: send posted before the receive exists
    dst2 = torch.zeros(nbytes, dtype=torch.uint8)
    ok, st = a.send_async(conn, 0, src.data_ptr(), nbytes)
    assert ok
    time.sleep(0.05)
    assert b.recv(conn_b, 0, dst2.data_ptr(), nbytes)
    assert a.wait(st, 10000)
    assert torch.equal(dst2, src)
    assert a.stats()["bytes_sent"] == 2 * nbytes and b.stats()["bytes_received"] == 2 * nbytes


def test_host_onesided_vector_ops_and_polling():
    a, b, conn, conn_b = _pair()
    sizes = [1000, 33, 1 << 18, 7]
    srcs = [torch.full((s,), i + 1, dtype=torch.uint8) for i, s in enumerate(sizes)]
    dsts = [torch.zeros(s, dtype=torch.uint8) for s in sizes]
    remote = a.deserialize_descs(b.get_serialized_descs(b.register_memory(dsts)))
    local = a.register_memory(srcs)
    ok, tid = a.transfer(conn, "write", local, remote)
    assert ok and a.wait(tid, 10000)
    for i, d in enumerate(dsts):
        assert bool((d == i + 1).all())
    back = [torch.zeros(s, dtype=torch.uint8) for s in sizes]
    ok, tid = a.transfer(conn, "read", a.register_memory(back), remote)
    assert ok
    done = False
    for _ in range(100000):
        ok, done = a.poll_async(tid)
        assert ok
        if done:
            break
    assert done
    for i, d in enumerate(back):
        assert bool((d == i + 1).all())
    ok, _ = a.poll_async(tid)  # handles are released once reported done
    assert not ok
    # a raw write larger than the advertised window is refused (transfer() itself clips to the window)
    big = torch.zeros(sizes[1] + 1, dtype=torch.uint8)
    ok, _ = a.write_async(conn, 0, big.data_ptr(), big.numel(), remote[1])
    assert not ok
    assert a.stats()["bytes_written"] == sum(sizes) and a.stats()["bytes_read"] == sum(sizes)


def test_host_notifications_and_wait_timeout():
    a, b, conn, conn_b = _pair()
    assert a.send_notif(conn, b"kv-ready:42")
    got = []
    t0 = time.time()
    while not got and time.time() - t0 < 5:
        got = b.get_notifs()
        time.sleep(0.005)
    assert got and got[0][1] == b"kv-ready:42"
    # a receive nobody sends to: wait() returns False after the timeout, the handle stays valid
    dst = torch.zeros(16, dtype=torch.uint8)
    ok, rt = b.recv_async(conn_b, 0, dst.data_ptr(), 16)
    assert ok
    t0 = time.time()
    assert not b.wait(rt, 150)
    assert 0.1 < time.time() - t0 < 2.0
    src = torch.ones(16, dtype=torch.uint8)
    assert a.send(conn, 0, src.data_ptr(), 16) and b.wait(rt, 5000) and bool((dst == 1).all())
    assert not b.wait(12345678, 10)  # unknown transfer id


def test_host_concurrent_streams_of_messages():
    """Several in-flight sends and receives on one connection complete in order of their sequence numbers."""
    a, b, conn, conn_b = _pair()
    n = 32
    srcs = [torch.full((1000 + i,), i, dtype=torch.uint8) for i in range(n)]
    dsts = [torch.zeros(1000 + i, dtype=torch.uint8) for i in range(n)]
    rts = []

    def receiver():
        for d in dsts:
            ok, rt = b.recv_async(conn_b, 0, d.data_ptr(), d.numel())
            assert ok
            rts.append(rt)

    th = threading.Thread(target=receiver)
    th.start()
    sts = []
    for s in srcs:
        ok, st = a.send_async(conn, 0, s.data_ptr(), s.numel())
        assert ok
        sts.append(st)
    th.join()
    for st in sts:
        assert a.wait(st, 10000)
    for rt in rts:
        assert b.wait(rt, 10000)
    for i, d in enumerate(dsts):
        assert bool((d == i).all())


def test_uccl_engine_c_api_host_mode(tmp_path):
    """The NIXL-plugin C surface (`uccl_engine_*`) driven from C++ against two host-mode engines."""
    import os
    import subprocess

    from uccl_b200 import _build

    _build.build()
    lib = _build.nccl_shim_path()  # carries the whole native core incl. the engine C API
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = tmp_path / "uccl_engine_test"
    cmd = ["g++", "-std=c++17", "-O1", os.path.join(root, "tests/cpp/uccl_engine_test.cc"),
           "-I" + os.path.join(root, "uccl_b200/csrc/p2p"), "-L" + str(lib.parent), "-luccl_b200_nccl",
           "-Wl,-rpath," + str(lib.parent), "-lpthread", "-o", str(exe)]
    subprocess.run(cmd, check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "uccl_engine_test: OK" in r.stdout, r.stdout + r.stderr


def _tcp_server(q_md, q_res, nbytes):
    import time

    import torch

    from uccl_b200.p2p import Endpoint

    e = Endpoint(-1)
    q_md.put(e.get_metadata())
    ok, ip, gpu, conn = e.accept(60000)
    buf = torch.zeros(nbytes, dtype=torch.uint8)
    win = torch.full((nbytes,), 7, dtype=torch.uint8)
    inbox = torch.zeros(nbytes, dtype=torch.uint8)
    okr = e.recv(conn, 0, buf.data_ptr(), nbytes)                 # two-sided receive (payload arrives over TCP)
    descs = e.register_memory([win, inbox])
    secret = torch.full((4096,), 9, dtype=torch.uint8)             # never registered / advertised
    e.send_notif(conn, e.get_serialized_descs(descs) + secret.data_ptr().to_bytes(8, "little"))
    back = torch.arange(1000, dtype=torch.int32)
    oks = e.send(conn, 0, back.data_ptr(), 4000)                  # and a message in the other direction
    t0 = time.time()
    fin = False
    while time.time() - t0 < 60 and not fin:
        for _, m in e.get_notifs():
            fin = fin or m == b"done"
        time.sleep(0.002)
    q_res.put((bool(ok), bool(okr), int(buf.sum().item()), bool(oks), int(inbox.to(torch.int64).sum().item()), fin,
               int(secret.to(torch.int64).sum().item())))


def _tcp_client(q_md, q_res, nbytes):
    import time

    import torch

    from uccl_b200.p2p import Endpoint

    e = Endpoint(-1)
    ok, conn = e.connect(remote_metadata=q_md.get(timeout=60))
    src = torch.ones(nbytes, dtype=torch.uint8)
    oks = e.send(conn, 0, src.data_ptr(), nbytes)
    blob = None
    t0 = time.time()
    while blob is None and time.time() - t0 < 60:
        for _, m in e.get_notifs():
            blob = m
        time.sleep(0.002)
    secret_addr = int.from_bytes(blob[-8:], "little")
    remote = e.deserialize_descs(blob[:-8])
    dst = torch.zeros(nbytes, dtype=torch.uint8)
    okr = e.read(conn, 0, dst.data_ptr(), nbytes, remote[0])       # one-sided read of the server's window
    three = torch.full((nbytes,), 3, dtype=torch.uint8)
    okw = e.write(conn, 0, three.data_ptr(), nbytes, remote[1])    # one-sided write, acknowledged by a flush
    got = torch.zeros(1000, dtype=torch.int32)
    okb = e.recv(conn, 0, got.data_ptr(), 4000)
    # a forged descriptor that points at memory the server never exposed: the write is dropped, the read refused
    from uccl_b200.p2p import XferDesc

    forged = bytearray(remote[1].raw)
    forged[72:80] = secret_addr.to_bytes(8, "little")
    forged[80:88] = (4096).to_bytes(8, "little")
    forged = XferDesc(bytes(forged))
    evil = torch.full((4096,), 1, dtype=torch.uint8)
    e.write(conn, 0, evil.data_ptr(), 4096, forged)
    leak = torch.zeros(4096, dtype=torch.uint8)
    ok_leak = e.read(conn, 0, leak.data_ptr(), 4096, forged)
    e.send_notif(conn, b"done")
    q_res.put((bool(ok), bool(oks), bool(okr), int(dst.to(torch.int64).sum().item()), bool(okw), bool(okb),
               bool(torch.equal(got, torch.arange(1000, dtype=torch.int32))), bool(ok_leak), int(leak.sum().item())))
    time.sleep(0.3)


def test_host_mode_between_processes_uses_the_tcp_data_path():
    """Two processes without any shared memory: payloads of send/recv, one-sided write (+flush/ack) and
    one-sided read (request/response) travel on the control connection (the reference's TCP backend role)."""
    import multiprocessing as mp

    nbytes = (3 << 20) + 17
    ctx = mp.get_context("spawn")
    q_md, q_s, q_c = ctx.Queue(), ctx.Queue(), ctx.Queue()
    ps = [ctx.Process(target=_tcp_server, args=(q_md, q_s, nbytes)), ctx.Process(target=_tcp_client, args=(q_md, q_c, nbytes))]
    [p.start() for p in ps]
    rs = q_s.get(timeout=180)
    rc = q_c.get(timeout=180)
    [p.join(30) for p in ps]
    assert rs == (True, True, nbytes, True, 3 * nbytes, True, 9 * 4096)     # the unexposed buffer is untouched
    assert rc == (True, True, True, 7 * nbytes, True, True, True, False, 0)  # and could not be read either


def _coll_worker(rank, world, port, q):
    import os

    import torch
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from uccl_b200 import collective as C

    ctx = C.init_collective(local_gpu_idx=-1, heap_bytes=128 << 20)
    peer = 1 - rank
    x = torch.full((5000,), float(rank + 1))
    y = torch.zeros(5000)
    if rank == 0:
        C.send(x, peer)
        C.recv(y, peer)
    else:
        C.recv(y, peer)
        C.send(x, peer)
    ok_sr = bool((y == peer + 1).all())
    # non-blocking + batch (ring step) + registration bookkeeping
    C.register_tensor(x)
    z = torch.zeros(5000)
    hs = C.batch_isend_irecv([ctx.P2POp("irecv", z, peer), ctx.P2POp("isend", x, peer)])
    C.wait_all(hs)
    ok_batch = bool((z == peer + 1).all()) and ctx.check_tensor_registered(x) is not None
    g = torch.zeros(2 * 5000)
    C.allgather(x, g)
    ok_ag = bool((g.view(2, -1)[0] == 1).all() and (g.view(2, -1)[1] == 2).all())
    a = torch.full((64,), float(rank))
    C.all_reduce(a, "sum")
    ok_ar = bool((a == 1.0).all())
    C.barrier()
    C.finalize_collective()
    q.put((rank, ok_sr, ok_batch, ok_ag, ok_ar))
    dist.destroy_process_group()


def test_collective_context_on_cpu_two_processes():
    """`uccl_b200.collective` (the `uccl.collective` surface: send/recv, isend/irecv, batch, allgather, native
    collectives) with host-mode endpoints and the host communicator, two processes rendezvousing over gloo."""
    import multiprocessing as mp
    import socket

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_coll_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in ps]
    got = sorted(q.get(timeout=240) for _ in range(2))
    [p.join(60) for p in ps]
    assert got == [(0, True, True, True, True), (1, True, True, True, True)]


def test_registration_type_tags_and_handles():
    """FloatType tags travel with registrations (reference: p2p/engine_api.cc:171-177,279-293), XferHandle / repr."""
    import torch

    from uccl_b200.p2p import Endpoint, FloatType, XferHandle

    e = Endpoint(-1)
    t = torch.zeros(64, dtype=torch.bfloat16)
    ok, mr = e.reg(t.data_ptr(), t.numel() * 2, FloatType.kBFloat16)
    assert ok and e.float_type(mr) == FloatType.kBFloat16
    ok2, mr2 = e.reg(t.data_ptr(), 16)
    assert ok2 and e.float_type(mr2) == FloatType.kUndefined
    d = e.register_memory([torch.zeros(8, dtype=torch.float32), torch.zeros(8, dtype=torch.int32)])
    assert e.float_type(d[0].mr_id) == FloatType.kFloat32 and e.float_type(d[1].mr_id) == FloatType.kUndefined
    e.dereg(mr)
    assert e.float_type(mr) == FloatType.kUndefined
    assert FloatType.from_tensor(torch.zeros(1, dtype=torch.float8_e4m3fn)) == FloatType.kFloat8E4M3FN
    h = XferHandle(3, "write", 17)
    assert h.conn_id == 3 and h.op_name == "write" and h.transfer_id == 17
    assert "host mode" in repr(e)


@pytest.mark.parametrize("san", ["thread", "address,undefined"])
def test_engine_concurrency_stress_under_sanitizers(tmp_path, san):
    """tests/cpp/p2p_engine_stress.cc: two-sided stream + one-sided vector writes / reads + notifications + connection
    churn at the same time between two host-mode endpoints, built with TSan resp. ASan + UBSan straight from the
    engine's sources (the copy kernel is stubbed: host mode never launches it).  TSan found -- and this test now
    guards -- the descriptor close racing with the engine thread's read and the unsynchronised transfer state."""
    import os
    import shutil
    import subprocess

    cudart = "/usr/local/cuda/lib64"
    if shutil.which("g++") is None or not os.path.exists(os.path.join(cudart, "libcudart.so")):
        pytest.skip("needs g++ and the CUDA runtime library")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    csrc = os.path.join(root, "uccl_b200", "csrc")
    exe = str(tmp_path / "p2p_engine_stress")
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-fsanitize=" + san, "-I" + csrc, "-I" + os.path.join(csrc, "p2p"),
           "-I/usr/local/cuda/include", os.path.join(root, "tests/cpp/p2p_engine_stress.cc"),
           os.path.join(root, "tests/cpp/p2p_kernel_stub.cc"), os.path.join(csrc, "p2p/endpoint.cc"), "-o", exe,
           "-L" + cudart, "-Wl,-rpath," + cudart, "-lcudart", "-lpthread"]
    b = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert b.returncode == 0, b.stderr[-3000:]
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0", TSAN_OPTIONS="halt_on_error=1 exitcode=66")
    r = subprocess.run([exe, "80"], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and "p2p_engine_stress: OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_endpoint_signature_audit_against_the_reference_binding():
    """Every method of the reference's nanobind `Endpoint` (p2p/engine_api.cc) exists with the same keyword names
    (`nb::arg(...)`) in the same order.  The binding's argument lists are stored in
    tests/golden/reference_signatures.json (oracle/extract_signatures.py)."""
    import inspect

    from helpers import reference_signatures
    from uccl_b200 import p2p
    from uccl_b200.p2p import Endpoint

    checked = 0
    for name, want in reference_signatures()["p2p_endpoint"].items():
        assert hasattr(Endpoint, name), f"Endpoint.{name} missing"
        if name == "get_metadata":
            continue  # the reference fills a caller-provided vector; here the bytes are returned
        have = [p for p in inspect.signature(getattr(Endpoint, name)).parameters if p != "self"]
        pos = [h for h in have]
        for i, w in enumerate(want):
            assert w in have, f"Endpoint.{name}: no parameter {w!r} (has {have})"
            if w not in ("remote_gpu_bdf",):  # an alias keyword placed after this library's own name for it
                assert pos.index(w) == i, f"Endpoint.{name}: {w!r} is argument {pos.index(w)}, the reference has it at {i}"
        checked += 1
    assert checked > 40 and hasattr(p2p, "get_oob_ip")
    e = Endpoint(-1)
    assert e.conn_id_of_rank(3) == 2 ** 64 - 1
    e.set_rank_conn(3, 17)
    assert e.conn_id_of_rank(3) == 17


def test_collective_signature_audit_against_the_reference():
    """Module functions and `CollectiveContext` methods of the reference's `uccl.collective` (p2p/collective.py) exist
    here with the same parameter names (stored in tests/golden/reference_signatures.json)."""
    import inspect

    import uccl_b200.collective as c
    from helpers import reference_signatures

    ref = reference_signatures()["collective"]
    n = 0
    for name, want in ref["functions"].items():
        have = list(inspect.signature(getattr(c, name)).parameters)
        assert not [p for p in want if p not in have], (name, want, have)
        n += 1
    for name, want in ref["CollectiveContext"].items():
        have = list(inspect.signature(getattr(c.CollectiveContext, name)).parameters)
        assert not [p for p in want if p not in have], (name, want, have)
        n += 1
    assert n > 25


def test_p2p_utils_helpers():
    """uccl_b200.p2p.utils: the helpers the reference ships next to its engine (p2p/utils.py)."""
    import random
    import socket
    import threading

    from uccl_b200.p2p.utils import (ClosedIntervalTree, create_socket_and_connect, recv_obj, send_obj,
                                     set_files_limit)

    soft, hard = set_files_limit(verbose=False)
    assert soft == hard or soft == -1
    # framed pickles over a real TCP connection made by the retrying connect (listener comes up late)
    srv = socket.socket()
    srv.bind(("127.0.0.1", 0))
    port = srv.getsockname()[1]
    got = {}

    def serve():
        import time

        time.sleep(0.3)
        srv.listen(1)
        c, _ = srv.accept()
        got["obj"] = recv_obj(c)
        got["none"] = recv_obj(c)
        send_obj(c, {"ok": True, "blob": b"x" * 100000})
        c.close()

    t = threading.Thread(target=serve)
    t.start()
    s = create_socket_and_connect("127.0.0.1", port, max_retries=20, initial_delay=0.05, backoff=1.5, max_delay=0.2)
    send_obj(s, ("meta", [1, 2, 3]))
    s.sendall(b"\x00" * 8)  # zero-length frame
    back = recv_obj(s)
    t.join()
    s.close()
    srv.close()
    assert got["obj"] == ("meta", [1, 2, 3]) and got["none"] is None and back["ok"] and len(back["blob"]) == 100000
    with pytest.raises(OSError):
        create_socket_and_connect("127.0.0.1", port, max_retries=1, initial_delay=0.01)
    # closed-interval index against brute force
    rng = random.Random(3)
    for _ in range(50):
        tree, ref = ClosedIntervalTree(), []
        for _ in range(rng.randint(1, 25)):
            a = rng.randint(0, 40)
            b = a + rng.randint(0, 15)
            d = rng.randint(0, 2)
            tree.add(a, b, d)
            ref.append((a, b, d))
        a, b, d = rng.choice(ref)
        n = tree.remove(a, b, d)
        assert n == sum(1 for r in ref if r == (a, b, d))
        ref = [r for r in ref if r != (a, b, d)]
        for _ in range(10):
            qa = rng.randint(0, 45)
            qb = qa + rng.randint(0, 10)
            assert sorted(tree.query_containing(qa, qb)) == sorted(r for r in ref if r[0] <= qa and r[1] >= qb)
            assert sorted(tree.query_overlap(qa, qb)) == sorted(r for r in ref if r[0] <= qb and r[1] >= qa)
            assert sorted(tree.query_exact_match(qa, qb)) == sorted(r for r in ref if r[:2] == (qa, qb))
        assert sorted(tree) == sorted(ref) and len(tree) == len(ref)
    with pytest.raises(ValueError):
        ClosedIntervalTree().add(5, 4, None)
