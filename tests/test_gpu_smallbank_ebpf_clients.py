"""-m gpu: the eBPF SmallBank tier (DINT_CFG_SMALLBANK_EBPF) under the transaction clients and across shards: clusters of
1 / 3 / 5 eBPF shards against one restatement per shard (tests/smallbank_ebpf_model.py) under the host SmallBank clients,
the GPU clients against the host clients and against a plain SmallBank cluster, the UDP front-end, and -- at the
reference's size, A = 24,000,000 -- shard 0's traffic of a populated and warmed three-shard cluster against the compiled
reference program populated and warmed the same way, then 600 rounds of 2^20 GPU clients with no error."""
import os
import socket
import subprocess
import time

import numpy as np
import pytest

import smallbank_ebpf_model as M
from dint_b200 import GpuCluster, GpuTxnClients, wire
from dint_b200.txn_workloads import Cluster, TxnWorkload
from golden_util import first_diff

pytestmark = pytest.mark.gpu
MSG = M.MSG
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "smallbank_ebpf")


def _models(G, n):
    oras = []
    for s in range(G):
        m = M.SmallbankEbpfModel(A=n, populated=n, shard=s, G=G)
        m.warmup()
        oras.append(m)
    return oras


@pytest.mark.parametrize("G", [1, 3, 5])
def test_cluster_serves_host_clients_like_one_model_per_shard(G):
    n, clients, rounds = 5000, 1300, 60
    cfg = dict(accts_sizing=n, accts_populate=n)

    def run(submit):
        wl = TxnWorkload(wire.SMALLBANK, n_clients=clients, n_shards=G, subscribers=n)
        trace = []
        for _ in range(rounds):
            rq, dst = wl.next()
            rs = submit(rq, dst)
            wl.feed(rs)
            trace.append((rq.copy(), dst.copy(), np.array(rs, copy=True)))
        return trace, wl.stats()

    oras = _models(G, n)
    want, st_want = run(Cluster([o.process for o in oras], MSG).submit)
    assert sum(o.stats["hits"] for o in oras) > 0 and sum(o.stats["write_backs"] for o in oras) > 0
    with GpuCluster(wire.SMALLBANK, G, devices=[0] * G, max_batch=4096, populate=True, smallbank_ebpf=True, **cfg) as cl:
        for s in range(G):
            assert cl.engine(s).smallbank_cache_stats() == _models(G, n)[s].stats, s
        got, st_got = run(lambda rq, dst: cl.submit(rq, dst))
        for r, ((q1, d1, s1), (q2, d2, s2)) in enumerate(zip(want, got)):
            assert np.array_equal(q1, q2) and np.array_equal(d1, d2), f"round {r}: clients diverged"
            assert first_diff(s2, s1, MSG) is None, f"round {r}: {first_diff(s2, s1, MSG)}"
        assert st_got == st_want
        for s in range(G):
            assert cl.engine(s).smallbank_cache_stats() == oras[s].stats, s


def test_gpu_clients_count_like_the_host_clients():
    n, clients, G, rounds = 5000, 2000, 3, 120
    oras = _models(G, n)
    ocl = Cluster([o.process for o in oras], MSG)
    wl = TxnWorkload(wire.SMALLBANK, n_clients=clients, n_shards=G, subscribers=n)
    with GpuCluster(wire.SMALLBANK, G, devices=[0] * G, populate=True, smallbank_ebpf=True, accts_sizing=n,
                    accts_populate=n) as cl:
        with GpuTxnClients(cl, clients, subscribers=n) as tc:
            for r in range(rounds):
                rq, dst = wl.next()
                if r % 10 == 0:
                    q, d, _ = tc.peek()
                    assert np.array_equal(q, rq) and np.array_equal(d, dst), f"round {r}: the clients diverged"
                wl.feed(ocl.submit(rq, dst))
                tc.run(1)
            st = tc.stats()
            assert {k: v for k, v in st.items() if k != "fallback_rounds"} == wl.stats()
            for s in range(G):
                assert cl.engine(s).smallbank_cache_stats() == oras[s].stats, s


@pytest.mark.parametrize("G", [3, 5])
def test_gpu_clients_see_the_plain_engine(G):
    """The clients' decisions depend only on the replies, and versions stay in step across replicas and between a set
    and its table -- so a commit miss's table version is the version the client sent, and the same GPU clients run
    byte-identical rounds on an eBPF cluster and on a plain SmallBank cluster, while the eBPF cluster's tier counts
    hits, table accesses and write-backs.  (One shard is left out: there a row is committed three times on one server,
    and the versions part.)"""
    n, clients, rounds = 20000, 8192, 150
    cfg = dict(accts_sizing=n, accts_populate=n)
    with GpuCluster(wire.SMALLBANK, G, devices=[0] * G, populate=True, smallbank_ebpf=True, **cfg) as ce, \
            GpuCluster(wire.SMALLBANK, G, devices=[0] * G, populate=True, **cfg) as cp:
        with GpuTxnClients(ce, clients, subscribers=n) as te, GpuTxnClients(cp, clients, subscribers=n) as tp:
            for r in range(rounds):
                te.run(1)
                tp.run(1)
                qe, de, re_ = te.peek()
                qp, dp, rp = tp.peek()
                assert np.array_equal(de, dp) and np.array_equal(qe, qp), f"round {r}: requests differ"
                assert first_diff(re_, rp, MSG) is None, f"round {r}: {first_diff(re_, rp, MSG)}"
            st = te.stats()
            assert st == tp.stats() and st["committed"] > 0
        for s in range(G):
            a, b = ce.engine(s).dump_log(), cp.engine(s).dump_log()
            assert a[1] == b[1] and np.array_equal(a[0], b[0]), s
            cs = ce.engine(s).smallbank_cache_stats()
            assert cs["hits"] > 0 and cs["table"] > 0 and cs["write_backs"] > 0, (s, cs)
            assert ce.engine(s).stats()["errors"] == 0


def test_udp_front_end_smallbank_ebpf():
    """dint_udp_server smallbank --smallbank-ebpf --populate P over loopback, one datagram at a time, against the model
    populated and warmed the same way (the golden's keys; requests the server refuses are left out)"""
    from dint_b200 import _build
    z = np.load(os.path.join(GOLDEN, "warm.npz"))
    P = int(z["populated"])
    rec = z["req"].reshape(-1, MSG)
    key = rec[:, 3:11].copy().view(np.uint64).reshape(-1)
    ok = ((rec[:, 2] < 2) & np.isin(rec[:, 1], [0, 1, 2, 3, 4, 5, 17]) & (key < P)) | (rec[:, 1] == 6)
    rec = rec[ok][:600]
    m = M.SmallbankEbpfModel(populated=P)
    m.warmup()
    want = m.process(rec.reshape(-1)).reshape(-1, MSG)
    assert (want[:, 1] != 0xFF).all()
    with socket.socket(socket.AF_INET, socket.SOCK_DGRAM) as s0:
        s0.bind(("127.0.0.1", 0))
        port = s0.getsockname()[1]
    args = [_build.UDP_SERVER, "smallbank", "--port", str(port), "--bind", "127.0.0.1", "--populate", str(P),
            "--smallbank-ebpf"]
    srv = subprocess.Popen(args, stderr=subprocess.PIPE)
    try:
        os.set_blocking(srv.stderr.fileno(), False)
        banner, t0 = b"", time.time()
        while b"sockets, batches" not in banner:           # printed once the engine exists and the sockets are bound
            assert srv.poll() is None and time.time() - t0 < 300, banner
            time.sleep(0.1)
            banner += srv.stderr.read() or b""
        c = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
        c.settimeout(5.0)
        c.connect(("127.0.0.1", port))
        got = np.empty_like(rec)
        for i in range(len(rec)):                           # one at a time: the replies depend on the order
            c.send(rec[i].tobytes())
            r = np.frombuffer(c.recv(256), dtype=np.uint8)
            assert r.size == MSG, (i, r.size)
            got[i] = r
        bad = np.flatnonzero((got != want).any(1))
        assert bad.size == 0, (bad.size, bad[:3])
    finally:
        srv.terminate()
        srv.wait(timeout=20)
    r = subprocess.run([_build.UDP_SERVER, "tatp", "--port", str(port), "--bind", "127.0.0.1", "--populate", "0",
                        "--smallbank-ebpf"], capture_output=True, timeout=120)
    assert r.returncode == 1 and b"dint_create failed" in r.stderr


@pytest.mark.skipif(not M.ref_available(), reason="oracle/_ref/smallbank_ebpf not built (reference sources absent)")
def test_full_size_shard0_equals_compiled_program_and_600_rounds():
    A, G, clients = M.REF_A, 3, 1 << 20
    per_rank = (clients + G - 1) // G
    with GpuCluster(wire.SMALLBANK, G, devices=[0] * G, max_batch=3 * per_rank, populate=True, smallbank_ebpf=True) as cl:
        c0 = cl.engine(0).smallbank_cache_stats()
        assert c0["table"] == c0["installs"] == 2 * A and c0["hits"] == 0
        wl = TxnWorkload(wire.SMALLBANK, n_clients=30000, n_shards=G, subscribers=A)
        stream, replies = [], []
        for _ in range(25):
            rq, dst = wl.next()
            rs = np.asarray(cl.submit(rq, dst)).reshape(-1, MSG)
            wl.feed(rs.reshape(-1))
            mine = np.asarray(dst) == 0
            stream.append(np.asarray(rq).reshape(-1, MSG)[mine])
            replies.append(rs[mine])
        stream, replies = np.concatenate(stream), np.concatenate(replies)
        assert len(stream) > 20000
        keys = stream[:, 3:11].copy().view(np.uint64).reshape(-1)
        tables = stream[:, 2]
        sel = tables < 2
        pick = np.unique(np.stack([keys[sel], tables[sel].astype(np.uint64)], 1), axis=0)[:3000]
        resp, sets, finds, locks, _ = M.run_ref_smallbank_ebpf(stream.reshape(-1), pick[:, 0], pick[:, 1], populate=A,
                                                             warmup=True, shard=0, G=G)
        assert first_diff(replies, resp, MSG) is None, first_diff(replies, resp, MSG)
        eng, H = cl.engine(0), M.hash_size(A)
        for i, (k, t) in enumerate(pick):
            k, t = int(k), int(t)
            h = M.fasthash64(k)
            assert np.array_equal(eng.smallbank_cache_set(t, h % H), sets[i]), i
            got = eng.kv_get(t, k)
            assert got is not None and finds[i]["found"] == 1 and got[1] == finds[i]["ver"], i
            assert bytes(got[0])[:8] == finds[i]["val"].tobytes(), i
            assert tuple(eng.lock_state(t, h % (4 * H))) == (locks[i]["num_ex"], locks[i]["num_sh"]), i
        with GpuTxnClients(cl, clients, subscribers=A) as tc:
            tc.run(600)
            assert tc.stats()["committed"] > 0
        for s in range(G):
            assert cl.engine(s).stats()["errors"] == 0, s
            assert cl.engine(s).smallbank_cache_stats()["hits"] > 0, s
