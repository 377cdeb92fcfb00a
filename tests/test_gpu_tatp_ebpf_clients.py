"""-m gpu: the eBPF TATP tier (DINT_CFG_TATP_EBPF) under the transaction clients and across shards: clusters of 1 / 3 / 5
eBPF shards against one restatement per shard (tests/tatp_ebpf_model.py) under the host TATP clients, the GPU clients
against the host clients, the UDP front-end, and -- at the reference's size, S = 7,000,000 -- shard 0's traffic of a
three-shard cluster against the compiled reference program populated the same way, then 600 rounds of 2^20 GPU
clients with no chain entry refused."""
import os
import socket
import subprocess
import time

import numpy as np
import pytest

import tatp_ebpf_model as M
from dint_b200 import GpuCluster, GpuTxnClients, wire
from dint_b200.txn_workloads import Cluster, TxnWorkload
from golden_util import first_diff

pytestmark = pytest.mark.gpu
MSG = M.MSG
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tatp_ebpf")


def _models(G, n, hk):
    oras = []
    for s in range(G):
        m = M.TatpEbpfModel(holder_keys=hk, S=n)
        m.populate(n, shard=s, G=G)
        oras.append(m)
    return oras


def test_single_shard_cluster_equals_model():
    """one eBPF shard fed the colliding-key trace directly (one shard cannot serve the transaction clients: a backup
    commit would meet the primary's own lock)"""
    n = 1500
    m = _models(1, n, True)[0]
    req = M.random_trace(M.colliding_groups(n, per_bucket=8, n_buckets=5, seed=3), 6000, seed=4)
    with GpuCluster(wire.TATP, 1, devices=[0], max_batch=8192, populate=True, tatp_ebpf=True, lock_holder_keys=True,
                    subs_sizing=n, subs_populate=n) as cl:
        got = cl.submit(req, np.zeros(req.size // MSG, dtype=np.uint8), check=False)
        assert first_diff(got, m.process(req), MSG) is None
        assert cl.engine(0).tatp_cache_stats() == m.stats


@pytest.mark.parametrize("G", [3, 5])
def test_cluster_serves_host_clients_like_one_model_per_shard(G):
    n, clients, rounds = 1500, 1300, 60
    cfg = dict(subs_sizing=n, subs_populate=n)

    def run(submit):
        wl = TxnWorkload(wire.TATP, n_clients=clients, n_shards=G, subscribers=n)
        trace = []
        for _ in range(rounds):
            rq, dst = wl.next()
            rs = submit(rq, dst)
            wl.feed(rs)
            trace.append((rq.copy(), dst.copy(), np.array(rs, copy=True)))
        return trace, wl.stats(), wl.lock_stats()

    oras = _models(G, n, True)
    want, st_want, ls_want = run(Cluster([o.process for o in oras], MSG).submit)
    assert sum(o.stats["table"] for o in oras) > 0 and sum(o.stats["hits"] for o in oras) > 0
    with GpuCluster(wire.TATP, G, devices=[0] * G, max_batch=4096, populate=True, tatp_ebpf=True, lock_holder_keys=True,
                    **cfg) as cl:
        got, st_got, ls_got = run(lambda rq, dst: cl.submit(rq, dst))
        for r, ((q1, d1, s1), (q2, d2, s2)) in enumerate(zip(want, got)):
            assert np.array_equal(q1, q2) and np.array_equal(d1, d2), f"round {r}: clients diverged"
            assert first_diff(s2, s1, MSG) is None, f"round {r}: {first_diff(s2, s1, MSG)}"
        assert st_got == st_want and ls_got == ls_want
        for s in range(G):
            assert cl.engine(s).tatp_cache_stats() == oras[s].stats, s


def test_gpu_clients_count_like_the_host_clients():
    n, clients, G, rounds = 1500, 2000, 3, 120
    oras = _models(G, n, True)
    ocl = Cluster([o.process for o in oras], MSG)
    wl = TxnWorkload(wire.TATP, n_clients=clients, n_shards=G, subscribers=n)
    with GpuCluster(wire.TATP, G, devices=[0] * G, populate=True, tatp_ebpf=True, lock_holder_keys=True,
                    subs_sizing=n, subs_populate=n) as cl:
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
            assert tc.lock_stats() == wl.lock_stats()
            for s in range(G):
                assert cl.engine(s).tatp_cache_stats() == oras[s].stats, s


@pytest.mark.parametrize("variant", M.VARIANTS)
def test_udp_front_end_tatp_ebpf(variant):
    """dint_udp_server tatp --tatp-ebpf [--lock-holder-keys] over loopback, at the reference's sizes"""
    from dint_b200 import _build
    g = np.load(os.path.join(GOLDEN, f"{variant}.npz"))
    rec = g["req"].reshape(-1, MSG)
    ok = (rec[:, 2] < 5) & np.isin(rec[:, 1], [0, 1, 2, 12, 13, 18, 19, 22, 23]) | np.isin(rec[:, 1], [14, 24])
    rec = rec[ok][:500]
    want = M.TatpEbpfModel(holder_keys=variant == "lock").process(rec.reshape(-1)).reshape(-1, MSG)
    with socket.socket(socket.AF_INET, socket.SOCK_DGRAM) as s0:
        s0.bind(("127.0.0.1", 0))
        port = s0.getsockname()[1]
    args = [_build.UDP_SERVER, "tatp", "--port", str(port), "--bind", "127.0.0.1", "--populate", "0", "--tatp-ebpf"]
    srv = subprocess.Popen(args + (["--lock-holder-keys"] if variant == "lock" else []), stderr=subprocess.PIPE)
    try:
        os.set_blocking(srv.stderr.fileno(), False)
        banner, t0 = b"", time.time()
        while b"sockets, batches" not in banner:           # printed once the engine exists and the sockets are bound
            assert srv.poll() is None and time.time() - t0 < 120, banner
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
    r = subprocess.run([_build.UDP_SERVER, "store", "--port", str(port), "--bind", "127.0.0.1", "--tatp-ebpf"],
                       capture_output=True, timeout=120)
    assert r.returncode == 1 and b"dint_create failed" in r.stderr


@pytest.mark.skipif(not M.ref_available(), reason="oracle/_ref/tatp_ebpf_* not built (reference sources absent)")
def test_full_size_shard0_equals_compiled_program_and_600_rounds_allocate():
    S, G, clients = M.REF_S, 3, 1 << 20
    per_rank = (clients + G - 1) // G
    with GpuCluster(wire.TATP, G, devices=[0] * G, max_batch=3 * per_rank, populate=True, tatp_ebpf=True) as cl:
        wl = TxnWorkload(wire.TATP, n_clients=30000, n_shards=G, subscribers=S)
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
        pick = np.unique(np.stack([keys, tables.astype(np.uint64)], 1), axis=0)[:3000]
        resp, sets, chains, finds, _, _ = M.run_ref_tatp_ebpf("shard", stream.reshape(-1), pick[:, 0], pick[:, 1],
                                                              populate=S, shard=0)
        assert first_diff(replies, resp, MSG) is None, first_diff(replies, resp, MSG)
        eng, H = cl.engine(0), M.hash_sizes(S)
        for i, (k, t) in enumerate(pick):
            b = M.fasthash64(int(k)) % H[int(t)]
            assert np.array_equal(eng.tatp_cache_set(int(t), b), sets[i]), i
            ch = eng.tatp_chain(int(t), b)
            assert len(ch) == chains[i]["n"] and ch.tobytes() == chains[i]["rec"][:len(ch)].tobytes(), i
        st0 = [cl.engine(s).tatp_cache_stats() for s in range(G)]
        assert all(st["failed"] == 0 for st in st0) and st0[0]["allocated"] > 0
        with GpuTxnClients(cl, clients, subscribers=S) as tc:
            tc.run(600)
            assert tc.stats()["committed"] > 0
        for s in range(G):
            st = cl.engine(s).tatp_cache_stats()
            assert st["failed"] == 0, (s, st)
            assert cl.engine(s).stats()["errors"] == 0
