"""-m gpu: re-sharding live TATP and SmallBank clusters (GpuTxnClients.drain, GpuCluster.reshard_txn,
GpuTxnClients.rebind; dint_cluster_reshard_txn).

The GPU clients run 20 rounds on three shards, drain, move to five shards, run 20 rounds, drain, move back to three and
run 20 more; the host clients (TxnWorkload) do the same against oracles re-placed through their wire handlers
(test_txn_reshard_cpu.place).  Every round's requests and replies, the drain round counts and the final counters must be
equal.  Rows are compared in bulk through state images (test_gpu_rebuild.shard_state)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as O
import test_txn_reshard_cpu as H
from golden_util import first_diff
from test_gpu_rebuild import regions, shard_state
from dint_b200 import GpuCluster, GpuTxnClients, wire
from dint_b200.engine import DintError
from dint_b200.txn_workloads import Cluster, TxnWorkload

pytestmark = pytest.mark.gpu
EINVAL = -22
TATP, SMALLBANK = wire.TATP, wire.SMALLBANK
GID0 = 5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _n_gpus():
    import torch
    return torch.cuda.device_count()


def _placements():
    """every shard on device 0; plus one shard per device when the box has five GPUs"""
    out = [("one_device", lambda G: [0] * G)]
    if _n_gpus() >= 5:
        out.append(("per_device", lambda G: list(range(G))))
    return out


def _rounds(wl, host, tc, k, tag):
    """k rounds of the host clients against `host` (a Cluster or GpuCluster) and of the GPU clients, compared"""
    msg = wl.msg
    for r in range(k):
        rq, dst = wl.next()
        q, d, _ = tc.peek()
        assert np.array_equal(q, rq) and np.array_equal(d, dst), f"{tag} round {r}: the clients diverged"
        rs = host.submit(rq, dst) if isinstance(host, Cluster) else host.submit(rq, dst=dst)
        wl.feed(rs)
        tc.run(1)
        _, _, got = tc.peek()
        assert first_diff(got, rs, msg) is None, f"{tag} round {r}: {first_diff(got, rs, msg)}"


def _host_drain(wl, host):
    wl.draining = True
    n = 0
    while True:
        rq, dst = wl.next()
        if not dst.size:
            break
        wl.feed(host.submit(rq, dst) if isinstance(host, Cluster) else host.submit(rq, dst=dst))
        n += 1
        assert n <= H.LONGEST[wl.kind]
    return n


def _cycle(kind, devs, oracle_side, **cfg_over):
    """3 -> 5 -> 3 with the GPU clients and the host clients side by side.  oracle_side: the host clients talk to oracles
    re-placed by test_txn_reshard_cpu.place; otherwise to GPU clusters re-placed by reshard_txn as well."""
    cfg = dict(H.oracle_cfg(kind), **cfg_over)
    wl = TxnWorkload(kind, n_clients=H.CLIENTS[kind], n_shards=3, subscribers=H.N[kind], gid0=GID0)
    if oracle_side:
        oras = [O.Oracle(kind, **H.oracle_cfg(kind)) for _ in range(3)]
        host = Cluster([o.process for o in oras], wire.MSG_SIZE[kind])
    else:
        host = GpuCluster(kind, 3, devices=devs(3), populate=True, **cfg)
    cl = GpuCluster(kind, 3, devices=devs(3), populate=True, **cfg)
    tc = GpuTxnClients(cl, H.CLIENTS[kind], subscribers=H.N[kind], gid0=GID0)
    try:
        _rounds(wl, host, tc, 20, "G=3")
        for G, G2 in ((3, 5), (5, 3)):
            n_host, n_gpu = _host_drain(wl, host), tc.drain()
            assert n_gpu == n_host >= 1, (n_gpu, n_host)
            assert wl.busy() == 0
            if oracle_side:
                oras = H.place(kind, H.rows_of(oras, kind, G), G2)
                host = Cluster([o.process for o in oras], wire.MSG_SIZE[kind])
            else:
                new = host.reshard_txn(G2, devices=devs(G2))
                host.close()
                host = new
            wl.set_shards(G2)
            wl.draining = False
            new = cl.reshard_txn(G2, devices=devs(G2))
            tc.rebind(new)
            cl.close()
            cl = new
            _rounds(wl, host, tc, 20, f"{G}->{G2}")
        st = tc.stats()
        assert st.pop("fallback_rounds") == 0
        assert st == wl.stats()
        assert tc.lock_stats() == wl.lock_stats()
        return st, tc.lock_stats()
    finally:
        tc.close()
        cl.close()
        if not oracle_side:
            host.close()


@pytest.mark.parametrize("kind", [TATP, SMALLBANK])
def test_live_cycle_equals_the_host_loop(kind):
    for name, devs in _placements():
        st, _ = _cycle(kind, devs, oracle_side=True)
        assert st["committed"] > 0, name


def test_holder_keys_across_a_reshard():
    _, locks = _cycle(TATP, lambda G: [0] * G, oracle_side=False, lock_holder_keys=True)
    assert locks["locks"] > 0


# ---- rows, through images ------------------------------------------------------------------------------------------
def _tables(d, G, kind):
    return [shard_state(os.path.join(d, f"shard-{r}.img"), kind)[1] for r in range(G)]


def _check_replaced(src_tabs, dst_tabs, kind, G, G2):
    """every destination shard holds {key: the old primary's row} over exactly the keys it replicates under G2"""
    for t in range(H.N_TABLES[kind]):
        prim = {}
        for s in range(G):
            prim.update({k: r for k, r in src_tabs[s][t].items() if k % G == s})
        for j in range(G2):
            want = {k: r for k, r in prim.items() if j in H.replicas(k, G2)}
            assert dst_tabs[j][t] == want, (t, j, len(dst_tabs[j][t]), len(want))


def _image_state(d, G):
    return [[x.tobytes() for x in regions(os.path.join(d, f"shard-{r}.img"))] for r in range(G)]


@pytest.mark.parametrize("kind", [TATP, SMALLBANK])
def test_rows_after_a_drain_and_source_unchanged(kind, tmp_path):
    cfg = H.oracle_cfg(kind)
    with GpuCluster(kind, 3, populate=True, **cfg) as cl:
        with GpuTxnClients(cl, H.CLIENTS[kind], subscribers=H.N[kind], gid0=GID0) as tc:
            tc.run(20)
            assert tc.drain() >= 1
            cl.save_image(str(tmp_path / "before"))
            with cl.reshard_txn(5) as dst:
                dst.save_image(str(tmp_path / "dst"))
                for r in range(5):                       # no lock comes along
                    assert not regions(os.path.join(tmp_path / "dst", f"shard-{r}.img"))[0].any()
            cl.save_image(str(tmp_path / "after"))
            assert _image_state(tmp_path / "before", 3) == _image_state(tmp_path / "after", 3)
            _check_replaced(_tables(tmp_path / "before", 3, kind), _tables(tmp_path / "dst", 5, kind), kind, 3, 5)
            assert tc.run(1) == 0                        # the source is still served


@pytest.mark.parametrize("kind", [TATP, SMALLBANK])
def test_populated_reshard_equals_a_populated_cluster(kind, tmp_path):
    cfg = H.oracle_cfg(kind)
    with GpuCluster(kind, 3, populate=True, **cfg) as cl, cl.reshard_txn(5) as dst, \
            GpuCluster(kind, 5, populate=True, **cfg) as fresh:
        dst.save_image(str(tmp_path / "dst"))
        fresh.save_image(str(tmp_path / "fresh"))
    assert _tables(tmp_path / "dst", 5, kind) == _tables(tmp_path / "fresh", 5, kind)


# ---- refusals ------------------------------------------------------------------------------------------------------
def _refused(fn, *words):
    with pytest.raises(DintError) as e:
        fn()
    assert e.value.code == EINVAL, str(e.value)
    for w in words:
        assert w in str(e.value), (w, str(e.value))


@pytest.mark.parametrize("kind", [TATP, SMALLBANK])
def test_refusals_leave_source_and_clients_usable(kind):
    cfg = H.oracle_cfg(kind)
    with GpuCluster(kind, 3, populate=True, **cfg) as cl, \
            GpuTxnClients(cl, H.CLIENTS[kind], subscribers=H.N[kind], gid0=GID0) as tc:
        tc.run(5)
        _refused(lambda: cl.reshard_txn(5), "shard", "locks", "drain")
        assert tc.run(1) == 0
        with GpuCluster(kind, 5, **cfg) as other:
            _refused(lambda: tc.rebind(other), "drain")
        assert tc.run(1) == 0
        for G2 in (0, 2, 9):
            _refused(lambda: cl.reshard_txn(G2))
            assert tc.run(1) == 0
        tc.drain()                                       # (no lock held: only the device list can refuse)
        mixed = [0, 0, 1] if _n_gpus() >= 2 else [0, 0, 99]
        _refused(lambda: cl.reshard_txn(3, devices=mixed))
        assert tc.run(1) == 0
        other_kind = SMALLBANK if kind == TATP else TATP
        with GpuCluster(other_kind, 3, **H.oracle_cfg(other_kind)) as other:
            _refused(lambda: tc.rebind(other), "kind")
        assert tc.run(1) == 0
    flag = "tatp_ebpf" if kind == TATP else "smallbank_ebpf"
    with GpuCluster(kind, 3, **{flag: True}, **cfg) as eb:
        _refused(lambda: eb.reshard_txn(5), "eBPF")


@pytest.mark.parametrize("kind", [wire.LOCK2PL, wire.FASST, wire.STORE, wire.LOG])
def test_refuses_other_kinds(kind):
    with GpuCluster(kind, 3) as cl:
        _refused(lambda: cl.reshard_txn(5), "dint_cluster_reshard")


# ---- the image tool --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", [TATP, SMALLBANK])
def test_image_tool_replicas_equals_live(kind, tmp_path):
    cfg = H.oracle_cfg(kind)
    with GpuCluster(kind, 3, populate=True, **cfg) as cl:
        with GpuTxnClients(cl, H.CLIENTS[kind], subscribers=H.N[kind], gid0=GID0) as tc:
            tc.run(15)
            tc.drain()
        cl.save_image(str(tmp_path / "src"))
        with cl.reshard_txn(5) as live:
            live.save_image(str(tmp_path / "live"))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "reshard_image.py"), str(tmp_path / "src"),
                        str(tmp_path / "tool"), "--shards", "5", "--replicas"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    with GpuCluster.open_image(str(tmp_path / "tool")) as opened:
        assert opened.G == 5
    assert _tables(tmp_path / "tool", 5, kind) == _tables(tmp_path / "live", 5, kind)


@pytest.mark.parametrize("kind", [TATP, SMALLBANK])
def test_image_tool_refuses_an_image_with_held_locks(kind, tmp_path):
    cfg = H.oracle_cfg(kind)
    with GpuCluster(kind, 3, populate=True, **cfg) as cl:
        with GpuTxnClients(cl, H.CLIENTS[kind], subscribers=H.N[kind], gid0=GID0) as tc:
            tc.run(5)
            cl.save_image(str(tmp_path / "src"))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "reshard_image.py"), str(tmp_path / "src"),
                        str(tmp_path / "dst"), "--shards", "5", "--replicas"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 1 and "locks" in r.stderr, r.stdout + r.stderr


@pytest.mark.slow
def test_bench_tool_small_size(tmp_path):
    out = tmp_path / "bench.json"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "txn_reshard_bench.py"), "--clients", str(1 << 18),
                        "--subscribers", "1000000", "--accounts", "4000000", "--rounds", "10", "--json", str(out)],
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
