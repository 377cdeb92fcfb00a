"""-m gpu: the TATP and SmallBank closed-loop clients resident on the GPU (dint_b200/csrc/txn_clients.cuh,
dint_txn_clients_*, GpuTxnClients) against a shard cluster.  Round for round they must emit what the host drivers
(TxnWorkload) emit and absorb what G oracle shard servers answer; at the end the counters, every shard's commit log
and (G = 3) every table's row count must be the oracles'.

TATP runs at G >= 3 only: on one shard the backups are the primary itself, and the backup commit of a record meets
the primary's own lock, which the reference server refuses (the oracle panics on it)."""
import numpy as np
import pytest

import oracle_lib as O
from dint_b200 import GpuCluster, GpuTxnClients, wire
from dint_b200.engine import DintError
from dint_b200.txn_workloads import Cluster, TxnWorkload
from golden_util import first_diff

pytestmark = pytest.mark.gpu
GID0 = 5


def _n_gpus():
    import torch
    return torch.cuda.device_count()


def _placements(G):
    """shards all on device 0; plus one shard per device when the box has enough GPUs"""
    out = [("one_device", [0] * G)]
    if G > 1 and _n_gpus() >= G:
        out.append(("per_device", list(range(G))))
    return out


def _cfg(kind, n):
    return dict(subs_populate=n) if kind == wire.TATP else dict(accts_populate=n)


def _without_fallback(st):
    return {k: v for k, v in st.items() if k != "fallback_rounds"}


def _parity(kind, n, clients, G, rounds, devs, max_batch=0):
    """Drives TxnWorkload + G oracles and the GPU clients side by side; returns the GPU clients' final stats."""
    msg = wire.MSG_SIZE[kind]
    oras = [O.Oracle(kind, **_cfg(kind, n)) for _ in range(G)]
    ocl = Cluster([o.process for o in oras], msg)
    wl = TxnWorkload(kind, n_clients=clients, n_shards=G, subscribers=n, gid0=GID0)
    with GpuCluster(kind, G, devices=devs, max_batch=max_batch, populate=True, **_cfg(kind, n)) as cl:
        with GpuTxnClients(cl, clients, subscribers=n, gid0=GID0) as tc:
            for r in range(rounds):
                rq, dst = wl.next()
                q, d, _ = tc.peek()
                assert np.array_equal(q, rq) and np.array_equal(d, dst), f"round {r}: the clients diverged"
                rs = ocl.submit(rq, dst)
                wl.feed(rs)
                tc.run(1)
                _, _, got = tc.peek()
                assert got.size == rs.size and first_diff(got, rs, msg) is None, f"round {r}: {first_diff(got, rs, msg)}"
            st = tc.stats()
            want = wl.stats()
            assert _without_fallback(st) == want and want["committed"] > 0
            for s in range(G):
                ring, appended = cl.engine(s).dump_log()
                assert appended == oras[s].log_appended() and np.array_equal(ring, oras[s].log_ring()), f"shard {s} log"
                if G == 3:                      # G > 3: a shard holds only the keys it is a replica of
                    for tb in range(5 if kind == wire.TATP else 2):
                        assert cl.engine(s).kv_count(tb) == oras[s].kv_count(tb), f"shard {s} table {tb}"
            return st


# client counts that G does not divide: the ranks hold blocks of different sizes
@pytest.mark.parametrize("kind,n,clients,G,rounds", [
    (wire.TATP, 3000, 1201, 3, 120), (wire.TATP, 2500, 1201, 4, 80), (wire.TATP, 2500, 1201, 5, 80),
    (wire.SMALLBANK, 5000, 1500, 1, 100), (wire.SMALLBANK, 5000, 1001, 3, 100), (wire.SMALLBANK, 4000, 1001, 8, 60)])
def test_gpu_txn_clients_match_host_clients_and_oracles(kind, n, clients, G, rounds):
    for name, devs in _placements(G):
        st = _parity(kind, n, clients, G, rounds, devs)
        assert st["fallback_rounds"] == 0, name


@pytest.mark.parametrize("kind,n,clients,G", [(wire.TATP, 3000, 1201, 3), (wire.SMALLBANK, 5000, 1001, 3)])
def test_gpu_txn_clients_fallback_rounds_match(kind, n, clients, G):
    """A cluster of max_batch 256: a rank's round exceeds the batch size, so every round is served one source rank at
    a time in pieces -- with the same replies and the same final state."""
    st = _parity(kind, n, clients, G, 40, [0] * G, max_batch=256)
    assert st["fallback_rounds"] > 0


def test_gpu_txn_clients_run_k_equals_k_runs_of_one():
    kind, n, clients, G, k = wire.SMALLBANK, 5000, 1001, 3, 40
    out = []
    for steps in ([1] * k, [k]):
        with GpuCluster(kind, G, devices=[0] * G, populate=True, **_cfg(kind, n)) as cl:
            with GpuTxnClients(cl, clients, subscribers=n) as tc:
                for s in steps:
                    tc.run(s)
                q, d, rs = tc.peek()
                tm = tc.times()
                assert tm["rounds"] == k and tm["wall_s"] > 0 and 0 < tm["device_s"]
                out.append((tc.stats(), q.copy(), d.copy(), rs.copy()))
    (s1, q1, d1, r1), (s2, q2, d2, r2) = out
    assert s1 == s2 and s1["rounds"] == k and s1["committed"] > 0
    assert np.array_equal(q1, q2) and np.array_equal(d1, d2) and np.array_equal(r1, r2)


def test_gpu_txn_clients_refuse_bad_arguments():
    with GpuCluster(wire.FASST, 1) as cl:
        with pytest.raises(DintError) as ei:
            GpuTxnClients(cl, 100, subscribers=1000)
        assert ei.value.code == -22
    with GpuCluster(wire.SMALLBANK, 1, populate=True, accts_populate=1000) as cl:
        for n_clients, subs in ((0, 1000), (100, 2)):
            with pytest.raises(DintError) as ei:
                GpuTxnClients(cl, n_clients, subscribers=subs)
            assert ei.value.code == -22
