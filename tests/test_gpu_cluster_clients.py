"""-m gpu: the lock_fasst, lock_2pl, store and log_server closed-loop clients on the GPU against a shard cluster
(dint_cluster_clients_*, GpuClusterClients).  A cluster of these kinds answers like ONE sequential server fed the
rank-major concatenation of its ranks' batches, and the clients are split over the ranks in contiguous blocks, so a
G-shard cluster must send and absorb, round for round, exactly what GpuClients with the same clients sends and absorbs on
one engine, end with the same counters, and leave the same server state.  Shards sit on device 0; on a box with G GPUs
the same tests also run with one shard per device."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from dint_b200 import DintError, Engine, GpuCluster, GpuClusterClients, GpuClients, lib, wire
from golden_util import first_diff

pytestmark = pytest.mark.gpu

SEED = 41
POP = 2000                       # store subscribers the engines populate


def _n_gpus():
    import torch
    return torch.cuda.device_count()


def _placements(G):
    """shards all on device 0; plus one shard per device when the box has enough GPUs"""
    out = [("one_device", [0] * G)]
    if G > 1 and _n_gpus() >= G:
        out.append(("per_device", list(range(G))))
    return out


def _block(n, G):
    """the largest rank's block of n clients over G ranks: the cluster's max_batch in these tests (at least 128)"""
    return max(-(-n // G), 128)


FAMILIES = {
    # name: (kind, server options of both sides, client family)
    "fasst_uniform": (wire.FASST, {}, dict(n_keys=60000)),
    "fasst_zipf_hot": (wire.FASST, {}, dict(n_keys=4800, zipf_theta=0.8)),
    "lock2pl_uniform": (wire.LOCK2PL, {}, dict(n_keys=50000)),
    "lock2pl_zipf_hot": (wire.LOCK2PL, {}, dict(n_keys=4800, zipf_theta=0.8)),
    "lock2pl_tiny": (wire.LOCK2PL, {}, dict(n_keys=7)),
    "store_parallel": (wire.STORE, dict(populate=True, subs_populate=POP), dict(store_subscribers=POP)),
    "store_contention": (wire.STORE, dict(populate=True, subs_populate=POP), dict(store_subscribers=POP, set_pct=50)),
    "store_hot": (wire.STORE, dict(populate=True, subs_populate=POP), dict(store_hot=True, n_keys=4800, zipf_theta=0.8, set_pct=50)),
    "store_misses": (wire.STORE, dict(populate=True, subs_populate=POP), dict(store_subscribers=3000, set_pct=50)),
    "log_default_ring": (wire.LOG, {}, {}),
    "log_ring1000": (wire.LOG, dict(log_ring=1000), {}),
}


def _drive(kind, eng, cl, n, rounds, fam, on_round=None):
    """GpuClients on `eng` next to GpuClusterClients on `cl`, `rounds` rounds: every round's requests (peek before it)
    and absorbed replies (peek after it) must be equal.  on_round(req) sees every round's requests.  Returns both
    sides' final counters."""
    msg = wire.MSG_SIZE[kind]
    with GpuClients(eng, n, seed=SEED, **fam) as one, GpuClusterClients(cl, n, seed=SEED, **fam) as cc:
        for r in range(rounds):
            want_req, _ = one.peek()
            got_req, _ = cc.peek()
            d = first_diff(got_req, want_req, msg)
            assert d is None, f"round {r}: requests differ: {d}"
            if on_round is not None:
                on_round(want_req)
            one.run(1)
            assert cc.run(1) == 0
            _, want_resp = one.peek()
            _, got_resp = cc.peek()
            d = first_diff(got_resp, want_resp, msg)
            assert d is None, f"round {r}: replies differ: {d}"
        a, b = one.stats(), cc.stats()
        t = cc.times()
    assert {k: v for k, v in b.items() if k != "fallback_rounds"} == a, (a, b)
    assert a["rounds"] == rounds and a["requests"] == rounds * n
    assert t["rounds"] == rounds and t["wall_s"] > 0 and t["device_s"] > 0
    return a, b


def _set_keys(req, out):
    """collects the keys of a store round's kSet requests"""
    rec = req.reshape(-1, 53)
    out.update(int(k) for k in rec[rec[:, 0] == 1, 1:9].copy().view(np.uint64).reshape(-1))


def _check_state(kind, eng, cl, G, fam, keys):
    if kind in (wire.FASST, wire.LOCK2PL):
        ids = range(fam["n_keys"]) if fam["n_keys"] <= 4800 else np.random.default_rng(2).integers(0, fam["n_keys"], size=256).tolist()
        for lid in ids:
            slot = eng.lock_slot(0, int(lid))
            assert cl.engine(slot % G).lock_state(0, slot) == eng.lock_state(0, slot), lid
    elif kind == wire.STORE:
        assert sum(cl.engine(s).kv_count(0) for s in range(G)) == eng.kv_count(0)
        if keys:
            rng = np.random.default_rng(1)
            for key in rng.choice(sorted(keys), size=min(128, len(keys)), replace=False):
                want = eng.kv_get(0, int(key))
                got = [v for v in (cl.engine(s).kv_get(0, int(key)) for s in range(G)) if v is not None]
                assert got == ([want] if want is not None else []), hex(int(key))


@pytest.mark.parametrize("G", [1, 2, 3, 8])
@pytest.mark.parametrize("name", list(FAMILIES))
def test_cluster_clients_equal_one_engine_round_for_round(name, G):
    kind, srv, fam = FAMILIES[name]
    n, rounds = 3000, 100
    for place, devs in _placements(G):
        rounds_req = []
        keys = set()

        def seen(req):
            rounds_req.append(req.copy())
            if kind == wire.STORE:
                _set_keys(req, keys)

        with Engine(kind, chunk=2048, **srv) as eng, \
                GpuCluster(kind, G, devices=devs, max_batch=_block(n, G), **srv) as cl:
            a, b = _drive(kind, eng, cl, n, rounds, fam, on_round=seen)
            assert a["committed"] > 0, place
            _check_state(kind, eng, cl, G, fam, keys)
            if name == "store_misses":
                assert a["not_exist"] > 0
            if name == "lock2pl_zipf_hot":
                assert a["lock_rejects"] > 0
            if kind == wire.LOG:
                # shard r's ring = a log server fed rank r's slice of every round
                msg = wire.MSG_SIZE[kind]
                for r in range(G):
                    lo, hi = n * r // G, n * (r + 1) // G
                    ora = O.Oracle(wire.LOG, **{k: v for k, v in srv.items() if k == "log_ring"})
                    for req in rounds_req:
                        ora.process(req[lo * msg:hi * msg])
                    ring, appended = cl.engine(r).dump_log()
                    assert appended == ora.log_appended() == rounds * (hi - lo), (place, r)
                    assert np.array_equal(ring, ora.log_ring()), (place, r)


@pytest.mark.parametrize("G", [2, 8])
def test_rounds_that_all_go_to_one_shard_are_served_in_pieces(G):
    """lock_fasst with ONE lock id: every record of every rank belongs to one shard, more than a slab holds, so every
    round is served one source rank at a time -- and still equals one engine."""
    n, rounds, fam = 3000, 30, dict(n_keys=1)
    with Engine(wire.FASST, chunk=2048) as eng, \
            GpuCluster(wire.FASST, G, devices=[0] * G, max_batch=-(-n // G)) as cl:
        a, b = _drive(wire.FASST, eng, cl, n, rounds, fam)
        assert b["fallback_rounds"] == rounds
        assert a["committed"] > 0
        slot = eng.lock_slot(0, 0)
        assert cl.engine(slot % G).lock_state(0, slot) == eng.lock_state(0, slot)


@pytest.mark.parametrize("name", ["fasst_zipf_hot", "store_contention", "log_default_ring"])
def test_ranks_without_clients_take_part(name):
    """5 clients over 8 ranks: ranks 0, 2 and 5 hold none; they still take part in every exchange."""
    kind, srv, fam = FAMILIES[name]
    G, n, rounds = 8, 5, 40
    with Engine(kind, chunk=2048, **srv) as eng, GpuCluster(kind, G, devices=[0] * G, max_batch=128, **srv) as cl:
        a, _ = _drive(kind, eng, cl, n, rounds, fam)
        assert a["committed"] > 0
        _check_state(kind, eng, cl, G, fam, set())


@pytest.mark.parametrize("name", ["fasst_zipf_hot", "lock2pl_zipf_hot", "store_hot", "log_default_ring"])
def test_many_rounds_in_one_call(name):
    """run(k) = k single rounds: same counters, same pending requests, same last replies."""
    kind, srv, fam = FAMILIES[name]
    G, n = 3, 20000
    with GpuCluster(kind, G, devices=[0] * G, max_batch=_block(n, G), **srv) as c1, \
            GpuCluster(kind, G, devices=[0] * G, max_batch=_block(n, G), **srv) as c2:
        with GpuClusterClients(c1, n, seed=5, **fam) as a, GpuClusterClients(c2, n, seed=5, **fam) as b:
            a.run(60)
            for _ in range(60):
                b.run(1)
            assert a.stats() == b.stats() and a.stats()["committed"] > 0 and a.stats()["rounds"] == 60
            ra, rb = a.peek(), b.peek()
            assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])
            assert a.times()["rounds"] == b.times()["rounds"] == 60


def test_cluster_clients_at_production_size():
    """2^20 lock_fasst clients at the reference's 24 M ids, 3 shards on one device, 20 rounds, every round compared
    with GpuClients on one engine; then a sample of lock words."""
    n, rounds, G, fam = 1 << 20, 20, 3, dict(n_keys=24_000_000)
    with Engine(wire.FASST) as eng, GpuCluster(wire.FASST, G, devices=[0] * G, max_batch=-(-n // G)) as cl:
        a, b = _drive(wire.FASST, eng, cl, n, rounds, fam)
        assert b["fallback_rounds"] == 0 and a["committed"] > 0
        _check_state(wire.FASST, eng, cl, G, fam, set())


def test_invalid_cluster_clients_are_refused():
    def refused(cl, n, **kw):
        with pytest.raises(DintError) as ex:
            GpuClusterClients(cl, n, **kw)
        assert ex.value.code == -22, kw
        return str(ex.value)

    with GpuCluster(wire.TATP, 3, devices=[0] * 3, max_batch=1024, subs_sizing=1000, subs_populate=1000) as cl:
        assert "txn_clients" in refused(cl, 100)
    with GpuCluster(wire.FASST, 2, devices=[0, 0], max_batch=128) as cl:
        refused(cl, 0)
        refused(cl, 257)                                  # a rank's block of 129 clients > max_batch
        for bad in (dict(n_keys=0), dict(read_pct=101)):
            refused(cl, 100, **bad)
        with GpuClusterClients(cl, 256) as ok:            # blocks of exactly max_batch
            assert ok.run(2) == 0 and ok.stats()["rounds"] == 2
    with GpuCluster(wire.LOCK2PL, 2, devices=[0, 0], max_batch=128) as cl:
        refused(cl, 100, n_keys=0)
    with GpuCluster(wire.STORE, 3, devices=[0] * 3, max_batch=128, subs_sizing=1000) as cl:
        for bad in (dict(set_pct=101), dict(store_subscribers=0), dict(store_hot=True, n_keys=0)):
            refused(cl, 100, **bad)
    with GpuCluster(wire.FASST, 1, max_batch=8) as cl:   # a fallback piece could not stay 16-byte aligned
        refused(cl, 8)
    h = C.c_void_p()
    assert lib().dint_cluster_clients_create(None, None, C.byref(h)) == -22
