"""-m gpu: re-sharding lock_2pl, lock_fasst and store clusters onto another shard count (dint_cluster_reshard,
GpuCluster.reshard) and moving closed-loop clients with them (dint_cluster_clients_rebind, GpuClusterClients.rebind).
A cluster of these kinds answers like ONE sequential server whatever its shard count, so after a re-shard the new
cluster -- and the untouched source -- must answer every later request as one server that saw the whole history.
Shards sit on device 0; on a box with enough GPUs the same tests also run with one shard per device."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as O
import store_ebpf_model as M
import trace_gen as T
from dint_b200 import DintError, Engine, GpuCluster, GpuClients, GpuClusterClients, wire
from dint_b200.workloads import REF
from golden_util import first_diff
from test_gpu_cluster_clients import FAMILIES, SEED, _block

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL = -22


def _n_gpus():
    import torch
    return torch.cuda.device_count()


def _placements(G, G2):
    """(name, source devices, destination devices): every shard on device 0; plus one shard per device when the box
    has enough GPUs for both"""
    out = [("one_device", [0] * G, [0] * G2)]
    if max(G, G2) > 1 and _n_gpus() >= max(G, G2):
        out.append(("per_device", list(range(G)), list(range(G2))))
    return out


def _trace(kind, n, seed, skew=False):
    if kind == wire.FASST:
        return T.fasst_random(n, 4800 if skew else 60000, seed=seed)
    if kind == wire.LOCK2PL:
        return T.lock2pl_random(n, 3000 if skew else 50000, seed=seed)
    return T.store_random(n, 500, seed=seed)


def _check_state(kind, cl, ora):
    """sampled lock_state of the owning shard, or the summed kv_count, against the oracle"""
    G = cl.G
    if kind in (wire.FASST, wire.LOCK2PL):
        for lid in np.random.default_rng(7).integers(0, 4800, size=128):
            slot = ora.lock_slot(0, int(lid))
            assert cl.engine(slot % G).lock_state(0, slot) == ora.lock_state(0, slot), lid
    else:
        assert sum(cl.engine(s).kv_count(0) for s in range(G)) == ora.kv_count(0)


@pytest.mark.parametrize("G,G2", [(1, 3), (3, 1), (2, 5), (3, 8), (8, 2), (3, 3)])
@pytest.mark.parametrize("kind", [wire.FASST, wire.LOCK2PL, wire.STORE])
def test_reshard_answers_like_one_server(kind, G, G2):
    msg = wire.MSG_SIZE[kind]
    cfg = dict(subs_populate=500) if kind == wire.STORE else {}
    max_batch = 4096
    prefix = [777, G * max_batch, 2 * G * max_batch + 129]
    suffix = [G2 * max_batch + 5, 50000, 333]
    for name, devs, devs2 in _placements(G, G2):
        ora = O.Oracle(kind, **cfg)
        with GpuCluster(kind, G, devices=devs, max_batch=max_batch, populate=True, **cfg) as src:
            for i, n in enumerate(prefix):
                req = _trace(kind, n, seed=10 + i, skew=(i % 2 == 1))
                d = first_diff(src.submit(req), ora.process(req), msg)
                assert d is None, f"{name} prefix call {i}: {d}"
            with src.reshard(G2, devices=devs2, max_batch=max_batch) as dst:
                assert dst.G == G2
                for i, n in enumerate(suffix):
                    req = _trace(kind, n, seed=20 + i, skew=(i % 2 == 0))
                    want = ora.process(req)
                    d = first_diff(dst.submit(req), want, msg)
                    assert d is None, f"{name} {G}->{G2} call {i}: {d}"
                    d = first_diff(src.submit(req), want, msg)      # the source was not changed by the re-shard
                    assert d is None, f"{name} source after {G}->{G2}, call {i}: {d}"
                _check_state(kind, dst, ora)
                _check_state(kind, src, ora)
                for s in range(G2):
                    assert dst.engine(s).stats()["errors"] == 0


def _fasst(types, lids):
    rec = np.zeros(len(lids), dtype=wire.MSG_DTYPE[wire.FASST])
    rec["type"] = types
    rec["lid"] = lids
    return wire.as_bytes(rec)


def _ver(reply):
    return reply[:, 5:9].copy().view(np.uint32).reshape(-1)


@pytest.mark.parametrize("G,G2", [(3, 5), (2, 1), (1, 8)])
def test_held_locks_and_versions_move(G, G2):
    """lock_fasst: locks granted before the re-shard and not yet committed are still held after it; their commit bumps
    the version a later kRead sees, and an abort frees them"""
    ids = np.random.default_rng(1).choice(1 << 20, size=3000, replace=False).astype(np.uint32)
    for name, devs, devs2 in _placements(G, G2):
        ora = O.Oracle(wire.FASST)
        with GpuCluster(wire.FASST, G, devices=devs, max_batch=4096) as src:
            def both(cl, req):
                got = cl.submit(req)
                d = first_diff(got, ora.process(req), 9)
                assert d is None, f"{name}: {d}"
                return got.reshape(-1, 9)

            both(src, T.fasst_random(20000, 60000, seed=3))
            held = ids[both(src, _fasst(1, ids))[:, 0] == 5]                 # granted (a slot shared with a held one is not)
            assert held.size > 2900
            commit, abort = held[: held.size // 2], held[held.size // 2:]
            with src.reshard(G2, devices=devs2, max_batch=4096) as dst:
                assert (both(dst, _fasst(1, held))[:, 0] == 6).all()         # a second acquire is rejected
                vb = _ver(both(dst, _fasst(0, commit)))
                assert (both(dst, _fasst(3, commit))[:, 0] == 8).all()       # commit: ver++ and release
                assert np.array_equal(_ver(both(dst, _fasst(0, commit))), vb + np.uint32(1))
                assert (both(dst, _fasst(1, commit))[:, 0] == 5).all()
                assert (both(dst, _fasst(2, abort))[:, 0] == 7).all()        # abort frees ...
                assert (both(dst, _fasst(1, abort))[:, 0] == 5).all()        # ... so the lock is granted again


def _store_tier_traffic(n, seed, fresh0, subs=1500):
    """kRead / kSet over subscribers (some absent) with kInserts of never-inserted keys mixed in"""
    rng = np.random.default_rng(seed)
    base = T.store_random(n, subs, seed=seed).reshape(-1, 53).copy()
    ins = rng.random(n) < 0.1
    fresh = (np.arange(int(ins.sum()), dtype=np.uint64) + np.uint64(fresh0)) | (np.uint64(1) << np.uint64(32))
    base[ins, 0] = 2
    base[ins, 1:9] = fresh.reshape(-1, 1).view(np.uint8)
    return base.reshape(-1), fresh


@pytest.mark.parametrize("G,G2", [(3, 5), (5, 1)])
@pytest.mark.parametrize("variant", M.VARIANTS)
def test_store_ebpf_tier_moves_whole(variant, G, G2):
    cfg = dict(subs_sizing=1000, subs_populate=1000, store_ebpf=variant)
    H = 1000 * 18 // 4
    for name, devs, devs2 in _placements(G, G2):
        with Engine(wire.STORE, device=0, chunk=4096, populate=True, **cfg) as one, \
                GpuCluster(wire.STORE, G, devices=devs, max_batch=4096, populate=True, **cfg) as src:
            keys = []
            for i in range(3):
                req, fresh = _store_tier_traffic(20000, 30 + i, 1_000_000 + 100_000 * i)
                keys.append(fresh)
                assert first_diff(src.submit(req), one.submit(req), 53) is None, f"{name} prefix {i}"
            st = one.store_cache_stats()
            assert st["write_backs" if variant != "wt" else "installs"] > 0 and st["hits"] > 0, st
            with src.reshard(G2, devices=devs2, max_batch=4096) as dst:
                for i in range(3):
                    req, fresh = _store_tier_traffic(20000, 40 + i, 2_000_000 + 100_000 * i)
                    keys.append(fresh)
                    want = one.submit(req)
                    got = dst.submit(req)
                    d = first_diff(got, want, 53)
                    assert d is None, f"{name} {variant} {G}->{G2} call {i}: {d}"
                shards = [dst.engine(s) for s in range(G2)]
                for b in np.random.default_rng(5).choice(H, size=256, replace=False):
                    assert np.array_equal(shards[b % G2].store_cache_set(int(b)), one.store_cache_set(int(b))), b
                assert sum(e.kv_count(0) for e in shards) == one.kv_count(0)
                allk = np.concatenate(keys)
                for k in np.random.default_rng(6).choice(allk, size=128, replace=False):
                    b = M.fasthash64(int(k)) % H
                    assert shards[b % G2].kv_get(0, int(k)) == one.kv_get(0, int(k)), hex(int(k))
                assert all(e.store_cache_stats()["hits"] > 0 for e in shards)


def _inserts(keys):
    rec = np.zeros(len(keys), dtype=wire.MSG_DTYPE[wire.STORE])
    rec["type"] = 2
    rec["key"] = keys
    rec["val"] = (np.asarray(keys, dtype=np.uint64) % np.uint64(251)).astype(np.uint8).reshape(-1, 1)
    return wire.as_bytes(rec)


def _reads(keys):
    rec = np.zeros(len(keys), dtype=wire.MSG_DTYPE[wire.STORE])
    rec["key"] = keys
    return wire.as_bytes(rec)


def test_capacity_grows_with_the_keys():
    """tables created at 2^10 entries, grown by the tombstone rehash to hold 6000 keys over 4 shards, re-sharded onto
    ONE shard: every key is kept, nothing is answered 0xFF, and the first call does not rehash"""
    keys = (np.arange(6000, dtype=np.uint64) * np.uint64(7919) + np.uint64(1)) | (np.uint64(3) << np.uint64(32))
    with GpuCluster(wire.STORE, 4, devices=[0] * 4, max_batch=1024, subs_populate=0, kv_capacity_log2=[10]) as src:
        for part in np.array_split(keys, 12):
            assert (src.submit(_inserts(part)).reshape(-1, 53)[:, 0] == 8).all()      # kInsertAck
        assert all(src.engine(s).stats()["kv_rebuilds"] > 0 for s in range(4))
        assert sum(src.engine(s).kv_count(0) for s in range(4)) == 6000
        want = src.submit(_reads(keys))
        with src.reshard(1, devices=[0], max_batch=1024) as dst:
            assert dst.engine(0).kv_count(0) == 6000
            got = dst.submit(_reads(keys))
            assert first_diff(got, want, 53) is None
            r = got.reshape(-1, 53)
            assert (r[:, 0] == 3).all()
            assert (r[:, 9] == (keys % np.uint64(251)).astype(np.uint8)).all()
            st = dst.engine(0).stats()
            assert st["errors"] == 0 and st["kv_rebuilds"] == 0, st


def test_refusals():
    def refused(fn):
        with pytest.raises(DintError) as ei:
            fn()
        assert ei.value.code == EINVAL, ei.value

    small = {wire.TATP: dict(subs_sizing=6000, subs_populate=40), wire.SMALLBANK: dict(accts_sizing=4000, accts_populate=4000),
             wire.LOG: dict(log_ring=4096)}
    for kind, cfg in small.items():
        with GpuCluster(kind, 3, devices=[0] * 3, max_batch=1024, **cfg) as cl:
            refused(lambda: cl.reshard(1, devices=[0]))
    with GpuCluster(wire.FASST, 2, devices=[0, 0], max_batch=1024, lock_slots=1 << 16) as cl:
        refused(lambda: cl.reshard(0))
        refused(lambda: cl.reshard(9, devices=[0] * 9))
        refused(lambda: cl.reshard(3, devices=[0, 0, 1] if _n_gpus() > 1 else [0, 0, -1]))
        with GpuCluster(wire.LOCK2PL, 2, devices=[0, 0], max_batch=1024, lock_slots=1 << 16) as other, \
                GpuClusterClients(cl, 500, n_keys=1000) as cc:
            cc.run(2)
            refused(lambda: cc.rebind(other))
            small_batch = cl.reshard(1, devices=[0], max_batch=128)     # a rank's block of 500 clients does not fit
            refused(lambda: cc.rebind(small_batch))
            small_batch.close()
            assert cc.run(1) == 0                                      # the clients are unchanged and still served


LIVE = {"fasst_ref": (wire.FASST, {}, dict(REF)), "lock2pl_ref": (wire.LOCK2PL, {}, dict(REF)),
        "store_contention": FAMILIES["store_contention"]}


@pytest.mark.parametrize("name", list(LIVE))
def test_live_closed_loop_follows_the_reshards(name):
    """G = 3 for 20 rounds, re-shard to 5 and rebind, 20 rounds, re-shard to 1 and rebind, 20 rounds: every round
    equals GpuClients on one engine, and so do the final counters"""
    kind, srv, fam = LIVE[name]
    n, msg = 3000, wire.MSG_SIZE[kind]
    steps = {20: 5, 40: 1}
    for place, devs, _ in _placements(3, 5):
        def devices(G):
            return [0] * G if place == "one_device" else list(range(G))

        with Engine(kind, chunk=2048, **srv) as eng, GpuClients(eng, n, seed=SEED, **fam) as one:
            cl = GpuCluster(kind, 3, devices=devs, max_batch=_block(n, 3), **srv)
            with GpuClusterClients(cl, n, seed=SEED, **fam) as cc:
                for r in range(60):
                    if r in steps:
                        G2 = steps[r]
                        new = cl.reshard(G2, devices=devices(G2), max_batch=_block(n, G2))
                        cc.rebind(new)
                        cl.close()
                        cl = new
                    want_req, _ = one.peek()
                    got_req, _ = cc.peek()
                    assert first_diff(got_req, want_req, msg) is None, f"{place} round {r}: requests differ"
                    one.run(1)
                    assert cc.run(1) == 0
                    _, want_resp = one.peek()
                    _, got_resp = cc.peek()
                    assert first_diff(got_resp, want_resp, msg) is None, f"{place} round {r}: replies differ"
                a, b = one.stats(), cc.stats()
                assert {k: v for k, v in b.items() if k != "fallback_rounds"} == a, (a, b)
                assert a["rounds"] == 60 and a["committed"] > 0
            cl.close()


def test_reshard_image_tool(tmp_path):
    cfg = dict(subs_populate=500)
    src, dst = str(tmp_path / "three"), str(tmp_path / "five")
    with Engine(wire.STORE, device=0, populate=True, **cfg) as one:
        with GpuCluster(wire.STORE, 3, devices=[0] * 3, max_batch=4096, populate=True, **cfg) as cl:
            req = _trace(wire.STORE, 30000, seed=1)
            assert first_diff(cl.submit(req), one.submit(req), 53) is None
            cl.save_image(src)
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "reshard_image.py"), src, dst, "--shards", "5",
                            "--device", "0"], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        with GpuCluster.open_image(dst, devices=[0] * 5, max_batch=4096) as cl5:
            assert cl5.G == 5
            for i in range(3):
                req = _trace(wire.STORE, 20000, seed=2 + i, skew=True)
                d = first_diff(cl5.submit(req), one.submit(req), 53)
                assert d is None, f"call {i}: {d}"
            assert sum(cl5.engine(s).kv_count(0) for s in range(5)) == one.kv_count(0)
    with GpuCluster.open_image(src, devices=[0] * 3) as cl3:
        assert cl3.G == 3


def _ref_round_trip(kind, srv, fam, tail):
    """50 rounds of 2^20 GPU clients on one engine and on a 3-shard cluster, the cluster re-sharded 3 -> 8 -> 1, then
    one 4 M-request batch on both"""
    n = 1 << 20
    with Engine(kind, **srv) as eng:
        with GpuClients(eng, n, seed=SEED, **fam) as one:
            one.run(50)
            one.stats()
        cl = GpuCluster(kind, 3, devices=[0] * 3, max_batch=n // 3 + 1, **srv)
        try:
            with GpuClusterClients(cl, n, seed=SEED, **fam) as cc:
                cc.run(50)
            for G2 in (8, 1):
                new = cl.reshard(G2, devices=[0] * G2)
                cl.close()
                cl = new
            req = tail()
            want = eng.submit(req)
            got = cl.submit(req)
            d = first_diff(got, want, wire.MSG_SIZE[kind])
            assert d is None, d
        finally:
            cl.close()


@pytest.mark.slow
def test_full_size_lock_fasst():
    _ref_round_trip(wire.FASST, {}, dict(REF), lambda: T.fasst_random(4 << 20, 24_000_000, seed=9))


@pytest.mark.slow
def test_full_size_store():
    srv = dict(populate=True)
    _ref_round_trip(wire.STORE, srv, dict(store_subscribers=2_000_000, set_pct=50),
                    lambda: T.store_random(4 << 20, 2_000_000, seed=9))
