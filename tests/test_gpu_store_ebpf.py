"""The store engine with the eBPF cache tier (DINT_CFG_STORE_EBPF_*) against the reference's eBPF store server: the
goldens made from its compiled XDP / TC programs, and, at the reference's sizes after the eBPF client's population,
the compiled programs themselves (oracle/_ref/store_ebpf_*) on random traces.  Replies, cache sets, table entries and
the table's key count must all be identical."""
import os

import numpy as np
import pytest

import store_ebpf_model as M
from dint_b200 import Engine, wire
from dint_b200.engine import DintError, GpuCluster

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "store_ebpf")
SUBS = 2_000_000                     # kSubscriberNum: 9,000,000 buckets, 24 M populated keys


def bucket(key):
    return M.fasthash64(int(key)) % M.REF_BUCKETS


def engine_state(engines, keys):
    """(sets, table) of `keys` read from the engine (or from the owning shard of a cluster's engines)"""
    sets = np.zeros((len(keys), M.CACHE_ENTRY), np.uint8)
    table = np.zeros(len(keys), dtype=M.TABLE_REC)
    for i, k in enumerate(keys):
        b = bucket(k)
        e = engines[b % len(engines)]
        sets[i] = e.store_cache_set(b)
        got = e.kv_get(0, int(k))
        if got is not None:
            val, ver = got
            table[i]["found"], table[i]["ver"] = 1, ver
            table[i]["val"] = np.frombuffer(bytes(val), dtype=np.uint8)
    return sets, table


def assert_same(got_resp, got_state, want_resp, want_sets, want_table):
    g, w = got_resp.reshape(-1, 53), want_resp.reshape(-1, 53)
    bad = np.flatnonzero((g != w).any(1))
    assert bad.size == 0, f"{bad.size} replies differ, first at {bad[0]}: {g[bad[0]][:1]} vs {w[bad[0]][:1]}"
    assert np.array_equal(got_state[0], want_sets)
    assert np.array_equal(got_state[1], want_table)


@pytest.mark.parametrize("variant", M.VARIANTS)
@pytest.mark.parametrize("chunk", [256, 4096, 1 << 20])
def test_golden_through_engine(variant, chunk):
    g = np.load(os.path.join(GOLDEN, f"{variant}.npz"))
    table = g["table"].reshape(-1).view(M.TABLE_REC)
    with Engine(wire.STORE, device=0, store_ebpf=variant, subs_populate=0, chunk=chunk) as eng:
        got = eng.submit(g["req"], check=False)
        assert_same(got, engine_state([eng], g["keys"]), g["resp"], g["sets"], table)
        assert eng.kv_count(0) == int(g["kv_count"])
        assert eng.stats()["errors"] == int((g["req"].reshape(-1, 53)[:, 0] > 2).sum())
        m = M.StoreEbpfModel(variant)         # the tier's counters, path by path, against the restatement's
        m.process(g["req"])
        assert eng.store_cache_stats() == m.stats


def ref_trace(seed):
    """Five segments over the populated store: GET only, 80/20 (client_ebpf.cc:61-63), 50/50, mostly absent keys, fresh
    inserts with reads of them, then 3000 requests on the keys of ONE bucket (a chunk's ordered replay overflows)."""
    rng = np.random.default_rng(seed)

    def keys(n, absent=False):
        s = rng.integers(0, SUBS, size=n).astype(np.uint64)
        sf = rng.integers(1, 5, size=n).astype(np.uint64) + (np.uint64(4) if absent else np.uint64(0))
        st = (rng.integers(0, 3, size=n) * 8).astype(np.uint64)
        return s | (sf << np.uint64(32)) | (st << np.uint64(40))

    segs = []
    for set_pct in (0, 20, 50):
        n = 20000
        segs.append(((rng.random(n) < set_pct / 100).astype(np.uint8), keys(n)))
    n = 8000
    k = keys(n)
    miss = rng.random(n) < 0.7
    k[miss] = keys(int(miss.sum()), absent=True)
    segs.append(((rng.random(n) < 0.4).astype(np.uint8), k))
    fresh = (np.arange(4000, dtype=np.uint64) + np.uint64(SUBS)) | (np.uint64(1) << np.uint64(32))
    t = np.concatenate([np.full(4000, 2, np.uint8), rng.integers(0, 2, size=4000).astype(np.uint8)])
    segs.append((t, np.concatenate([fresh, rng.choice(fresh, size=4000)])))
    hot = M.colliding_keys(M.REF_BUCKETS, 6, 1, seed=seed, key_space=1 << 30)[0]
    segs.append((rng.integers(0, 2, size=3000).astype(np.uint8), rng.choice(hot, size=3000)))
    types = np.concatenate([s[0] for s in segs])
    ks = np.concatenate([s[1] for s in segs])
    n = types.size
    req = M.make_req(types, ks, rng.integers(0, 256, size=(n, 40), dtype=np.uint8), rng.integers(0, 9, size=n, dtype=np.uint32))
    touched = np.unique(ks)      # state is compared on a sample of the touched keys and on every key of the hot bucket
    return req, np.unique(np.concatenate([rng.choice(touched, size=min(3000, touched.size), replace=False), hot]))


@pytest.mark.skipif(not M.ref_available(), reason="oracle/_ref/store_ebpf_* not built")
@pytest.mark.parametrize("variant", M.VARIANTS)
def test_reference_sizes_against_compiled_programs(variant):
    req, keys = ref_trace(7)
    want = M.run_ref_store_ebpf(variant, req, keys, populate=SUBS)
    with Engine(wire.STORE, device=0, store_ebpf=variant, chunk=4096, populate=True) as eng:
        eng.reset_stats()
        before = eng.store_cache_stats()
        got = eng.submit(req)
        assert_same(got, engine_state([eng], keys), *want[:3])
        assert eng.kv_count(0) == want[3]
        st, cs = eng.stats(), eng.store_cache_stats()
        d = {k: cs[k] - before[k] for k in cs}
        assert st["conflicted"] > 0 and st["ordered_fallbacks"] > 0      # bucket replay and the radix fallback both ran
        assert d["hits"] > 0 and d["table"] > 0 and d["installs"] > 0
        if variant != "wt":
            assert d["write_backs"] > 0
        if variant == "wb_bloom":
            assert d["bloom_negatives"] > 0


@pytest.mark.parametrize("variant", M.VARIANTS)
def test_snapshot_restores_the_cache(variant):
    g = np.load(os.path.join(GOLDEN, f"{variant}.npz"))
    req = g["req"].reshape(-1, 53)
    req = req[req[:, 0] <= 2]
    a, b = req[:1500].reshape(-1), req[1500:].reshape(-1)
    with Engine(wire.STORE, device=0, store_ebpf=variant, subs_populate=0, chunk=4096) as eng:
        eng.submit(a)
        snap = eng.snapshot()
        rb = eng.submit(b)
        sb = engine_state([eng], g["keys"])
        eng.restore(snap)
        eng.sync()
        assert_same(eng.submit(b), engine_state([eng], g["keys"]), rb, *sb)
        eng.free_snapshot(snap)


@pytest.mark.parametrize("variant", M.VARIANTS)
def test_three_shards_equal_one_engine(variant):
    req, keys = ref_trace(11)
    cfg = dict(store_ebpf=variant, subs_populate=3000)
    with Engine(wire.STORE, device=0, chunk=4096, populate=True, **cfg) as one, \
            GpuCluster(wire.STORE, 3, devices=[0, 0, 0], populate=True, **cfg) as cl:
        want = one.submit(req)
        got = cl.submit(req)
        shards = [cl.engine(i) for i in range(3)]
        assert_same(got, engine_state(shards, keys), want, *engine_state([one], keys))
        assert sum(e.kv_count(0) for e in shards) == one.kv_count(0)


def test_refused_for_other_kinds():
    for kind in (wire.LOCK2PL, wire.FASST, wire.LOG, wire.TATP, wire.SMALLBANK):
        with pytest.raises(DintError) as ei:
            Engine(kind, device=0, store_ebpf="wb")
        assert ei.value.code == -22
    with pytest.raises(DintError):
        GpuCluster(wire.FASST, 1, devices=[0], store_ebpf="wt")
    with Engine(wire.STORE, device=0, subs_populate=0) as eng:      # option off: no tier to inspect
        with pytest.raises(DintError):
            eng.store_cache_stats()
        with pytest.raises(DintError):
            eng.store_cache_set(0)
