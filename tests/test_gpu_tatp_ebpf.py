"""The tatp engine with the eBPF cache tier (DINT_CFG_TATP_EBPF, with and without holder keys) against the reference's
eBPF TATP shard server: the goldens made from its compiled XDP / TC programs at the reference's sizes, and the plain
restatement in tests/tatp_ebpf_model.py on small populated engines.  Replies, cache sets, chains, table finds, lock and
holder words, the log ring and the tier's counters must all be identical."""
import os

import numpy as np
import pytest

import tatp_ebpf_model as M
from dint_b200 import Engine, wire
from dint_b200.engine import DintError

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tatp_ebpf")


def submit(eng, req, path):
    if path == "host":
        return eng.submit(req, check=False)
    import torch
    return eng.submit_tensor(torch.from_numpy(np.ascontiguousarray(req)).cuda()).cpu().numpy().reshape(-1)


def engine_state(eng, H, keys, tables, holder_keys):
    """(sets, chains, finds, locks) as run_ref_tatp_ebpf dumps them, read through the C ABI"""
    n = len(keys)
    sets = np.zeros((n, M.CACHE_ENTRY), np.uint8)
    chains = np.zeros(n, dtype=M.CHAIN_DUMP)
    finds = np.zeros(n, dtype=M.FIND_REC)
    locks = np.zeros(n, dtype=M.LOCK_REC)
    for i, (k, t) in enumerate(zip(keys, tables)):
        k, t = int(k), int(t)
        h = M.fasthash64(k)
        sets[i] = eng.tatp_cache_set(t, h % H[t])
        ch = eng.tatp_chain(t, h % H[t])
        chains[i]["n"] = len(ch)
        chains[i]["rec"][:len(ch)] = ch.view(M.CHAIN_REC)
        got = eng.kv_get(t, k)
        if got is not None:
            finds[i]["found"], finds[i]["ver"] = 1, got[1]
            finds[i]["val"] = np.frombuffer(bytes(got[0]), dtype=np.uint8)
        slot = h % (4 * H[t])
        assert eng.lock_slot(t, k) == slot
        locks[i]["lock"] = eng.lock_state(t, slot)[0]
        locks[i]["holder"] = eng.lock_holder(t, slot) if holder_keys else 0
    return sets, chains, finds, locks


def assert_replies(got, want):
    g, w = np.asarray(got).reshape(-1, M.MSG), np.asarray(want).reshape(-1, M.MSG)
    bad = np.flatnonzero((g != w).any(1))
    assert bad.size == 0, f"{bad.size} replies differ, first at {bad[0]}: {g[bad[0]][:12]} vs {w[bad[0]][:12]}"


def assert_state(got, want):
    for name, a, b in zip(("sets", "chains", "finds", "locks"), got, want):
        bad = np.flatnonzero((np.asarray(a).reshape(len(a), -1).view(np.uint8) != np.asarray(b).reshape(len(b), -1).view(np.uint8)).any(1))
        assert bad.size == 0, f"{name}: {bad.size} keys differ, first at {bad[0]}"


@pytest.mark.parametrize("variant", M.VARIANTS)
@pytest.mark.parametrize("chunk", [256, 4096, 65536])
@pytest.mark.parametrize("path", ["host", "device"])
def test_golden_through_engine(variant, chunk, path):
    g = np.load(os.path.join(GOLDEN, f"{variant}.npz"))
    hk = variant == "lock"
    with Engine(wire.TATP, device=0, tatp_ebpf=True, lock_holder_keys=hk, subs_populate=0, chunk=chunk) as eng:
        got = submit(eng, g["req"], path)
        assert_replies(got, g["resp"])
        want = (g["sets"], g["chains"].view(M.CHAIN_DUMP), g["finds"].view(M.FIND_REC), g["locks"].view(M.LOCK_REC))
        assert_state(engine_state(eng, M.hash_sizes(M.REF_S), g["keys"], g["tables"], hk), want)
        ring, appended = eng.dump_log()
        assert appended == len(g["log"])
        np.testing.assert_array_equal(ring[:appended], g["log"])
        m = M.TatpEbpfModel(holder_keys=hk)
        m.process(g["req"])
        assert eng.tatp_cache_stats() == m.stats
        assert eng.stats()["errors"] == m.paths["invalid"]
        st = eng.stats()
        n = len(g["req"]) // M.MSG
        assert 0 < st["conflicted"] < n                    # the solo path and the bucket replay both answered
        if chunk == 65536:
            assert st["ordered_fallbacks"] >= 1             # one chunk, fifteen buckets: the radix fallback ran


def small_traffic(S, keys_by_table, n, seed):
    """TATP-shaped traffic over populated rows: reads, lock / commit / abort pairs, inserts of fresh call forwarding
    rows, and deletes followed by reads in the same bucket"""
    rng = np.random.default_rng(seed)
    ty, tb, ks = [], [], []
    for _ in range(n):
        t = int(rng.integers(0, 5))
        k = int(keys_by_table[t][rng.integers(0, len(keys_by_table[t]))])
        r = rng.random()
        if r < 0.45:
            ty += [M.READ]; tb += [t]; ks += [k]
        elif r < 0.65:
            ty += [M.ACQUIRE_LOCK, M.COMMIT_PRIM, M.COMMIT_BCK, M.COMMIT_LOG]; tb += [t] * 4; ks += [k] * 4
        elif r < 0.72:
            ty += [M.ACQUIRE_LOCK, M.ABORT]; tb += [t] * 2; ks += [k] * 2
        elif r < 0.85:
            k = int(rng.integers(0, S)) | (int(rng.integers(1, 5)) << 32) | (int(rng.integers(0, 3)) * 8 << 40)
            ty += [M.READ, M.INSERT_PRIM, M.INSERT_BCK, M.READ]; tb += [4] * 4; ks += [k] * 4
        else:
            ty += [M.DELETE_PRIM, M.DELETE_BCK, M.DELETE_LOG, M.READ, M.READ]; tb += [t] * 5
            ks += [k, k, k, k, int(keys_by_table[t][rng.integers(0, len(keys_by_table[t]))])]
    m = len(ty)
    vals = rng.integers(0, 256, size=(m, 40), dtype=np.uint8)
    vers = rng.integers(0, 1 << 32, size=m, dtype=np.uint64).astype(np.uint32)
    return M.make_req(ty, tb, ks, vals, vers), np.array(ks, dtype=np.uint64), np.array(tb, dtype=np.uint8)


@pytest.mark.parametrize("variant", M.VARIANTS)
def test_small_populated_engine_equals_model(variant):
    S, hk = 6000, variant == "lock"
    m = M.TatpEbpfModel(holder_keys=hk, S=S)
    m.populate(S)
    rows = M.population(S)
    keys_by_table = [[k for t, k, _ in rows if t == tt] for tt in range(5)]
    groups = M.colliding_groups(S, per_bucket=8, n_buckets=6, seed=7)
    reqs = [M.random_trace(groups, 6000, seed=11)] + [small_traffic(S, keys_by_table, 4000, seed=s)[0] for s in (1, 2)]
    with Engine(wire.TATP, device=0, tatp_ebpf=True, lock_holder_keys=hk, subs_sizing=S, subs_populate=S,
                chunk=4096) as eng:
        eng.populate()
        assert eng.tatp_cache_stats() == m.stats
        for req in reqs:
            assert_replies(eng.submit(req, check=False), m.process(req))
        keys = np.array([k for _, k, _ in rows[::3]] + [k for g in groups for grp in g for k in grp], dtype=np.uint64)
        tables = np.array([t for t, _, _ in rows[::3]] + [t for t, g in enumerate(groups) for grp in g for _ in grp],
                          dtype=np.uint8)
        assert_state(engine_state(eng, M.hash_sizes(S), keys, tables, hk), m.state(keys, tables))
        assert eng.tatp_cache_stats() == m.stats
        assert m.paths["read_bloom_neg_false"] > 0 and m.paths["insert_duplicate"] > 0
        for t in range(5):
            assert eng.kv_count(t) == sum(sum(e[3]) for ch in m.table[t].values() for e in ch)
        d = eng.stats()
        assert d["conflicted"] > 0 and d["ordered_fallbacks"] > 0


def test_snapshot_restore_replays_the_same():
    g = np.load(os.path.join(GOLDEN, "lock.npz"))
    req = g["req"].reshape(-1, M.MSG)
    first, second = req[:4000].reshape(-1), req[4000:].reshape(-1)
    with Engine(wire.TATP, device=0, tatp_ebpf=True, lock_holder_keys=True, subs_populate=0, chunk=4096) as eng:
        eng.submit(first, check=False)
        snap = eng.snapshot()
        a = eng.submit(second, check=False).copy()
        import torch
        eng.restore(snap)
        torch.cuda.synchronize()
        b = eng.submit(second, check=False)
        np.testing.assert_array_equal(a, b)
        assert_replies(b, g["resp"].reshape(-1, M.MSG)[4000:])


def test_refusals():
    with pytest.raises(DintError):
        Engine(wire.STORE, device=0, tatp_ebpf=True, subs_populate=0)
    with pytest.raises(DintError):
        Engine(wire.SMALLBANK, device=0, tatp_ebpf=True, accts_populate=0)
    with pytest.raises(DintError):
        Engine(wire.TATP, device=0, tatp_ebpf=True, subs_populate=0, n_shards=2, shard_id=0)
    with Engine(wire.TATP, device=0, subs_sizing=6000, subs_populate=0) as plain:
        with pytest.raises(DintError):
            plain.tatp_cache_set(0, 0)
        with pytest.raises(DintError):
            plain.tatp_cache_stats()
    with Engine(wire.TATP, device=0, tatp_ebpf=True, subs_sizing=6000, subs_populate=0) as eng:
        with pytest.raises(DintError):
            eng.store_cache_set(0)
        with pytest.raises(DintError):
            eng.tatp_cache_set(5, 0)
        with pytest.raises(DintError):
            eng.tatp_cache_set(4, M.hash_sizes(6000)[4])
