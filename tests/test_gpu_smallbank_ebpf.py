"""The smallbank engine with the eBPF cache tier (DINT_CFG_SMALLBANK_EBPF) against the reference's eBPF SmallBank shard
server: the goldens made from its compiled XDP / TC programs at the reference's sizes (cold: the tables populated, the
cache empty, as dint_load leaves it; warm: after dint_populate's warm-up), and the plain restatement in
tests/smallbank_ebpf_model.py on a colliding-key trace.  Replies, cache sets, table finds, lock units, the log ring and
the tier's counters must all be identical."""
import os

import numpy as np
import pytest

import smallbank_ebpf_model as M
from dint_b200 import Engine, wire
from dint_b200.engine import DintError

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "smallbank_ebpf")


def submit(eng, req, path):
    if path == "host":
        return eng.submit(req, check=False)
    import torch
    return eng.submit_tensor(torch.from_numpy(np.ascontiguousarray(req)).cuda()).cpu().numpy().reshape(-1)


def load_accounts(eng, populated):
    """kvs_insert of accounts [0, populated) into both tables, the cache left cold"""
    keys = np.arange(populated, dtype=np.uint64)
    for t in range(2):
        vals = np.frombuffer(M.initial_value(t) * populated, dtype=np.uint8)
        eng.load(t, keys, vals)


def engine_for(z, chunk):
    P, warm = int(z["populated"]), bool(z["warm"])
    eng = Engine(wire.SMALLBANK, device=0, smallbank_ebpf=True, accts_populate=P, chunk=chunk)
    if warm:
        eng.populate()
    else:
        load_accounts(eng, P)
    return eng


def engine_state(eng, H, keys, tables):
    """(sets, finds, locks) as run_ref_smallbank_ebpf dumps them, read through the C ABI"""
    n = len(keys)
    sets = np.zeros((n, M.CACHE_ENTRY), np.uint8)
    finds = np.zeros(n, dtype=M.FIND_REC)
    locks = np.zeros(n, dtype=M.LOCK_REC)
    for i, (k, t) in enumerate(zip(keys, tables)):
        k, t = int(k), int(t)
        h = M.fasthash64(k)
        sets[i] = eng.smallbank_cache_set(t, h % H)
        got = eng.kv_get(t, k)
        if got is not None:
            finds[i]["found"], finds[i]["ver"] = 1, got[1]
            finds[i]["val"] = np.frombuffer(bytes(got[0])[:8], dtype=np.uint8)
        slot = h % (4 * H)
        assert eng.lock_slot(t, k) == slot
        locks[i]["num_ex"], locks[i]["num_sh"] = eng.lock_state(t, slot)
    return sets, finds, locks


def assert_replies(got, want):
    g, w = np.asarray(got).reshape(-1, M.MSG), np.asarray(want).reshape(-1, M.MSG)
    bad = np.flatnonzero((g != w).any(1))
    assert bad.size == 0, f"{bad.size} replies differ, first at {bad[0]}: {g[bad[0]]} vs {w[bad[0]]}"


def assert_state(got, want):
    for name, a, b in zip(("sets", "finds", "locks"), got, want):
        bad = np.flatnonzero((np.asarray(a).reshape(len(a), -1).view(np.uint8) != np.asarray(b).reshape(len(b), -1).view(np.uint8)).any(1))
        assert bad.size == 0, f"{name}: {bad.size} keys differ, first at {bad[0]}"


@pytest.mark.parametrize("name", ["cold", "warm"])
@pytest.mark.parametrize("chunk", [256, 4096, 65536])
@pytest.mark.parametrize("path", ["host", "device"])
def test_golden_through_engine(name, chunk, path):
    z = np.load(os.path.join(GOLDEN, f"{name}.npz"))
    m = M.SmallbankEbpfModel(populated=int(z["populated"]))
    if bool(z["warm"]):
        m.warmup()
    with engine_for(z, chunk) as eng:
        assert eng.smallbank_cache_stats() == m.stats
        s0 = eng.stats()                                   # (the warm-up of dint_populate is counted too)
        got = submit(eng, z["req"], path)
        assert_replies(got, z["resp"])
        want = (z["sets"], z["finds"].view(M.FIND_REC), z["locks"].view(M.LOCK_REC))
        assert_state(engine_state(eng, M.hash_size(), z["keys"], z["tables"]), want)
        ring, appended = eng.dump_log()
        assert appended == len(z["log"])
        np.testing.assert_array_equal(ring[:appended], z["log"])
        m.process(z["req"])
        assert eng.smallbank_cache_stats() == m.stats
        bad = m.paths["invalid_type"] + m.paths["invalid_table"] + m.paths["missing_key"] + m.paths["missing_key_after_write_back"]
        st = eng.stats()
        assert st["errors"] - s0["errors"] == bad
        n = len(z["req"]) // M.MSG
        assert 0 < st["conflicted"] - s0["conflicted"] < n                    # the solo path and the bucket replay both answered


def test_colliding_trace_equals_model():
    """a longer trace over more colliding buckets, on an engine sized for the accounts it holds (A = 600,000)"""
    A = 600_000
    groups = M.colliding_groups(A, A=A, per_bucket=5, n_buckets=12, seed=5)
    keys, tables = M.group_keys(groups)
    req = M.random_trace(groups, 30000, seed=6)
    m = M.SmallbankEbpfModel(A=A, populated=A)
    m.warmup()
    with Engine(wire.SMALLBANK, device=0, smallbank_ebpf=True, accts_sizing=A, accts_populate=A, chunk=8192,
                populate=True) as eng:
        assert eng.smallbank_cache_stats() == m.stats
        assert_replies(eng.submit(req, check=False), m.process(req))
        assert_state(engine_state(eng, M.hash_size(A), keys, tables), m.state(keys, tables))
        assert eng.smallbank_cache_stats() == m.stats
        for t in range(2):
            assert eng.kv_count(t) == A
        assert eng.stats()["conflicted"] > 0


def test_snapshot_restore_replays_the_same():
    z = np.load(os.path.join(GOLDEN, "warm.npz"))
    req = z["req"].reshape(-1, M.MSG)
    first, second = req[:3000].reshape(-1), req[3000:].reshape(-1)
    with engine_for(z, 4096) as eng:
        eng.submit(first, check=False)
        snap = eng.snapshot()
        a = eng.submit(second, check=False).copy()
        import torch
        eng.restore(snap)
        torch.cuda.synchronize()
        b = eng.submit(second, check=False)
        np.testing.assert_array_equal(a, b)
        assert_replies(b, z["resp"].reshape(-1, M.MSG)[3000:])


def test_refusals_and_the_plain_engine():
    with pytest.raises(DintError):
        Engine(wire.TATP, device=0, smallbank_ebpf=True, subs_populate=0)
    with pytest.raises(DintError):
        Engine(wire.STORE, device=0, smallbank_ebpf=True, subs_populate=0)
    with pytest.raises(DintError):
        Engine(wire.SMALLBANK, device=0, smallbank_ebpf=True, accts_populate=0, n_shards=2, shard_id=0)
    with Engine(wire.SMALLBANK, device=0, accts_sizing=6000, accts_populate=6000, populate=True) as plain:
        with pytest.raises(DintError):
            plain.smallbank_cache_set(0, 0)
        with pytest.raises(DintError):
            plain.smallbank_cache_stats()
        req = M.make_req([M.WARMUP_READ, M.WARMUP_READ], [0, 1], [5, 7])
        got = plain.submit(req, check=False).reshape(-1, M.MSG)
        assert got[:, 1].tolist() == [0xFF, 0xFF]          # the UDP server knows no kWarmupRead
    with Engine(wire.SMALLBANK, device=0, smallbank_ebpf=True, accts_sizing=6000, accts_populate=0) as eng:
        with pytest.raises(DintError):
            eng.store_cache_set(0)
        with pytest.raises(DintError):
            eng.smallbank_cache_set(2, 0)
        with pytest.raises(DintError):
            eng.smallbank_cache_set(1, M.hash_size(6000))
