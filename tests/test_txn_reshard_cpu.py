"""CPU: draining the host TATP / SmallBank clients (TxnWorkload.draining, busy, set_shards) against the oracles, then
re-placing every row on its replicas under another shard count and resuming; the placement rule of
dint_cluster_reshard_txn (dint_test_txn_reshard_dests); and the image tool's --replicas refusals.

The re-placed reference is built through the oracle's own wire handlers from its rows: a TATP row is inserted with
kInsertBck (version 0) on an empty oracle and written again with kCommitBck until it has the old primary's version; a
SmallBank row (every account is populated and none is ever deleted) gets the kCommitBck writes alone.  kCommitBck sets
the value and bumps the version by one, as the engine does."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as O
from dint_b200 import engine as E, wire
from dint_b200.txn_workloads import Cluster, TxnWorkload

TATP, SMALLBANK = wire.TATP, wire.SMALLBANK
N = {TATP: 1500, SMALLBANK: 3000}
CLIENTS = {TATP: 900, SMALLBANK: 1100}
N_TABLES = {TATP: 5, SMALLBANK: 2}
VALSZ = {TATP: 40, SMALLBANK: 8}
# the longest transaction, in rounds: TATP insert_call_forwarding (read secondary, read special facility, read + lock,
# verify, log, backups, primary), SmallBank's acquire, log, backups, primary, release.  A drain ends within L + 1 rounds
# emitted: at most L served, then the empty one.
LONGEST = {TATP: 7, SMALLBANK: 5}
ROUNDS_BEFORE, ROUNDS_AFTER = 20, 30


def oracle_cfg(kind):
    n = N[kind]
    return dict(subs_sizing=n, subs_populate=n) if kind == TATP else dict(accts_sizing=n, accts_populate=n)


def sub_nbr(s):
    r = 0
    for g in range(3):
        i = s % 1000
        s //= 1000
        r |= (((i // 100) % 10) << 8 | ((i // 10) % 10) << 4 | (i % 10)) << (12 * g)
    return r


def universe(kind):
    """every (table, key) a client or the population can touch"""
    n = N[kind]
    if kind == SMALLBANK:
        return [(t, a) for t in range(2) for a in range(n)]
    out = [(0, s) for s in range(n)] + [(1, sub_nbr(s)) for s in range(n)]
    out += [(t, s | (x << 32)) for t in (2, 3) for s in range(n) for x in range(1, 5)]
    out += [(4, s | (x << 32) | (st << 40)) for s in range(n) for x in range(1, 5) for st in (0, 8, 16)]
    return out


def replicas(key, G):
    return sorted({(key % G + i) % G for i in range(3)})


def rows_of(oras, kind, G):
    """{(table, key): (value bytes, version)} from each key's primary"""
    out = {}
    for t, k in universe(kind):
        r = oras[k % G].kv_get(t, k)
        if r is not None:
            out[(t, k)] = (r[0][:VALSZ[kind]], r[1])
    return out


def place(kind, rows, G2):
    """G2 oracles holding each row on its replicas under G2, built through the wire handlers (module docstring)"""
    oras = [O.Oracle(kind, populate=kind == SMALLBANK, **oracle_cfg(kind)) for _ in range(G2)]
    per = [[] for _ in range(G2)]
    ins, bck = (wire.Tatp.kInsertBck, wire.Tatp.kCommitBck) if kind == TATP else (None, wire.Smallbank.kCommitBck)
    for (t, k), (val, ver) in rows.items():
        types = ([ins] if kind == TATP else []) + [bck] * ver
        for s in replicas(k, G2):
            per[s] += [(ty, t, k, val) for ty in types]
    for o, recs in zip(oras, per):
        if not recs:
            continue
        a = np.zeros(len(recs), wire.MSG_DTYPE[kind])
        a["type"] = [r[0] for r in recs]
        a["table"] = [r[1] for r in recs]
        a["key"] = np.array([r[2] for r in recs], np.uint64)
        a["val"] = np.frombuffer(b"".join(r[3] for r in recs), np.uint8).reshape(len(recs), -1)
        o.process(wire.as_bytes(a))
    return oras


def serve(wl, cl, rounds):
    for _ in range(rounds):
        rq, dst = wl.next()
        assert dst.size and int(dst.max()) < len(cl.servers)
        wl.feed(cl.submit(rq, dst))


def drain(wl, cl):
    """serve rounds with the clients draining until one is empty; returns the rounds served (still draining)"""
    wl.draining = True
    served = 0
    for _ in range(LONGEST[wl.kind] + 1):
        rq, dst = wl.next()
        if not dst.size:
            break
        wl.feed(cl.submit(rq, dst))
        served += 1
    else:
        pytest.fail(f"the drain did not end within {LONGEST[wl.kind] + 1} rounds")
    return served


def check_drained(wl, oras, kind, G):
    assert wl.busy() == 0
    for t, k in universe(kind):
        reps = replicas(k, G)
        for s in reps:
            st = oras[s].lock_state(t, oras[s].lock_slot(t, k))
            assert st == (0, 0) if kind == SMALLBANK else st[0] == 0, (t, k, s, st)
        first = oras[reps[0]].kv_get(t, k)
        for s in reps[1:]:
            assert oras[s].kv_get(t, k) == first, (t, k, s)


def run_host(kind, G):
    """20 rounds, then a drain; returns (workload, oracles, drain rounds)"""
    oras = [O.Oracle(kind, **oracle_cfg(kind)) for _ in range(G)]
    wl = TxnWorkload(kind, n_clients=CLIENTS[kind], n_shards=G, subscribers=N[kind], gid0=5)
    cl = Cluster([o.process for o in oras], wire.MSG_SIZE[kind])
    serve(wl, cl, ROUNDS_BEFORE)
    assert wl.busy() == CLIENTS[kind]
    n = drain(wl, cl)
    assert 1 <= n <= LONGEST[kind]
    return wl, oras, n


@pytest.mark.parametrize("kind,G", [(TATP, 3), (TATP, 5), (SMALLBANK, 1), (SMALLBANK, 3), (SMALLBANK, 8)])
def test_drain_reaches_a_lock_free_replica_consistent_point(kind, G):
    wl, oras, n = run_host(kind, G)
    check_drained(wl, oras, kind, G)
    st = wl.stats()
    assert st["rounds"] == ROUNDS_BEFORE + n             # the empty round is not counted
    rq, dst = wl.next()                                  # still draining: nothing starts
    assert dst.size == 0 and wl.busy() == 0 and wl.stats() == st
    wl.draining = False                                  # resumed: every client begins in this emission
    rq, dst = wl.next()
    assert wl.busy() == CLIENTS[kind] and wl.stats()["txns"] == st["txns"] + CLIENTS[kind]


@pytest.mark.parametrize("kind,G,G2", [(TATP, 3, 5), (TATP, 5, 3), (TATP, 3, 4),
                                       (SMALLBANK, 3, 1), (SMALLBANK, 1, 3), (SMALLBANK, 3, 8)])
def test_replace_and_resume(kind, G, G2):
    wl, oras, n = run_host(kind, G)
    rows = rows_of(oras, kind, G)
    new = place(kind, rows, G2)
    assert rows_of(new, kind, G2) == rows
    before = wl.stats()
    wl.set_shards(G2)
    wl.draining = False
    cl = Cluster([o.process for o in new], wire.MSG_SIZE[kind])
    serve(wl, cl, ROUNDS_AFTER)                          # (an oracle that meets an error raises)
    st = wl.stats()
    assert st["committed"] > before["committed"]
    assert st["rounds"] == ROUNDS_BEFORE + n + ROUNDS_AFTER
    assert st["txns"] > before["txns"]


def test_set_shards_only_between_transactions():
    wl = TxnWorkload(TATP, n_clients=64, n_shards=3, subscribers=1000)
    with pytest.raises(ValueError):
        wl.set_shards(5)                                 # every client is mid-transaction
    assert wl.n_shards == 3
    oras = [O.Oracle(TATP, **oracle_cfg(TATP)) for _ in range(3)]
    cl = Cluster([o.process for o in oras], wire.MSG_SIZE[TATP])
    drain(wl, cl)
    wl.draining = False
    for bad in (0, 2, 9):
        with pytest.raises(ValueError):
            wl.set_shards(bad)
    assert wl.n_shards == 3
    wl.set_shards(4)
    assert wl.n_shards == 4


def test_replica_dests_hook_matches_the_rule():
    L = E.lib()
    rng = np.random.default_rng(3)
    keys = [0, 1, 2, 7, 8, 255, 2**32 - 1, 2**32, 2**63 + 5, 2**64 - 1] + [int(k) for k in rng.integers(0, 2**63, 60)]
    shard_counts = (1, 3, 4, 5, 6, 7, 8)
    for G in shard_counts:
        for G2 in shard_counts:
            for src in range(G):
                for k in keys:
                    want = sum(1 << s for s in replicas(k, G2)) if k % G == src else 0
                    assert L.dint_test_txn_reshard_dests(k, G, G2, src) == want, (k, G, G2, src)
    assert L.dint_test_txn_reshard_dests(5, 0, 3, 0) == 0 and L.dint_test_txn_reshard_dests(5, 3, 9, 2) == 0


TOOL = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "reshard_image.py")


@pytest.mark.parametrize("kind", [TATP, SMALLBANK])
@pytest.mark.parametrize("shards", [0, 2, 9])
def test_image_tool_replicas_refuses_bad_shard_counts(kind, shards, tmp_path):
    from test_reshard_cpu import _manifest
    src = str(tmp_path / "src")
    _manifest(src, kind, 3)
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, TOOL, src, str(tmp_path / "dst"), "--shards", str(shards), "--replicas"],
                       capture_output=True, text=True, timeout=120, env=env)
    assert r.returncode == 2 and "1 or 3..8" in r.stderr, r.stdout + r.stderr
    assert not os.path.exists(tmp_path / "dst")


def test_image_tool_replicas_refuses_other_kinds(tmp_path):
    from test_reshard_cpu import _manifest
    src = str(tmp_path / "src")
    _manifest(src, wire.STORE, 3)
    r = subprocess.run([sys.executable, TOOL, src, str(tmp_path / "dst"), "--shards", "5", "--replicas"],
                       capture_output=True, text=True, timeout=120, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 2 and "store" in r.stderr, r.stdout + r.stderr
