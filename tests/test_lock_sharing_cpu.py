"""CPU: the same-key / false-sharing split of refused TATP locks (DINT_CFG_LOCK_HOLDER_KEYS, include/dint_b200.h;
tatp/ebpf/lock_kern.c:289-298) as far as it goes without a GPU: the model the GPU tests compare the engine with
(tests/lock_sharing_model.py), and the host clients' counters (TxnWorkload.lock_stats, the counters behind
tatp/caladan/client_lock.cc:403-428)."""
import numpy as np
import pytest

import lock_sharing_model as M
import oracle_lib as O
import trace_gen as T
from dint_b200 import wire
from dint_b200.txn_workloads import Cluster, TxnWorkload
from dint_b200.wire import Tatp

S = 2000            # subs_sizing: lock moduli of a few thousand slots, so that keys share slots often
CFG = dict(subs_sizing=S, subs_populate=S)


def test_wire_names_and_constructor_spelling():
    from dint_b200 import engine as E
    assert Tatp.kRejectLock == 8 and Tatp.kRejectLockSameKey == 28
    assert E.default_cfg(wire.TATP).flags == 0
    assert E.default_cfg(wire.TATP, lock_holder_keys=True).flags == E.DINT_CFG_LOCK_HOLDER_KEYS == 1
    assert E.default_cfg(wire.TATP, lock_holder_keys=False).flags == 0


def test_model_slots_are_the_servers_slots():
    ora = O.Oracle(wire.TATP, populate=False, **CFG)
    model = M.HolderModel(S)
    rng = np.random.default_rng(1)
    for tb in range(5):
        for key in [0, 1, 2**40 + 5, 2**64 - 1] + [int(k) for k in rng.integers(0, 2**63, size=200)]:
            assert model.slot(tb, key) == ora.lock_slot(tb, key)
    for tb in range(5):
        for a, b in M.colliding_pairs(S, tb, 8):
            assert a != b and ora.lock_slot(tb, a) == ora.lock_slot(tb, b)


def test_scripted_trace_has_both_reject_kinds_where_lock_kern_puts_them():
    """The expected types are written out by hand from tatp/ebpf/lock_kern.c:289-298,338."""
    (a, b), (c, d) = M.colliding_pairs(S, Tatp.kCallForwarding, 2)
    L, A = Tatp.kAcquireLock, Tatp.kAbort
    script = [
        (L, a, 7),     # free slot: granted, holder = a
        (L, a, 28),    # the same key again: a true conflict
        (L, b, 8),     # a foreign key on the held slot: false sharing
        (A, a, 9),     # release: the bit clears, the holder word stays a
        (L, b, 7),     # a stale holder word under a clear bit grants (and becomes b)
        (L, a, 8),     # the old key now meets a foreign holder: 8, not 28
        (L, b, 28),
        (A, b, 9),
        (L, a, 7),     # stale word b, clear bit: granted to a
        (L, a, 28),
        (L, c, 7),     # another slot is untouched by all of this
        (L, d, 8),
    ]
    req = M.lock_records([s[0] for s in script], [s[1] for s in script], table=Tatp.kCallForwarding)
    ora = M.HolderOracle(**CFG)
    got = ora.process(req)
    assert list(wire.as_records(wire.TATP, got)["type"]) == [s[2] for s in script]
    plain = O.Oracle(wire.TATP, **CFG).process(req)
    assert np.array_equal(M.to_option_off(got), plain)
    slot = ora.model.slot(Tatp.kCallForwarding, a)
    assert ora.model.held(Tatp.kCallForwarding, slot) and ora.model.holder(Tatp.kCallForwarding, slot) == a
    assert ora.lock_state(Tatp.kCallForwarding, slot)[0] == 1


def test_random_trace_splits_rejects_and_keeps_the_option_off_stream():
    ora = M.HolderOracle(subs_sizing=60, subs_populate=40)
    plain = O.Oracle(wire.TATP, subs_sizing=60, subs_populate=40)
    req = T.tatp_random(30000, 40, seed=5, oracle=plain)
    got, off = ora.process(req), plain.process(req)        # the model asserts every lock decision on the way
    locks, sharing, same = M.count_lock_replies(req, got)
    assert sharing > 100 and same > 100
    assert np.array_equal(M.to_option_off(got), off)
    assert M.count_lock_replies(req, off) == (locks, sharing + same, 0)
    with pytest.raises(ValueError):                        # 28 is a reply type: as a REQUEST it is still invalid
        plain.process(M.lock_records([28], [1]))


def _closed_loop(servers, G, n, clients, rounds, gid0=3):
    cl = Cluster(servers, wire.MSG_SIZE[wire.TATP])
    wl = TxnWorkload(wire.TATP, n_clients=clients, n_shards=G, subscribers=n, gid0=gid0)
    trace, seen = [], np.zeros(3, dtype=np.int64)
    for _ in range(rounds):
        rq, dst = wl.next()
        rs = cl.submit(rq, dst)
        wl.feed(rs)
        seen += M.count_lock_replies(rq, rs)
        trace.append((rq.copy(), dst.copy(), rs.copy()))
    return trace, wl.stats(), wl.lock_stats(), seen


@pytest.mark.parametrize("G", [3, 5])
def test_host_clients_count_what_the_reply_stream_holds(G):
    n, clients, rounds = 1500, 1300, 300
    cfg = dict(subs_sizing=n, subs_populate=n)
    on = [M.HolderOracle(**cfg) for _ in range(G)]
    t_on, st_on, ls_on, seen = _closed_loop([o.process for o in on], G, n, clients, rounds)
    assert (ls_on["locks"], ls_on["reject_sharing"], ls_on["reject_same_key"]) == tuple(seen)
    assert ls_on["reject_sharing"] > 50 and ls_on["reject_same_key"] > 50
    refused = sum(int((wire.as_records(wire.TATP, rs)["type"][wire.as_records(wire.TATP, rq)["type"] == 1] != 7).sum())
                  for rq, _, rs in t_on)
    assert ls_on["reject_sharing"] + ls_on["reject_same_key"] == refused
    # a same-key reject aborts the transaction exactly as a plain reject does: against servers without the option the
    # clients emit the same records, round for round, and only the split of the counters differs
    off = [O.Oracle(wire.TATP, **cfg) for _ in range(G)]
    t_off, st_off, ls_off, _ = _closed_loop([o.process for o in off], G, n, clients, rounds)
    assert st_on == st_off and st_on["committed"] > 0
    for r, ((q1, d1, s1), (q2, d2, s2)) in enumerate(zip(t_on, t_off)):
        assert np.array_equal(q1, q2) and np.array_equal(d1, d2), f"round {r}: the clients diverged"
        assert np.array_equal(M.to_option_off(s1), s2), f"round {r}"
    assert ls_off == dict(locks=ls_on["locks"], reject_sharing=refused, reject_same_key=0)


def test_smallbank_clients_count_no_locks():
    n = 2000
    oras = [O.Oracle(wire.SMALLBANK, accts_populate=n) for _ in range(3)]
    cl = Cluster([o.process for o in oras], wire.MSG_SIZE[wire.SMALLBANK])
    wl = TxnWorkload(wire.SMALLBANK, n_clients=300, n_shards=3, subscribers=n)
    for _ in range(30):
        rq, dst = wl.next()
        wl.feed(cl.submit(rq, dst))
    assert wl.stats()["committed"] > 0
    assert wl.lock_stats() == dict(locks=0, reject_sharing=0, reject_same_key=0)
