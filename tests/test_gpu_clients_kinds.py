"""-m gpu: the lock_2pl, store and log_server closed-loop clients resident on the GPU (dint_b200/csrc/clients.cuh,
dint_clients_create_cfg) must take, round for round, the decisions of the host-side restatement of the reference's
clients (workloads.cc, restating lock_2pl/caladan/client.cc:181-230, store/caladan/client_udp.cc:135-208 and
log_server/caladan/trace_init.sh:15-19) driving the oracle server: same requests on the wire every round, same replies
absorbed, same counters, and the same server state at the end."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from dint_b200 import DintError, Engine, GpuClients, lib, wire
from dint_b200.workloads import Workload
from golden_util import first_diff

pytestmark = pytest.mark.gpu

SEED = 77
POP = 2000                       # store subscribers the small engines and oracles populate


def _drive(kind, eng, ora, n, rounds, fam, on_round=None):
    """GpuClients on `eng` next to Workload + `ora`, `rounds` rounds; every round's requests (peek before the round)
    and absorbed replies (peek after it) must equal the host clients'.  on_round(req) sees every round's requests.
    Returns the final counters, equal on both sides."""
    msg = wire.MSG_SIZE[kind]
    wl = Workload(kind, n_clients=n, seed=SEED, **fam)
    with GpuClients(eng, n, seed=SEED, **fam) as gc:
        for r in range(rounds):
            want_req = wl.next()
            got_req, _ = gc.peek()
            d = first_diff(got_req, want_req, msg)
            assert d is None, f"round {r}: requests differ: {d}"
            want_resp = ora.process(want_req)
            wl.feed(want_resp)
            gc.run(1)
            _, got_resp = gc.peek()
            d = first_diff(got_resp, want_resp, msg)
            assert d is None, f"round {r}: replies differ: {d}"
            if on_round is not None:
                on_round(want_req)
        a, b = gc.stats(), wl.stats()
    assert a == b, (a, b)
    assert a["rounds"] == rounds and a["requests"] == rounds * n and a["committed"] > 0
    return a


def _set_keys(req, out):
    """collects the keys of a store round's kSet requests"""
    rec = req.reshape(-1, 53)
    out.update(int(k) for k in rec[rec[:, 0] == 1, 1:9].copy().view(np.uint64).reshape(-1))


def _check_kv_sample(eng, ora, keys, k=256):
    assert keys, "no kSet was sent"
    rng = np.random.default_rng(1)
    sample = rng.choice(sorted(keys), size=min(k, len(keys)), replace=False)
    for key in sample:
        assert eng.kv_get(0, int(key)) == ora.kv_get(0, int(key)), hex(int(key))


LOCK2PL_FAMS = [dict(n_keys=50000, zipf_theta=0.0), dict(n_keys=4800, zipf_theta=0.8), dict(n_keys=7, zipf_theta=0.0)]


@pytest.mark.parametrize("fam", LOCK2PL_FAMS, ids=["uniform", "zipf_hot", "tiny"])
def test_lock2pl_clients_reproduce_the_host_clients_round_for_round(fam):
    n, rounds = 3000, 120
    ora = O.Oracle(wire.LOCK2PL)
    with Engine(wire.LOCK2PL, chunk=2048) as eng:
        st = _drive(wire.LOCK2PL, eng, ora, n, rounds, fam)
        assert st["validation_aborts"] == 0 and st["not_exist"] == 0
        if fam["n_keys"] <= 4800:
            assert st["lock_rejects"] > 0
        if fam["zipf_theta"] > 0:
            assert eng.stats()["conflicted"] > 0         # the ordered replay ran under the clients
            for lid in range(fam["n_keys"]):
                slot = ora.lock_slot(0, lid)
                assert eng.lock_state(0, slot) == ora.lock_state(0, slot), lid


STORE_FAMS = {
    "parallel": dict(store_subscribers=POP),
    "contention": dict(store_subscribers=POP, set_pct=50),
    "hot": dict(store_hot=True, n_keys=4800, zipf_theta=0.8, set_pct=50),
    "misses": dict(store_subscribers=3000, set_pct=50),
}


@pytest.mark.parametrize("name", list(STORE_FAMS))
def test_store_clients_reproduce_the_host_clients_round_for_round(name):
    fam = STORE_FAMS[name]
    n, rounds = 3000, 120
    ora = O.Oracle(wire.STORE, subs_populate=POP)
    keys = set()
    with Engine(wire.STORE, chunk=2048, populate=True, subs_populate=POP) as eng:
        st = _drive(wire.STORE, eng, ora, n, rounds, fam, on_round=lambda req: _set_keys(req, keys))
        assert st["validation_aborts"] == st["lock_rejects"] == 0
        if name == "misses":
            assert st["not_exist"] > 0
        elif name == "parallel":
            assert st["not_exist"] == 0 and not keys
        else:
            assert st["not_exist"] == 0
            _check_kv_sample(eng, ora, keys)
        assert eng.kv_count(0) == ora.kv_count(0)


@pytest.mark.parametrize("ring", [None, 1000], ids=["default_ring", "ring1000"])
def test_log_clients_reproduce_the_host_clients_round_for_round(ring):
    n, rounds = 3000, 120
    cfg = {} if ring is None else dict(log_ring=ring)
    ora = O.Oracle(wire.LOG, **cfg)
    with Engine(wire.LOG, chunk=2048, **cfg) as eng:
        st = _drive(wire.LOG, eng, ora, n, rounds, {})
        assert st["committed"] == rounds * n
        got_ring, appended = eng.dump_log()
        assert appended == ora.log_appended() == rounds * n
        if ring is not None:
            assert n > ring                               # the ring wraps inside every round
        assert np.array_equal(got_ring, ora.log_ring())


RUN_K = {
    "lock2pl_zipf": (wire.LOCK2PL, dict(n_keys=4800, zipf_theta=0.8)),
    "store_contention": (wire.STORE, dict(store_subscribers=POP, set_pct=50)),
    "store_hot": (wire.STORE, dict(store_hot=True, n_keys=4800, zipf_theta=0.8, set_pct=50)),
    "log": (wire.LOG, {}),
}


@pytest.mark.parametrize("name", list(RUN_K))
def test_clients_many_rounds_in_one_call(name):
    """run(k) = k rounds back to back on the stream; the counters and the pending requests equal k single rounds."""
    kind, fam = RUN_K[name]
    n = 20000
    cfg = dict(populate=True, subs_populate=POP) if kind == wire.STORE else {}
    with Engine(kind, **cfg) as e1, Engine(kind, **cfg) as e2:
        with GpuClients(e1, n, seed=5, **fam) as a, GpuClients(e2, n, seed=5, **fam) as b:
            a.run(60)
            for _ in range(60):
                b.run(1)
            assert a.stats() == b.stats() and a.stats()["committed"] > 0 and a.stats()["rounds"] == 60
            ra, rb = a.peek(), b.peek()
            assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])


@pytest.mark.parametrize("name", ["lock2pl_ref", "store_contention"])
def test_clients_at_production_size(name):
    """2^20 clients, 20 rounds: lock_2pl at the reference's 24 M ids on 36 M lock slots, store contention over 200,000
    populated subscribers; every round compared with the host clients."""
    n, rounds = 1 << 20, 20
    if name == "lock2pl_ref":
        ora = O.Oracle(wire.LOCK2PL)
        with Engine(wire.LOCK2PL) as eng:
            st = _drive(wire.LOCK2PL, eng, ora, n, rounds, dict(n_keys=24_000_000))
            assert st["lock_rejects"] > 0
            rng = np.random.default_rng(3)
            for lid in rng.integers(0, 24_000_000, size=256).tolist():
                slot = ora.lock_slot(0, lid)
                assert eng.lock_state(0, slot) == ora.lock_state(0, slot), lid
    else:
        subs = 200_000
        ora = O.Oracle(wire.STORE, subs_populate=subs)
        keys = set()
        with Engine(wire.STORE, populate=True, subs_populate=subs) as eng:
            _drive(wire.STORE, eng, ora, n, rounds, dict(store_subscribers=subs, set_pct=50),
                   on_round=lambda req: _set_keys(req, keys))
            _check_kv_sample(eng, ora, keys)


def test_create_cfg_equals_create_for_lock_fasst():
    """dint_clients_create (lock_fasst, positional arguments) is dint_clients_create_cfg with the same family."""
    n, fam = 5000, dict(n_keys=4800, zipf_theta=0.8, read_pct=70)
    with Engine(wire.FASST) as e1, Engine(wire.FASST) as e2:
        with GpuClients(e1, n, seed=9, **fam) as a:
            b = GpuClients.__new__(GpuClients)
            b.engine, b.n, b.kind, b.msg = e2, n, wire.FASST, wire.MSG_SIZE[wire.FASST]
            h = C.c_void_p()
            assert lib().dint_clients_create(e2.h, n, 9, fam["n_keys"], fam["zipf_theta"], fam["read_pct"], C.byref(h)) == 0
            b.h = h
            try:
                for _ in range(30):
                    ra, rb = a.peek(), b.peek()
                    assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])
                    a.run(1)
                    b.run(1)
                assert a.stats() == b.stats() and a.stats()["not_exist"] == 0
                out = (C.c_uint64 * 5)()
                assert lib().dint_clients_stats(b.h, out) == 0
                s = b.stats()
                assert list(out) == [s["requests"], s["committed"], s["validation_aborts"], s["lock_rejects"], s["rounds"]]
            finally:
                b.close()


def test_invalid_clients_are_refused():
    with Engine(wire.TATP, subs_sizing=1000, subs_populate=1000) as eng:
        with pytest.raises(DintError) as ex:
            GpuClients(eng, 100)
        assert ex.value.code == -22 and "tatp" in str(ex.value)
    with Engine(wire.LOCK2PL, lock_slots=1 << 16) as eng:
        for bad in (dict(n_clients=0), dict(n_keys=0), dict(read_pct=101)):
            args = dict(n_clients=100)
            args.update(bad)
            with pytest.raises(DintError) as ex:
                GpuClients(eng, args.pop("n_clients"), **args)
            assert ex.value.code == -22, bad
        h = C.c_void_p()
        assert lib().dint_clients_create(eng.h, 100, 1, 100, 0.0, 80, C.byref(h)) == -22   # lock_fasst only
    with Engine(wire.STORE, subs_sizing=1000, subs_populate=1000) as eng:
        for bad in (dict(set_pct=101), dict(store_subscribers=0), dict(store_hot=True, n_keys=0)):
            with pytest.raises(DintError) as ex:
                GpuClients(eng, 100, **bad)
            assert ex.value.code == -22, bad
