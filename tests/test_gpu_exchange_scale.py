"""-m gpu: the multi-GPU exchange and the GPU transaction clients at the sizes production runs them, and over long runs.

The other suites drive k_route_dispatch / k_route_combine, the shard step (shard_run / shard_engine) and the TATP /
SmallBank clients on the GPU (k_txn_step / k_txn_scan / k_txn_compact) with batches of a few tiles.  Whole branches of
those kernels only run at larger sizes or after many calls, and each case here is sized to reach one of them:

  A  the dispatch look-back's second window of group descriptors (a tile index >= 1056, i.e. 33 groups of 32 tiles),
     against numpy, for every record size and both tile sizes (2048 records for 6 / 9 bytes, 256 for 23 / 53 / 55);
  B  the cluster at max_batch 2^19 .. 2^22 (>= 2048 dispatch tiles per rank) and engine chunks of G x cap records,
     with a skewed call whose recovery rounds put a whole chunk on one lock slot (the radix fallback of k_ordered);
  C  the GPU clients with 80 k clients per rank (313 tiles: two passes of k_txn_scan) and 2^20 clients, ranks that hold
     no client, and 600 rounds (route_seq, 1..255, wraps twice and clears the look-back descriptors);
  D  commit-log rings (tatp, smallbank) smaller than one chunk's appends, on one engine and across the exchange;
  E  a KV table rehashed inside the exchange step (kv_maintain in shard_engine -> run_device): once doubled, once only
     cleared of tombstones.

Everything is compared bit for bit with numpy or with the oracle (one sequential server, or G shard servers)."""
import numpy as np
import pytest

import oracle_lib as O
import trace_gen as T
from dint_b200 import Engine, GpuCluster, GpuTxnClients, wire
from dint_b200.engine import lib
from dint_b200.txn_workloads import Cluster, TxnWorkload
from dint_b200.wire import Tatp
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


def _pop(kind, n):
    return dict(subs_populate=n) if kind == wire.TATP else dict(accts_populate=n)


# ---------------------------------------------------------------- A: dispatch / combine at large tile counts ------
def _route_records(kind, n, seed):
    """n valid wire records of `kind` whose keys spread over many lock slots / table groups, and the engine config."""
    rng = np.random.default_rng(seed)
    if kind == wire.FASST:
        return T.fasst_random(n, 10**6, seed=seed), {}
    if kind == wire.LOCK2PL:
        return T.lock2pl_random(n, 10**5, seed=seed), {}
    if kind == wire.STORE:
        return T.store_random(n, 500, seed=seed), dict(subs_populate=500)
    if kind == wire.SMALLBANK:
        return T.smallbank_random(n, 300000, seed=seed), dict(accts_populate=300)
    # tatp: a valid trace of 4096 records, resampled to n with the subscriber id of every key redrawn (the type / table
    # pairs stay those of valid requests; the keys spread over 2^20 subscribers)
    base = wire.as_records(wire.TATP, T.tatp_random(4096, 300, seed=seed))
    rec = base[rng.integers(0, base.size, size=n)].copy()
    rec["key"] = (rec["key"] & np.uint64(0xFFFFFFFF00000000)) | rng.integers(0, 1 << 20, size=n).astype(np.uint64)
    return wire.as_bytes(rec), dict(subs_populate=300)


def _tilebase_want(owner, n_tiles, recs, world):
    """[n_tiles][world]: records owned by shard o in the tiles before t"""
    pad = np.full(n_tiles * recs, 0xFF, dtype=np.uint8)
    pad[: owner.size] = owner
    tiles = pad.reshape(n_tiles, recs)
    cnt = np.stack([(tiles == o).sum(1) for o in range(world)], axis=1).astype(np.int64)
    return np.cumsum(cnt, axis=0) - cnt


def _dispatch_and_check(eng, req, n, world, rank, want_owner, owner_in, cap, what):
    """One dispatch into back-to-back slabs of `cap` records and one combine of those slabs, checked against numpy:
    owner bytes, tilebase, every slab (its first min(count, cap) records in request order, then 0xFE padding), the
    overflow count and the combine (identity; 0xFF for records that are undeliverable or did not fit)."""
    import torch
    msg = wire.MSG_SIZE[eng.kind]
    recs = lib().dint_route_tile_records(eng.h)
    n_tiles = (n + recs - 1) // recs
    d = torch.from_numpy(req).cuda()
    slabs = torch.zeros(world * cap * msg, dtype=torch.uint8, device="cuda")
    flags = torch.zeros(2, dtype=torch.int32, device="cuda")
    ptrs = Engine.slab_ptrs(slabs.data_ptr(), world, cap * msg)
    state = eng.route_dispatch(d, n, world, rank, cap, ptrs, flags,
                               owner_in=None if owner_in is None else torch.from_numpy(owner_in).cuda())
    own_want = np.where(want_owner < world, want_owner, 255).astype(np.uint8)
    own = state[0].cpu().numpy()[:n]
    assert np.array_equal(own, own_want), f"{what}: owner bytes"
    tb = state[1].cpu().numpy()[: n_tiles * 8].reshape(n_tiles, 8)[:, :world]
    tb_want = _tilebase_want(own_want, n_tiles, recs, world)
    bad = np.argwhere(tb != tb_want)
    assert bad.size == 0, f"{what}: tilebase[{bad[0][0]}][{bad[0][1]}] = {tb[tuple(bad[0])]}, want {tb_want[tuple(bad[0])]}"
    rec = req.reshape(n, msg)
    got = slabs.cpu().numpy().reshape(world, cap, msg)
    counts = np.bincount(own_want[own_want < world], minlength=world)[:world]
    for o in range(world):
        k = min(int(counts[o]), cap)
        assert np.array_equal(got[o, :k], rec[own_want == o][:k]), f"{what}: slab {o}"
        assert (got[o, k:] == 0xFE).all(), f"{what}: padding of slab {o}"
    assert flags.cpu().tolist() == [int(np.maximum(counts - cap, 0).sum()), 0], f"{what}: flags"
    out = torch.empty(n * msg, dtype=torch.uint8, device="cuda")
    eng.route_combine(ptrs, state, n, world, cap, out)
    back = out.cpu().numpy().reshape(n, msg)
    served = own_want < world
    for o in range(world):
        served[np.flatnonzero(own_want == o)[cap:]] = False             # dropped by a full slab
    assert np.array_equal(back[served], rec[served]), f"{what}: combine"
    assert (back[~served] == 0xFF).all(), f"{what}: error replies"


@pytest.mark.parametrize("world", [1, 3, 8])
@pytest.mark.parametrize("kind", [wire.LOCK2PL, wire.FASST, wire.SMALLBANK, wire.STORE, wire.TATP])
def test_route_dispatch_combine_at_large_tile_counts(kind, world):
    """1024 tiles (32 full groups: one window), 1025 (a 33rd group, nobody before it in the second window), 1057 (a
    tile that reads the second window) and 4100 with a ragged last tile (129 groups, the last one of 4 tiles);
    computed owners and client-chosen owners of which a few name a shard that does not exist."""
    from dint_b200.shard import owners_cpu
    rank = world - 1
    _, cfg = _route_records(kind, 1, 0)
    rng = np.random.default_rng(world)
    with Engine(kind, n_shards=world, shard_id=rank, chunk=4096, **cfg) as eng:
        recs = lib().dint_route_tile_records(eng.h)
        assert recs == (2048 if wire.MSG_SIZE[kind] <= 12 else 256)
        for tiles in (1024, 1025, 1057, 4100):
            n = tiles * recs if tiles != 4100 else (tiles - 1) * recs + recs // 3 + 5
            req, _ = _route_records(kind, n, seed=tiles)
            for by_dst in (False, True):
                if by_dst:
                    want = rng.integers(0, world, n).astype(np.uint8)
                    want[rng.integers(0, n, 7)] = rng.integers(world, 256, 7).astype(np.uint8)
                    owner_in = want
                else:
                    want = owners_cpu(kind, eng.cfg, world, rank, req)
                    owner_in = None
                counts = np.bincount(want[want < world], minlength=world)[:world]
                cap = (int(counts.max()) + 16 + 15) // 16 * 16
                _dispatch_and_check(eng, req, n, world, rank, want, owner_in, cap,
                                    f"{wire.KIND_NAMES[kind]} world {world} tiles {tiles} {'owner_in' if by_dst else 'computed'}")


def test_route_dispatch_over_capacity_at_2000_tiles():
    """Slabs of 80 % of the mean: every slab overflows.  The overflow count is the sum of the excesses, a slab holds
    exactly its first `cap` records, the tilebase is still the exact prefix, and the dropped records come back 0xFF."""
    from dint_b200.shard import owners_cpu
    world, rank = 3, 1
    with Engine(wire.FASST, n_shards=world, shard_id=rank, chunk=4096) as eng:
        n = 2000 * 2048 - 77
        req, _ = _route_records(wire.FASST, n, seed=9)
        want = owners_cpu(wire.FASST, eng.cfg, world, rank, req)
        cap = int(0.8 * n / world) // 16 * 16
        assert (np.bincount(want, minlength=world) > cap).all()
        _dispatch_and_check(eng, req, n, world, rank, want, None, cap, "over capacity")


# ---------------------------------------------------------------- B: the cluster at production batch sizes ---------
def _lock_or_store_trace(kind, n, seed, one_key=False):
    if kind == wire.FASST:
        return T.fasst_random(n, 1 if one_key else 10**6, seed=seed)
    if kind == wire.LOCK2PL:
        return T.lock2pl_random(n, 1 if one_key else 10**6, seed=seed)
    return T.store_random(n, 1 if one_key else 5000, seed=seed)


@pytest.mark.parametrize("kind,G,max_batch", [(wire.FASST, 2, 1 << 22), (wire.FASST, 8, 1 << 22),
                                              (wire.LOCK2PL, 3, 1 << 22), (wire.STORE, 4, 1 << 19)])
def test_cluster_answers_like_one_server_at_production_batch_sizes(kind, G, max_batch):
    """Every rank dispatches max_batch records (>= 2048 tiles) and every engine runs chunks of G x cap records.  The
    second call puts 1.5 x max_batch records on one key (lock id 0, or one store subscriber): the lock kinds overflow the
    owner's slab and are served again in recovery rounds of cap records per rank -- G x cap >= one engine chunk on one
    lock slot, which lock_fasst serves through the radix fallback of k_ordered."""
    cfg = dict(subs_populate=5000) if kind == wire.STORE else {}
    msg = wire.MSG_SIZE[kind]
    assert max_batch // (2048 if msg <= 12 else 256) > 1056
    for name, devs in _placements(G):
        ora = O.Oracle(kind, **cfg)
        with GpuCluster(kind, G, devices=devs, max_batch=max_batch, populate=True, **cfg) as cl:
            calls = [_lock_or_store_trace(kind, G * max_batch + 129, seed=1),
                     _lock_or_store_trace(kind, 3 * max_batch // 2 + 7, seed=2, one_key=True)]
            for i, req in enumerate(calls):
                want = ora.process(req)
                got = cl.submit(req)
                d = first_diff(got, want, msg)
                assert d is None, f"{name} G={G} call {i} (n={req.size // msg}): {d}"
            rng = np.random.default_rng(7)
            if kind in (wire.FASST, wire.LOCK2PL):
                assert cl.overflow_retries() >= 1, name
                for lid in [0] + rng.integers(0, 10**6, size=63).tolist():
                    slot = ora.lock_slot(0, int(lid))
                    assert cl.engine(slot % G).lock_state(0, slot) == ora.lock_state(0, slot), (name, lid)
                if kind == wire.FASST:
                    owner = ora.lock_slot(0, 0) % G
                    assert cl.engine(owner).stats()["ordered_fallbacks"] > 0, name
            else:
                assert sum(cl.engine(s).kv_count(0) for s in range(G)) == ora.kv_count(0), name
            assert all(cl.engine(s).stats()["errors"] == 0 for s in range(G)), name


# ---------------------------------------------------------------- C / D / E: the GPU clients against G oracles -----
def _parity(kind, n, clients, G, rounds, devs, max_batch=0, between=None, **cfg_over):
    """Drives TxnWorkload + G oracles and GpuTxnClients side by side, checking every round's requests and replies, then
    the counters, every shard's log ring and (G = 3) every table's row count.  between(r, cl, ocl): called after the
    clients emitted round r and before it is served, on the cluster and on the oracles alike.  Returns the clients'
    stats and every shard's engine stats."""
    msg = wire.MSG_SIZE[kind]
    ora_cfg = {k: v for k, v in cfg_over.items() if k != "kv_capacity_log2"}
    oras = [O.Oracle(kind, **_pop(kind, n), **ora_cfg) for _ in range(G)]
    ocl = Cluster([o.process for o in oras], msg)
    wl = TxnWorkload(kind, n_clients=clients, n_shards=G, subscribers=n, gid0=GID0)
    with GpuCluster(kind, G, devices=devs, max_batch=max_batch, populate=True, **_pop(kind, n), **cfg_over) as cl:
        with GpuTxnClients(cl, clients, subscribers=n, gid0=GID0) as tc:
            for r in range(rounds):
                rq, dst = wl.next()
                q, d, _ = tc.peek()
                assert np.array_equal(q, rq) and np.array_equal(d, dst), f"round {r}: the clients diverged"
                if between is not None:
                    between(r, cl, ocl)
                rs = ocl.submit(rq, dst)
                wl.feed(rs)
                tc.run(1)
                _, _, got = tc.peek()
                assert got.size == rs.size and first_diff(got, rs, msg) is None, f"round {r}: {first_diff(got, rs, msg)}"
            st = tc.stats()
            want = wl.stats()
            assert {k: v for k, v in st.items() if k != "fallback_rounds"} == want and want["committed"] > 0
            for s in range(G):
                ring, appended = cl.engine(s).dump_log()
                assert appended == oras[s].log_appended() and np.array_equal(ring, oras[s].log_ring()), f"shard {s} log"
                if G == 3:                      # G > 3: a shard holds only the keys it is a replica of
                    for tb in range(5 if kind == wire.TATP else 2):
                        assert cl.engine(s).kv_count(tb) == oras[s].kv_count(tb), f"shard {s} table {tb}"
            return st, [cl.engine(s).stats() for s in range(G)]


@pytest.mark.parametrize("kind,n", [(wire.TATP, 300000), (wire.SMALLBANK, 300000)])
def test_gpu_txn_clients_at_80k_clients_per_rank(kind, n):
    """240,007 clients over 3 ranks: 80,002 clients = 313 tiles per rank, so k_txn_scan carries its sum from its
    first pass of 256 tiles into the second, and k_txn_compact runs 313 CTAs."""
    for name, devs in _placements(3):
        st, _ = _parity(kind, n, 240007, 3, 12, devs, max_batch=1 << 20)
        assert st["fallback_rounds"] == 0, name


@pytest.mark.slow
def test_gpu_txn_clients_at_the_benchmark_shape():
    """2^20 TATP clients over 3 ranks (1366 tiles in k_txn_scan) with rounds of about a million records per rank: each
    rank's dispatch passes 1056 tiles of 256 records and reads the look-back's second window."""
    for name, devs in _placements(3):
        st, _ = _parity(wire.TATP, 300000, 1 << 20, 3, 4, devs, max_batch=1 << 21)
        assert st["rounds"] == 4, name


@pytest.mark.parametrize("clients", [1, 2, 4])
@pytest.mark.parametrize("kind,n", [(wire.TATP, 3000), (wire.SMALLBANK, 5000)])
def test_gpu_txn_clients_with_ranks_that_hold_no_client(kind, n, clients):
    """n_clients < G: a rank holds no client and launches no client kernel, but still takes part in every exchange."""
    for name, devs in _placements(3):
        st, _ = _parity(kind, n, clients, 3, 30, devs)
        assert st["rounds"] == 30, name


def test_gpu_txn_clients_long_run():
    """600 rounds, one dispatch per rank each: route_seq wraps twice (every look-back descriptor is cleared at the wrap)
    and the three buffer sets of the step are each reused 200 times."""
    for name, devs in _placements(3):
        st, eng = _parity(wire.SMALLBANK, 5000, 1001, 3, 600, devs)
        assert st["rounds"] == 600 and st["fallback_rounds"] == 0, name
        assert all(e["errors"] == 0 for e in eng), name


# ---------------------------------------------------------------- D: log rings that wrap --------------------------
@pytest.mark.parametrize("chunk", [256, 4096])
@pytest.mark.parametrize("ring", [1, 7, 1000])
@pytest.mark.parametrize("kind", [wire.TATP, wire.SMALLBANK])
def test_log_ring_wraps_on_one_engine(kind, ring, chunk):
    """About 3,000 log appends, tens to hundreds per chunk: an append that a later append of
    the same chunk overwrites is skipped (log_keep), and the ring must still be the oracle's, entry for entry."""
    msg = wire.MSG_SIZE[kind]
    if kind == wire.TATP:
        ora = O.Oracle(kind, subs_populate=300, log_ring=ring)
        req = T.tatp_random(30000, 300, seed=ring + chunk, oracle=ora)
        cfg = dict(subs_populate=300)
    else:
        ora = O.Oracle(kind, accts_populate=3000, log_ring=ring)
        req = T.smallbank_random(30000, 3000, seed=ring + chunk)
        cfg = dict(accts_populate=3000)
    want = ora.process(req)
    assert ora.log_appended() > 2 * ring
    with Engine(kind, log_ring=ring, chunk=chunk, populate=True, **cfg) as eng:
        got = eng.submit(req)
        assert first_diff(got, want, msg) is None, first_diff(got, want, msg)
        ring_got, appended = eng.dump_log()
        assert appended == ora.log_appended()
        assert np.array_equal(ring_got, ora.log_ring())


@pytest.mark.parametrize("ring", [7, 1000])
@pytest.mark.parametrize("kind,n,clients", [(wire.TATP, 3000, 1201), (wire.SMALLBANK, 5000, 1001)])
def test_log_ring_wraps_across_the_exchange(kind, n, clients, ring):
    """Host clients through cluster.submit, then the GPU clients: every step appends across slab boundaries and
    padding records, and the ring of 7 wraps inside one step."""
    msg = wire.MSG_SIZE[kind]
    G = 3
    for name, devs in _placements(G):
        oras = [O.Oracle(kind, log_ring=ring, **_pop(kind, n)) for _ in range(G)]
        ocl = Cluster([o.process for o in oras], msg)
        wl = TxnWorkload(kind, n_clients=clients, n_shards=G, subscribers=n)
        with GpuCluster(kind, G, devices=devs, max_batch=2048, populate=True, log_ring=ring, **_pop(kind, n)) as cl:
            for r in range(40):
                rq, dst = wl.next()
                want = ocl.submit(rq, dst)
                got = cl.submit(rq, dst)
                assert first_diff(got, want, msg) is None, f"{name} round {r}: {first_diff(got, want, msg)}"
                wl.feed(want)
            for s in range(G):
                ring_got, appended = cl.engine(s).dump_log()
                assert appended == oras[s].log_appended() > 2 * ring, f"{name} shard {s}"
                assert np.array_equal(ring_got, oras[s].log_ring()), f"{name} shard {s}"
        _parity(kind, n, clients, G, 40, devs, log_ring=ring)


# ---------------------------------------------------------------- E: KV rehash inside the exchange step -----------
E_SUBS = 2500              # 9,283 call-forwarding rows per shard ...
E_CAP_LOG2 = 14            # ... fill 57 % of 16,384 entries
E_CHURN = 1024             # call-forwarding rows inserted, read and deleted again per churn call and shard


def _e_cfg():
    rows = O.Oracle(wire.TATP, subs_populate=E_SUBS).kv_count(Tatp.kCallForwarding)
    assert 0.40 <= rows / (1 << E_CAP_LOG2) <= 0.65, rows       # the first rehash doubles, the next ones only reclaim
    return dict(kv_capacity_log2=[0, 0, 0, 0, E_CAP_LOG2])


class _Churn:
    """Calls of ever-new call-forwarding keys: insert (kInsertBck), read, delete (kDeleteBck), read a key that never
    existed -- none takes a lock.  Every record goes once to each of the three shards, so their tables churn alike."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.next_sid = 1 << 24

    def call(self, m=E_CHURN):
        keys = (np.arange(self.next_sid, self.next_sid + m, dtype=np.uint64) | (np.uint64(1) << np.uint64(32)) |
                (np.uint64(8) << np.uint64(40)))
        self.next_sid += m
        rec = np.zeros(4 * m, dtype=wire.MSG_DTYPE[wire.TATP])
        rec["table"] = Tatp.kCallForwarding
        rec["key"] = np.concatenate([keys, keys, keys, keys + np.uint64(1 << 20)])
        rec["type"] = np.concatenate([np.full(m, Tatp.kInsertBck), np.full(m, Tatp.kRead), np.full(m, Tatp.kDeleteBck),
                                      np.full(m, Tatp.kRead)]).astype(np.uint8)
        rec["val"] = self.rng.integers(0, 256, size=(4 * m, 40))
        req = np.tile(wire.as_bytes(rec), 3)
        dst = np.repeat(np.arange(3, dtype=np.uint8), 4 * m)
        return req, dst


def _check_rehashed(cl, oras, what):
    for s in range(3):
        st = cl.engine(s).stats()
        assert st["errors"] == 0, f"{what} shard {s}: {st}"
        assert st["kv_rebuilds"] >= 2, f"{what} shard {s}: {st}"
        for tb in range(5):
            assert cl.engine(s).kv_count(tb) == oras[s].kv_count(tb), f"{what} shard {s} table {tb}"


def test_kv_rehash_inside_the_exchange_step():
    """30 closed-loop rounds, then 60 churn calls (61,440 inserts; an insert that meets a tombstone on its probe path
    reuses it, so FULL + TOMB grows by less than one per insert): FULL + TOMB entries pass 70 % of the call-forwarding
    table, which shard_engine rehashes between the flag wait and the chunk launches -- first into a doubled table (live
    rows above 35 %), later in place (live rows below 35 %).  The replies stay the oracles'."""
    cfg = _e_cfg()
    msg = wire.MSG_SIZE[wire.TATP]
    oras = [O.Oracle(wire.TATP, subs_populate=E_SUBS) for _ in range(3)]
    ocl = Cluster([o.process for o in oras], msg)
    wl = TxnWorkload(wire.TATP, n_clients=1201, n_shards=3, subscribers=E_SUBS)
    churn = _Churn(5)
    with GpuCluster(wire.TATP, 3, devices=[0] * 3, max_batch=4096, populate=True, subs_populate=E_SUBS, **cfg) as cl:
        for r in range(30):
            rq, dst = wl.next()
            want = ocl.submit(rq, dst)
            got = cl.submit(rq, dst)
            assert first_diff(got, want, msg) is None, f"round {r}: {first_diff(got, want, msg)}"
            wl.feed(want)
        for i in range(60):
            rq, dst = churn.call()
            want = ocl.submit(rq, dst)
            got = cl.submit(rq, dst)
            assert first_diff(got, want, msg) is None, f"churn call {i}: {first_diff(got, want, msg)}"
        _check_rehashed(cl, oras, "cluster")


def test_kv_rehash_inside_the_exchange_step_under_gpu_clients():
    """The GPU clients for 150 rounds on such a cluster, with a churn call between the emission and the service of every
    second round: the table passes 70 % in steps that serve the clients' rounds too, with per-round parity."""
    cfg = _e_cfg()
    churn = _Churn(6)

    def between(r, cl, ocl):
        if r % 2 == 0:
            rq, dst = churn.call()
            want = ocl.submit(rq, dst)
            got = cl.submit(rq, dst)
            assert first_diff(got, want, wire.MSG_SIZE[wire.TATP]) is None, f"churn before round {r}"

    _, eng = _parity(wire.TATP, E_SUBS, 1201, 3, 150, [0] * 3, max_batch=4096, between=between, **cfg)
    for s, st in enumerate(eng):
        assert st["errors"] == 0 and st["kv_rebuilds"] >= 2, (s, st)
