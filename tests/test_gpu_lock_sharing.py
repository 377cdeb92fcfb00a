"""-m gpu: the same-key / false-sharing split of refused TATP locks (DINT_CFG_LOCK_HOLDER_KEYS, include/dint_b200.h;
tatp/ebpf/lock_kern.c:289-298) through the C ABI: the engine against the option-on model of
tests/lock_sharing_model.py on every route a lock request can take (solo in k_apply, bucket replay, radix fallback --
the engine's counters prove which one answered), the option-off engine on the same traces, snapshots, shard clusters,
the clients on the GPU and the UDP front-end."""
import os
import socket
import subprocess
import time

import numpy as np
import pytest

import lock_sharing_model as M
import oracle_lib as O
import trace_gen as T
from dint_b200 import Engine, GpuCluster, GpuTxnClients, wire
from dint_b200.engine import DintError
from dint_b200.txn_workloads import Cluster, TxnWorkload
from dint_b200.wire import Tatp
from golden_util import first_diff

pytestmark = pytest.mark.gpu
MSG = wire.MSG_SIZE[wire.TATP]
L, A = Tatp.kAcquireLock, Tatp.kAbort
S, NSUBS = 60, 40          # subs_sizing / subs_populate of the single-engine tests: lock moduli of 80 .. 336 slots
ROUTE_KEYS = ("conflicted", "ordered_fallbacks", "bucket_split_tasks")


def _types(resp):
    return wire.as_records(wire.TATP, resp)["type"]


class _Served:
    """An engine and the server it must equal, fed the same calls; host path or device path."""

    def __init__(self, eng, ora, device_path):
        self.eng, self.ora, self.device_path = eng, ora, device_path

    def __call__(self, req, what):
        want = self.ora.process(req)
        before = self.eng.stats()
        if self.device_path:
            import torch
            got = self.eng.submit_tensor(torch.from_numpy(np.ascontiguousarray(req)).cuda()).cpu().numpy()
        else:
            got = self.eng.submit(req)
        after = self.eng.stats()
        assert first_diff(got, want, MSG) is None, f"{what}: {first_diff(got, want, MSG)}"
        return _types(got), {k: after[k] - before[k] for k in ROUTE_KEYS}


def _route_calls(pairs):
    """Three calls of at most 256 lock requests (one chunk at every chunk size) on table 0, after every a_i was granted:
    solo      every slot once: the holder's key again (28) or the key that shares its slot (8);
    bucket    per slot, far apart in the call: abort a, acquire b (7), b again (28), a (8);
    fallback  200 requests on ONE slot, more than a bucket holds, plus a few on three others."""
    h = len(pairs) // 2
    solo = M.lock_records([L] * len(pairs), [a for a, _ in pairs[:h]] + [b for _, b in pairs[h:]])
    bp = pairs[:32]
    bucket = M.lock_records([A] * 32 + [L] * 96, [a for a, _ in bp] + [b for _, b in bp] * 2 + [a for a, _ in bp])
    rng = np.random.default_rng(11)
    ty, keys = [], []
    for j, n in ((40, 200), (41, 18), (42, 18), (43, 18)):
        a, b = pairs[j]
        for x in rng.random(n):
            ty.append(A if x < 0.3 else L)
            keys.append(a if x < 0.65 else b)
    order = rng.permutation(len(ty))
    fallback = M.lock_records(np.array(ty)[order], np.array(keys, dtype=np.uint64)[order])
    return solo, bucket, fallback


@pytest.mark.parametrize("device_path", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("chunk", [256, 4096, 1 << 16])
@pytest.mark.parametrize("option", [True, False], ids=["holder_keys", "plain"])
def test_engine_answers_like_the_model_on_every_route(option, chunk, device_path):
    cfg = dict(subs_sizing=S, subs_populate=NSUBS, log_ring=512)
    big = dict(cfg, subs_sizing=40000)        # the route calls want 64 slots of their own: a second engine, larger moduli
    for c, routes in ((big, True), (cfg, False)):
        ora = M.HolderOracle(**c) if option else O.Oracle(wire.TATP, **c)
        with Engine(wire.TATP, populate=True, chunk=chunk, lock_holder_keys=option, **c) as eng:
            serve = _Served(eng, ora, device_path)
            if routes:
                pairs = M.colliding_pairs(c["subs_sizing"], 0, 64)
                solo, bucket, fallback = _route_calls(pairs)
                ty, d = serve(M.lock_records([L] * 64, [a for a, _ in pairs]), "grants")
                assert (ty == 7).all() and d["conflicted"] == 0
                ty, d = serve(solo, "solo")
                assert d["conflicted"] == 0, d                       # nothing was listed: k_apply answered all of it
                assert list(ty) == ([28] * 32 + [8] * 32 if option else [8] * 64)
                ty, d = serve(bucket, "bucket")
                assert d["conflicted"] == 128 and d["ordered_fallbacks"] == 0, d      # all listed, none through the radix sort
                assert list(ty) == [9] * 32 + [7] * 32 + ([28] if option else [8]) * 32 + [8] * 32
                ty, d = serve(fallback, "fallback")
                assert d["conflicted"] == len(ty) and d["ordered_fallbacks"] == 1, d  # all listed, all through the radix sort
                assert ((ty == 28).sum() > 20) == option and (ty == 8).sum() > 20
            # random traffic of every request type over a handful of slots, several chunks per call
            plain = ora.ora if option else ora
            for seed, n in ((1, 20000), (2, 70000), (3, 3000)):
                req = T.tatp_random(n, NSUBS, seed=seed, oracle=plain)
                ty, d = serve(req, f"random {seed}")
                assert d["conflicted"] > 0
                assert ((ty == 28).sum() > 0) == option
            # final state: lock bits and holder words of every slot, rows, log
            mods = M.lock_moduli(c["subs_sizing"])
            rng = np.random.default_rng(5)
            for tb in range(5):
                slots = range(mods[tb]) if mods[tb] <= 400 else [int(s) for s in rng.integers(0, mods[tb], size=100)]
                if routes and tb == 0:
                    slots = list(slots) + [M.HolderModel(c["subs_sizing"]).slot(0, a) for a, _ in pairs]
                for s in slots:
                    assert eng.lock_state(tb, s)[0] == ora.lock_state(tb, s)[0], (tb, s)
                    if option:
                        assert eng.lock_state(tb, s)[0] == ora.model.held(tb, s)
                        assert eng.lock_holder(tb, s) == ora.model.holder(tb, s), (tb, s)
            if not option:
                with pytest.raises(DintError) as ei:
                    eng.lock_holder(0, 0)
                assert ei.value.code == -22
            for tb, key in T.tatp_key_universe(NSUBS):
                assert eng.kv_get(tb, key) == ora.kv_get(tb, key), (tb, key)
            ring, appended = eng.dump_log()
            assert appended == ora.log_appended() and np.array_equal(ring, ora.log_ring())


def test_snapshot_carries_the_holder_words():
    """After the restore the lock bit of the slot is set either way; only the restored holder word tells the engine
    that the refused key is the holder's own."""
    cfg = dict(subs_sizing=S, subs_populate=NSUBS)
    (a, b), = M.colliding_pairs(S, 0, 1)
    with Engine(wire.TATP, populate=True, lock_holder_keys=True, **cfg) as eng:
        assert list(_types(eng.submit(M.lock_records([L], [a])))) == [7]
        snap = eng.snapshot()
        assert list(_types(eng.submit(M.lock_records([A, L, L], [a, b, a])))) == [9, 7, 8]
        slot = eng.lock_slot(0, a)
        assert eng.lock_holder(0, slot) == b
        eng.restore(snap, stream=0)
        eng.sync()
        assert eng.lock_holder(0, slot) == a and eng.lock_state(0, slot)[0] == 1
        rest = M.lock_records([L, L, A, L], [a, b, a, b])
        assert list(_types(eng.submit(rest))) == [28, 8, 9, 7]
        eng.free_snapshot(snap)


def test_option_is_refused_for_other_kinds():
    for kind in (wire.FASST, wire.LOCK2PL, wire.SMALLBANK):
        with pytest.raises(DintError) as ei:
            Engine(kind, lock_holder_keys=True)
        assert ei.value.code == -22
    with pytest.raises(DintError) as ei:
        GpuCluster(wire.FASST, 2, devices=[0, 0], lock_holder_keys=True)
    assert ei.value.code == -22


def test_single_shard_cluster_splits_rejects():
    """One shard cannot serve the transaction clients (a backup commit would meet the primary's own lock), so it is fed
    shard traffic directly."""
    cfg = dict(subs_sizing=S, subs_populate=NSUBS)
    ora = M.HolderOracle(**cfg)
    with GpuCluster(wire.TATP, 1, devices=[0], max_batch=2048, populate=True, lock_holder_keys=True, **cfg) as cl:
        for seed in (7, 8):
            req = T.tatp_random(9000, NSUBS, seed=seed, oracle=ora.ora)
            want = ora.process(req)
            got = cl.submit(req, np.zeros(req.size // MSG, dtype=np.uint8))
            assert first_diff(got, want, MSG) is None, first_diff(got, want, MSG)
            assert (_types(got) == 28).sum() > 0 and (_types(got) == 8).sum() > 0


@pytest.mark.parametrize("G", [3, 5])
def test_cluster_serves_host_clients_like_option_on_shard_servers(G):
    n, clients, rounds = 1500, 1300, 80
    cfg = dict(subs_sizing=n, subs_populate=n)

    def run(submit):
        wl = TxnWorkload(wire.TATP, n_clients=clients, n_shards=G, subscribers=n)
        trace = []
        for _ in range(rounds):
            rq, dst = wl.next()
            rs = submit(rq, dst)
            wl.feed(rs)
            trace.append((rq.copy(), dst.copy(), np.array(rs, copy=True)))
        return trace, wl.stats(), wl.lock_stats()

    oras = [M.HolderOracle(**cfg) for _ in range(G)]
    want, st_want, ls_want = run(Cluster([o.process for o in oras], MSG).submit)
    assert ls_want["reject_sharing"] > 0 and ls_want["reject_same_key"] > 0
    with GpuCluster(wire.TATP, G, devices=[0] * G, max_batch=2048, populate=True, lock_holder_keys=True, **cfg) as cl:
        got, st_got, ls_got = run(lambda rq, dst: cl.submit(rq, dst))
        for r, ((q1, d1, s1), (q2, d2, s2)) in enumerate(zip(want, got)):
            assert np.array_equal(q1, q2) and np.array_equal(d1, d2), f"round {r}: clients diverged"
            assert first_diff(s2, s1, MSG) is None, f"round {r}: {first_diff(s2, s1, MSG)}"
        assert st_got == st_want and ls_got == ls_want
        for s in range(G):                                 # a shard indexes its holders by the slot itself
            for tb in range(5):
                for slot, (held, key) in list(oras[s].model.state[tb].items())[:40]:
                    assert cl.engine(s).lock_state(tb, slot)[0] == held and cl.engine(s).lock_holder(tb, slot) == key


def test_gpu_clients_count_locks_like_the_host_clients():
    """2000 clients on 3 ranks: 666 / 667 / 667, three k_txn_step tiles each, the last one partial."""
    n, clients, G, rounds, gid0 = 1500, 2000, 3, 150, 5
    cfg = dict(subs_sizing=n, subs_populate=n)
    oras = [M.HolderOracle(**cfg) for _ in range(G)]
    ocl = Cluster([o.process for o in oras], MSG)
    wl = TxnWorkload(wire.TATP, n_clients=clients, n_shards=G, subscribers=n, gid0=gid0)
    with GpuCluster(wire.TATP, G, devices=[0] * G, populate=True, lock_holder_keys=True, **cfg) as cl:
        with GpuTxnClients(cl, clients, subscribers=n, gid0=gid0) as tc:
            for r in range(rounds):
                rq, dst = wl.next()
                if r % 10 == 0:
                    q, d, _ = tc.peek()
                    assert np.array_equal(q, rq) and np.array_equal(d, dst), f"round {r}: the clients diverged"
                wl.feed(ocl.submit(rq, dst))
                tc.run(1)
            st, ls, want = tc.stats(), tc.lock_stats(), wl.lock_stats()
            assert {k: v for k, v in st.items() if k != "fallback_rounds"} == wl.stats() and st["fallback_rounds"] == 0
            assert ls == want
            assert want["reject_sharing"] > 100 and want["reject_same_key"] > 100
            assert want["locks"] > want["reject_sharing"] + want["reject_same_key"]
    # against servers without the option the same clients see no 28 and count every refusal as sharing
    with GpuCluster(wire.TATP, G, devices=[0] * G, populate=True, **cfg) as cl:
        with GpuTxnClients(cl, clients, subscribers=n, gid0=gid0) as tc:
            tc.run(rounds)
            off = tc.lock_stats()
            assert off == dict(locks=want["locks"], reject_sharing=want["reject_sharing"] + want["reject_same_key"], reject_same_key=0)


def test_udp_front_end_sends_type_28():
    """dint_udp_server tatp --lock-holder-keys at the reference's table sizes: a client that speaks
    tatp/caladan/proto.h gets kRejectLockSameKey on the wire."""
    from dint_b200 import _build
    (a, b), = M.colliding_pairs(7_000_000, 0, 1)
    script = [(L, a, 7), (L, a, 28), (L, b, 8), (A, a, 9), (L, b, 7), (L, a, 8), (L, b, 28)]
    with socket.socket(socket.AF_INET, socket.SOCK_DGRAM) as s0:
        s0.bind(("127.0.0.1", 0))
        port = s0.getsockname()[1]
    srv = subprocess.Popen([_build.UDP_SERVER, "tatp", "--port", str(port), "--bind", "127.0.0.1", "--lock-holder-keys",
                            "--populate", "30"], stderr=subprocess.PIPE)
    try:
        os.set_blocking(srv.stderr.fileno(), False)
        banner, t0 = b"", time.time()
        while b"sockets, batches" not in banner:           # printed once the engine exists and the sockets are bound
            assert srv.poll() is None and time.time() - t0 < 120, banner
            time.sleep(0.1)
            banner += srv.stderr.read() or b""
        c = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
        c.settimeout(5.0)
        c.connect(("127.0.0.1", port))
        for i, (ty, key, want) in enumerate(script):
            rec = M.lock_records([ty], [key])
            c.send(rec.tobytes())
            got = np.frombuffer(c.recv(256), dtype=np.uint8)
            assert got.size == MSG and got[1] == want and np.array_equal(got[2:], rec[2:]), (i, got[1], want)
    finally:
        srv.terminate()
        srv.wait(timeout=20)
    # the flag belongs to tatp: another kind's server refuses to start
    r = subprocess.run([_build.UDP_SERVER, "lock_fasst", "--port", str(port), "--bind", "127.0.0.1", "--lock-holder-keys"],
                       capture_output=True, timeout=120)
    assert r.returncode == 1 and b"dint_create failed" in r.stderr
