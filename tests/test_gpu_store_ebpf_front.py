"""The eBPF store's cache tier beyond the engine's own tests: run-time table sizes against the restatement, the GPU
store clients against an engine with the tier, and dint_udp_server --store-ebpf behind a loopback socket."""
import os
import socket
import subprocess
import time

import numpy as np
import pytest

import store_ebpf_model as M
from dint_b200 import Engine, GpuClients, wire

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "store_ebpf")


@pytest.mark.parametrize("variant", M.VARIANTS)
def test_small_tables_equal_restatement(variant):
    """subs_sizing 1000: 4,500 buckets instead of the reference's 9,000,000, populated through the tier"""
    S, P = 1000, 200
    buckets = S * 18 // 4
    rng = np.random.default_rng(5)
    pop = [k for k, _ in M.population(P)]
    coll = np.concatenate(M.colliding_keys(buckets, 6, 20, seed=9, key_space=1 << 40))
    keys = np.concatenate([rng.choice(np.array(pop, dtype=np.uint64), size=300), coll])
    n = 6000
    k = rng.choice(keys, size=n)
    t = rng.choice([0, 0, 1, 2], size=n).astype(np.uint8)
    seen = set(pop)
    for i in range(n):                 # every key inserted at most once (see include/dint_b200.h)
        if t[i] == 2:
            if int(k[i]) in seen:
                t[i] = 0
            else:
                seen.add(int(k[i]))
    req = M.make_req(t, k, rng.integers(0, 256, size=(n, 40), dtype=np.uint8), rng.integers(0, 5, size=n, dtype=np.uint32))
    m = M.StoreEbpfModel(variant, buckets=buckets)
    m.populate(P)
    m.stats = dict.fromkeys(m.stats, 0)
    want = m.process(req)
    with Engine(wire.STORE, device=0, store_ebpf=variant, subs_sizing=S, subs_populate=P, chunk=1024, populate=True) as eng:
        before = eng.store_cache_stats()
        got = eng.submit(req)
        g, w = got.reshape(-1, 53), want.reshape(-1, 53)
        bad = np.flatnonzero((g != w).any(1))
        assert bad.size == 0, (bad.size, bad[:3])
        after = eng.store_cache_stats()
        assert {k: after[k] - before[k] for k in after} == m.stats
        probe = np.unique(keys)
        want_sets, want_table = m.state(probe)
        for i, key in enumerate(probe):
            assert np.array_equal(eng.store_cache_set(M.fasthash64(int(key)) % buckets), want_sets[i]), i
            got_kv = eng.kv_get(0, int(key))
            assert (got_kv is not None) == bool(want_table[i]["found"])
            if got_kv is not None:
                assert got_kv[1] == want_table[i]["ver"] and got_kv[0] == want_table[i]["val"].tobytes()
        assert eng.kv_count(0) == m.kv_count()


@pytest.mark.parametrize("family", [dict(set_pct=0), dict(set_pct=20), dict(set_pct=50, store_subscribers=3000)])
def test_gpu_store_clients_same_counters_with_the_tier(family):
    """The store clients decide on reply types only, so against the tier they must send the same requests and count
    the same commits and not-exists as against the UDP server's store (store_subscribers=3000 > the 2000 populated:
    a third of the keys are absent)."""
    fam = dict(store_subscribers=2000, **family) if "store_subscribers" not in family else family
    results = {}
    for v in (None,) + M.VARIANTS:
        with Engine(wire.STORE, device=0, subs_sizing=20000, subs_populate=2000, populate=True, store_ebpf=v) as eng, \
                GpuClients(eng, 4096, seed=77, **fam) as gc:
            gc.run(40, 0)
            eng.sync()
            st = gc.stats()
            results[v] = (st, gc.peek()[0].copy())
            if v is not None:
                cs = eng.store_cache_stats()
                assert cs["hits"] > 0 and cs["table"] > 0
    base, base_req = results[None]
    assert base["requests"] > 0 and base["committed"] > 0
    if fam["store_subscribers"] > 2000:
        assert base["not_exist"] > 0
    for v in M.VARIANTS:
        st, rq = results[v]
        assert {k: st[k] for k in ("requests", "committed", "not_exist")} == \
            {k: base[k] for k in ("requests", "committed", "not_exist")}, v
        assert np.array_equal(rq.reshape(-1, 53)[:, :9], base_req.reshape(-1, 53)[:, :9]), v   # next requests: type + key


@pytest.mark.parametrize("variant", M.VARIANTS)
def test_udp_front_end_store_ebpf(variant):
    """dint_udp_server store --store-ebpf over loopback answers a short trace as the reference's eBPF server does"""
    from dint_b200 import _build
    g = np.load(os.path.join(GOLDEN, f"{variant}.npz"))
    rec = g["req"].reshape(-1, 53)
    rec = rec[rec[:, 0] <= 2][:400]
    want = M.StoreEbpfModel(variant).process(rec.reshape(-1)).reshape(-1, 53)
    with socket.socket(socket.AF_INET, socket.SOCK_DGRAM) as s0:
        s0.bind(("127.0.0.1", 0))
        port = s0.getsockname()[1]
    srv = subprocess.Popen([_build.UDP_SERVER, "store", "--port", str(port), "--bind", "127.0.0.1", "--populate", "0",
                            "--store-ebpf", variant.replace("_", "-")], stderr=subprocess.PIPE)
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
        got = np.empty_like(rec)
        for i in range(len(rec)):                           # one at a time: the replies depend on the order
            c.send(rec[i].tobytes())
            got[i] = np.frombuffer(c.recv(256), dtype=np.uint8)
        bad = np.flatnonzero((got != want).any(1))
        assert bad.size == 0, (bad.size, bad[:3])
    finally:
        srv.terminate()
        srv.wait(timeout=20)
    # the option belongs to the store: another kind's server refuses to start
    r = subprocess.run([_build.UDP_SERVER, "lock_fasst", "--port", str(port), "--bind", "127.0.0.1", "--store-ebpf", "wt"],
                       capture_output=True, timeout=120)
    assert r.returncode == 1 and b"dint_create failed" in r.stderr
