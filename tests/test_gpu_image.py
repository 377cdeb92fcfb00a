"""State images on the GPU (dint_image_save / dint_image_open, dint_cluster_image_*): every kind and option is saved
after a trace that reaches the ordered replay, opened next to the original, and both must then answer one continuation
trace byte for byte and hold the same log, tables, lock words and cache sets.  Also: the checksums the device computed
equal the documented ones (tests/test_image_cpu.py's reader), an unpopulated engine, a rehashed KV table, a wrapped log
ring, the D2D snapshot of the same moment, corrupted and truncated files, shard clusters after GPU client rounds, the
UDP front-end's --image-out / --image-in, and (slow) a full-size eBPF TATP cluster too large to snapshot on the device."""
import os
import shutil
import signal
import socket
import subprocess
import time

import numpy as np
import pytest

import test_image_cpu as R
import trace_gen as T
import tatp_ebpf_model as TM
from dint_b200 import Engine, GpuCluster, GpuClusterClients, GpuTxnClients, wire
from dint_b200.engine import DintError, read_image_header

pytestmark = pytest.mark.gpu
EINVAL, EIO = -22, -5

SMALL = dict(log_ring=4096, chunk=4096)
# name -> (kind, engine options, populate, trace(seed))
CASES = {
    "lock_2pl": (wire.LOCK2PL, dict(lock_slots=1 << 16), False, lambda s: T.lock2pl_random(20000, 64, seed=s)),
    "lock_fasst": (wire.FASST, dict(lock_slots=1 << 16), False, lambda s: T.fasst_random(20000, 64, seed=s)),
    "log_server": (wire.LOG, dict(), False, lambda s: T.log_random(9000, seed=s)),          # > log_ring: wraps
    "store": (wire.STORE, dict(subs_sizing=1000, subs_populate=100), True, lambda s: T.store_random(20000, 100, seed=s)),
    "store_wb_bloom": (wire.STORE, dict(subs_sizing=1000, subs_populate=100, store_ebpf="wb_bloom"), True,
                       lambda s: T.store_random(20000, 100, seed=s)),
    "store_wb": (wire.STORE, dict(subs_sizing=1000, subs_populate=100, store_ebpf="wb"), True,
                 lambda s: T.store_random(20000, 100, seed=s)),
    "store_wt": (wire.STORE, dict(subs_sizing=1000, subs_populate=100, store_ebpf="wt"), True,
                 lambda s: T.store_random(20000, 100, seed=s)),
    "tatp": (wire.TATP, dict(subs_sizing=6000, subs_populate=40), True, lambda s: T.tatp_random(6000, 40, seed=s)),
    "tatp_holder": (wire.TATP, dict(subs_sizing=6000, subs_populate=40, lock_holder_keys=True), True,
                    lambda s: T.tatp_random(6000, 40, seed=s)),
    "tatp_ebpf": (wire.TATP, dict(subs_sizing=6000, subs_populate=40, tatp_ebpf=True), True,
                  lambda s: T.tatp_random(6000, 40, seed=s)),
    "tatp_ebpf_holder": (wire.TATP, dict(subs_sizing=6000, subs_populate=40, tatp_ebpf=True, lock_holder_keys=True), True,
                         lambda s: T.tatp_random(6000, 40, seed=s)),
    "smallbank": (wire.SMALLBANK, dict(accts_sizing=4000, accts_populate=4000), True,
                  lambda s: T.smallbank_random(20000, 300, seed=s)),
    "smallbank_ebpf": (wire.SMALLBANK, dict(accts_sizing=4000, accts_populate=4000, smallbank_ebpf=True), True,
                       lambda s: T.smallbank_random(20000, 300, seed=s)),
}


def make(name, populate=None):
    kind, opts, pop, _ = CASES[name]
    eng = Engine(kind, device=0, **SMALL, **opts)
    if pop if populate is None else populate:
        eng.populate()
    return eng


def sample_keys(name, rng, n=64):
    kind, opts = CASES[name][:2]
    if kind == wire.STORE:
        return [(0, int(T.store_key(int(s), int(rng.integers(1, 5)), int(rng.integers(0, 3)) * 8))) for s in rng.integers(0, 100, n)]
    if kind == wire.TATP:
        u = T.tatp_key_universe(40)
        return [u[i] for i in rng.integers(0, len(u), n)]
    if kind == wire.SMALLBANK:
        return [(int(rng.integers(0, 2)), int(k)) for k in rng.integers(0, 300, n)]
    return [(0, int(k)) for k in rng.integers(0, 64, n)]


def assert_same_state(name, a, b):
    """dump_log, kv_get / kv_count, lock_state / lock_holder and the cache sets and chains of sampled keys"""
    kind, opts = CASES[name][:2]
    rng = np.random.default_rng(5)
    if kind in (wire.LOG, wire.TATP, wire.SMALLBANK):
        la, na = a.dump_log()
        lb, nb = b.dump_log()
        assert na == nb and np.array_equal(la, lb)
    keys = sample_keys(name, rng)
    if kind in (wire.STORE, wire.TATP, wire.SMALLBANK):
        for t in range(5 if kind == wire.TATP else 2 if kind == wire.SMALLBANK else 1):
            assert a.kv_count(t) == b.kv_count(t), t
        for t, k in keys:
            assert a.kv_get(t, k) == b.kv_get(t, k), (t, k)
    if kind in (wire.LOCK2PL, wire.FASST):
        for _, k in keys:
            slot = a.lock_slot(0, k)
            assert a.lock_state(0, slot) == b.lock_state(0, slot), k
    if kind in (wire.TATP, wire.SMALLBANK):
        for t, k in keys:
            slot = a.lock_slot(t, k)
            assert slot == b.lock_slot(t, k)
            assert a.lock_state(t, slot) == b.lock_state(t, slot), (t, k)
            if opts.get("lock_holder_keys"):
                assert a.lock_holder(t, slot) == b.lock_holder(t, slot), (t, k)
    if opts.get("store_ebpf"):
        for bkt in rng.integers(0, 4500, 64):
            assert np.array_equal(a.store_cache_set(int(bkt)), b.store_cache_set(int(bkt))), bkt
    if opts.get("tatp_ebpf"):
        H = TM.hash_sizes(6000)
        for t, k in keys:
            bkt = TM.fasthash64(k) % H[t]
            assert np.array_equal(a.tatp_cache_set(t, bkt), b.tatp_cache_set(t, bkt)), (t, k)
            assert a.tatp_chain(t, bkt).tobytes() == b.tatp_chain(t, bkt).tobytes(), (t, k)
    if opts.get("smallbank_ebpf"):
        H = 4000 * 3 // 2 // 4
        for bkt in rng.integers(0, H, 64):
            for t in range(2):
                assert np.array_equal(a.smallbank_cache_set(t, int(bkt)), b.smallbank_cache_set(t, int(bkt))), bkt


def assert_checksums(path):
    """every block's stored checksum is the documented sum over its bitmap words and lines"""
    img = R.read_image(path)
    for reg in img["regions"]:
        for blk in reg["blocks"]:
            assert R.recompute_checksum(path, blk) == blk["checksum"]
    return img


@pytest.mark.parametrize("name", list(CASES))
def test_round_trip(name, tmp_path):
    trace = CASES[name][3]
    path = str(tmp_path / f"{name}.img")
    with make(name) as a:
        a.submit(trace(1), check=False)
        st = a.stats()
        if CASES[name][0] != wire.LOG:
            assert st["conflicted"] > 0, st                  # the first trace reached the ordered replay
        a.save_image(path)
        assert not os.path.exists(path + ".tmp")
        img = assert_checksums(path)
        assert img["kind"] == CASES[name][0]
        with Engine.open_image(path, device=0) as b:
            assert b.stats()["requests"] == 0
            assert_same_state(name, a, b)
            nxt = trace(2)
            ra = a.submit(nxt, check=False)
            rb = b.submit(nxt, check=False)
            assert np.array_equal(ra, rb)
            assert_same_state(name, a, b)
        if CASES[name][0] == wire.LOG:
            assert a.dump_log()[1] > a.cfg.log_ring         # the ring wrapped before the save
        # the image is smaller than the raw state: zero lines are left out
        assert img["size"] < sum(r["bytes"] for r in img["regions"]) + 4096


def test_unpopulated_engine(tmp_path):
    path = str(tmp_path / "empty.img")
    with make("tatp_ebpf", populate=False) as a:
        a.save_image(path)
        img = assert_checksums(path)
        assert all(len(b["line_index"]) == 0 for r in img["regions"] for b in r["blocks"])
        with Engine.open_image(path) as b:
            req = CASES["tatp_ebpf"][3](3)
            assert np.array_equal(a.submit(req, check=False), b.submit(req, check=False))
            assert_same_state("tatp_ebpf", a, b)


def churn(m, start, seed):
    from dint_b200.wire import Tatp
    rng = np.random.default_rng(seed)
    keys = np.arange(start, start + m, dtype=np.uint64) | (np.uint64(1) << np.uint64(32)) | (np.uint64(8) << np.uint64(40))
    rec = np.zeros(3 * m, dtype=wire.MSG_DTYPE[wire.TATP])
    rec["table"] = Tatp.kCallForwarding
    rec["key"] = np.concatenate([keys, keys, keys])
    rec["type"] = np.concatenate([np.full(m, Tatp.kInsertBck), np.full(m, Tatp.kRead), np.full(m, Tatp.kRead)]).astype(np.uint8)
    rec["val"] = rng.integers(0, 256, size=(3 * m, 40))
    return wire.as_bytes(rec)


def test_image_after_a_rehash_opens_at_the_saved_capacity(tmp_path):
    path = str(tmp_path / "rehash.img")
    with Engine(wire.TATP, device=0, populate=True, subs_populate=20, kv_capacity_log2=[0, 0, 0, 0, 10], **SMALL) as a:
        for c in range(6):                                  # live keys outgrow 35 % of 1024 entries: the table doubles
            a.submit(churn(200, 1000 + 200 * c, c))
        assert a.stats()["kv_rebuilds"] > 0
        a.save_image(path)
        hdr = R.read_image(path)
        assert hdr["kv_capacity"][4] > 1024
        with Engine.open_image(path) as b:
            for c in range(6, 9):
                req = churn(200, 1000 + 200 * c, c)
                assert np.array_equal(a.submit(req), b.submit(req))
            assert a.kv_count(4) == b.kv_count(4)
            req = T.tatp_random(3000, 20, seed=4)
            assert np.array_equal(a.submit(req, check=False), b.submit(req, check=False))


def test_snapshot_and_image_of_the_same_moment_agree(tmp_path):
    import torch
    path = str(tmp_path / "snap.img")
    trace = CASES["smallbank_ebpf"][3]
    with make("smallbank_ebpf") as a:
        a.submit(trace(1), check=False)
        snap = a.snapshot()
        a.save_image(path)
        nxt = trace(2)
        ra = a.submit(nxt, check=False).copy()
        a.restore(snap)
        torch.cuda.synchronize()
        rs = a.submit(nxt, check=False).copy()
        a.free_snapshot(snap)
        with Engine.open_image(path) as b:
            rb = b.submit(nxt, check=False)
        assert np.array_equal(ra, rs) and np.array_equal(ra, rb)


def test_corrupt_and_truncated_images_are_refused(tmp_path):
    path = str(tmp_path / "ok.img")
    with make("tatp_holder") as a:
        a.submit(CASES["tatp_holder"][3](1), check=False)
        a.save_image(path)
    img = R.read_image(path)
    # the last region with stored lines: flip one byte in the middle of its lines
    r, reg = [(i, x) for i, x in enumerate(img["regions"]) if any(len(b["line_index"]) for b in x["blocks"])][-1]
    b, blk = [(i, x) for i, x in enumerate(reg["blocks"]) if len(x["line_index"])][-1]
    data = bytearray(open(path, "rb").read())
    bad = str(tmp_path / "flip.img")
    data[blk["lines_off"] + blk["stored"] // 2] ^= 0x40
    open(bad, "wb").write(bytes(data))
    with pytest.raises(DintError) as ei:
        Engine.open_image(bad)
    assert ei.value.code == EIO and f"region {r} block {b}: checksum mismatch" in str(ei.value)
    # truncated in the middle of that block
    cut = str(tmp_path / "cut.img")
    open(cut, "wb").write(open(path, "rb").read()[:blk["lines_off"] + blk["stored"] // 2])
    with pytest.raises(DintError) as ei:
        Engine.open_image(cut)
    assert ei.value.code == EIO and f"region {r} block {b}: short read" in str(ei.value)
    # a configuration this build lays out differently (another lock-slot count: other region sizes)
    data = bytearray(open(path, "rb").read())
    cfg = read_image_header(path)["cfg"]
    cfg.subs_sizing = 6001
    data[16:92] = bytes(cfg)
    other = str(tmp_path / "other.img")
    open(other, "wb").write(bytes(data))
    with pytest.raises(DintError) as ei:
        Engine.open_image(other)
    assert ei.value.code == EINVAL and "this build lays out" in str(ei.value)


def test_small_explicit_table_capacity(tmp_path):
    """an explicit kv_capacity_log2 below the automatic minimum of 2^10 saves and opens like any other"""
    path = str(tmp_path / "small.img")
    with Engine(wire.STORE, device=0, populate=True, subs_sizing=1000, subs_populate=10, kv_capacity_log2=[9], **SMALL) as a:
        a.submit(T.store_random(4000, 10, seed=1), check=False)
        a.save_image(path)
        assert R.read_image(path)["kv_capacity"][0] == 512
        with Engine.open_image(path) as b:
            req = T.store_random(4000, 10, seed=2)
            assert np.array_equal(a.submit(req, check=False), b.submit(req, check=False))


def test_trailing_bytes_are_refused(tmp_path):
    path = str(tmp_path / "t.img")
    with make("lock_fasst") as a:
        a.save_image(path)
    with open(path, "ab") as f:
        f.write(b"\0")
    with pytest.raises(DintError) as ei:
        Engine.open_image(path)
    assert ei.value.code == EINVAL and "bytes after the last block" in str(ei.value)


# ---- clusters ------------------------------------------------------------------------------------------------------
def test_cluster_save_that_stops_part_way_leaves_nothing_to_open(tmp_path):
    """saving over an earlier cluster image: the old manifest goes before the first shard is replaced, so a save that
    fails at shard 1 leaves a directory that is refused, not one of shards saved at two moments"""
    G, d = 3, str(tmp_path / "again")
    with GpuCluster(wire.FASST, G, devices=[0] * G, max_batch=8192, lock_slots=1 << 16) as a:
        a.submit(T.fasst_random(20000, 64, seed=1))
        a.save_image(d)
        with GpuCluster.open_image(d, devices=[0] * G) as b:
            req = T.fasst_random(2000, 64, seed=2)
            assert np.array_equal(a.submit(req), b.submit(req))
        a.submit(T.fasst_random(20000, 64, seed=3))
        os.mkdir(os.path.join(d, "shard-1.img.tmp"))      # shard 1's image cannot be written
        with pytest.raises(DintError) as ei:
            a.save_image(d)
        assert ei.value.code == EIO and "shard-1.img.tmp" in str(ei.value)
    assert not os.path.exists(os.path.join(d, "manifest"))
    with pytest.raises(DintError) as ei:
        GpuCluster.open_image(d, devices=[0] * G)
    assert ei.value.code == EIO and "manifest" in str(ei.value)
    with pytest.raises(DintError) as ei:
        GpuCluster.open_image(d)
    assert ei.value.code == EIO and "manifest" in str(ei.value)


def test_cluster_lock_fasst(tmp_path):
    G, d = 3, str(tmp_path / "fasst")
    with GpuCluster(wire.FASST, G, devices=[0] * G, max_batch=8192, lock_slots=1 << 18) as a:
        with GpuClusterClients(a, 6000, n_keys=4096, read_pct=50) as cc:
            cc.run(8)
        a.save_image(d)
        assert sorted(os.listdir(d)) == ["manifest"] + [f"shard-{r}.img" for r in range(G)]
        with GpuCluster.open_image(d, devices=[0] * G, max_batch=8192) as b:
            req = T.fasst_random(30000, 4096, seed=9)
            assert np.array_equal(a.submit(req), b.submit(req))

            for k in range(0, 4096, 7):
                slot = a.engine(0).lock_slot(0, k)
                s = slot % G
                assert a.engine(s).lock_state(0, slot) == b.engine(s).lock_state(0, slot), k
        with pytest.raises(DintError) as ei:
            GpuCluster.open_image(d, devices=[0, 0])
        assert ei.value.code == EINVAL
        os.remove(os.path.join(d, "shard-1.img"))
        with pytest.raises(DintError) as ei:
            GpuCluster.open_image(d, devices=[0] * G)
        assert ei.value.code == EIO and "shard-1.img" in str(ei.value)


@pytest.mark.parametrize("kind", ["tatp_ebpf", "smallbank_ebpf"])
def test_cluster_txn_ebpf(kind, tmp_path):
    G, d, n = 3, str(tmp_path / kind), 3000
    over = dict(tatp_ebpf=True, subs_sizing=n, subs_populate=n) if kind == "tatp_ebpf" else \
        dict(smallbank_ebpf=True, accts_sizing=n, accts_populate=n)
    k = wire.TATP if kind == "tatp_ebpf" else wire.SMALLBANK
    with GpuCluster(k, G, devices=[0] * G, populate=True, **over) as a:
        with GpuTxnClients(a, 4000, subscribers=n) as tc:
            tc.run(20)
            a.save_image(d)
            with GpuCluster.open_image(d, devices=[0] * G) as b:
                rq, dst, _ = tc.peek()
                for _ in range(3):                       # the clients' pending round, submitted to both (three times)
                    ra = a.submit(rq, dst=dst, check=False)
                    rb = b.submit(rq, dst=dst, check=False)
                    assert np.array_equal(ra, rb)
                for s in range(G):
                    x, y = a.engine(s), b.engine(s)
                    for t in range(2):
                        for key in range(0, n, 37):
                            assert x.kv_get(t, key) == y.kv_get(t, key)


# ---- the UDP front-end ---------------------------------------------------------------------------------------------
def _start(args):
    srv = subprocess.Popen(args, stderr=subprocess.PIPE)
    os.set_blocking(srv.stderr.fileno(), False)
    banner, t0 = b"", time.time()
    while b"sockets, batches" not in banner:
        assert srv.poll() is None and time.time() - t0 < 120, banner
        time.sleep(0.1)
        banner += srv.stderr.read() or b""
    return srv


def _send(port, rec, msg):
    got = np.empty_like(rec)
    with socket.socket(socket.AF_INET, socket.SOCK_DGRAM) as c:
        c.settimeout(5.0)
        c.connect(("127.0.0.1", port))
        for i in range(len(rec)):
            c.send(rec[i].tobytes())
            r = np.frombuffer(c.recv(256), dtype=np.uint8)
            assert r.size == msg
            got[i] = r
    return got


def test_udp_front_end_image_out_then_in(tmp_path):
    from dint_b200 import _build
    msg = wire.MSG_SIZE[wire.FASST]
    a_req = T.fasst_random(400, 32, seed=21).reshape(-1, msg)
    b_req = T.fasst_random(400, 32, seed=22).reshape(-1, msg)
    img = str(tmp_path / "srv.img")
    with socket.socket(socket.AF_INET, socket.SOCK_DGRAM) as s0:
        s0.bind(("127.0.0.1", 0))
        port = s0.getsockname()[1]
    base = [_build.UDP_SERVER, "lock_fasst", "--port", str(port), "--bind", "127.0.0.1"]
    srv = _start(base + ["--image-out", img])
    try:
        _send(port, a_req, msg)
    finally:
        srv.send_signal(signal.SIGTERM)
        assert srv.wait(timeout=120) == 0
    assert os.path.exists(img)
    srv = _start(base + ["--image-in", img])
    try:
        got = _send(port, b_req, msg)
    finally:
        srv.terminate()
        srv.wait(timeout=60)
    with Engine(wire.FASST, device=0) as e:
        e.submit(a_req.reshape(-1))
        want = e.submit(b_req.reshape(-1)).reshape(-1, msg)
    assert np.array_equal(got, want)
    r = subprocess.run([_build.UDP_SERVER, "lock_2pl", "--port", str(port), "--bind", "127.0.0.1", "--image-in", img],
                       capture_output=True, timeout=120)
    assert r.returncode == 2 and b"lock_fasst" in r.stderr
    # server_shard <id>: the image must be that shard's
    shard = str(tmp_path / "shard1.img")
    with Engine(wire.TATP, device=0, subs_sizing=6000, subs_populate=0, txn_shards=3, txn_shard_id=1, **SMALL) as e:
        e.save_image(shard)
    for args in (["--shards", "3", "--shard-id", "0"], []):
        r = subprocess.run([_build.UDP_SERVER, "tatp", "--port", str(port), "--bind", "127.0.0.1", "--image-in", shard, *args],
                           capture_output=True, timeout=120)
        assert r.returncode == 2 and b"holds shard 1 of 3" in r.stderr, r.stderr


# ---- full size -----------------------------------------------------------------------------------------------------
@pytest.mark.slow
def test_full_size_tatp_ebpf_cluster(tmp_path):
    """three eBPF TATP shards at S = 7,000,000 on one H100 (48 GB: no room for a device-to-device snapshot) after 100
    rounds of 2^20 GPU clients: save, serve a recorded host batch, close, open, serve it again"""
    from dint_b200.txn_workloads import TxnWorkload
    S, G, clients = 7_000_000, 3, 1 << 20
    free = shutil.disk_usage(str(tmp_path)).free
    if free < 24 << 30:                                 # the three images take 18.2 GB (tools/image_bench.py)
        pytest.skip(f"{free >> 30} GiB free under {tmp_path}; the images need about 18 GiB")
    d = str(tmp_path / "full")
    wl = TxnWorkload(wire.TATP, n_clients=4096, n_shards=G, subscribers=S)
    rq, dst = wl.next()
    try:
        with GpuCluster(wire.TATP, G, devices=[0] * G, max_batch=(clients + G - 1) // G * 3, populate=True, tatp_ebpf=True) as a:
            with GpuTxnClients(a, clients, subscribers=S) as tc:
                tc.run(100)
            a.save_image(d)
            want = a.submit(rq, dst=dst, check=False).copy()
        with GpuCluster.open_image(d, devices=[0] * G, max_batch=(clients + G - 1) // G * 3) as b:
            got = b.submit(rq, dst=dst, check=False)
        assert np.array_equal(got, want)
    finally:
        shutil.rmtree(d, ignore_errors=True)
