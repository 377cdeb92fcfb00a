"""Rebuilding lost tatp / smallbank shards from their replicas (dint_cluster_rebuild, dint_cluster_image_open_rebuild).

Rows are compared in bulk through state images: a shard image holds every KV table's entries, so the FULL entries of a
table, as {key: version + value bytes}, are the table's rows whatever the capacity or insertion order.  The pre-damage
copy of a lost shard is the image saved before the damage.  Also: later GPU client traffic on a rebuilt cluster against
one opened from the pre-damage image, the mid-transaction rule, damaged image directories, every refusal, the UDP
front-end's --rebuild-lost, and (slow) three full-size TATP shards."""
import os
import shutil
import signal
import socket
import subprocess

import numpy as np
import pytest

import test_image_cpu as R
import trace_gen as T
from test_gpu_image import _send, _start
from dint_b200 import Engine, GpuCluster, GpuTxnClients, wire
from dint_b200 import engine as E
from dint_b200.engine import DintError

pytestmark = pytest.mark.gpu
EINVAL, EIO = -22, -5
TATP, SMALLBANK = wire.TATP, wire.SMALLBANK
N = {TATP: 20_000, SMALLBANK: 50_000}
SIZES = {TATP: dict(subs_sizing=N[TATP], subs_populate=N[TATP]), SMALLBANK: dict(accts_sizing=N[SMALLBANK], accts_populate=N[SMALLBANK])}
N_TABLES = {TATP: 5, SMALLBANK: 2}
ENT, VALSZ = {TATP: 64, SMALLBANK: 32}, {TATP: 40, SMALLBANK: 8}
Tt, Sb = wire.Tatp, wire.Smallbank


def source(key, G, lost):
    for i in range(3):
        s = (key % G + i) % G
        if not (lost >> s) & 1:
            return s
    return -1


def replicates(key, G, shard):
    return (shard - key % G) % G <= 2


# ---- reading shard images --------------------------------------------------------------------------------------------
def regions(path):
    """the raw bytes of every region of a state image"""
    img, data, out = R.read_image(path), open(path, "rb").read(), []
    for reg in img["regions"]:
        buf = np.zeros(len(reg["blocks"]) * R.BLOCK + R.LINE, np.uint8)
        for b, blk in enumerate(reg["blocks"]):
            idx = blk["line_index"]
            lines = np.zeros(len(idx) * R.LINE, np.uint8)
            lines[:blk["stored"]] = np.frombuffer(data, np.uint8, blk["stored"], blk["lines_off"])
            buf[b * R.BLOCK: b * R.BLOCK + R.lines_of(blk["raw"]) * R.LINE].reshape(-1, R.LINE)[idx] = lines.reshape(-1, R.LINE)
        out.append(buf[:reg["bytes"]])
    return out


def shard_state(path, kind):
    """(the lock region, [{key: version + value bytes} per table]) of a tatp / smallbank shard image (no holder keys,
    no eBPF tier: region 0 is the lock state, region 1 + 2 t table t's entries)"""
    regs = regions(path)
    tabs = []
    for t in range(N_TABLES[kind]):
        e = regs[1 + 2 * t].reshape(-1, ENT[kind])
        full = e[:, 12:16].copy().view("<u4").ravel() == 1
        keys = e[full, 0:8].copy().view("<u8").ravel()
        rows = np.concatenate([e[full, 8:12], e[full, 16:16 + VALSZ[kind]]], axis=1)
        assert len(np.unique(keys)) == len(keys), "a key stored twice"
        tabs.append({int(k): r.tobytes() for k, r in zip(keys, rows)})
    return regs[0], tabs


def shard_tables(d, r, kind):
    return shard_state(os.path.join(d, f"shard-{r}.img"), kind)[1]


# ---- host-built whole transactions -----------------------------------------------------------------------------------
def submit(cl, kind, rows, check=True):
    """rows: (type, table, key, value or None, destination shard); returns the reply records"""
    a = np.zeros(len(rows), wire.MSG_DTYPE[kind])
    if not rows:
        return a
    a["type"] = [r[0] for r in rows]
    a["table"] = [r[1] for r in rows]
    a["key"] = np.array([r[2] for r in rows], np.uint64)
    for i, r in enumerate(rows):
        if r[3] is not None:
            a["val"][i] = r[3]
    dst = np.array([r[4] for r in rows], np.uint8)
    return wire.as_records(kind, cl.submit(wire.as_bytes(a), dst=dst, check=check))


def whole_txns(cl, kind, G, ops):
    """ops: (op, table, key, value), op "upd" / "ins" / "del", distinct (table, key).  Each is locked on its primary,
    logged on its three replicas, then written to the backups, then to the primary, and released: every record served.
    Returns the ops whose lock was granted (the others are dropped)."""
    if kind == TATP:
        rep = submit(cl, kind, [(Tt.kAcquireLock, t, k, None, k % G) for _, t, k, _ in ops])
        ops = [o for o, r in zip(ops, rep["type"]) if r == Tt.kGrantLock]
        bt = {"upd": Tt.kCommitBck, "ins": Tt.kInsertBck, "del": Tt.kDeleteBck}
        pt = {"upd": Tt.kCommitPrim, "ins": Tt.kInsertPrim, "del": Tt.kDeletePrim}
        lt = {"upd": Tt.kCommitLog, "ins": Tt.kCommitLog, "del": Tt.kDeleteLog}
    else:
        rep = submit(cl, kind, [(Sb.kAcquireExclusive, t, k, None, k % G) for _, t, k, _ in ops])
        ops = [o for o, r in zip(ops, rep["type"]) if r == Sb.kGrantExclusive]
        bt, pt, lt = {"upd": Sb.kCommitBck}, {"upd": Sb.kCommitPrim}, {"upd": Sb.kCommitLog}
    submit(cl, kind, [(lt[op], t, k, v, (k % G + i) % G) for op, t, k, v in ops for i in range(3)])
    submit(cl, kind, [(bt[op], t, k, v, (k % G + i) % G) for op, t, k, v in ops for i in (1, 2)])
    submit(cl, kind, [(pt[op], t, k, v, k % G) for op, t, k, v in ops])
    if kind == SMALLBANK:
        submit(cl, kind, [(Sb.kReleaseExclusive, t, k, None, k % G) for _, t, k, _ in ops])
    return ops


def traffic(cl, kind, G, seed=1):
    """two rounds of whole transactions: updates of every table, and for tatp call-forwarding deletes and inserts
    (existence is read from the primaries first, so no insert meets an existing row)"""
    rng = np.random.default_rng(seed)
    if kind == SMALLBANK:
        for _ in range(2):
            pairs = {(int(rng.integers(0, 2)), int(k)) for k in rng.integers(0, N[kind], 3000)}
            whole_txns(cl, kind, G, [("upd", t, k, rng.integers(0, 256, 8, dtype=np.uint8)) for t, k in sorted(pairs)])
        return
    u = T.tatp_key_universe(N[kind])
    cands = [u[i] for i in rng.choice(len(u), 6000, replace=False)]
    rep = submit(cl, kind, [(Tt.kRead, t, k, None, k % G) for t, k in cands])
    have = [c for c, r in zip(cands, rep["type"]) if r == Tt.kGrantRead]
    miss = [c for c, r in zip(cands, rep["type"]) if r == Tt.kNotExist and c[0] == Tt.kCallForwarding]
    cf = [c for c in have if c[0] == Tt.kCallForwarding]
    val = lambda: rng.integers(0, 256, 40, dtype=np.uint8)
    upd = [c for c in have if c[0] != Tt.kCallForwarding]
    ops = [("upd", t, k, val()) for t, k in upd[:2000]] + [("del", t, k, val()) for t, k in cf[:400]] + \
          [("ins", t, k, val()) for t, k in miss[:400]]
    done = whole_txns(cl, kind, G, ops)
    deleted = [(t, k) for op, t, k, _ in done if op == "del"]
    whole_txns(cl, kind, G, [("upd", t, k, val()) for t, k in upd[2000:3000]] + [("ins", t, k, val()) for t, k in deleted[:200]])


def damage(cl, kind, j, tabs):
    """junk commits and deletes served by shard j's engine alone: a rebuild that read it would carry them"""
    rng = np.random.default_rng(99)
    eng = cl.engine(j)
    rows = []
    for t, tab in enumerate(tabs):
        for k in list(tab)[:200]:
            rows.append((Tt.kCommitPrim if kind == TATP else Sb.kCommitPrim, t, k))
        if kind == TATP:
            rows += [(Tt.kDeletePrim, t, k) for k in list(tab)[200:300]]
    a = np.zeros(len(rows), wire.MSG_DTYPE[kind])
    a["type"], a["table"] = [r[0] for r in rows], [r[1] for r in rows]
    a["key"] = np.array([r[2] for r in rows], np.uint64)
    a["val"] = rng.integers(0, 256, a["val"].shape)
    eng.submit(wire.as_bytes(a), check=False)


def check_rebuilt(cl, kind, j, pre, post):
    """shard j of `post` (an image of the rebuilt cluster) holds exactly the rows of shard j of `pre`, its locks are
    free, and kv_count / kv_get on the live engine agree"""
    lock, tabs = shard_state(os.path.join(post, f"shard-{j}.img"), kind)
    want = shard_tables(pre, j, kind)
    assert not lock.any(), "a rebuilt shard's lock state starts free"
    eng = cl.engine(j)
    for t in range(N_TABLES[kind]):
        assert tabs[t] == want[t], (j, t, len(tabs[t]), len(want[t]))
        assert eng.kv_count(t) == len(want[t])
        for k in list(want[t])[::max(1, len(want[t]) // 50)]:
            val, ver = eng.kv_get(t, k)
            assert np.uint32(ver).tobytes() + val[:VALSZ[kind]] == want[t][k]


def make(kind, G, **over):
    return GpuCluster(kind, G, devices=[0] * G, populate=True, **SIZES[kind], **over)


MASKS = {3: [0b10, 0b001, 0b100, 0b011], 4: [0b10, 0b0001, 0b0100, 0b1000], 5: [0b10, 0b00001, 0b00100, 0b01000, 0b10000, 0b00101],
         8: [0b10, 0b1, 0b100, 0b1000, 0b10000, 0b100000, 0b1000000, 0b10000000, 0b110]}


def _bits(m):
    return [r for r in range(8) if (m >> r) & 1]


# ---- 1 + 2: rows at a replica-consistent point, then later traffic ---------------------------------------------------
@pytest.mark.parametrize("G", [3, 4, 5, 8])
@pytest.mark.parametrize("kind", [TATP, SMALLBANK], ids=["tatp", "smallbank"])
def test_rows_equal_and_later_traffic_is_answered_identically(kind, G, tmp_path):
    pre, post = str(tmp_path / "pre"), str(tmp_path / "post")
    with make(kind, G) as cl:
        traffic(cl, kind, G)
        cl.save_image(pre)
        for n, mask in enumerate(MASKS[G]):
            # the first mask on the live cluster after its traffic, the others on clusters opened from the same moment
            c = cl if n == 0 else GpuCluster.open_image(pre, devices=[0] * G)
            try:
                for j in _bits(mask):
                    damage(c, kind, j, shard_tables(pre, j, kind))
                c.rebuild(_bits(mask))
                shutil.rmtree(post, ignore_errors=True)
                c.save_image(post)
                for r in range(G):
                    if (mask >> r) & 1:
                        check_rebuilt(c, kind, r, pre, post)
                    else:
                        assert shard_tables(post, r, kind) == shard_tables(pre, r, kind)
            finally:
                if c is not cl:
                    c.close()
        # 2: the rebuilt cluster (shard 1) and one opened from the pre-damage image answer the same clients alike
        with GpuCluster.open_image(pre, devices=[0] * G) as ref:
            got = []
            for c in (cl, ref):
                with GpuTxnClients(c, 4096, subscribers=N[kind]) as tc:
                    tc.run(50)
                    got.append((tc.peek(), tc.stats(), tc.lock_stats()))
            (pa, sa, la), (pb, sb, lb) = got
            assert all(np.array_equal(x, y) for x, y in zip(pa, pb))
            assert sa == sb and la == lb
            a_dir, b_dir = str(tmp_path / "a"), str(tmp_path / "b")
            cl.save_image(a_dir)
            ref.save_image(b_dir)
            for r in range(G):
                assert shard_tables(a_dir, r, kind) == shard_tables(b_dir, r, kind), r


# ---- 3: the mid-transaction rule -------------------------------------------------------------------------------------
@pytest.mark.parametrize("G", [3, 5])
@pytest.mark.parametrize("kind", [TATP, SMALLBANK], ids=["tatp", "smallbank"])
def test_mid_transaction_rule(kind, G, tmp_path):
    mid, post = str(tmp_path / "mid"), str(tmp_path / "post")
    j = 1
    with make(kind, G) as cl:
        with GpuTxnClients(cl, 4096, subscribers=N[kind]) as tc:
            tc.run(30)
        cl.save_image(mid)
        cl.rebuild([j])
        cl.save_image(post)
    lock, got = shard_state(os.path.join(post, f"shard-{j}.img"), kind)
    assert not lock.any(), "every lock of a rebuilt shard is free"
    tabs = [shard_tables(mid, r, kind) for r in range(G)]
    differ = []
    for t in range(N_TABLES[kind]):
        want = {}
        for s in range(G):
            if s != j:
                want.update({k: row for k, row in tabs[s][t].items() if replicates(k, G, j) and source(k, G, 1 << j) == s})
        assert got[t] == want, t                          # every rebuilt row is its lowest-role surviving copy
        keys = set(want) | set(tabs[j][t])
        for k in keys:
            copies = {tabs[s][t].get(k) for s in range(G) if s != j and replicates(k, G, s)}
            if len(copies) == 1 and got[t].get(k) != tabs[j][t].get(k):
                differ.append((t, k))
    # a row whose surviving copies agree differs from the lost one only where the lost shard was the primary and still
    # held the key's lock: the backups were one write ahead
    with GpuCluster.open_image(mid, devices=[0] * G) as old:
        e = old.engine(j)
        for t, k in differ:
            assert k % G == j and any(e.lock_state(t, e.lock_slot(t, k))), (t, k)


# ---- 4: damaged image directories ------------------------------------------------------------------------------------
def _flip(path, region):
    img = R.read_image(path)
    blk = img["regions"][region]["blocks"][0]
    with open(path, "r+b") as f:
        f.seek(blk["lines_off"] + 5)
        b = f.read(1)
        f.seek(blk["lines_off"] + 5)
        f.write(bytes([b[0] ^ 0x40]))


def test_image_directories(tmp_path):
    kind, G = TATP, 4
    pre = str(tmp_path / "pre")
    with make(kind, G) as cl:
        traffic(cl, kind, G)
        cl.save_image(pre)

    def copy(name):
        d = str(tmp_path / name)
        shutil.copytree(pre, d)
        return d
    d1 = copy("missing1")
    os.remove(os.path.join(d1, "shard-1.img"))
    with pytest.raises(DintError) as ei:
        GpuCluster.open_image(d1, devices=[0] * G)
    assert ei.value.code == EIO
    fixed = str(tmp_path / "fixed")
    with GpuCluster.open_image(d1, devices=[0] * G, rebuild=True) as c:
        assert c.rebuilt == [1]
        t = E.rebuild_times()
        assert t["wall_s"] > 0 and t["kernel_s"] > 0
        c.save_image(fixed)
        check_rebuilt(c, kind, 1, pre, fixed)
    with GpuCluster.open_image(fixed, devices=[0] * G) as c:       # the repaired directory is whole again
        assert c.engine(1).kv_count(0) == len(shard_tables(pre, 1, kind)[0])
    d2 = copy("flipped2")
    _flip(os.path.join(d2, "shard-2.img"), 1)
    with GpuCluster.open_image(d2, devices=[0] * G, rebuild=True) as c:
        assert c.rebuilt == [2]
        out = str(tmp_path / "fixed2")
        c.save_image(out)
        check_rebuilt(c, kind, 2, pre, out)
    d3 = copy("three")                                              # three consecutive shards: no replica left
    os.remove(os.path.join(d3, "shard-0.img"))
    _flip(os.path.join(d3, "shard-1.img"), 1)
    _flip(os.path.join(d3, "shard-2.img"), 3)
    with pytest.raises(DintError) as ei:
        GpuCluster.open_image(d3, devices=[0] * G, rebuild=True)
    assert ei.value.code == EIO and "{0, 1, 2}" in str(ei.value), str(ei.value)
    d4 = copy("foreign")
    with Engine(SMALLBANK, device=0, accts_sizing=1000, accts_populate=100) as e:
        e.save_image(os.path.join(d4, "shard-1.img"))
    with pytest.raises(DintError) as ei:
        GpuCluster.open_image(d4, devices=[0] * G, rebuild=True)
    assert ei.value.code == EINVAL
    d5 = copy("nomanifest")
    os.remove(os.path.join(d5, "manifest"))
    with pytest.raises(DintError) as ei:
        GpuCluster.open_image(d5, devices=[0] * G, rebuild=True)
    assert ei.value.code == EIO


# ---- 5: refusals -----------------------------------------------------------------------------------------------------
def _probe(cl, kind, G):
    rng = np.random.default_rng(3)
    if kind == TATP:
        rows = [(Tt.kRead, 0, int(k), None, int(k) % G) for k in rng.integers(0, 1000, 300)]
        rows += [(Tt.kAcquireLock, 0, int(k), None, int(k) % G) for k in rng.integers(0, 1000, 300)]
        return wire.as_bytes(submit(cl, kind, rows)).copy()
    if kind == SMALLBANK:
        rows = [(Sb.kAcquireShared, int(k) & 1, int(k), None, int(k) % G) for k in rng.integers(0, 1000, 300)]
        return wire.as_bytes(submit(cl, kind, rows)).copy()
    req = {wire.FASST: T.fasst_random(300, 64, seed=3), wire.STORE: T.store_random(300, 100, seed=3),
           wire.LOCK2PL: T.lock2pl_random(300, 64, seed=3), wire.LOG: T.log_random(300, seed=3)}[kind]
    return cl.submit(req).copy()


@pytest.mark.parametrize("kind,G,over,mask,why", [
    (TATP, 5, {}, 0, "empty"), (TATP, 5, {}, 1 << 5, "outside"), (SMALLBANK, 5, {}, 0b00111, "without a replica"),
    (TATP, 3, {}, 0b111, "without a replica"), (TATP, 1, {}, 1, "one-shard"),
    (TATP, 3, dict(tatp_ebpf=True), 0b10, "eBPF"), (SMALLBANK, 3, dict(smallbank_ebpf=True), 0b10, "eBPF"),
    (wire.FASST, 3, dict(lock_slots=1 << 12), 0b10, "no replicas"), (wire.LOCK2PL, 3, dict(lock_slots=1 << 12), 0b10, "no replicas"),
    (wire.STORE, 3, dict(subs_sizing=1000, subs_populate=100), 0b10, "no replicas"), (wire.LOG, 3, {}, 0b10, "no replicas"),
    (TATP, 4, {}, 0b10, "attached"),
])
def test_refusals_leave_the_cluster_unchanged(kind, G, over, mask, why):
    """the refused cluster then answers a probe trace exactly as a twin that was never asked"""
    sizes = {TATP: dict(subs_sizing=2000, subs_populate=2000), SMALLBANK: dict(accts_sizing=2000, accts_populate=2000)}
    opts = {**sizes.get(kind, {}), **over}
    with GpuCluster(kind, G, devices=[0] * G, populate=True, **opts) as cl, \
            GpuCluster(kind, G, devices=[0] * G, populate=True, **opts) as twin:
        tcs = [GpuTxnClients(c, 256, subscribers=2000) for c in (cl, twin)] if why == "attached" else []
        for tc in tcs:
            tc.run(3)
        rc = E.lib().dint_cluster_rebuild(cl.h, mask)
        assert rc == EINVAL and why in E.lib().dint_last_error().decode(), E.lib().dint_last_error()
        for tc in tcs:
            tc.close()
        assert np.array_equal(_probe(cl, kind, G), _probe(twin, kind, G))


# ---- 6: the UDP front-end --------------------------------------------------------------------------------------------
def _ports(n):
    for base in range(31000, 60000, 97):
        socks = []
        try:
            for i in range(n):
                s = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
                socks.append(s)
                s.bind(("127.0.0.1", base + i))
            return base
        except OSError:
            continue
        finally:
            for s in socks:
                s.close()
    raise RuntimeError("no free ports")


def test_udp_front_end_rebuild_lost(tmp_path):
    from dint_b200 import _build
    kind, G = TATP, 3
    whole = str(tmp_path / "whole")
    with make(kind, G) as cl:
        traffic(cl, kind, G)
        cl.save_image(whole)
    torn = str(tmp_path / "torn")
    shutil.copytree(whole, torn)
    os.remove(os.path.join(torn, "shard-1.img"))
    rng = np.random.default_rng(8)
    u = T.tatp_key_universe(N[kind])
    rec = np.zeros(600, wire.MSG_DTYPE[kind])
    for i, c in enumerate(rng.choice(len(u), 300)):
        t, k = u[c]
        rec[2 * i]["type"], rec[2 * i]["table"], rec[2 * i]["key"] = Tt.kRead, t, k
        rec[2 * i + 1]["type"], rec[2 * i + 1]["table"], rec[2 * i + 1]["key"] = Tt.kAcquireLock, t, k
    msg = wire.MSG_SIZE[kind]
    raw = wire.as_bytes(rec).reshape(-1, msg)
    port = _ports(G)
    base = [_build.UDP_SERVER, "tatp", "--port", str(port), "--bind", "127.0.0.1", "--gpus", str(G), "--devices", "0,0,0"]
    got = {}
    for name, d, extra in (("torn", torn, ["--rebuild-lost"]), ("whole", whole, [])):
        srv = _start(base + ["--image-in", d, *extra])
        try:
            out = np.empty_like(raw)
            for i in range(len(raw)):
                out[i] = _send(port + int(rec[i]["key"]) % G, raw[i:i + 1], msg)[0]
            got[name] = out
        finally:
            srv.send_signal(signal.SIGTERM)
            assert srv.wait(timeout=120) == 0
    assert np.array_equal(got["torn"], got["whole"])
    assert (wire.as_records(kind, got["whole"].reshape(-1))["type"] == Tt.kGrantRead).sum() > 0
    r = subprocess.run(base + ["--image-in", torn], capture_output=True, timeout=120)   # without the flag: stops
    assert r.returncode == 1 and b"shard-1.img" in r.stderr


# ---- 7: full size ----------------------------------------------------------------------------------------------------
@pytest.mark.slow
def test_full_size_tatp_shard_rebuilt():
    """three TATP shards at S = 7,000,000 after population: shard 1 rebuilt holds the lost shard's rows (every table's
    count, and the value and version of 20,000 sampled keys, present or absent)"""
    S, G = 7_000_000, 3
    rng = np.random.default_rng(5)
    sample = []
    for s, ty, st in zip(rng.integers(0, S, 4000).tolist(), rng.integers(1, 5, 4000).tolist(), rng.integers(0, 3, 4000).tolist()):
        sample += [(Tt.kSubscriber, s), (Tt.kAccessInfo, s | ty << 32), (Tt.kSpecialFacility, s | ty << 32),
                   (Tt.kCallForwarding, s | ty << 32 | (8 * st) << 40)]
    with GpuCluster(TATP, G, devices=[0] * G, populate=True) as cl:
        e = cl.engine(1)
        counts = [e.kv_count(t) for t in range(5)]
        want = [e.kv_get(t, k) for t, k in sample]
        cl.rebuild([1])
        e = cl.engine(1)
        assert [e.kv_count(t) for t in range(5)] == counts
        assert [e.kv_get(t, k) for t, k in sample] == want
