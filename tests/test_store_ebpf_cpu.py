"""The eBPF store server's cache tier without a GPU: the plain restatement (tests/store_ebpf_model.py) against the
goldens made from the reference's compiled XDP / TC programs, against those programs on random traces when
oracle/_ref holds them, and the option's plumbing."""
import os

import numpy as np
import pytest

import store_ebpf_model as M
from dint_b200 import engine as E
from dint_b200 import wire

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "store_ebpf")


def load_golden(v):
    g = np.load(os.path.join(GOLDEN, f"{v}.npz"))
    return g["req"], g["resp"], g["keys"], g["sets"], g["table"].reshape(-1).view(M.TABLE_REC), int(g["kv_count"])


@pytest.mark.parametrize("variant", M.VARIANTS)
def test_model_equals_golden(variant):
    req, resp, keys, sets, table, count = load_golden(variant)
    m = M.StoreEbpfModel(variant)
    got = m.process(req)
    assert np.array_equal(got, resp)
    s, t = m.state(keys)
    assert np.array_equal(s, sets) and np.array_equal(t, table)
    assert m.kv_count() == count


@pytest.mark.parametrize("variant", M.VARIANTS)
def test_golden_covers_every_path(variant):
    req, resp, keys, sets, table, count = load_golden(variant)
    m = M.StoreEbpfModel(variant)
    seen = set()
    q, r = req.reshape(-1, 53), resp.reshape(-1, 53)
    for i in range(q.shape[0]):
        b = M.fasthash64(int(q[i, 1:9].view(np.uint64)[0])) % m.buckets
        before = {k: v for k, v in m.stats.items()}
        s = m._set(b)
        valid, dirty = list(s["valid"]), list(s["dirty"])
        m.request(q[i].tobytes())
        d = {k: m.stats[k] - before[k] for k in before}
        t, rt = q[i, 0], r[i, 0]
        if t == M.INSERT:
            slot = next((j for j in range(4) if not valid[j]), None)
            seen.add("insert_free" if slot is not None else
                     "insert_dirty" if d["write_backs"] else "insert_clean")
        elif t > 2:
            seen.add("unknown")
        elif d["hits"]:
            seen.add("read_hit" if t == M.READ else "set_hit")
        elif d["bloom_negatives"]:
            seen.add("bloom_negative")
        elif t == M.READ:
            if rt == M.NOT_EXIST:
                seen.add("false_positive")
            if d["write_backs"]:
                seen.add("read_miss_write_back")
        else:
            seen.add("set_miss_found" if rt == M.SET_ACK else "set_absent")
    want = {"insert_free", "read_hit", "false_positive", "set_miss_found", "set_absent", "unknown"}
    if variant != "wt":
        want |= {"insert_clean", "insert_dirty", "read_miss_write_back", "set_hit"}
    if variant == "wb_bloom":
        want.add("bloom_negative")
    assert want <= seen, want - seen
    if variant == "wb_bloom":     # a false positive carries the eviction flag, not the request's ver
        fp = (q[:, 0] == M.READ) & (r[:, 0] == M.NOT_EXIST) & (q[:, 49:53] != r[:, 49:53]).any(1)
        assert fp.any()


@pytest.mark.skipif(not M.ref_available(), reason="oracle/_ref/store_ebpf_* not built (reference sources absent)")
@pytest.mark.parametrize("variant", M.VARIANTS)
@pytest.mark.parametrize("seed", [1, 2])
def test_model_equals_compiled_reference(variant, seed):
    rng = np.random.default_rng(seed)
    keys = np.concatenate(M.colliding_keys(M.REF_BUCKETS, 6, 10, seed=100 + seed))
    n = 2500
    k = rng.choice(keys, size=n)
    t = rng.choice([0, 0, 1, 2, 7], size=n).astype(np.uint8)
    req = M.make_req(t, k, rng.integers(0, 256, size=(n, 40), dtype=np.uint8), rng.integers(0, 3, size=n, dtype=np.uint32))
    resp, sets, table, count = M.run_ref_store_ebpf(variant, req, keys, populate=1200)
    m = M.StoreEbpfModel(variant)
    m.populate(1200)
    assert np.array_equal(m.process(req), resp)
    s, tb = m.state(keys)
    assert np.array_equal(s, sets) and np.array_equal(tb, table)
    assert m.kv_count() == count


def test_flag_values_and_names():
    assert E.DINT_CFG_STORE_EBPF_MASK == 6
    assert {v: E.default_cfg(wire.STORE, store_ebpf=v).flags for v in M.VARIANTS} == {"wb_bloom": 2, "wb": 4, "wt": 6}
    assert E.default_cfg(wire.STORE, store_ebpf=None).flags == 0
    assert E.default_cfg(wire.STORE, store_ebpf="wt", lock_holder_keys=True).flags == 7
    with pytest.raises(ValueError):
        E.default_cfg(wire.STORE, store_ebpf="write-back")
    assert wire.StoreEbpf.NOT_EXIST == wire.Store.kNotExist == 7


def test_header_documents_flags():
    h = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dint_b200.h")).read()
    for name, val in (("WB_BLOOM", "(1u << 1)"), ("WB", "(2u << 1)"), ("WT", "(3u << 1)"), ("MASK", "(3u << 1)")):
        assert f"#define DINT_CFG_STORE_EBPF_{name} {val}" in h
    assert "int dint_store_cache_set(" in h and "int dint_store_cache_stats(" in h


def test_udp_server_rejects_unknown_variant():
    import subprocess
    from dint_b200 import _build
    r = subprocess.run([_build.UDP_SERVER, "store", "--store-ebpf", "write-back"], capture_output=True, timeout=60)
    assert r.returncode == 2 and b"--store-ebpf takes" in r.stderr
