"""The eBPF TATP shard server's restatement (tests/tatp_ebpf_model.py) against the reference's compiled programs, and the
DINT_CFG_TATP_EBPF plumbing that needs no GPU."""
import os

import numpy as np
import pytest

import tatp_ebpf_model as M
from dint_b200 import engine as E
from dint_b200 import wire

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tatp_ebpf")


def _golden(variant):
    return np.load(os.path.join(GOLDEN, f"{variant}.npz"))


@pytest.mark.parametrize("variant", M.VARIANTS)
def test_model_equals_golden(variant):
    z = _golden(variant)
    m = M.TatpEbpfModel(holder_keys=variant == "lock")
    np.testing.assert_array_equal(m.process(z["req"]), z["resp"])
    sets, chains, finds, locks = m.state(z["keys"], z["tables"])
    np.testing.assert_array_equal(sets, z["sets"])
    np.testing.assert_array_equal(chains.view(np.uint8).reshape(z["chains"].shape), z["chains"])
    np.testing.assert_array_equal(finds.view(np.uint8).reshape(z["finds"].shape), z["finds"])
    np.testing.assert_array_equal(locks.view(np.uint8).reshape(z["locks"].shape), z["locks"])
    np.testing.assert_array_equal(m.log_dump(), z["log"])


@pytest.mark.parametrize("variant", M.VARIANTS)
def test_golden_covers_every_path(variant):
    m = M.TatpEbpfModel(holder_keys=variant == "lock")
    m.process(_golden(variant)["req"])
    need = M.REQUIRED_PATHS_LOCK if variant == "lock" else M.REQUIRED_PATHS
    assert not set(need) - set(m.paths), sorted(set(need) - set(m.paths))
    assert m.stats["freed"] > 0 and m.stats["reused"] > 0 and m.stats["allocated"] > 0


@pytest.mark.skipif(not M.ref_available(), reason="oracle/_ref/tatp_ebpf_* not built (reference sources absent)")
@pytest.mark.parametrize("variant", M.VARIANTS)
@pytest.mark.parametrize("seed", [1, 2])
def test_model_equals_compiled_reference(variant, seed):
    groups = M.colliding_groups(M.REF_S, per_bucket=6, n_buckets=4, seed=100 + seed)
    req = M.random_trace(groups, 3000, seed=seed)
    keys = np.array([k for g in groups for grp in g for k in grp], dtype=np.uint64)
    tables = np.array([t for t, g in enumerate(groups) for grp in g for _ in grp], dtype=np.uint8)
    resp, sets, chains, finds, locks, log = M.run_ref_tatp_ebpf(variant, req, keys, tables)
    m = M.TatpEbpfModel(holder_keys=variant == "lock")
    np.testing.assert_array_equal(m.process(req), resp)
    ms, mc, mf, ml = m.state(keys, tables)
    np.testing.assert_array_equal(ms, sets)
    np.testing.assert_array_equal(mc, chains)
    np.testing.assert_array_equal(mf, finds)
    np.testing.assert_array_equal(ml, locks)
    np.testing.assert_array_equal(m.log_dump(), log)


@pytest.mark.skipif(not M.ref_available(), reason="oracle/_ref/tatp_ebpf_* not built (reference sources absent)")
def test_population_equals_compiled_reference():
    """the eBPF client's population stream (600 threads, fastrand per thread), served by both, at a small S: the
    compiled programs keep the reference's bucket counts, so the model is run with them too"""
    S = 1800
    keys, tables = [], []
    for t, key, _ in M.population(S)[::7]:
        keys.append(key)
        tables.append(t)
    for shard in (0, 2):
        _, sets, chains, finds, locks, _ = M.run_ref_tatp_ebpf("shard", np.zeros(0, np.uint8), keys, tables, populate=S,
                                                              shard=shard)
        m = M.TatpEbpfModel()
        m.populate(S, shard=shard)
        ms, mc, mf, ml = m.state(keys, tables)
        np.testing.assert_array_equal(ms, sets)
        np.testing.assert_array_equal(mc, chains)
        np.testing.assert_array_equal(mf, finds)


def test_flag_values_and_names():
    assert E.DINT_CFG_TATP_EBPF == 8
    assert not E.DINT_CFG_TATP_EBPF & (E.DINT_CFG_LOCK_HOLDER_KEYS | E.DINT_CFG_STORE_EBPF_MASK)
    assert wire.TatpEbpf.REJECT_LOCK_SAME_KEY == wire.Tatp.kRejectLockSameKey
    assert wire.TatpEbpf.DELETE_BCK_ACK == wire.Tatp.kDeleteBckAck == M.DELETE_BCK_ACK
    assert E.TATP_CHAIN_REC.itemsize == 212 and E.TATP_CACHE_STATS == M.STATS
    for name in ("dint_tatp_cache_set", "dint_tatp_chain", "dint_tatp_cache_stats"):
        assert name in E.ABI_SYMBOLS


def test_header_documents_flag():
    h = open(os.path.join(ROOT, "include", "dint_b200.h")).read()
    assert "#define DINT_CFG_TATP_EBPF (1u << 3)" in h
    assert "#define DINT_TATP_CHAIN_REC_BYTES 212" in h
    for name in ("dint_tatp_cache_set", "dint_tatp_chain", "dint_tatp_cache_stats"):
        assert f"int {name}(" in h


def test_hash_sizes():
    assert M.hash_sizes(M.REF_S) == [2625000, 2625000, 6562500, 6562500, 6562500]


def test_udp_server_parses_tatp_ebpf():
    """--tatp-ebpf takes no value (like --lock-holder-keys) and is listed in the usage line"""
    import subprocess
    from dint_b200 import _build
    r = subprocess.run([_build.UDP_SERVER, "tatp", "--tatp-ebpf", "--no-such-option", "1"], capture_output=True, timeout=60)
    assert r.returncode == 2 and b"unknown option --no-such-option" in r.stderr
    r = subprocess.run([_build.UDP_SERVER], capture_output=True, timeout=60)
    assert b"[--tatp-ebpf]" in r.stderr
    assert E.default_cfg(wire.TATP, tatp_ebpf=True, lock_holder_keys=True).flags == 9
    assert E.default_cfg(wire.TATP, tatp_ebpf=False).flags == 0
