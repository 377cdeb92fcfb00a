"""The eBPF SmallBank shard server's restatement (tests/smallbank_ebpf_model.py) against the reference's compiled
program, and the DINT_CFG_SMALLBANK_EBPF plumbing that needs no GPU."""
import os

import numpy as np
import pytest

import smallbank_ebpf_model as M
from dint_b200 import engine as E
from dint_b200 import wire

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "smallbank_ebpf")
NAMES = ("cold", "warm")


def golden(name):
    return np.load(os.path.join(GOLDEN, f"{name}.npz"))


def model_for(z):
    m = M.SmallbankEbpfModel(populated=int(z["populated"]))
    if bool(z["warm"]):
        m.warmup()
    return m


def assert_model_state(m, z):
    sets, finds, locks = m.state(z["keys"], z["tables"])
    np.testing.assert_array_equal(sets, z["sets"])
    np.testing.assert_array_equal(finds.view(np.uint8).reshape(z["finds"].shape), z["finds"])
    np.testing.assert_array_equal(locks.view(np.uint8).reshape(z["locks"].shape), z["locks"])
    np.testing.assert_array_equal(m.log_dump(), z["log"])


@pytest.mark.parametrize("name", NAMES)
def test_model_equals_golden(name):
    z = golden(name)
    m = model_for(z)
    np.testing.assert_array_equal(m.process(z["req"]), z["resp"])
    assert_model_state(m, z)


def test_goldens_cover_every_path():
    paths = set()
    for name in NAMES:
        m = model_for(golden(name))
        m.process(golden(name)["req"])
        paths |= set(m.paths)
    assert not set(M.REQUIRED_PATHS) - paths, sorted(set(M.REQUIRED_PATHS) - paths)


@pytest.mark.skipif(not M.ref_available(), reason="oracle/_ref/smallbank_ebpf not built (reference sources absent)")
@pytest.mark.parametrize("warm", [False, True])
@pytest.mark.parametrize("seed", [1, 2])
def test_model_equals_compiled_reference(warm, seed):
    populated = 3_000_000
    groups = M.colliding_groups(populated, per_bucket=5, n_buckets=3, seed=100 + seed)
    keys, tables = M.group_keys(groups)
    req = M.random_trace(groups, 2500, seed=seed)
    resp, sets, finds, locks, log = M.run_ref_smallbank_ebpf(req, keys, tables, populate=populated, warmup=warm)
    m = M.SmallbankEbpfModel(populated=populated)
    if warm:
        m.warmup()
    np.testing.assert_array_equal(m.process(req), resp)
    ms, mf, ml = m.state(keys, tables)
    np.testing.assert_array_equal(ms, sets)
    np.testing.assert_array_equal(mf, finds)
    np.testing.assert_array_equal(ml, locks)
    np.testing.assert_array_equal(m.log_dump(), log)


@pytest.mark.skipif(not M.ref_available(), reason="oracle/_ref/smallbank_ebpf not built (reference sources absent)")
@pytest.mark.parametrize("shard,G", [(0, 3), (2, 3), (1, 5), (4, 7)])
def test_warmup_equals_compiled_reference(shard, G):
    """the warm-up stream as shard `shard` of G sees it: the model's closed form against the program served one warm-up
    read at a time, on sets sampled over the populated accounts"""
    populated = 200_000
    keys = np.arange(0, populated, 37, dtype=np.uint64)
    keys = np.concatenate([keys, keys])
    tables = np.repeat(np.array([0, 1], np.uint8), len(keys) // 2)
    _, sets, finds, _, _ = M.run_ref_smallbank_ebpf(np.zeros(0, np.uint8), keys, tables, populate=populated, warmup=True,
                                                    shard=shard, G=G)
    m = M.SmallbankEbpfModel(populated=populated, shard=shard, G=G)
    m.warmup()
    ms, mf, _ = m.state(keys, tables)
    np.testing.assert_array_equal(ms, sets)
    held = mf["found"] == 1     # every shard of the reference populates every account; the engine (and the model),
    assert held.any()           # with G > 3, only the accounts the shard replicates
    np.testing.assert_array_equal(mf[held], finds[held])
    assert sets[:, 80:84].any()


def test_flag_values_and_names():
    assert E.DINT_CFG_SMALLBANK_EBPF == 16
    assert not E.DINT_CFG_SMALLBANK_EBPF & (E.DINT_CFG_LOCK_HOLDER_KEYS | E.DINT_CFG_STORE_EBPF_MASK | E.DINT_CFG_TATP_EBPF)
    S = wire.SmallbankEbpf
    assert (S.WARMUP_READ, S.WARMUP_READ_ACK, S.RETRY) == (17, 18, 16) == (M.WARMUP_READ, M.WARMUP_READ_ACK, M.RETRY)
    assert S.COMMIT_LOG_ACK == wire.Smallbank.kCommitLogAck and S.WARMUP_READ == wire.Smallbank.kWarmupRead
    assert E.SMALLBANK_CACHE_ENTRY_BYTES == M.CACHE_ENTRY and E.SMALLBANK_CACHE_STATS == M.STATS
    for name in ("dint_smallbank_cache_set", "dint_smallbank_cache_stats"):
        assert name in E.ABI_SYMBOLS


def test_header_documents_flag():
    h = open(os.path.join(ROOT, "include", "dint_b200.h")).read()
    assert "#define DINT_CFG_SMALLBANK_EBPF (1u << 4)" in h
    assert "#define DINT_SMALLBANK_CACHE_ENTRY_BYTES 96" in h
    for name in ("dint_smallbank_cache_set", "dint_smallbank_cache_stats"):
        assert f"int {name}(" in h


def test_hash_size_and_replicas():
    assert M.hash_size() == 9_000_000
    assert M.replicates(0, 3, 10).tolist() == list(range(10))
    assert M.replicates(1, 5, 12).tolist() == [0, 1, 4, 5, 6, 9, 10, 11]   # a % 5 in {4, 0, 1}


def test_udp_server_parses_smallbank_ebpf():
    """--smallbank-ebpf takes no value (like --tatp-ebpf) and is listed in the usage line"""
    import subprocess
    from dint_b200 import _build
    r = subprocess.run([_build.UDP_SERVER, "smallbank", "--smallbank-ebpf", "--no-such-option", "1"], capture_output=True,
                       timeout=60)
    assert r.returncode == 2 and b"unknown option --no-such-option" in r.stderr
    r = subprocess.run([_build.UDP_SERVER], capture_output=True, timeout=60)
    assert b"[--smallbank-ebpf]" in r.stderr
    assert E.default_cfg(wire.SMALLBANK, smallbank_ebpf=True).flags == 16
    assert E.default_cfg(wire.SMALLBANK, smallbank_ebpf=False).flags == 0
