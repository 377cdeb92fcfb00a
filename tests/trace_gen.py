"""Seeded request-trace generators for the parity tests (valid traces only: nothing the reference
would panic() on, and -- as the reference's clients guarantee -- no insert of a key that exists).

Contention is deliberate: keys are drawn from small sets so the same slot / key appears many times
inside one batch and the ordered (intra-batch conflict) path of the engine is exercised.
"""
import numpy as np

import oracle_lib as O
from dint_b200 import wire
from dint_b200.wire import Tatp, Smallbank


def fasst_random(n, n_keys, seed, weights=(0.5, 0.25, 0.1, 0.15)):
    rng = np.random.default_rng(seed)
    rec = np.zeros(n, dtype=wire.MSG_DTYPE[wire.FASST])
    rec["type"] = rng.choice(4, size=n, p=weights)
    rec["lid"] = rng.integers(0, n_keys, size=n)
    rec["ver"] = rng.integers(0, 2**32, size=n, dtype=np.uint64).astype(np.uint32)
    return wire.as_bytes(rec)


def lock2pl_random(n, n_keys, seed, p_release=0.45):
    rng = np.random.default_rng(seed)
    rec = np.zeros(n, dtype=wire.MSG_DTYPE[wire.LOCK2PL])
    rec["action"] = (rng.random(n) < p_release).astype(np.uint8)      # includes release-without-hold (u32 wrap)
    rec["lid"] = rng.integers(0, n_keys, size=n)
    rec["type"] = rng.integers(0, 2, size=n)
    return wire.as_bytes(rec)


def log_random(n, seed):
    rng = np.random.default_rng(seed)
    rec = np.zeros(n, dtype=wire.MSG_DTYPE[wire.LOG])
    rec["key"] = rng.integers(0, 7010000, size=n)
    rec["val"] = rng.integers(0, 256, size=(n, 40))
    rec["ver"] = rng.integers(0, 128, size=n)
    return wire.as_bytes(rec)


def store_key(s_id, sf, st):
    return np.uint64(s_id) | (np.uint64(sf) << np.uint64(32)) | (np.uint64(st) << np.uint64(40))


def store_random(n, n_subs, seed, p_set=0.3, p_miss=0.1):
    """kRead / kSet over subscribers [0, n_subs); a fraction of keys does not exist (sf_type 5..7)."""
    rng = np.random.default_rng(seed)
    rec = np.zeros(n, dtype=wire.MSG_DTYPE[wire.STORE])
    rec["type"] = (rng.random(n) < p_set).astype(np.uint8)
    s_id = rng.integers(0, n_subs, size=n).astype(np.uint64)
    sf = rng.integers(1, 5, size=n).astype(np.uint64)
    miss = rng.random(n) < p_miss
    sf[miss] += 4
    st = (rng.integers(0, 3, size=n) * 8).astype(np.uint64)
    rec["key"] = s_id | (sf << np.uint64(32)) | (st << np.uint64(40))
    rec["val"] = rng.integers(0, 256, size=(n, 40))
    rec["ver"] = rng.integers(0, 2**32, size=n, dtype=np.uint64).astype(np.uint32)
    return wire.as_bytes(rec)


def smallbank_random(n, n_accts, seed):
    rng = np.random.default_rng(seed)
    rec = np.zeros(n, dtype=wire.MSG_DTYPE[wire.SMALLBANK])
    rec["ord"] = rng.integers(0, 256, size=n)
    rec["type"] = rng.choice(7, size=n, p=[0.2, 0.2, 0.15, 0.15, 0.1, 0.1, 0.1])
    rec["table"] = rng.integers(0, 2, size=n)
    rec["key"] = rng.integers(0, n_accts, size=n)
    rec["val"] = rng.integers(0, 256, size=(n, 8))
    rec["ver"] = rng.integers(0, 2**32, size=n, dtype=np.uint64).astype(np.uint32)
    return wire.as_bytes(rec)


def tatp_key_universe(n_subs):
    """Candidate (table, key) pairs over subscribers [0, n_subs): some exist after populate, some do not."""
    cands = []
    for s in range(n_subs):
        cands.append((Tatp.kSubscriber, s))
        for t in (1, 2, 3, 4):
            cands.append((Tatp.kAccessInfo, s | (t << 32)))
            cands.append((Tatp.kSpecialFacility, s | (t << 32)))
            for st in (0, 8, 16):
                cands.append((Tatp.kCallForwarding, s | (t << 32) | (st << 40)))
    return cands


def tatp_random(n, n_subs, seed, oracle=None):
    """Valid random TATP shard traffic.  Existence is tracked sequentially, starting from the
    populated state of `oracle` (an oracle_lib.Oracle(TATP) with the same subs_populate)."""
    rng = np.random.default_rng(seed)
    own = oracle is None
    if own:
        oracle = O.Oracle(wire.TATP, subs_populate=n_subs)
    cands = tatp_key_universe(n_subs)
    exists = {c: oracle.kv_get(c[0], c[1]) is not None for c in cands}
    if own:
        oracle.close()
    rec = np.zeros(n, dtype=wire.MSG_DTYPE[wire.TATP])
    rec["ord"] = rng.integers(0, 256, size=n)
    rec["val"] = rng.integers(0, 256, size=(n, 40))
    rec["ver"] = rng.integers(0, 2**32, size=n, dtype=np.uint64).astype(np.uint32)
    pick = rng.integers(0, len(cands), size=n)
    u = rng.random(n)
    for i in range(n):
        tb, key = cands[pick[i]]
        x = u[i]
        if x < 0.30: ty = Tatp.kRead
        elif x < 0.42: ty = Tatp.kAcquireLock
        elif x < 0.50: ty = Tatp.kAbort
        elif x < 0.56: ty = Tatp.kCommitLog
        elif x < 0.60: ty = Tatp.kDeleteLog
        elif exists[(tb, key)]:
            if x < 0.72: ty = Tatp.kCommitPrim
            elif x < 0.84: ty = Tatp.kCommitBck
            elif tb != Tatp.kCallForwarding: ty = Tatp.kCommitBck
            elif x < 0.92: ty = Tatp.kDeletePrim
            else: ty = Tatp.kDeleteBck
            if ty in (Tatp.kDeletePrim, Tatp.kDeleteBck):
                exists[(tb, key)] = False
        else:
            ty = Tatp.kInsertPrim if x < 0.80 else Tatp.kInsertBck
            exists[(tb, key)] = True
        rec["type"][i] = ty
        rec["table"][i] = tb
        rec["key"][i] = key
    return wire.as_bytes(rec)


# seeded traces whose replies from the unmodified reference server binaries are stored under
# tests/golden/reference_replay/<name>.npz (tools/make_golden.py); (name, kind, trace)
REFERENCE_REPLAY = [
    ("fasst_random", wire.FASST, lambda: fasst_random(20000, 64, seed=11)),
    ("lock2pl_random", wire.LOCK2PL, lambda: lock2pl_random(20000, 64, seed=12)),
    ("log_random", wire.LOG, lambda: log_random(5000, seed=13)),
    ("fasst_single_datagram", wire.FASST, lambda: fasst_random(1, 1, seed=14)),
    ("fasst_one_slot", wire.FASST, lambda: fasst_random(6000, 1, seed=15)),                        # every request on ONE lock slot
    ("lock2pl_release_wrap", wire.LOCK2PL, lambda: lock2pl_random(6000, 1, seed=16, p_release=0.7)),  # releases without a hold
    ("lock2pl_full_u32_ids", wire.LOCK2PL, lambda: lock2pl_random(3000, 2**32 - 1, seed=17)),       # ids over the whole u32 range
]
