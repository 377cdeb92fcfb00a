"""TEST INFRASTRUCTURE: what a TATP server that keeps holder keys (DINT_CFG_LOCK_HOLDER_KEYS, include/dint_b200.h)
must answer, stated without any server code.

The reference's eBPF lock server keeps `struct txn_lock {u64 lock_bit; u64 key}` per lock slot
(tatp/ebpf/lock_kern.c:12-16): a granted kAcquireLock records the holder's key (:292), a refused one is answered
kRejectLockSameKey (28) when the holder's key is the request's and kRejectLock (8) when it is another key that shares
the slot (:296-298); releases clear the bit and leave the key (:338,423,609,1119,1196).

HolderModel is a dict slot -> [held, holder key] per table, walked over a trace in order.  The slot is the pure-Python
fasthash64 below modulo the table's lock modulus (tatp/udp/tatp.h:12-14: 4 x hash_size).  It predicts every lock
decision itself and checks it against the reply stream it is given, so it also cross-checks the servers' lock bits.

HolderOracle composes the two pinned pieces into the option-on server: the sequential restatement of
tatp/udp/server_shard.cc (oracle_lib.Oracle, pinned by the unmodified reference binary and the goldens), whose refused
acquires all read 8, and the model, which turns the same-key ones into 28.  Rewriting every 28 of its stream back to 8
therefore gives the option-off stream by construction.
"""
import numpy as np

import oracle_lib as O
from dint_b200 import wire

M64 = (1 << 64) - 1
LOCK, ABORT, GRANT, REJECT, REJECT_SAME_KEY = 1, 2, 7, 8, 28
RELEASING = {12: 15, 18: 20, 22: 25}      # kCommitPrim / kInsertPrim / kDeletePrim -> their ack (0xFF: nothing applied)


def _mix(h):
    h ^= h >> 23
    h = (h * 0x2127599BF4325C37) & M64
    return h ^ (h >> 47)


def fasthash64_u64(x, seed=0xDEADBEEF):
    """fasthash64 of one 8-byte little-endian word (tatp/udp/utils.h; Zilong Tan's public fast-hash)."""
    m = 0x880355F21E6D1965
    h = (seed ^ (8 * m)) & M64
    h ^= _mix(x & M64)
    h = (h * m) & M64
    return _mix(h)


def lock_moduli(subs_sizing):
    """kKeysPerEntry (4) x hash_size of the five tables (tatp/udp/server_shard.cc:75-79, tatp.h:12-14)."""
    S = subs_sizing
    hs = [S * 3 // 2 // 4, S * 3 // 2 // 4, S * 15 // 4 // 4, S * 15 // 4 // 4, S * 45 // 8 // 4]
    return [4 * h for h in hs]


def colliding_pairs(subs_sizing, table, n_pairs, start=0):
    """n_pairs pairs of keys (a, b), a != b, that share a lock slot of `table`; every pair on a slot of its own."""
    mod = lock_moduli(subs_sizing)[table]
    first, pairs, used = {}, [], set()
    k = start
    while len(pairs) < n_pairs:
        s = fasthash64_u64(k) % mod
        if s in first and s not in used:
            pairs.append((first[s], k))
            used.add(s)
        first.setdefault(s, k)
        k += 1
    return pairs


def lock_records(types, keys, table=0):
    rec = np.zeros(len(types), dtype=wire.MSG_DTYPE[wire.TATP])
    rec["type"], rec["key"], rec["table"] = types, keys, table
    return wire.as_bytes(rec)


class HolderModel:
    def __init__(self, subs_sizing):
        self.mod = lock_moduli(subs_sizing)
        self.state = [dict() for _ in range(5)]      # slot -> [held, holder key]

    def slot(self, table, key):
        return fasthash64_u64(key) % self.mod[table]

    def holder(self, table, slot):
        return self.state[table].get(slot, [False, 0])[1]

    def held(self, table, slot):
        return self.state[table].get(slot, [False, 0])[0]

    def apply(self, req, resp):
        """resp: the replies of a server WITHOUT holder keys to req.  Returns the replies of one with them."""
        q = wire.as_records(wire.TATP, req)
        out = np.array(resp, dtype=np.uint8, copy=True).reshape(-1)
        r = wire.as_records(wire.TATP, out)
        touches = np.isin(q["type"], [LOCK, ABORT, 12, 18, 22]) & (q["table"] < 5)
        for i in np.flatnonzero(touches):
            ty, tb, key, got = int(q["type"][i]), int(q["table"][i]), int(q["key"][i]), int(r["type"][i])
            st = self.state[tb].setdefault(self.slot(tb, key), [False, 0])
            if ty == LOCK:
                assert got == (REJECT if st[0] else GRANT), f"request {i}: the server's lock bit disagrees with the model"
                if st[0]:
                    if st[1] == key:
                        r["type"][i] = REJECT_SAME_KEY
                else:
                    st[0], st[1] = True, key
            elif ty == ABORT or got == RELEASING[ty]:
                st[0] = False
        return out


class HolderOracle:
    """One option-on TATP shard server: oracle_lib.Oracle + HolderModel (see the module docstring)."""

    def __init__(self, **cfg):
        self.ora = O.Oracle(wire.TATP, **cfg)
        self.model = HolderModel(self.ora.cfg.subs_sizing)

    def process(self, req):
        req = np.ascontiguousarray(req, dtype=np.uint8)
        return self.model.apply(req, self.ora.process(req))

    def __getattr__(self, name):                      # kv_get, lock_state, log_ring, ...: the plain oracle's
        return getattr(self.ora, name)


def to_option_off(resp):
    """invariant 1: an option-on reply stream with every 28 rewritten to 8 is the option-off stream"""
    out = np.array(resp, dtype=np.uint8, copy=True).reshape(-1)
    r = wire.as_records(wire.TATP, out)
    r["type"][r["type"] == REJECT_SAME_KEY] = REJECT
    return out


def count_lock_replies(req, resp):
    """(locks requested, refused through sharing, refused by the same key) read off a raw request / reply stream"""
    q, r = wire.as_records(wire.TATP, req), wire.as_records(wire.TATP, resp)
    t = r["type"][q["type"] == LOCK]
    return int(t.size), int((t == REJECT).sum()), int((t == REJECT_SAME_KEY).sum())
