"""The reference's eBPF SmallBank shard server (smallbank/ebpf), for tests of the engine's DINT_CFG_SMALLBANK_EBPF option.

Two independent statements of it:

* run_ref_smallbank_ebpf(): the reference's own XDP / TC programs (shard_kern.c) and kvs.h, compiled unmodified by
  oracle/smallbank_ebpf.mk into oracle/_ref/smallbank_ebpf and driven one request at a time
  (oracle/smallbank_ebpf_replay.c).  Its sizes are the reference's (A = 24,000,000 accounts); a prefix of them is
  populated.
* SmallbankEbpfModel: a plain restatement in Python with a run-time account count, so that small engines can be checked
  too.  Pinned to the compiled program by tests/golden/smallbank_ebpf/*.npz and, where oracle/_ref exists, by random
  traces.

The table side needs no chain layout: population inserts each account once, so kvs_get / kvs_set find that one copy.
The model keeps only the rows that changed since population; the populated ones are implied.
"""
import collections
import os
import struct
import subprocess
import tempfile

import numpy as np

from store_ebpf_model import M64, fasthash64, fasthash64_np  # noqa: F401  (re-exported)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
REF_BIN = os.path.join(REF_DIR, "smallbank_ebpf")
MSG = 23
CACHE_ENTRY = 96            # struct cache_entry, smallbank/ebpf/utils.h:82-89
FIND_REC = np.dtype([("found", "<u4"), ("ver", "<u4"), ("val", "u1", (8,))])
LOCK_REC = np.dtype([("lock", "<u8"), ("num_ex", "<u4"), ("num_sh", "<u4")])
LOG_ENTRY = 32
REF_A = 24_000_000

(ACQUIRE_SHARED, ACQUIRE_EXCLUSIVE, RELEASE_SHARED, RELEASE_EXCLUSIVE, COMMIT_PRIM, COMMIT_BCK, COMMIT_LOG,
 GRANT_SHARED, REJECT_SHARED, GRANT_EXCLUSIVE, REJECT_EXCLUSIVE, RELEASE_SHARED_ACK, RELEASE_EXCLUSIVE_ACK,
 COMMIT_PRIM_ACK, COMMIT_BCK_ACK, COMMIT_LOG_ACK, RETRY, WARMUP_READ, WARMUP_READ_ACK) = range(19)
STATS = ("hits", "table", "write_backs", "installs")
U32 = 0xffffffff


def hash_size(A=REF_A):
    """bucket count of each table (smallbank/ebpf/utils.h:16-17)"""
    return A * 3 // 2 // 4


def initial_value(table):
    """the value population writes (smallbank.h:44-66): {u32 magic = 97 / 98; float bal = 1e9}"""
    return struct.pack("<If", 97 + table, 1e9)


def replicates(shard, G, accounts):
    """the accounts [0, accounts) shard `shard` of G holds, ascending: all of them when G <= 3, else those whose
    primary a % G is shard, shard - 1 or shard - 2 (mod G)"""
    a = np.arange(accounts, dtype=np.uint64)
    if G > 3:
        a = a[(np.uint64(shard + G) - a % np.uint64(G)) % np.uint64(G) <= 2]
    return a


def ref_available():
    return os.path.exists(REF_BIN)


def run_ref_smallbank_ebpf(req, keys=(), tables=(), populate=0, warmup=False, shard=0, G=3):
    """Replies of the compiled reference server to `req` (n*23 uint8), after populating accounts [0, populate) and, with
    `warmup`, serving the warm-up stream of shard `shard` of G.  Returns (replies [n*23], sets [k, 96], finds FIND_REC [k],
    locks LOCK_REC [k], log [m, 32]) for the (key, table) pairs, after the trace."""
    req = np.ascontiguousarray(req, dtype=np.uint8).reshape(-1)
    kt = np.zeros((len(keys), 2), dtype=np.uint64)
    kt[:, 0] = np.asarray(keys, dtype=np.uint64)
    kt[:, 1] = np.asarray(tables, dtype=np.uint64)
    with tempfile.TemporaryDirectory() as d:
        p = {n: os.path.join(d, n) for n in ("req", "resp", "keys", "sets", "finds", "locks", "log")}
        req.tofile(p["req"])
        kt.tofile(p["keys"])
        cmd = [REF_BIN, p["req"], p["resp"], "--populate", str(populate), "--shard", str(shard), "--shards", str(G),
               "--dump", p["keys"], p["sets"], p["finds"], p["locks"], p["log"]]
        if warmup:
            cmd.append("--warmup")
        subprocess.run(cmd, check=True, capture_output=True)
        resp = np.fromfile(p["resp"], dtype=np.uint8)
        sets = np.fromfile(p["sets"], dtype=np.uint8).reshape(-1, CACHE_ENTRY)
        finds = np.fromfile(p["finds"], dtype=FIND_REC)
        locks = np.fromfile(p["locks"], dtype=LOCK_REC)
        log = np.fromfile(p["log"], dtype=np.uint8).reshape(-1, LOG_ENTRY)
    return resp, sets, finds, locks, log


class SmallbankEbpfModel:
    """One server thread of smallbank/ebpf: XDP (shard_kern.c), the user-space dispatch (shard_user.c:139-189) over the
    tables of smallbank/ebpf/kvs.h, and TC egress -- with hash_size(A) buckets and accounts [0, populated) in the
    tables -- of them, with G = txn_shards > 3, only those shard `shard` replicates."""

    def __init__(self, A=REF_A, populated=0, shard=0, G=3, log_ring=1_000_000):
        self.H = hash_size(A)
        self.populated, self.shard, self.G = populated, shard, G
        self.cache = [dict(), dict()]     # bucket -> dict(key, val, ver, valid, dirty: [4])
        self.warm = [None, None]          # after warmup(): per table (sorted buckets, slot keys [n, 4], slots used [n])
        self.rows = [dict(), dict()]      # key -> [val, ver]: the rows that changed since population
        self.locks = [dict(), dict()]     # lock slot -> [num_ex, num_sh] (u32)
        self.log_ring = log_ring
        self.log = {}
        self.log_cnt = 0
        self.stats = dict.fromkeys(STATS, 0)
        self.paths = collections.Counter()   # which path of the server each request took (coverage of a trace)

    # ---- smallbank/ebpf/kvs.h: None = the key is absent (kvs_get / kvs_set would panic) ------------------------------
    def kvs_get(self, t, key):
        if key in self.rows[t]:
            return tuple(self.rows[t][key])
        held = key < self.populated and (self.G <= 3 or (self.shard - key % self.G) % self.G <= 2)
        return (initial_value(t), 0) if held else None

    def kvs_set(self, t, key, val, ver):
        got = self.kvs_get(t, key)
        if got is None:
            return None
        nv = ver if ver != 0 else (got[1] + 1) & U32
        self.rows[t][key] = [val, nv]
        return nv

    # ---- the cache sets -------------------------------------------------------------------------------------------
    def _set(self, t, b):
        s = self.cache[t].get(b)
        if s is None:
            s = dict(key=[0] * 4, val=[bytes(8)] * 4, ver=[0] * 4, valid=[0] * 4, dirty=[0] * 4)
            w = self.warm[t]
            if w is not None:
                i = int(np.searchsorted(w[0], b))
                if i < len(w[0]) and int(w[0][i]) == b:
                    for j in range(int(w[2][i])):
                        s["key"][j], s["val"][j], s["valid"][j] = int(w[1][i][j]), initial_value(t), 1
            self.cache[t][b] = s
        return s

    @staticmethod
    def _victim(s):
        for i in range(4):
            if not s["valid"][i]:
                return i, "invalid"
        for i in range(4):
            if not s["dirty"][i]:
                return i, "clean"
        return 0, "dirty"

    def request(self, rec):
        """rec: 23 bytes; returns the 23-byte reply"""
        r = bytearray(rec)
        ty, t = r[1], r[2]
        key = int.from_bytes(r[3:11], "little")
        val = bytes(r[11:19])
        if ty == COMMIT_LOG:                                   # shard_kern.c:566-583: any table byte
            e = bytearray(LOG_ENTRY)
            e[0] = t
            e[8:16], e[16:24], e[24:28] = r[3:11], val, r[19:23]
            self.log[self.log_cnt % self.log_ring] = bytes(e)
            self.log_cnt += 1
            self.paths["log_table_ge2" if t >= 2 else "log"] += 1
            r[1] = COMMIT_LOG_ACK
            return bytes(r)
        if t >= 2 or ty not in (ACQUIRE_SHARED, ACQUIRE_EXCLUSIVE, RELEASE_SHARED, RELEASE_EXCLUSIVE, COMMIT_PRIM,
                                COMMIT_BCK, WARMUP_READ):
            self.paths["invalid_table" if t >= 2 else "invalid_type"] += 1
            r[1] = 0xFF
            return bytes(r)
        h = fasthash64(key)
        if ty <= RELEASE_EXCLUSIVE:                            # the lock unit, :96-392
            lk = self.locks[t].setdefault(h % (4 * self.H), [0, 0])
            # the counters are ints compared with > 0 (:138, :255): a count a stray release took below zero refuses
            # nothing, where the UDP server's unsigned == 0 test refuses
            ex, sh = (lk[0] ^ 0x80000000) - 0x80000000, (lk[1] ^ 0x80000000) - 0x80000000
            if ty == ACQUIRE_SHARED and ex > 0:
                self.paths["reject_shared"] += 1
                r[1] = REJECT_SHARED
                return bytes(r)
            if ty == ACQUIRE_EXCLUSIVE and (ex > 0 or sh > 0):
                self.paths["reject_exclusive"] += 1
                r[1] = REJECT_EXCLUSIVE
                return bytes(r)
            if ty in (RELEASE_SHARED, RELEASE_EXCLUSIVE):
                i = 1 if ty == RELEASE_SHARED else 0
                if lk[i] == 0:
                    self.paths["release_below_zero"] += 1
                lk[i] = (lk[i] - 1) & U32
                r[1] = RELEASE_SHARED_ACK if ty == RELEASE_SHARED else RELEASE_EXCLUSIVE_ACK
                return bytes(r)
            if ex < 0 or (ty == ACQUIRE_EXCLUSIVE and sh < 0):
                self.paths["grant_below_zero"] += 1
            i = 1 if ty == ACQUIRE_SHARED else 0
            lk[i] = (lk[i] + 1) & U32                          # counted before the cache is looked at
        commit = ty in (COMMIT_PRIM, COMMIT_BCK)
        name = "commit" if commit else "warmup" if ty == WARMUP_READ else "grant"
        ack = {ACQUIRE_SHARED: GRANT_SHARED, ACQUIRE_EXCLUSIVE: GRANT_EXCLUSIVE, COMMIT_PRIM: COMMIT_PRIM_ACK,
               COMMIT_BCK: COMMIT_BCK_ACK, WARMUP_READ: WARMUP_READ_ACK}[ty]
        st = self.stats
        s = self._set(t, h % self.H)
        hit = next((i for i in range(4) if s["valid"][i] and s["key"][i] == key), -1)
        if hit >= 0:
            st["hits"] += 1
            self.paths[name + "_hit"] += 1
            if commit:                                         # the reply echoes the client's ver
                s["val"][hit] = val
                s["ver"][hit] = (s["ver"][hit] + 1) & U32
                s["dirty"][hit] = 1
                r[1] = ack
            else:                                              # a warm-up hit is answered kGrantShared
                r[11:19], r[19:23] = s["val"][hit], s["ver"][hit].to_bytes(4, "little")
                r[1] = GRANT_EXCLUSIVE if ty == ACQUIRE_EXCLUSIVE else GRANT_SHARED
            return bytes(r)
        st["table"] += 1
        v, vk = self._victim(s)
        self.paths["%s_miss_%s" % (name, vk)] += 1
        wrote_back = False
        if s["valid"][v] and s["dirty"][v]:                    # kvs_set(key2, val2, ver2)
            st["write_backs"] += 1
            wrote_back = True
            if s["ver"][v] == 0:
                self.paths["write_back_ver0"] += 1
            self.kvs_set(t, s["key"][v], s["val"][v], s["ver"][v])
        if commit:
            nv = self.kvs_set(t, key, val, 0)
            got = None if nv is None else (val, nv)
        else:
            got = self.kvs_get(t, key)
        if got is None:                                        # the reference panics: answered 0xFF, nothing installed
            self.paths["missing_key" + ("_after_write_back" if wrote_back else "")] += 1
            r[1] = 0xFF
            return bytes(r)
        st["installs"] += 1
        r[11:19], r[19:23] = got[0], got[1].to_bytes(4, "little")
        s["key"][v], s["val"][v], s["ver"][v], s["valid"][v], s["dirty"][v] = key, got[0], got[1], 1, 0
        r[1] = ack
        return bytes(r)

    def process(self, req):
        raw = np.ascontiguousarray(req, dtype=np.uint8).reshape(-1)
        out = bytearray(raw.size)
        for i in range(raw.size // MSG):
            out[i * MSG:(i + 1) * MSG] = self.request(raw[i * MSG:(i + 1) * MSG].tobytes())
        return np.frombuffer(bytes(out), dtype=np.uint8)

    def warmup(self):
        """the eBPF client's warm-up stream over the populated accounts, as this shard sees it, on a cold cache:
        every request is a miss (no key repeats in a table) that installs into the first invalid slot, else slot 0
        (every slot is clean), so a bucket ends with its first keys in slots 1-3 and its last in slot 0.  Computed per
        bucket in closed form rather than one request at a time."""
        assert not any(self.cache) and not any(self.rows) and self.warm == [None, None], "warm-up of a fresh server only"
        acc = replicates(self.shard, self.G, self.populated)
        for t in range(2):
            b = fasthash64_np(acc) % np.uint64(self.H)
            order = np.argsort(b, kind="stable")
            bs, ks = b[order], acc[order]
            starts = np.flatnonzero(np.r_[True, bs[1:] != bs[:-1]]) if bs.size else np.zeros(0, np.int64)
            counts = np.diff(np.r_[starts, bs.size])
            slots = np.zeros((starts.size, 4), dtype=np.uint64)
            for j in range(4):
                has = counts > j
                slots[has, j] = ks[starts[has] + j]
            last = counts > 4
            slots[last, 0] = ks[starts[last] + counts[last] - 1]
            self.warm[t] = (bs[starts], slots, np.minimum(counts, 4))
            self.stats["table"] += int(acc.size)
            self.stats["installs"] += int(acc.size)

    # ---- state, in the compiled oracle's dump formats -----------------------------------------------------------
    def cache_entry(self, t, b):
        """struct cache_entry of bucket b of table t (96 uint8, lock = 0)"""
        s = self._set(t, b)
        out = bytearray(CACHE_ENTRY)
        for i in range(4):
            out[8 * i:8 * i + 8] = s["key"][i].to_bytes(8, "little")
            out[32 + 8 * i:40 + 8 * i] = s["val"][i]
            out[64 + 4 * i:68 + 4 * i] = s["ver"][i].to_bytes(4, "little")
            out[80 + i], out[84 + i] = s["valid"][i], s["dirty"][i]
        return np.frombuffer(bytes(out), dtype=np.uint8)

    def state(self, keys, tables):
        """(sets, finds, locks) as run_ref_smallbank_ebpf dumps them"""
        n = len(keys)
        sets = np.zeros((n, CACHE_ENTRY), np.uint8)
        finds = np.zeros(n, dtype=FIND_REC)
        locks = np.zeros(n, dtype=LOCK_REC)
        for i, (k, t) in enumerate(zip(keys, tables)):
            k, t = int(k), int(t)
            h = fasthash64(k)
            sets[i] = self.cache_entry(t, h % self.H)
            got = self.kvs_get(t, k)
            if got is not None:
                finds[i]["found"], finds[i]["ver"] = 1, got[1]
                finds[i]["val"] = np.frombuffer(got[0], dtype=np.uint8)
            locks[i]["num_ex"], locks[i]["num_sh"] = self.locks[t].get(h % (4 * self.H), [0, 0])
        return sets, finds, locks

    def log_dump(self):
        """the first min(appends, ring) entries of the log ring, [m, 32] uint8"""
        m = min(self.log_cnt, self.log_ring)
        out = np.zeros((m, LOG_ENTRY), np.uint8)
        for i in range(m):
            out[i] = np.frombuffer(self.log[i], dtype=np.uint8)
        return out


def make_req(types, tables, keys, vals=None, vers=None, ords=None):
    """n packed 23-byte smallbank messages"""
    n = len(types)
    rec = np.zeros((n, MSG), dtype=np.uint8)
    if ords is not None:
        rec[:, 0] = np.asarray(ords, dtype=np.uint8)
    rec[:, 1] = np.asarray(types, dtype=np.uint8)
    rec[:, 2] = np.asarray(tables, dtype=np.uint8)
    rec[:, 3:11] = np.asarray(keys, dtype=np.uint64).reshape(-1, 1).view(np.uint8)
    if vals is not None:
        rec[:, 11:19] = np.asarray(vals, dtype=np.uint8).reshape(n, 8)
    if vers is not None:
        rec[:, 19:23] = np.asarray(vers, dtype=np.uint32).reshape(-1, 1).view(np.uint8)
    return rec.reshape(-1)


def colliding_groups(populated, A=REF_A, per_bucket=5, n_buckets=4, seed=0):
    """per table: n_buckets groups of per_bucket populated accounts (< populated) that share one bucket of hash_size(A),
    each followed by one key the tables lack (in [populated, 2 * populated)) of the same bucket"""
    H = np.uint64(hash_size(A))
    out = []
    for t in range(2):
        k = np.arange(2 * populated, dtype=np.uint64)
        b = fasthash64_np(k) % H
        miss = dict(zip(b[populated:].tolist(), k[populated:].tolist()))
        pb = b[:populated]
        order = np.argsort(pb, kind="stable")
        bs = pb[order]
        starts = np.flatnonzero(np.r_[True, bs[1:] != bs[:-1]])
        counts = np.diff(np.r_[starts, bs.size])
        cand = [int(s) for s, c in zip(starts, counts) if c >= per_bucket and int(bs[s]) in miss]
        rng = np.random.default_rng(seed + t)
        pick = rng.choice(len(cand), size=n_buckets, replace=False)
        groups = []
        for p in sorted(pick):
            s = cand[p]
            groups.append([int(x) for x in k[order[s:s + per_bucket]]] + [miss[int(bs[s])]])
        out.append(groups)
    return out


def random_trace(groups, n, seed=0):
    """n requests over the colliding key groups of both tables: lock pairs (acquire, then commit / release), stray
    releases, commits without a lock, warm-up reads, log appends (some with a table >= 2), and requests the server
    refuses (unknown types, a table >= 2).  The last key of a group is one the tables lack."""
    rng = np.random.default_rng(seed)
    ty, tb, ks = [], [], []
    while len(ty) < n:
        t = int(rng.integers(0, 2))
        g = groups[t][rng.integers(0, len(groups[t]))]
        k = g[rng.integers(0, len(g))] if rng.random() < 0.08 else g[rng.integers(0, len(g) - 1)]
        r = rng.random()
        if r < 0.22:
            ty += [ACQUIRE_SHARED, RELEASE_SHARED] if rng.random() < 0.8 else [ACQUIRE_SHARED]
        elif r < 0.45:
            ty += [ACQUIRE_EXCLUSIVE, COMMIT_PRIM, COMMIT_BCK, RELEASE_EXCLUSIVE] if rng.random() < 0.85 else [ACQUIRE_EXCLUSIVE]
        elif r < 0.62:
            ty += [COMMIT_PRIM if rng.random() < 0.5 else COMMIT_BCK]
        elif r < 0.77:
            ty += [WARMUP_READ]
        elif r < 0.81:
            ty += [RELEASE_SHARED if rng.random() < 0.5 else RELEASE_EXCLUSIVE]
        elif r < 0.9:
            ty += [COMMIT_LOG]
            if rng.random() < 0.2:
                t = int(rng.integers(2, 256))
        elif r < 0.95:
            ty += [int(rng.choice([7, 9, 11, 13, 15, 16, 18, 19, 40, 255]))]
        else:
            ty += [int(rng.choice([ACQUIRE_SHARED, RELEASE_EXCLUSIVE, COMMIT_PRIM, WARMUP_READ]))]
            t = int(rng.integers(2, 256))
        while len(tb) < len(ty):
            tb.append(t)
            ks.append(k)
    ty, tb, ks = ty[:n], tb[:n], ks[:n]
    vals = rng.integers(0, 256, size=(n, 8), dtype=np.uint8)
    vers = rng.integers(0, 1 << 32, size=n, dtype=np.uint64).astype(np.uint32)
    vers[rng.random(n) < 0.3] = 0
    ords = rng.integers(0, 256, size=n, dtype=np.uint8)
    return make_req(ty, tb, ks, vals, vers, ords)


def group_keys(groups):
    """(keys, tables) of every key of the groups"""
    keys = np.array([k for g in groups for grp in g for k in grp], dtype=np.uint64)
    tables = np.array([t for t, g in enumerate(groups) for grp in g for _ in grp], dtype=np.uint8)
    return keys, tables


# every path of the server the two golden traces must reach together (SmallbankEbpfModel.paths).  A dirty slot with
# version 0 ("write_back_ver0") needs 2^32 commits of one cached row and is left out.
REQUIRED_PATHS = (
    "reject_shared", "reject_exclusive", "grant_below_zero", "grant_hit", "grant_miss_invalid", "grant_miss_clean", "grant_miss_dirty",
    "commit_hit", "commit_miss_invalid", "commit_miss_clean", "commit_miss_dirty", "release_below_zero",
    "warmup_hit", "warmup_miss_invalid", "warmup_miss_clean", "warmup_miss_dirty", "log", "log_table_ge2",
    "invalid_type", "invalid_table", "missing_key", "missing_key_after_write_back")
