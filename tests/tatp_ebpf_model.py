"""The reference's eBPF TATP shard server (tatp/ebpf), for tests of the engine's DINT_CFG_TATP_EBPF option.

Two independent statements of it:

* run_ref_tatp_ebpf(): the reference's own XDP / TC programs (shard_kern.c, or lock_kern.c with holder keys) and kvs.h,
  compiled unmodified by oracle/tatp_ebpf.mk into oracle/_ref/tatp_ebpf_{shard,lock} and driven one request at a time
  (oracle/tatp_ebpf_replay.c).  Its sizes are the reference's (S = 7,000,000).
* TatpEbpfModel: a plain restatement in Python with run-time bucket counts, so that small engines can be checked too.
  Pinned to the compiled programs by tests/golden/tatp_ebpf/*.npz and, where oracle/_ref exists, by random traces.
"""
import collections
import os
import subprocess
import tempfile

import numpy as np

from store_ebpf_model import M64, _FH_M, _mix, fasthash64, fasthash64_np  # noqa: F401  (re-exported)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
VARIANTS = ("shard", "lock")
MSG = 55
CACHE_ENTRY = 232           # struct cache_entry, tatp/ebpf/utils.h:103-111
CHAIN_REC = np.dtype([("key", "<u8", (4,)), ("ver", "<u4", (4,)), ("valid", "u1", (4,)), ("val", "u1", (4, 40))])
CHAIN_DUMP = np.dtype([("n", "<u4"), ("rec", CHAIN_REC, (8,))])
FIND_REC = np.dtype([("found", "<u4"), ("ver", "<u4"), ("val", "u1", (40,))])
LOCK_REC = np.dtype([("lock", "<u8"), ("holder", "<u8")])
LOG_ENTRY = 64
REF_S = 7000000

(READ, ACQUIRE_LOCK, ABORT, GRANT_READ, NOT_EXIST, GRANT_LOCK, REJECT_LOCK, ABORT_ACK) = 0, 1, 2, 4, 6, 7, 8, 9
COMMIT_PRIM, COMMIT_BCK, COMMIT_LOG, COMMIT_PRIM_ACK, COMMIT_BCK_ACK, COMMIT_LOG_ACK = 12, 13, 14, 15, 16, 17
INSERT_PRIM, INSERT_BCK, INSERT_PRIM_ACK, INSERT_BCK_ACK = 18, 19, 20, 21
DELETE_PRIM, DELETE_BCK, DELETE_LOG, DELETE_PRIM_ACK, DELETE_BCK_ACK, DELETE_LOG_ACK = 22, 23, 24, 25, 26, 27
REJECT_LOCK_SAME_KEY = 28
STATS = ("hits", "bloom_negatives", "table", "write_backs", "installs", "allocated", "reused", "freed", "failed")


def hash_sizes(S):
    """bucket count of each table (tatp/ebpf/utils.h:17-21: call_forwarding has S*15/4/4, not the UDP server's S*45/8/4)"""
    return [S * 3 // 2 // 4, S * 3 // 2 // 4, S * 15 // 4 // 4, S * 15 // 4 // 4, S * 15 // 4 // 4]


def fasthash64_key_array(keys):
    """fasthash64(&head->key, 32, 0xdeadbeef) of a chain entry's 4-key array (shard_user.c:98)"""
    h = 0xdeadbeef ^ ((32 * _FH_M) & M64)
    for k in keys:
        h ^= _mix(k)
        h = (h * _FH_M) & M64
    return _mix(h)


def ref_available():
    return all(os.path.exists(os.path.join(REF_DIR, f"tatp_ebpf_{v}")) for v in VARIANTS)


def run_ref_tatp_ebpf(variant, req, keys=(), tables=(), populate=0, shard=0):
    """Replies of the compiled reference server to `req` (n*55 uint8), after serving the eBPF client's population of
    `populate` subscribers as shard `shard` of three.  Returns (replies [n*55], sets [k, 232], chains CHAIN_DUMP [k],
    finds FIND_REC [k], locks LOCK_REC [k], log [m, 64]) for the (key, table) pairs, after the trace."""
    binary = os.path.join(REF_DIR, f"tatp_ebpf_{variant}")
    req = np.ascontiguousarray(req, dtype=np.uint8).reshape(-1)
    kt = np.zeros((len(keys), 2), dtype=np.uint64)
    kt[:, 0] = np.asarray(keys, dtype=np.uint64)
    kt[:, 1] = np.asarray(tables, dtype=np.uint64)
    with tempfile.TemporaryDirectory() as d:
        p = {n: os.path.join(d, n) for n in ("req", "resp", "keys", "sets", "chains", "finds", "locks", "log")}
        req.tofile(p["req"])
        kt.tofile(p["keys"])
        cmd = [binary, p["req"], p["resp"], "--shard", str(shard),
               "--dump", p["keys"], p["sets"], p["chains"], p["finds"], p["locks"], p["log"]]
        if populate:
            cmd += ["--populate", str(populate)]
        subprocess.run(cmd, check=True, capture_output=True)
        resp = np.fromfile(p["resp"], dtype=np.uint8)
        sets = np.fromfile(p["sets"], dtype=np.uint8).reshape(-1, CACHE_ENTRY)
        chains = np.fromfile(p["chains"], dtype=CHAIN_DUMP)
        finds = np.fromfile(p["finds"], dtype=FIND_REC)
        locks = np.fromfile(p["locks"], dtype=LOCK_REC)
        log = np.fromfile(p["log"], dtype=np.uint8).reshape(-1, LOG_ENTRY)
    return resp, sets, chains, finds, locks, log


def _fastrand(seed):
    seed = (seed * 1103515245 + 12345) & M64
    return seed, (seed >> 32) & 0xffffffff


def _select_types(seed):
    seed, r = _fastrand(seed)
    n, used, out = r % 4 + 1, set(), []
    while len(out) < n:
        seed, r = _fastrand(seed)
        v = r % 4 + 1
        if v not in used:
            used.add(v)
            out.append(v)
    return seed, out


def _sub_nbr(s):
    r = 0
    for g in range(3):
        i = s % 1000
        s //= 1000
        r |= (((i // 100) % 10) << 8 | ((i // 10) % 10) << 4 | (i % 10)) << (12 * g)
    return r


def population(subscribers):
    """(table, key, 40-byte value) rows of the eBPF client's population stream, in the order one server sees them
    (tatp/caladan/client_ebpf_shard.cc:96-339: 600 populate threads in thread order, fastrand restarting per thread and
    running on through the four tables of the thread's slice)."""
    threads, out = 600, []
    sl = subscribers // threads
    for w in range(threads):
        seed = 0xdeadbeef
        lo, hi = w * sl, (subscribers if w == threads - 1 else (w + 1) * sl)
        for s in range(lo, hi):
            v = bytearray(40)
            v[0:8] = _sub_nbr(s).to_bytes(8, "little")
            for i in range(5):
                seed, r = _fastrand(seed)
                v[15 + i] = r & 0xff
            for i in range(10):
                seed, r = _fastrand(seed)
                v[20 + i] = r & 0xff
            seed, r = _fastrand(seed)
            v[30:32] = (r & 0xffff).to_bytes(2, "little")
            seed, r = _fastrand(seed)
            v[32:36] = (97).to_bytes(4, "little")
            v[36:40] = r.to_bytes(4, "little")
            out.append((0, s, bytes(v)))
        for s in range(lo, hi):
            v = bytearray(40)
            v[0:4] = s.to_bytes(4, "little")
            v[4] = 98
            out.append((1, _sub_nbr(s), bytes(v)))
        for s in range(lo, hi):
            seed, ty = _select_types(seed)
            for t in ty:
                v = bytearray(40)
                v[0] = 99
                out.append((2, s | (t << 32), bytes(v)))
        for s in range(lo, hi):
            seed, ty = _select_types(seed)
            for t in ty:
                v = bytearray(40)
                v[3] = 100
                seed, r = _fastrand(seed)
                v[0] = 1 if r % 100 < 85 else 0
                out.append((3, s | (t << 32), bytes(v)))
                for st in (0, 8, 16):
                    seed, r = _fastrand(seed)
                    if r % 2 == 0:
                        continue
                    v = bytearray(40)
                    v[1] = 101
                    seed, r = _fastrand(seed)
                    v[0] = r % 24 + 1
                    out.append((4, s | (t << 32) | (st << 40), bytes(v)))
    return out


class TatpEbpfModel:
    """One server thread of tatp/ebpf: XDP (shard_kern.c / lock_kern.c), the user-space dispatch (shard_user.c:171-247)
    over the chained tables of tatp/ebpf/kvs.h, and TC egress -- with hash_sizes(S) buckets."""

    def __init__(self, holder_keys=False, S=REF_S, log_ring=1000000):
        self.holder_keys = holder_keys
        self.H = hash_sizes(S)
        self.cache = [dict() for _ in range(5)]     # bucket -> dict(key, val, ver, valid, dirty: [4]; bloom)
        self.table = [dict() for _ in range(5)]     # bucket -> chain, head first: [keys[4], vals[4], vers[4], valid[4]]
        self.locks = [dict() for _ in range(5)]     # lock slot -> [lock_bit, holder]
        self.log_ring = log_ring
        self.log = {}                               # ring index -> 64-byte entry
        self.log_cnt = 0
        self.stats = dict.fromkeys(STATS, 0)
        self.freed = collections.Counter()      # (table, bucket) -> entries on the bucket's free list
        self.paths = collections.Counter()      # which path of the server each request took (coverage of a trace)

    # ---- tatp/ebpf/kvs.h ------------------------------------------------------------------------------------
    def _chain(self, t, key):
        return self.table[t].setdefault(fasthash64(key) % self.H[t], [])

    def kvs_get(self, t, key):
        for e in self._chain(t, key):
            for i in range(4):
                if e[0][i] == key and e[3][i]:
                    return e[1][i], e[2][i]
        return None

    def kvs_insert(self, t, key, val):
        ch = self._chain(t, key)
        if self.kvs_get(t, key) is not None:
            self.paths["insert_duplicate"] += 1
        for e in ch:
            for i in range(4):
                if not e[3][i]:
                    e[0][i], e[1][i], e[2][i], e[3][i] = key, val, 0, 1
                    return
        b = fasthash64(key) % self.H[t]
        if self.freed[t, b]:
            self.freed[t, b] -= 1
            self.stats["reused"] += 1
        else:
            self.stats["allocated"] += 1
        ch.insert(0, [[key, 0, 0, 0], [val, bytes(40), bytes(40), bytes(40)], [0, 0, 0, 0], [1, 0, 0, 0]])

    def kvs_set(self, t, key, val, ver):
        for e in self._chain(t, key):
            for i in range(4):
                if e[0][i] == key and e[3][i]:
                    e[1][i] = val
                    e[2][i] = ver if ver != 0 else (e[2][i] + 1) & 0xffffffff
                    return e[2][i]
        self.kvs_insert(t, key, val)
        return 0

    def kvs_delete(self, t, key):
        ch = self._chain(t, key)
        for n, e in enumerate(ch):
            for i in range(4):
                if e[0][i] == key and e[3][i]:
                    e[3][i] = 0
                    if not any(e[3]):
                        del ch[n]
                        self.freed[t, fasthash64(key) % self.H[t]] += 1
                        self.stats["freed"] += 1
                    self.paths["delete_freed" if not any(e[3]) else "delete_kept"] += 1
                    return

    def bloom_of_chain(self, t, b):
        bf = 0
        for e in self.table[t].get(b, []):
            bf |= 1 << (fasthash64_key_array(e[0]) >> 58)
        return bf

    # ---- the cache tier and the locks -------------------------------------------------------------------------
    def _set(self, t, b):
        s = self.cache[t].get(b)
        if s is None:
            s = self.cache[t][b] = dict(key=[0] * 4, val=[bytes(40)] * 4, ver=[0] * 4, valid=[0] * 4, dirty=[0] * 4,
                                        bloom=0)
        return s

    def _lock(self, t, h):
        return self.locks[t].setdefault(h % (4 * self.H[t]), [0, 0])

    @staticmethod
    def _victim(s):
        for i in range(4):
            if not s["valid"][i]:
                return i
        for i in range(4):
            if not s["dirty"][i]:
                return i
        return 0

    def request(self, rec):
        """rec: 55 bytes; returns the first 55 bytes of the reply"""
        r = bytearray(rec)
        ty, t = r[1], r[2]
        key = int.from_bytes(r[3:11], "little")
        val = bytes(r[11:51])
        st = self.stats
        if ty in (COMMIT_LOG, DELETE_LOG):                     # shard_kern.c:914-936
            e = bytearray(self.log.get(self.log_cnt % self.log_ring, bytes(LOG_ENTRY)))
            e[0], e[1] = int(ty == DELETE_LOG), t
            e[8:16] = r[3:11]
            if ty == COMMIT_LOG:
                e[16:56] = val
            e[56:60] = r[51:55]
            self.log[self.log_cnt % self.log_ring] = bytes(e)
            self.log_cnt += 1
            self.paths["log_commit" if ty == COMMIT_LOG else "log_delete"] += 1
            r[1] = COMMIT_LOG_ACK if ty == COMMIT_LOG else DELETE_LOG_ACK
            return bytes(r)
        if t >= 5 or ty not in (READ, ACQUIRE_LOCK, ABORT, COMMIT_PRIM, COMMIT_BCK, INSERT_PRIM, INSERT_BCK,
                                DELETE_PRIM, DELETE_BCK):
            self.paths["invalid"] += 1
            r[1] = 0xFF
            return bytes(r)
        h = fasthash64(key)
        if ty == ACQUIRE_LOCK:                                 # :251-296 (lock_kern.c:289-298)
            lk = self._lock(t, h)
            self.paths["acquire_" + ("grant" if lk[0] == 0 else "same_key" if lk[1] == key else "reject")] += 1
            if lk[0] == 0:
                lk[0] = 1
                if self.holder_keys:
                    lk[1] = key
                r[1] = GRANT_LOCK
            else:
                r[1] = REJECT_LOCK_SAME_KEY if self.holder_keys and lk[1] == key else REJECT_LOCK
            return bytes(r)
        if ty == ABORT:                                        # :298-336
            self._lock(t, h)[0] = 0
            self.paths["abort"] += 1
            r[1] = ABORT_ACK
            return bytes(r)
        prim = ty in (COMMIT_PRIM, INSERT_PRIM, DELETE_PRIM)
        b = h % self.H[t]
        s = self._set(t, b)
        bit = 1 << (h >> 58)
        hit = next((i for i in range(4) if s["valid"][i] and s["key"][i] == key), -1)
        v = self._victim(s)
        evict = bool(s["valid"][v] and s["dirty"][v])
        old = (s["key"][v], s["val"][v], s["ver"][v])

        def unlock():
            if prim:
                self._lock(t, h)[0] = 0

        if ty == READ:                                         # :140-249, TC :964-1045
            if hit >= 0:
                st["hits"] += 1
                self.paths["read_hit"] += 1
                r[11:51] = s["val"][hit]
                r[51:55] = s["ver"][hit].to_bytes(4, "little")
                s["bloom"] |= bit
                r[1] = GRANT_READ
                return bytes(r)
            if not s["bloom"] & bit:
                st["bloom_negatives"] += 1
                self.paths["read_bloom_neg" + ("_false" if self.kvs_get(t, key) is not None else "")] += 1
                r[1] = NOT_EXIST
                return bytes(r)
            st["table"] += 1
            if evict:
                st["write_backs"] += 1
                self.kvs_set(t, *old)
            got = self.kvs_get(t, key)
            self.paths["read_table_%s_%s" % ("hit" if got else "miss", "dirty" if evict else "clean")] += 1
            if got is None:
                r[51:55] = int(evict).to_bytes(4, "little")
                r[1] = NOT_EXIST
                return bytes(r)
            st["installs"] += 1
            r[11:51], r[51:55] = got[0], got[1].to_bytes(4, "little")
            s["key"][v], s["val"][v], s["ver"][v], s["dirty"][v], s["valid"][v] = key, got[0], got[1], 0, 1
            s["bloom"] |= bit
            r[1] = GRANT_READ
            return bytes(r)
        if ty in (COMMIT_PRIM, COMMIT_BCK):                    # :338-474, :659-761, TC :1047-1119, :1193-1232
            ack = COMMIT_PRIM_ACK if prim else COMMIT_BCK_ACK
            self.paths["commit_%s_%s" % ("prim" if prim else "bck", "hit" if hit >= 0 else "miss")] += 1
            if hit >= 0:
                st["hits"] += 1
                unlock()
                s["val"][hit] = val
                s["ver"][hit] = (s["ver"][hit] + 1) & 0xffffffff
                s["dirty"][hit] = 1
                r[1] = ack
                return bytes(r)
            st["table"] += 1
            st["installs"] += 1
            s["key"][v], s["val"][v], s["dirty"][v] = key, val, 0
            if evict:
                st["write_backs"] += 1
                self.paths["commit_write_back_ver%s" % ("0" if old[2] == 0 else "n")] += 1
                self.kvs_set(t, *old)
            nv = self.kvs_set(t, key, val, 0)
            unlock()
            s["ver"][v], s["valid"][v] = nv, 1
            r[51:55] = nv.to_bytes(4, "little")
            r[1] = ack
            return bytes(r)
        if ty in (INSERT_PRIM, INSERT_BCK):                    # :476-608, :763-863, TC :1121-1191, :1234-1271
            s["bloom"] |= bit
            st["installs"] += 1
            self.paths["insert_evict" if evict else "insert_cache_only"] += 1
            s["key"][v], s["val"][v], s["ver"][v] = key, val, 0
            if evict:
                st["table"] += 1
                st["write_backs"] += 1
                s["dirty"][v] = 0
                self.kvs_insert(t, key, val)
                self.kvs_set(t, *old)
            else:
                s["valid"][v], s["dirty"][v] = 1, 1
            unlock()
            r[1] = INSERT_PRIM_ACK if prim else INSERT_BCK_ACK
            return bytes(r)
        # DELETE_PRIM / DELETE_BCK: :610-657, :865-912, shard_user.c:207-219,235-246, TC :1121-1191, :1234-1271
        st["table"] += 1
        self.paths["delete"] += 1
        if hit >= 0:
            s["valid"][hit] = 0
        self.kvs_delete(t, key)
        bf = self.bloom_of_chain(t, b)
        s["bloom"] = bf
        unlock()
        r[11:19] = bf.to_bytes(8, "little")
        r[1] = DELETE_PRIM_ACK if prim else DELETE_BCK_ACK
        return bytes(r)

    def process(self, req):
        raw = np.ascontiguousarray(req, dtype=np.uint8).reshape(-1)
        out = bytearray(raw.size)
        for i in range(raw.size // MSG):
            out[i * MSG:(i + 1) * MSG] = self.request(raw[i * MSG:(i + 1) * MSG].tobytes())
        return np.frombuffer(bytes(out), dtype=np.uint8)

    def populate(self, subscribers, shard=0, G=3):
        """the population stream as shard `shard` of G sees it: every row when G <= 3 (kInsertPrim where key % 3 ==
        shard), else only the rows whose primary key % G is shard, shard - 1 or shard - 2 (mod G)"""
        Ge = G if G > 3 else 3
        for t, key, val in population(subscribers):
            if G > 3 and (shard - key % G) % G > 2:
                continue
            ty = INSERT_PRIM if key % Ge == shard else INSERT_BCK
            self.request(bytes([0, ty, t]) + key.to_bytes(8, "little") + val + bytes(4))

    # ---- state, in the compiled oracle's dump formats -----------------------------------------------------------
    def cache_entry(self, t, b):
        """struct cache_entry of bucket b of table t (232 uint8, lock = 0)"""
        s = self.cache[t].get(b)
        out = bytearray(CACHE_ENTRY)
        if s is not None:
            for i in range(4):
                out[8 * i:8 * i + 8] = s["key"][i].to_bytes(8, "little")
                out[32 + 40 * i:72 + 40 * i] = s["val"][i]
                out[192 + 4 * i:196 + 4 * i] = s["ver"][i].to_bytes(4, "little")
                out[208 + i], out[212 + i] = s["valid"][i], s["dirty"][i]
            out[216:224] = s["bloom"].to_bytes(8, "little")
        return np.frombuffer(bytes(out), dtype=np.uint8)

    def chain(self, t, b):
        """the chain of bucket b of table t, head first, as CHAIN_REC records"""
        ch = self.table[t].get(b, [])
        out = np.zeros(len(ch), dtype=CHAIN_REC)
        for n, e in enumerate(ch):
            out[n]["key"], out[n]["ver"], out[n]["valid"] = e[0], e[2], e[3]
            out[n]["val"] = np.frombuffer(b"".join(e[1]), dtype=np.uint8).reshape(4, 40)
        return out

    def state(self, keys, tables):
        """(sets, chains, finds, locks) as run_ref_tatp_ebpf dumps them"""
        n = len(keys)
        sets = np.zeros((n, CACHE_ENTRY), np.uint8)
        chains = np.zeros(n, dtype=CHAIN_DUMP)
        finds = np.zeros(n, dtype=FIND_REC)
        locks = np.zeros(n, dtype=LOCK_REC)
        for i, (k, t) in enumerate(zip(keys, tables)):
            k, t = int(k), int(t)
            h = fasthash64(k)
            b = h % self.H[t]
            sets[i] = self.cache_entry(t, b)
            ch = self.chain(t, b)
            chains[i]["n"] = len(ch)
            chains[i]["rec"][:len(ch)] = ch
            got = self.kvs_get(t, k)
            if got is not None:
                finds[i]["found"], finds[i]["ver"] = 1, got[1]
                finds[i]["val"] = np.frombuffer(got[0], dtype=np.uint8)
            lk = self.locks[t].get(h % (4 * self.H[t]), [0, 0])
            locks[i]["lock"], locks[i]["holder"] = lk
        return sets, chains, finds, locks

    def log_dump(self):
        """the first min(appends, ring) entries of the log ring, [m, 64] uint8"""
        m = min(self.log_cnt, self.log_ring)
        out = np.zeros((m, LOG_ENTRY), np.uint8)
        for i in range(m):
            out[i] = np.frombuffer(self.log[i], dtype=np.uint8)
        return out


def make_req(types, tables, keys, vals=None, vers=None, ords=None):
    """n packed 55-byte tatp messages"""
    n = len(types)
    rec = np.zeros((n, MSG), dtype=np.uint8)
    if ords is not None:
        rec[:, 0] = np.asarray(ords, dtype=np.uint8)
    rec[:, 1] = np.asarray(types, dtype=np.uint8)
    rec[:, 2] = np.asarray(tables, dtype=np.uint8)
    rec[:, 3:11] = np.asarray(keys, dtype=np.uint64).reshape(-1, 1).view(np.uint8)
    if vals is not None:
        rec[:, 11:51] = np.asarray(vals, dtype=np.uint8).reshape(n, 40)
    if vers is not None:
        rec[:, 51:55] = np.asarray(vers, dtype=np.uint32).reshape(-1, 1).view(np.uint8)
    return rec.reshape(-1)


def colliding_groups(S, per_bucket=8, n_buckets=3, seed=0):
    """per table: n_buckets groups of `per_bucket` distinct keys that share one bucket of hash_sizes(S)"""
    from store_ebpf_model import colliding_keys
    return [colliding_keys(H, per_bucket, n_buckets, seed=seed + t) for t, H in enumerate(hash_sizes(S))]


def random_trace(groups, n, seed=0):
    """n requests over the colliding key groups of every table: reads, locks, commits, inserts and deletes of both
    forms, log appends and a few requests the server refuses (unknown type, table >= 5)"""
    rng = np.random.default_rng(seed)
    types = np.array([READ, ACQUIRE_LOCK, ABORT, COMMIT_PRIM, COMMIT_BCK, INSERT_PRIM, INSERT_BCK, DELETE_PRIM,
                      DELETE_BCK, COMMIT_LOG, DELETE_LOG, 3])
    weights = np.array([30, 8, 5, 8, 8, 9, 9, 5, 5, 3, 2, 1], dtype=float)
    ty = rng.choice(types, size=n, p=weights / weights.sum())
    tb = rng.integers(0, 5, size=n)
    tb[rng.random(n) < 0.005] = 5
    keys = np.zeros(n, dtype=np.uint64)
    for i in range(n):
        g = groups[min(int(tb[i]), 4)]
        grp = g[rng.integers(0, len(g))]
        j = rng.integers(0, len(grp))
        keys[i] = grp[j]
        if j == len(grp) - 1 and ty[i] in (INSERT_PRIM, INSERT_BCK):   # the last key of a group is never inserted
            ty[i] = READ
    vals = rng.integers(0, 256, size=(n, 40), dtype=np.uint8)
    vers = rng.integers(0, 1 << 32, size=n, dtype=np.uint64).astype(np.uint32)
    vers[rng.random(n) < 0.3] = 0
    ords = rng.integers(0, 256, size=n, dtype=np.uint8)
    return make_req(ty, tb, keys, vals, vers, ords)


# every path of the server a golden trace must reach (TatpEbpfModel.paths)
REQUIRED_PATHS = (
    "read_hit", "read_bloom_neg", "read_bloom_neg_false", "read_table_hit_clean", "read_table_hit_dirty",
    "read_table_miss_clean", "read_table_miss_dirty", "commit_prim_hit", "commit_prim_miss", "commit_bck_hit",
    "commit_bck_miss", "commit_write_back_ver0", "commit_write_back_vern", "insert_cache_only", "insert_evict",
    "insert_duplicate", "delete", "delete_freed", "delete_kept", "acquire_grant", "acquire_reject",
    "abort", "log_commit", "log_delete", "invalid")
REQUIRED_PATHS_LOCK = REQUIRED_PATHS + ("acquire_same_key",)   # only a server that keeps holder keys tells it apart
