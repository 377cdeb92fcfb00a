"""The reference's eBPF store server (store/ebpf), for tests of the engine's DINT_CFG_STORE_EBPF_* option.

Two independent statements of it:

* run_ref_store_ebpf(): the reference's own XDP / TC programs and kvs.h, compiled unmodified by oracle/store_ebpf.mk
  into oracle/_ref/store_ebpf_{wb_bloom,wb,wt} and driven one request at a time (oracle/store_ebpf_replay.c).  Its
  sizes are the reference's (9,000,000 buckets).
* StoreEbpfModel: a plain restatement in Python with a run-time bucket count, so that small engines can be checked
  too.  Pinned to the compiled programs by tests/golden/store_ebpf/*.npz and, where oracle/_ref exists, by random traces.
"""
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
VARIANTS = ("wb_bloom", "wb", "wt")
MSG = 53
CACHE_ENTRY = 232           # struct cache_entry, store/ebpf/utils.h:58-66
TABLE_REC = np.dtype([("found", "<u4"), ("ver", "<u4"), ("val", "u1", (40,))])
READ, SET, INSERT, GRANT_READ, SET_ACK, NOT_EXIST, INSERT_ACK = 0, 1, 2, 3, 5, 7, 8
REF_BUCKETS = 9000000       # KVS_HASH_SIZE, store/ebpf/utils.h:13

M64 = (1 << 64) - 1
_FH_M = 0x880355f21e6d1965


def _mix(h):
    h ^= h >> 23
    h = (h * 0x2127599bf4325c37) & M64
    return h ^ (h >> 47)


def fasthash64(key):
    """fasthash64(&key, 8, 0xdeadbeef), store/ebpf/utils.h:129-159"""
    h = 0xdeadbeef ^ ((8 * _FH_M) & M64)
    h ^= _mix(key)
    h = (h * _FH_M) & M64
    return _mix(h)


def fasthash64_np(keys):
    """vectorised fasthash64 of a uint64 array"""
    with np.errstate(over="ignore"):
        k = np.asarray(keys, dtype=np.uint64)

        def mix(h):
            h = h ^ (h >> np.uint64(23))
            h = h * np.uint64(0x2127599bf4325c37)
            return h ^ (h >> np.uint64(47))
        h = np.uint64(0xdeadbeef ^ ((8 * _FH_M) & M64)) ^ mix(k)
        h = h * np.uint64(_FH_M)
        return mix(h)


def ref_available():
    return all(os.path.exists(os.path.join(REF_DIR, f"store_ebpf_{v}")) for v in VARIANTS)


def run_ref_store_ebpf(variant, req, keys=(), populate=0):
    """Replies of the compiled reference server to `req` (n*53 uint8), after serving the eBPF client's population of
    `populate` subscribers.  Returns (replies uint8 [n*53], sets uint8 [len(keys), 232], table TABLE_REC [len(keys)],
    kv_count): the cache_entry of each key's bucket and kvs_get of each key, after the trace."""
    binary = os.path.join(REF_DIR, f"store_ebpf_{variant}")
    req = np.ascontiguousarray(req, dtype=np.uint8).reshape(-1)
    keys = np.ascontiguousarray(keys, dtype=np.uint64).reshape(-1)
    with tempfile.TemporaryDirectory() as d:
        p = {n: os.path.join(d, n) for n in ("req", "resp", "keys", "sets", "table")}
        req.tofile(p["req"])
        keys.tofile(p["keys"])
        cmd = [binary, p["req"], p["resp"], p["keys"], p["sets"], p["table"]]
        if populate:
            cmd += ["--populate", str(populate)]
        out = subprocess.run(cmd, check=True, capture_output=True, text=True).stdout
        resp = np.fromfile(p["resp"], dtype=np.uint8)
        sets = np.fromfile(p["sets"], dtype=np.uint8).reshape(-1, CACHE_ENTRY)
        table = np.fromfile(p["table"], dtype=TABLE_REC)
    count = int(out.split()[1])
    return resp, sets, table, count


def population(subscribers):
    """(key, 40-byte value) pairs of the eBPF client's kInsert stream, in the order one server sees them
    (store/caladan/client_ebpf.cc:137-180, 600 populate threads in thread order, fastrand restarting per thread)."""
    threads, out = 600, []
    sl = subscribers // threads
    for w in range(threads):
        seed = 0xdeadbeef
        lo, hi = w * sl, (subscribers if w == threads - 1 else (w + 1) * sl)
        for s in range(lo, hi):
            for sf in range(1, 5):
                for st in (0, 8, 16):
                    seed = (seed * 1103515245 + 12345) & M64
                    val = bytearray(40)
                    val[0] = ((seed >> 32) & 0xffffffff) % 24 + 1
                    val[1] = 0x5a
                    out.append((s | (sf << 32) | (st << 40), bytes(val)))
    return out


class StoreEbpfModel:
    """One server thread of store/ebpf: XDP (store*_kern.c), the user-space dispatch (store*_user.c:127-165) over the
    chained table of store/ebpf/kvs.h, and TC egress -- with `buckets` in place of KVS_HASH_SIZE."""

    def __init__(self, variant, buckets=REF_BUCKETS):
        assert variant in VARIANTS
        self.variant, self.buckets = variant, buckets
        self.wt, self.bloom_on = variant == "wt", variant == "wb_bloom"
        self.cache = {}     # bucket -> dict(key=[4], val=[4], ver=[4], valid=[4], dirty=[4], bloom=int)
        self.table = {}     # bucket -> list of kvs_entry (head first): [keys[4], vals[4], vers[4], valid[4]]
        self.stats = dict(hits=0, bloom_negatives=0, table=0, write_backs=0, installs=0)

    # ---- store/ebpf/kvs.h --------------------------------------------------------------------------------------
    def _chain(self, key):
        return self.table.setdefault(fasthash64(key) % self.buckets, [])

    def kvs_get(self, key):
        for e in self._chain(key):
            for i in range(4):
                if e[0][i] == key and e[3][i]:
                    return e[1][i], e[2][i]
        return None

    def kvs_set(self, key, val):
        for e in self._chain(key):
            for i in range(4):
                if e[0][i] == key and e[3][i]:
                    e[1][i] = val
                    e[2][i] = (e[2][i] + 1) & 0xffffffff
                    return e[2][i]
        return 0

    def kvs_insert(self, key, val):
        ch = self._chain(key)
        for e in ch:
            for i in range(4):
                if not e[3][i]:
                    e[0][i], e[1][i], e[2][i], e[3][i] = key, val, 0, 1
                    return
        ch.insert(0, [[key, 0, 0, 0], [val, bytes(40), bytes(40), bytes(40)], [0, 0, 0, 0], [1, 0, 0, 0]])

    def kvs_set_evict(self, key, val, ver):
        for e in self._chain(key):
            for i in range(4):
                if e[0][i] == key and e[3][i]:
                    e[1][i], e[2][i] = val, ver
                    return
        self.kvs_insert(key, val)

    def kv_count(self):
        return sum(sum(e[3]) for ch in self.table.values() for e in ch)

    # ---- the cache tier -----------------------------------------------------------------------------------------
    def _set(self, b):
        s = self.cache.get(b)
        if s is None:
            s = self.cache[b] = dict(key=[0] * 4, val=[bytes(40)] * 4, ver=[0] * 4, valid=[0] * 4, dirty=[0] * 4, bloom=0)
        return s

    def _victim(self, s):
        for i in range(4):
            if not s["valid"][i]:
                return i
        if not self.wt:
            for i in range(4):
                if not s["dirty"][i]:
                    return i
        return 0

    def _write_back(self, s, v):
        self.stats["write_backs"] += 1
        return s["key"][v], s["val"][v], s["ver"][v]

    def request(self, rec):
        """rec: 53 bytes; returns the 53-byte reply"""
        r = bytearray(rec)
        t = r[0]
        key = int.from_bytes(r[1:9], "little")
        val = bytes(r[9:49])
        ver = int.from_bytes(r[49:53], "little")
        if t > 2:
            r[0] = 0xFF
            return bytes(r)
        h = fasthash64(key)
        s = self._set(h % self.buckets)
        bit = 1 << (h >> 58)
        hit = next((i for i in range(4) if s["valid"][i] and s["key"][i] == key), -1)
        v = self._victim(s)
        evict = not self.wt and s["valid"][v] and s["dirty"][v]

        def install(i, k, vv, ve):
            s["key"][i], s["val"][i], s["ver"][i] = k, vv, ve
            self.stats["installs"] += 1

        if t == INSERT:
            if self.wt:
                free = next((i for i in range(4) if not s["valid"][i]), -1)
                if free >= 0:
                    install(free, key, val, ver)
                    s["valid"][free], s["dirty"][free] = 1, 0
                self.kvs_insert(key, val)
                self.stats["table"] += 1
            else:
                if self.bloom_on:
                    s["bloom"] |= bit
                if evict:
                    old = self._write_back(s, v)
                    install(v, key, val, 0)
                    s["dirty"][v] = 0
                    self.kvs_insert(key, val)
                    self.kvs_set_evict(*old)
                    self.stats["table"] += 1
                else:
                    install(v, key, val, 0)
                    s["valid"][v], s["dirty"][v] = 1, 1
            r[0] = INSERT_ACK
            return bytes(r)
        if hit >= 0 and (t == READ or not self.wt):
            self.stats["hits"] += 1
            if t == READ:
                r[9:49] = s["val"][hit]
                r[49:53] = s["ver"][hit].to_bytes(4, "little")
                r[0] = GRANT_READ
            else:
                s["val"][hit] = val
                s["ver"][hit] = (s["ver"][hit] + 1) & 0xffffffff
                s["dirty"][hit] = 1
                r[0] = SET_ACK
            if self.bloom_on:
                s["bloom"] |= bit
            return bytes(r)
        if self.bloom_on and not s["bloom"] & bit:
            self.stats["bloom_negatives"] += 1
            r[0] = NOT_EXIST
            return bytes(r)
        self.stats["table"] += 1
        if evict:
            self.kvs_set_evict(*self._write_back(s, v))
        if t == READ:
            got = self.kvs_get(key)
            if got is not None:
                r[9:49] = got[0]
                r[49:53] = got[1].to_bytes(4, "little")
                r[0] = GRANT_READ
                install(v, key, got[0], got[1])
                s["valid"][v] = 1
                if not self.wt:
                    s["dirty"][v] = 0
                if self.bloom_on:
                    s["bloom"] |= bit
            else:
                if not self.wt:
                    r[49:53] = (1 if evict else 0).to_bytes(4, "little")
                    s["dirty"][v] = 0
                r[0] = NOT_EXIST
            return bytes(r)
        if self.wt and hit >= 0:
            s["valid"][hit] = 0
        nv = self.kvs_set(key, val)
        r[49:53] = nv.to_bytes(4, "little")
        r[0] = SET_ACK if nv else NOT_EXIST
        if not self.wt:
            if nv:
                install(v, key, val, nv)
                s["valid"][v] = 1
                if self.bloom_on:
                    s["bloom"] |= bit
            s["dirty"][v] = 0
        return bytes(r)

    def process(self, req):
        raw = np.ascontiguousarray(req, dtype=np.uint8).reshape(-1)
        out = bytearray(raw.size)
        for i in range(raw.size // MSG):
            out[i * MSG:(i + 1) * MSG] = self.request(raw[i * MSG:(i + 1) * MSG].tobytes())
        return np.frombuffer(bytes(out), dtype=np.uint8)

    def populate(self, subscribers):
        for key, val in population(subscribers):
            self.request(bytes([INSERT]) + key.to_bytes(8, "little") + val + bytes(4))

    def cache_entry(self, bucket):
        """struct cache_entry of `bucket` (232 uint8, lock = 0)"""
        s = self.cache.get(bucket)
        out = bytearray(CACHE_ENTRY)
        if s is not None:
            for i in range(4):
                out[8 * i:8 * i + 8] = s["key"][i].to_bytes(8, "little")
                out[32 + 40 * i:72 + 40 * i] = s["val"][i]
                out[192 + 4 * i:196 + 4 * i] = s["ver"][i].to_bytes(4, "little")
                out[208 + i], out[212 + i] = s["valid"][i], s["dirty"][i]
            out[216:224] = s["bloom"].to_bytes(8, "little")
        return np.frombuffer(bytes(out), dtype=np.uint8)

    def state(self, keys):
        """(sets [len(keys), 232], table TABLE_REC [len(keys)]) as run_ref_store_ebpf dumps them"""
        sets = np.stack([self.cache_entry(fasthash64(int(k)) % self.buckets) for k in keys]) if len(keys) else \
            np.zeros((0, CACHE_ENTRY), np.uint8)
        table = np.zeros(len(keys), dtype=TABLE_REC)
        for i, k in enumerate(keys):
            got = self.kvs_get(int(k))
            if got is not None:
                table[i]["found"], table[i]["ver"] = 1, got[1]
                table[i]["val"] = np.frombuffer(got[0], dtype=np.uint8)
        return sets, table


def make_req(types, keys, vals=None, vers=None):
    """n packed 53-byte store messages"""
    n = len(types)
    rec = np.zeros((n, MSG), dtype=np.uint8)
    rec[:, 0] = np.asarray(types, dtype=np.uint8)
    rec[:, 1:9] = np.asarray(keys, dtype=np.uint64).reshape(-1, 1).view(np.uint8)
    if vals is not None:
        rec[:, 9:49] = np.asarray(vals, dtype=np.uint8).reshape(n, 40)
    if vers is not None:
        rec[:, 49:53] = np.asarray(vers, dtype=np.uint32).reshape(-1, 1).view(np.uint8)
    return rec.reshape(-1)


def colliding_keys(buckets, per_bucket, n_buckets, seed=0, key_space=1 << 40):
    """n_buckets groups of `per_bucket` distinct keys that share one bucket (fasthash64 % buckets)"""
    rng = np.random.default_rng(seed)
    groups = {}
    while True:
        k = np.unique(rng.integers(0, key_space, size=1 << 22, dtype=np.uint64))
        b = fasthash64_np(k) % np.uint64(buckets)
        order = np.argsort(b, kind="stable")
        bs, ks = b[order], k[order]
        starts = np.flatnonzero(np.r_[True, bs[1:] != bs[:-1]])
        counts = np.diff(np.r_[starts, bs.size])
        for st, c in zip(starts[counts >= per_bucket], counts[counts >= per_bucket]):
            bk = int(bs[st])
            if bk not in groups:
                groups[bk] = ks[st:st + per_bucket].copy()
                if len(groups) == n_buckets:
                    return list(groups.values())
