"""-m gpu: every route of the ordered replay, reached on purpose and proven reached.

Requests that conflict inside a chunk are listed by K2 and replayed in index order by one of three routes
(DESIGN.md section 3): the per-warp bucket replay (single pass, or bucket by bucket when a warp task holds more
than one shared-memory slice), or the radix-sort fallback of k_ordered when a bucket overflows (for lock_fasst a
segmented scan over 2048-entry sort tiles).  Uniform random traces reach some of these by luck.  Here the traces are
built so that each case takes a known route, and every case checks three things against one oracle fed the same
requests in the same order: bit-exact replies, bit-exact final state, and the engine's path counters.

The expected counters come from `Model`, a Python restatement of K1/K2's classification (flag nibbles, folded to
flags_mask) and of the route choice (bucket_of, the task size `gsz`, kBucketCap).  Each case also asserts on the
model's verdict that the route it was designed for is the one taken, so a wrong copy of the engine's constants
fails loudly instead of silently testing another route.
"""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
import trace_gen as T
from dint_b200 import engine as E, wire
from dint_b200.engine import Engine, DintError
from properties import fasthash64_u32, _mix

LOCK2PL, FASST, LOG, STORE, TATP, SMALLBANK = range(6)
KEYED = [LOCK2PL, FASST, STORE, TATP, SMALLBANK]
ALL_KINDS = KEYED + [LOG]
NAMES = wire.KIND_NAMES

RA, WA, WL = 1, 2, 4                # what a request touches in its group (engine.cuh C_RA / C_WA / C_WL)
BUCKET_CAP, BUCKET_FILL, SORT_TILE = 128, 64, 2048
HOST_MIN_SLICE, HOST_MAX_SLICE = 131072, 1 << 18
FOLD = 1 << 25                      # flag nibbles of the default 36 M-slot lock table

# KV-kind configurations small enough that the oracle populates in well under a second
KV_CFG = {STORE: dict(subs_sizing=20000, subs_populate=1000),
          TATP: dict(subs_sizing=20000, subs_populate=1000),
          SMALLBANK: dict(accts_sizing=20000, accts_populate=5000)}
ORACLE_KEYS = ("lock_slots", "log_ring", "subs_sizing", "subs_populate", "accts_sizing", "accts_populate")


def fasthash64_u64(x, seed=0xDEADBEEF):
    """Vectorised fasthash64(&x, 8, seed): one 8-byte block, no tail (the KV kinds' key hash)."""
    with np.errstate(over="ignore"):
        m = np.uint64(0x880355F21E6D1965)
        h = np.uint64(seed) ^ (np.uint64(8) * m)
        h = (h ^ _mix(np.asarray(x, dtype=np.uint64))) * m
        return _mix(h)


def bucket_of(g, log2p):
    """kernels.cuh bucket_of: multiplicative hash of the group id onto 2^log2p buckets."""
    g = np.asarray(g, dtype=np.uint64)
    if log2p == 0:
        return np.zeros(g.shape, dtype=np.int64)
    return (((g * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)) >> np.uint64(32 - log2p)).astype(np.int64)


def host_slices(n, max_slice):
    """The slices dint_submit cuts an n-request call into (each one is a chunk of its own)."""
    L = E.lib()
    L.dint_test_host_slices.restype = C.c_uint32
    L.dint_test_host_slices.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_int, C.POINTER(C.c_uint32), C.c_uint32]
    cap = 1 << 12
    buf = (C.c_uint32 * cap)()
    k = L.dint_test_host_slices(n, HOST_MIN_SLICE, max_slice, 1, buf, cap)
    assert k <= cap
    return [int(x) for x in buf[:k]]


class Geo:
    """Group space, flag folding, radix passes and bucket count of an engine with this configuration
    (engine.cu create_impl, kv.cuh kv_create_tables)."""

    def __init__(self, kind, **cfg):
        d = E.default_cfg(kind, **cfg)
        self.kind = kind
        self.chunk = ((d.chunk or (1 << 20)) + 127) // 128 * 128
        S, A = d.subs_sizing, d.accts_sizing
        if kind in (LOCK2PL, FASST):
            mods = [d.lock_slots]
        elif kind == STORE:
            mods = [S * 18 // 4]
        elif kind == TATP:
            mods = [4 * h for h in (S * 3 // 2 // 4, S * 3 // 2 // 4, S * 15 // 4 // 4, S * 15 // 4 // 4, S * 45 // 8 // 4)]
        elif kind == SMALLBANK:
            mods = [4 * (A * 3 // 2 // 4)] * 2
        else:
            mods = []
        self.mods = np.array(mods, dtype=np.uint64)
        self.base = np.concatenate([[0], np.cumsum(mods)[:-1]]).astype(np.int64) if mods else np.zeros(0, np.int64)
        groups = int(sum(mods))
        fl = 25
        while fl > 10 and (1 << (fl - 1)) >= groups * 2 + 2048:
            fl -= 1
        self.flags_mask = (1 << fl) - 1
        bits = 1
        while (1 << bits) < groups:
            bits += 1
        self.sort_passes = (bits + 7) // 8
        lg = 0
        while (BUCKET_FILL << lg) < self.chunk:
            lg += 1
        self.bucket_log2 = lg

    def group(self, table, key):
        """group id of (table, key); lock kinds: key = lock id"""
        if self.kind in (LOCK2PL, FASST):
            return (fasthash64_u32(np.asarray(key, dtype=np.uint64)) % self.mods[0]).astype(np.int64)
        tb = np.asarray(table, dtype=np.int64)
        return self.base[tb] + (fasthash64_u64(key) % self.mods[tb]).astype(np.int64)

    def slot(self, table, key):
        """the slot lock_state() takes: the group id minus its table's base"""
        g = self.group(table, key)
        return g - self.base[np.asarray(table, dtype=np.int64)] if self.kind in (TATP, SMALLBANK) else g


# what each request type touches (engine.cuh / kv.cuh type_info); -1 = a log append, no group
TATP_MASK = {0: RA, 1: WL, 2: WL, 12: WA | WL, 18: WA | WL, 22: WA | WL, 13: WA, 19: WA, 23: WA, 14: -1, 24: -1}
SB_MASK = {0: RA | WL, 1: RA | WL, 2: WL, 3: WL, 4: WA, 5: WA, 6: -1}


def classify(geo, raw):
    """(group id or -1, touch mask) of every request of a valid trace"""
    kind = geo.kind
    rec = wire.as_records(kind, raw)
    n = len(rec)
    if kind == LOG:
        return np.full(n, -1, np.int64), np.zeros(n, np.int64)
    if kind == LOCK2PL:
        return geo.group(0, rec["lid"]), np.full(n, WL, np.int64)
    if kind == FASST:
        t = rec["type"]
        return geo.group(0, rec["lid"]), np.select([t == 0, t == 3], [RA, WA | WL], WL).astype(np.int64)
    if kind == STORE:
        return geo.group(np.zeros(n, np.int64), rec["key"]), np.where(rec["type"] == 0, RA, WA).astype(np.int64)
    table = TATP_MASK if kind == TATP else SB_MASK
    lut = np.zeros(256, np.int64)
    for k, v in table.items():
        lut[k] = v
    mask = lut[rec["type"]]
    is_log = mask < 0
    tb = np.where(is_log, 0, rec["table"]).astype(np.int64)
    g = np.where(is_log, -1, geo.group(tb, rec["key"]))
    return g, np.where(is_log, 0, mask)


def model(geo, raw, chunks):
    """Expected path counters of one call cut into `chunks`, and per chunk the route it takes."""
    g, mask = classify(geo, raw)
    assert sum(chunks) == len(g)
    exp = dict(conflicted=0, ordered_fallbacks=0, bucket_split_tasks=0, writerless_chunks=0)
    routes = []
    P = 1 << geo.bucket_log2
    off = 0
    for n in chunks:
        gg, mm = g[off:off + n], mask[off:off + n]
        off += n
        act = (gg >= 0) & (mm != 0)
        if not (act & (mm != RA)).any():
            exp["writerless_chunks"] += 1
            routes.append(dict(route="writerless", nc=0))
            continue
        ga, m = gg[act], mm[act]
        _, inv = np.unique(ga & geo.flags_mask, return_inverse=True)
        has_r = np.bincount(inv, weights=(m & RA) != 0) > 0
        n_wa = np.bincount(inv, weights=(m & WA) != 0)
        n_wl = np.bincount(inv, weights=(m & WL) != 0)
        f_wa, w2, f_r = (n_wa >= 1)[inv], ((n_wa >= 2) | (n_wl >= 2))[inv], has_r[inv]
        listed = (((m & RA) != 0) & f_wa) | (((m & WA) != 0) & (f_r | w2)) | (((m & WL) != 0) & w2)
        lg = ga[listed]
        nc = len(lg)
        exp["conflicted"] += nc
        if nc == 0:
            routes.append(dict(route="solo", nc=0))
            continue
        cnt = np.bincount(bucket_of(lg, geo.bucket_log2), minlength=P)
        if cnt.max() > BUCKET_CAP:
            exp["ordered_fallbacks"] += 1
            routes.append(dict(route="radix", nc=nc))
            continue
        gsz = 1
        while gsz < 32 and nc * gsz * 2 <= 16 * P:
            gsz <<= 1
        tasks = np.concatenate([cnt, np.zeros(-P % gsz, np.int64)]).reshape(-1, gsz).sum(axis=1)
        split = int((tasks > BUCKET_CAP).sum())
        exp["bucket_split_tasks"] += split
        routes.append(dict(route="split" if split else "bucket", nc=nc, tasks=tasks[tasks > 0]))
    return exp, routes


def call_chunks(geo, n, path):
    if n == 0:
        return []
    if path == "host":
        return host_slices(n, min(HOST_MAX_SLICE, geo.chunk))
    return [min(geo.chunk, n - o) for o in range(0, n, geo.chunk)]


# ---------------------------------------------------------------- traces -----------------------------------------
def records(kind, table, key, ty, rng):
    n = len(ty)
    rec = np.zeros(n, dtype=wire.MSG_DTYPE[kind])
    ty = np.asarray(ty)
    if kind == LOCK2PL:
        rec["action"], rec["lid"], rec["type"] = ty >> 1, key, ty & 1
        return wire.as_bytes(rec)
    rec["type"] = ty
    rec["ver"] = rng.integers(0, 2**32, size=n, dtype=np.uint64).astype(np.uint32)
    if kind == FASST:
        rec["lid"] = key
        return wire.as_bytes(rec)
    rec["key"] = key
    rec["val"] = rng.integers(0, 256, size=rec["val"].shape)
    if kind in (TATP, SMALLBANK):
        rec["ord"] = rng.integers(0, 256, size=n)
        rec["table"] = table
    return wire.as_bytes(rec)


# request types: a read-only one (C_RA alone; None: the kind has none), one writer that is solo when alone in its
# group, the mix of a hot group and the two types forced into every hot group so that ALL its requests are listed
READ = {LOCK2PL: None, FASST: 0, STORE: 0, TATP: 0, SMALLBANK: None}
LONE_WRITER = {LOCK2PL: 1, FASST: 3, STORE: 1, TATP: 13, SMALLBANK: 0}
HOT_MIX = {LOCK2PL: [0, 1, 2, 3], FASST: [0, 1, 2, 3], STORE: [0, 1], TATP: [0, 1, 2, 12, 13], SMALLBANK: [0, 1, 2, 3, 4, 5]}
HOT_FORCED = {LOCK2PL: [0, 1], FASST: [3, 3], STORE: [1, 1], TATP: [12, 12], SMALLBANK: [0, 1]}
LOG_TYPE = {TATP: 14, SMALLBANK: 6}


def hot_types(kind, m, rng):
    """types of m >= 2 requests on one group such that every one of them is listed"""
    assert m >= 2
    t = rng.choice(HOT_MIX[kind], size=m)
    t[rng.choice(m, size=2, replace=False)] = HOT_FORCED[kind]
    return t


def cold_types(kind, m, rng, read_only=False):
    """types of m requests, each alone on its group: reads, and (unless read_only) some lone writers"""
    if READ[kind] is None:
        assert not read_only
        return np.full(m, LONE_WRITER[kind])
    t = np.full(m, READ[kind])
    if not read_only:
        t[rng.random(m) < 0.3] = LONE_WRITER[kind]
    return t


class Pool:
    """Keys that exist after populate (KV kinds) or lock ids, one per group, with their group ids."""

    def __init__(self, geo, ora, n_lids=1 << 20):
        kind = geo.kind
        if kind in (LOCK2PL, FASST):
            tb, key = np.zeros(n_lids, np.int64), np.arange(n_lids, dtype=np.uint64)
        elif kind == STORE:
            s = np.arange(ora.cfg.subs_populate, dtype=np.uint64)
            key = np.concatenate([T.store_key(s, sf, st) for sf in (1, 2, 3, 4) for st in (0, 8, 16)])
            tb = np.zeros(len(key), np.int64)
        elif kind == TATP:
            cands = [c for c in T.tatp_key_universe(ora.cfg.subs_populate) if ora.kv_get(c[0], c[1]) is not None]
            tb = np.array([c[0] for c in cands], np.int64)
            key = np.array([c[1] for c in cands], np.uint64)
        else:
            a = np.arange(ora.cfg.accts_populate, dtype=np.uint64)
            tb, key = np.repeat([0, 1], len(a)), np.tile(a, 2)
        g = geo.group(tb, key)
        _, first = np.unique(g, return_index=True)
        self.geo, self.tb, self.key, self.g = geo, tb[first], key[first], g[first]
        self.nib = self.g & geo.flags_mask
        self.bucket = bucket_of(self.g, geo.bucket_log2)

    def pick(self, m, rng, used, where=None):
        """m pool entries on distinct flag nibbles outside `used` (updated), optionally restricted to a bool mask"""
        idx = rng.permutation(len(self.g))
        if where is not None:
            idx = idx[where[idx]]
        idx = idx[~np.isin(self.nib[idx], np.fromiter(used, np.int64, len(used)))]
        _, first = np.unique(self.nib[idx], return_index=True)
        idx = idx[np.sort(first)][:m]
        assert len(idx) == m, f"pool too small: {len(idx)} < {m}"
        used.update(int(x) for x in self.nib[idx])
        return idx


class Chunk:
    """Requests of one chunk, accumulated as (table, key, type) and laid out in a random order."""

    def __init__(self, kind, pool, rng):
        self.kind, self.pool, self.rng = kind, pool, rng
        self.tb, self.key, self.ty, self.hot = [], [], [], []

    def add(self, idx, types, hot):
        idx = np.broadcast_to(idx, np.shape(types))
        self.tb.append(self.pool.tb[idx])
        self.key.append(self.pool.key[idx])
        self.ty.append(np.asarray(types))
        self.hot.append(np.full(len(types), hot))

    def hot_group(self, idx, m):
        self.add(idx, hot_types(self.kind, m, self.rng), True)

    def cold(self, m, used, read_only=False):
        self.add(self.pool.pick(m, self.rng, used), cold_types(self.kind, m, self.rng, read_only), False)

    def logs(self, m):
        if self.kind in LOG_TYPE and m:
            self.tb.append(self.rng.integers(0, 2, m))
            self.key.append(self.rng.integers(0, 2**40, m).astype(np.uint64))
            self.ty.append(np.full(m, LOG_TYPE[self.kind]))
            self.hot.append(np.zeros(m, bool))

    def build(self, edges_hot=False):
        tb, key, ty, hot = (np.concatenate(x) for x in (self.tb, self.key, self.ty, self.hot))
        order = self.rng.permutation(len(ty))
        if edges_hot:                       # a hot request on the first and on the last position
            h = np.nonzero(hot[order])[0]
            assert len(h) >= 2
            pos = [0, len(order) - 1]
            for p, q in zip(pos, self.rng.choice(h, size=2, replace=False)):
                order[[p, q]] = order[[q, p]]
        return records(self.kind, tb[order], key[order], ty[order], self.rng)


# ---------------------------------------------------------------- running a case ---------------------------------
def cfg_for(kind, **over):
    cfg = dict(KV_CFG.get(kind, {}))
    cfg.update(over)
    return cfg


def make_oracle(kind, cfg):
    return O.Oracle(kind, **{k: v for k, v in cfg.items() if k in ORACLE_KEYS})


def first_diff(a, b, msg):
    a, b = a.reshape(-1, msg), b.reshape(-1, msg)
    bad = np.nonzero((a != b).any(axis=1))[0]
    if bad.size == 0:
        return None
    i = int(bad[0])
    return f"{bad.size} of {a.shape[0]} replies differ; first at {i}: got {a[i].tolist()} want {b[i].tolist()}"


def submit(eng, path, raw):
    if path == "host":
        return eng.submit(raw)
    import torch
    if raw.size == 0:
        return raw.copy()
    d = torch.from_numpy(raw.copy()).cuda()
    out = eng.submit_tensor(d)
    eng.sync()
    torch.cuda.synchronize()
    return out.cpu().numpy()


PATH_KEYS = ("conflicted", "ordered_fallbacks", "bucket_split_tasks", "writerless_chunks")


def serve(eng, ora, geo, calls):
    """Feed (path, raw) calls to the engine and the oracle; replies must match and the path counters must match
    the model.  Returns the model's routes per call."""
    all_routes = []
    for path, raw in calls:
        before = eng.stats()
        want = ora.process(raw)
        got = submit(eng, path, raw)
        d = first_diff(got, want, eng.msg)
        assert d is None, f"{NAMES[geo.kind]} {path} call of {raw.size // eng.msg}: {d}"
        exp, routes = model(geo, raw, call_chunks(geo, raw.size // eng.msg, path))
        after = eng.stats()
        got_c = {k: after[k] - before[k] for k in PATH_KEYS}
        assert got_c == exp, f"{NAMES[geo.kind]} {path}: path counters {got_c} != model {exp} ({[r['route'] for r in routes]})"
        assert after["errors"] == 0
        all_routes.append(routes)
    return all_routes


def check_state(eng, ora, geo, raws, max_keys=1500):
    """Final state, bit for bit: lock words / counters of every touched group (the busiest first), KV rows, table
    sizes, log ring."""
    kind = geo.kind
    if kind == LOG or kind in LOG_TYPE:
        ring, appended = eng.dump_log()
        assert appended == ora.log_appended()
        assert np.array_equal(ring, ora.log_ring())
    if kind == LOG:
        return
    g, mask = classify(geo, np.concatenate(raws))
    rec = wire.as_records(kind, np.concatenate(raws))
    keep = g >= 0
    if kind in (LOCK2PL, FASST):
        tb, key = np.zeros(len(rec), np.int64), rec["lid"].astype(np.uint64)
    elif kind == STORE:
        tb, key = np.zeros(len(rec), np.int64), rec["key"]
    else:
        tb, key = rec["table"].astype(np.int64), rec["key"]
    u, first, cnt = np.unique(g[keep], return_index=True, return_counts=True)
    sel = np.nonzero(keep)[0][first[np.argsort(-cnt, kind="stable")][:max_keys]]
    for t, k in zip(tb[sel], key[sel]):
        t, k = int(t), int(k)
        if kind != STORE:                         # a store group has no state of its own
            s = int(geo.slot(t, k))
            a, b = eng.lock_state(t, s), ora.lock_state(t, s)
            if kind == TATP:
                a, b = a[0], b[0]                 # TATP groups hold a lock bit only
            assert a == b, (NAMES[kind], t, hex(k), s, a, b)
        if kind in (STORE, TATP, SMALLBANK):
            x, y = eng.kv_get(t, k), ora.kv_get(t, k)
            if kind == SMALLBANK and x is not None and y is not None:
                x, y = (x[0][:8], x[1]), (y[0][:8], y[1])
            assert x == y, (NAMES[kind], t, hex(k))
    for t in range(len(geo.mods) if kind != STORE else 1):
        if kind in (STORE, TATP, SMALLBANK):
            assert eng.kv_count(t) == ora.kv_count(t), t


def run_calls(kind, cfg, calls, populate=True):
    geo = Geo(kind, **cfg)
    ora = make_oracle(kind, cfg)
    with Engine(kind, populate=populate and kind in KV_CFG, **cfg) as eng:
        routes = serve(eng, ora, geo, calls)
        check_state(eng, ora, geo, [r for _, r in calls])
    return routes


def setup(kind, seed, **over):
    cfg = cfg_for(kind, **over)
    geo = Geo(kind, **cfg)
    ora = make_oracle(kind, cfg)
    pool = Pool(geo, ora)
    ora.close()
    return cfg, geo, pool, np.random.default_rng(seed)


# ---------------------------------------------------------------- CPU: the Python copies of the engine's hashes --
def test_python_group_ids_match_the_oracle():
    """Geo.group must be the slot the oracle (and so the reference) computes; the path model rests on it."""
    rng = np.random.default_rng(1)
    lids = rng.integers(0, 2**32, 300, dtype=np.uint64)
    for kind in (LOCK2PL, FASST):
        for slots in (200, 60000, 16_000_000, 36_000_000):
            geo, ora = Geo(kind, lock_slots=slots), O.Oracle(kind, populate=False, lock_slots=slots)
            assert geo.group(0, lids).tolist() == [ora.lock_slot(0, int(x)) for x in lids]
    keys = rng.integers(0, 2**64, 200, dtype=np.uint64)
    for kind in (TATP, SMALLBANK):
        cfg = {k: v for k, v in KV_CFG[kind].items() if k.endswith("sizing")}
        geo, ora = Geo(kind, **cfg), O.Oracle(kind, populate=False, **cfg)
        for t in range(len(geo.mods)):
            assert geo.slot(np.full(len(keys), t), keys).tolist() == [ora.lock_slot(t, int(k)) for k in keys]
    assert Geo(FASST).sort_passes == 4 and Geo(FASST).flags_mask == FOLD - 1
    assert [Geo(FASST, lock_slots=s).sort_passes for s in (200, 60000, 16_000_000)] == [1, 2, 3]


def test_model_route_choice():
    """The route model on hand-made group lists: one chunk of 4096 has 64 buckets."""
    geo = Geo(FASST, lock_slots=1 << 20, chunk=4096)
    assert geo.bucket_log2 == 6
    lids = np.arange(1 << 16, dtype=np.uint64)
    g = geo.group(0, lids)
    b = bucket_of(g, 6)
    rng = np.random.default_rng(0)

    def trace(groups_sizes):
        parts = [np.repeat(lids[[int(np.nonzero(b == bk)[0][j])]], m) for bk, j, m in groups_sizes]
        lid = np.concatenate(parts)
        return records(FASST, 0, lid, np.full(len(lid), 3), rng)

    exp, r = model(geo, trace([(0, 0, 100), (0, 1, 20)]), [120])
    assert exp["conflicted"] == 120 and r[0]["route"] == "bucket" and r[0]["tasks"].tolist() == [120]
    exp, r = model(geo, trace([(2, 0, 70), (3, 0, 70)]), [140])
    assert r[0]["route"] == "split" and exp["bucket_split_tasks"] == 1
    exp, r = model(geo, trace([(5, 0, 129)]), [129])
    assert r[0]["route"] == "radix" and exp["ordered_fallbacks"] == 1
    exp, r = model(geo, records(FASST, 0, lids[:50], np.zeros(50, np.int64), rng), [50])
    assert r[0]["route"] == "writerless" and exp["writerless_chunks"] == 1


# ---------------------------------------------------------------- 1. path matrix ---------------------------------
def matrix_trace(kind, pool, case, rng):
    P = 1 << pool.geo.bucket_log2
    used = set()
    ch = Chunk(kind, pool, rng)
    per_bucket = np.bincount(pool.bucket, minlength=P)
    if case == "bucket":            # one task of <= 32 pairs (rank sort), one of 33..128 (bitonic sort)
        ba = int(np.argmax(per_bucket[:P // 2]))
        bb = P // 2 + int(np.argmax(per_bucket[P // 2:]))
        for i in pool.pick(3, rng, used, pool.bucket == ba):
            ch.hot_group(i, 8)
        for i in pool.pick(2, rng, used, pool.bucket == bb):
            ch.hot_group(i, 40)
    elif case == "split":           # two adjacent buckets of 70 pairs: a task of 140 > kBucketCap, no bucket over it;
        gsz = 1                     # the second one is the task's last bucket
        while gsz < 32 and 140 * gsz * 2 <= 16 * P:
            gsz <<= 1
        ends = np.arange(gsz - 2, P, gsz)
        b0 = int(ends[np.argmax((per_bucket[ends] >= 2) & (per_bucket[ends + 1] >= 2))])
        assert per_bucket[b0] >= 2 and per_bucket[b0 + 1] >= 2
        for b in (b0, b0 + 1):
            for i in pool.pick(2, rng, used, pool.bucket == b):
                ch.hot_group(i, 35)
    elif case == "radix":           # one group of 200 listed requests overflows its bucket
        ch.hot_group(pool.pick(1, rng, used)[0], 200)
        for i in pool.pick(3, rng, used):
            ch.hot_group(i, 10)
    ch.cold(1500, used)
    ch.logs(100)
    return ch.build()


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [4096, 1 << 16])
@pytest.mark.parametrize("kind", KEYED, ids=[NAMES[k] for k in KEYED])
def test_path_matrix(kind, chunk):
    """(a) solo only, (b) bucket replay in one pass with both sorts, (c) bucket replay task split bucket by bucket,
    (d) radix fallback -- each one chunk, each proven by the counters."""
    cfg, geo, pool, rng = setup(kind, seed=100 + kind + chunk, chunk=chunk)
    traces = {case: matrix_trace(kind, pool, case, rng) for case in ("solo", "bucket", "split", "radix")}
    routes = {}
    for case, raw in traces.items():
        exp, r = model(geo, raw, call_chunks(geo, raw.size // wire.MSG_SIZE[kind], "host"))
        assert len(r) == 1
        routes[case] = (exp, r[0])
    exp, r = routes["solo"]
    assert exp["conflicted"] == 0 and r["route"] == "solo"
    exp, r = routes["bucket"]
    assert r["route"] == "bucket" and exp["conflicted"] == 3 * 8 + 2 * 40
    assert r["tasks"].min() <= 32 and 32 < r["tasks"].max() <= BUCKET_CAP
    exp, r = routes["split"]
    assert r["route"] == "split" and exp["bucket_split_tasks"] == 1 and exp["ordered_fallbacks"] == 0
    assert exp["conflicted"] == 4 * 35
    exp, r = routes["radix"]
    assert r["route"] == "radix" and exp["ordered_fallbacks"] == 1 and exp["conflicted"] == 200 + 3 * 10
    run_calls(kind, cfg, [("host", raw) for raw in traces.values()])


# ---------------------------------------------------------------- 2. radix pass count ----------------------------
def digit_pairs(geo, lids, rng):
    """per 8-bit digit d of the group id: two lock ids whose groups differ in digit d only"""
    g = geo.group(0, lids)
    out = []
    for d in range(geo.sort_passes):
        rest = g & ~np.int64(0xFF << (8 * d))
        order = np.lexsort((g, rest))
        rs, gs = rest[order], g[order]
        hit = np.nonzero((rs[1:] == rs[:-1]) & (gs[1:] != gs[:-1]))[0]
        assert hit.size, d
        j = int(rng.choice(hit))
        out.append((lids[order[j]], lids[order[j + 1]]))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("slots,passes", [(200, 1), (60000, 2), (16_000_000, 3), (36_000_000, 4)])
@pytest.mark.parametrize("kind", [LOCK2PL, FASST], ids=["lock_2pl", "lock_fasst"])
def test_radix_pass_count(kind, slots, passes):
    """Fallback chunks on group spaces of 1-4 radix digits.  For every digit two hot groups that differ in that digit
    only, their requests alternating: a pass that does not run leaves them interleaved and the replay wrong."""
    cfg = dict(lock_slots=slots, chunk=1 << 16)
    geo = Geo(kind, **cfg)
    assert geo.sort_passes == passes
    rng = np.random.default_rng(slots + kind)
    lids = np.arange(1 << 22 if slots > 1 << 20 else 1 << 16, dtype=np.uint64)
    tys, ids = [], []
    for a, b in digit_pairs(geo, lids, rng):
        ta, tb_ = hot_types(kind, 150, rng), hot_types(kind, 150, rng)
        tys.append(np.stack([ta, tb_], axis=1).reshape(-1))
        ids.append(np.tile([a, b], 150))
    lid, ty = np.concatenate(ids), np.concatenate(tys)
    raw = records(kind, 0, lid, ty, rng)
    exp, r = model(geo, raw, [len(ty)])
    assert r[0]["route"] == "radix" and exp["conflicted"] == len(ty)
    # a second call on the state the first left behind
    run_calls(kind, cfg, [("host", raw), ("device", records(kind, 0, lid[::-1].copy(), ty, rng))])


# ---------------------------------------------------------------- 3./4. folding and the segmented scan -----------
def fold_pairs(geo, n_lids, rng):
    """(low lid, high lid) pairs whose slots s, s + 2^25 share a flag nibble (default 36 M slots)"""
    lids = np.arange(n_lids, dtype=np.uint64)
    g = geo.group(0, lids)
    lo = np.nonzero(g < geo.mods[0] - FOLD)[0]
    hi_of = {int(x): i for i, x in zip(np.nonzero(g >= FOLD)[0], g[g >= FOLD])}
    pairs = [(int(lids[i]), int(lids[hi_of[int(g[i]) + FOLD]]), int(g[i])) for i in lo if int(g[i]) + FOLD in hi_of]
    rng.shuffle(pairs)
    return lids, g, pairs


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [LOCK2PL, FASST], ids=["lock_2pl", "lock_fasst"])
def test_false_conflicts_from_flag_folding(kind):
    """A lone request on slot s shares its flag nibble with hot writers on slot s + 2^25: it is listed as a group of
    its own (a false conflict) and must still be answered exactly."""
    cfg = dict(chunk=1 << 16)
    geo = Geo(kind, **cfg)
    rng = np.random.default_rng(40 + kind)
    lids, g, pairs = fold_pairs(geo, 1 << 22, rng)
    pairs = pairs[:20]
    lone_t = np.full(20, READ[kind] if READ[kind] is not None else LONE_WRITER[kind])
    lone_t[10:] = LONE_WRITER[kind]
    ids = [np.array([p[0] for p in pairs], np.uint64)]
    tys = [lone_t]
    for _, hi, _ in pairs:
        ids.append(np.full(3, hi, np.uint64))
        tys.append(hot_types(kind, 3, rng))
    used = {p[2] for p in pairs}
    free = np.nonzero(~np.isin(g & geo.flags_mask, list(used)) & (g < FOLD))[0]
    cold = rng.choice(free, 1000, replace=False)
    _, first = np.unique(g[cold], return_index=True)
    cold = cold[first]
    ids.append(lids[cold])
    tys.append(cold_types(kind, len(cold), rng))
    lid, ty = np.concatenate(ids), np.concatenate(tys)
    order = rng.permutation(len(ty))
    raw = records(kind, 0, lid[order], ty[order], rng)
    exp, r = model(geo, raw, [len(ty)])
    assert exp["conflicted"] == 20 * 3 + 20 and r[0]["route"] == "bucket"
    run_calls(kind, cfg, [("host", raw)])


@pytest.mark.gpu
def test_fasst_segmented_scan_tile_boundaries():
    """lock_fasst radix fallback: run heads at sorted positions 2047, 2048 and 2049 (around the first sort-tile edge),
    a run that covers three whole 2048-entry sort tiles, single-request runs between long ones, all four request types
    at the tile edges, and runs that start from a pre-chunk state (lock = 1, ver != 0) left by an earlier call."""
    kind = FASST
    cfg = dict(chunk=1 << 16)
    geo = Geo(kind, **cfg)
    rng = np.random.default_rng(3)
    lids, g, pairs = fold_pairs(geo, 1 << 22, rng)
    lone_region = geo.mods[0] - FOLD
    # five lone (single-request) runs: the low side of fold pairs, spread over the low slots
    pairs.sort(key=lambda p: p[2])
    at = [int(q * len(pairs)) for q in (0.2, 0.4, 0.6, 0.8)]
    lone = [pairs[i] for i in (at[0], at[0] + 1, at[1], at[2], at[3])]
    assert lone[0][2] < lone[1][2]
    ls = [p[2] for p in lone]
    fold_slots = {p[2] for p in pairs} | {p[2] + FOLD for p in pairs}
    plain = np.nonzero((g < lone_region) & ~np.isin(g, list(fold_slots)))[0]

    def plain_in(lo, hi, k):
        c = plain[(g[plain] > lo) & (g[plain] < hi)]
        c = c[np.unique(g[c], return_index=True)[1]]
        return [int(lids[i]) for i in rng.choice(c, k, replace=False)]

    # runs in sorted (slot) order: (lid, length); None length = a lone run
    r1 = plain_in(0, ls[0], 3)
    r1.sort(key=lambda x: int(geo.group(0, x)))
    runs = [(r1[0], 1000), (r1[1], 600), (r1[2], 447),                   # 2047 entries
            (lone[0][0], 1), (lone[1][0], 1),                            # heads at 2047 and 2048
            (plain_in(ls[1], ls[2], 1)[0], 8300),                        # head at 2049, covers tiles 2, 3 and 4
            (lone[2][0], 1), (plain_in(ls[2], ls[3], 1)[0], 300),
            (lone[3][0], 1), (plain_in(ls[3], ls[4], 1)[0], 2),
            (lone[4][0], 1), (plain_in(ls[4], lone_region, 1)[0], 40)]
    runs += [(p[1], 3) for p in lone]                                    # the fold partners sort last
    slots = [int(geo.group(0, x)) for x, _ in runs]
    assert slots == sorted(slots) and len(set(slots)) == len(slots)
    heads = np.concatenate([[0], np.cumsum([m for _, m in runs])[:-1]])
    assert heads[3:6].tolist() == [2047, 2048, 2049]
    assert heads[5] + runs[5][1] > 5 * SORT_TILE
    nc = int(sum(m for _, m in runs))
    # types by sorted position: random, every tile edge cycles through all four types, lone runs are 0..3 + 0
    types = []
    for j, (lid, m) in enumerate(runs):
        if m == 1:
            types.append(np.array([[0, 1, 2, 3, 0][[3, 4, 6, 8, 10].index(j)]]))
        elif j >= 12:
            types.append(np.array([3, 3, 0]))
        else:
            types.append(rng.choice(4, size=m, p=[0.3, 0.3, 0.15, 0.25]))
    flat = np.concatenate(types)
    for k, e in enumerate(range(SORT_TILE, nc, SORT_TILE)):
        for d in range(-2, 2):
            if 0 <= e + d < nc and e + d not in heads[[3, 4, 6, 8, 10]]:
                flat[e + d] = (k + d) % 4
    flat[heads[5]:heads[5] + 3] = [0, 1, 0]      # the long run starts from lock = 1: read, rejected acquire, read
    # index order: runs interleaved at random, each run in its own order
    label = rng.permutation(np.repeat(np.arange(len(runs)), [m for _, m in runs]))
    lid = np.array([x for x, _ in runs], np.uint64)[label]
    ty = np.empty(nc, np.int64)
    for j in range(len(runs)):
        ty[label == j] = flat[heads[j]:heads[j] + runs[j][1]]
    raw = records(kind, 0, lid, ty, rng)
    exp, r = model(geo, raw, [nc])
    assert r[0]["route"] == "radix" and exp["conflicted"] == nc
    # the earlier call: three commits and an acquire leave lock = 1, ver = 3 on some of these slots
    pre_ids = np.repeat(np.array([runs[i][0] for i in (3, 4, 5, 7, 11, 0)], np.uint64), 4)
    pre = records(kind, 0, pre_ids, np.tile([3, 3, 3, 1], 6), rng)
    run_calls(kind, cfg, [("host", pre), ("host", raw)])


# ---------------------------------------------------------------- 5. chunk transitions ---------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("chunk", [256, 4096])
@pytest.mark.parametrize("kind", KEYED, ids=[NAMES[k] for k in KEYED])
def test_chunk_transitions(kind, chunk, path):
    """One call of six chunks: radix fallback -> bucket -> writer-free -> solo -> fallback -> bucket, with the same hot
    groups on both sides of every chunk boundary (flag-set alternation, the listed counts cleared one launch early and
    the writer-free skip of K2 all hand over between them)."""
    cfg, geo, pool, rng = setup(kind, seed=500 + kind + chunk, chunk=chunk)
    hot = pool.pick(3, rng, set())
    hot_nibs = {int(x) for x in pool.nib[hot]}
    big = 150
    parts = []
    for route in ("radix", "bucket", "writerless", "solo", "radix", "bucket"):
        ch = Chunk(kind, pool, rng)
        used = set(hot_nibs)
        if route == "radix":
            ch.hot_group(hot[0], big)
            ch.hot_group(hot[1], 10)
            ch.hot_group(hot[2], 10)
        elif route == "bucket":
            for i, m in zip(hot, (20, 10, 10)):
                ch.hot_group(i, m)
        elif route == "writerless" and READ[kind] is not None:
            for i in hot:
                ch.add(i, np.full(3, READ[kind]), True)
        else:
            for i in hot:
                ch.add(i, [LONE_WRITER[kind]], True)
        n_hot = sum(len(t) for t in ch.ty)
        n_log = 8 if kind in LOG_TYPE else 0
        ch.cold(chunk - n_hot - n_log, used, read_only=route == "writerless" and READ[kind] is not None)
        ch.logs(n_log)
        parts.append(ch.build(edges_hot=True))
    raw = np.concatenate(parts)
    exp, r = model(geo, raw, call_chunks(geo, raw.size // wire.MSG_SIZE[kind], path))
    want_routes = ["radix", "bucket", "writerless" if READ[kind] is not None else "solo", "solo", "radix", "bucket"]
    assert [x["route"] for x in r] == want_routes
    assert exp["ordered_fallbacks"] == 2 and exp["writerless_chunks"] == (READ[kind] is not None)
    run_calls(kind, cfg, [(path, raw)])


# ---------------------------------------------------------------- 6. default configuration, sliced host path ----
def background(kind, pool, n, rng):
    """random traffic over the pool: every type of hot_types, contention wherever keys repeat"""
    if kind == LOG:
        return T.log_random(n, seed=int(rng.integers(1 << 30)))
    idx = rng.integers(0, len(pool.g), n)
    ty = rng.choice(HOT_MIX[kind], size=n)
    if kind in LOG_TYPE:
        ty[rng.random(n) < 0.05] = LOG_TYPE[kind]
    return records(kind, pool.tb[idx], pool.key[idx], ty, rng)


def straddle(kind, pool, raw, boundaries, rng):
    """overwrite three requests on each side of every boundary with one hot group (listed on both sides)"""
    if kind == LOG:
        return raw
    msg = wire.MSG_SIZE[kind]
    out = raw.copy().reshape(-1, msg)
    n = len(out)
    hot = pool.pick(len(boundaries), rng, set())
    for b, i in zip(boundaries, hot):
        for lo, hi in ((b - 3, b), (b, b + 3)):
            lo, hi = max(lo, 0), min(hi, n)
            if hi - lo >= 2:
                out[lo:hi] = records(kind, pool.tb[[i] * (hi - lo)], pool.key[[i] * (hi - lo)],
                                     hot_types(kind, hi - lo, rng), rng).reshape(-1, msg)
    return out.reshape(-1)


SIZES = [131071, 131073, 300001, 1_500_000, 3_000_000]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ALL_KINDS, ids=[NAMES[k] for k in ALL_KINDS])
def test_default_config_sliced_host_path(kind):
    """The production host path: the default 2^20 chunk, so every call is cut into 128 K - 256 K slices smaller than
    the chunk (one of them ragged in the middle of a 300001-request call), with hot groups on both sides of every
    slice boundary."""
    cfg = {k: v for k, v in KV_CFG.get(kind, {}).items() if k.endswith("populate")}
    geo = Geo(kind, **cfg)
    ora = make_oracle(kind, cfg)
    pool = Pool(geo, ora) if kind != LOG else None
    rng = np.random.default_rng(600 + kind)
    calls = []
    for n in SIZES:
        sl = host_slices(n, HOST_MAX_SLICE)
        assert max(sl) < geo.chunk and (n < 300000 or len(set(sl)) > 1)
        calls.append(("host", straddle(kind, pool, background(kind, pool, n, rng), np.cumsum(sl)[:-1], rng)))
    with Engine(kind, populate=kind in KV_CFG, **cfg) as eng:
        serve(eng, ora, geo, calls)
        check_state(eng, ora, geo, [r for _, r in calls], max_keys=800)


@pytest.mark.gpu
def test_host_and_device_calls_share_one_engine():
    """A host call, device calls of ragged sizes on the torch stream, another host call: one oracle fed the
    concatenation."""
    kind = FASST
    cfg, geo, pool, rng = setup(kind, seed=7, chunk=1 << 16)
    ora = make_oracle(kind, cfg)
    calls = [("host", background(kind, pool, 200001, rng))]
    calls += [("device", background(kind, pool, n, rng)) for n in (1, 129, 65537, 131071, 3)]
    calls.append(("host", background(kind, pool, 300001, rng)))
    with Engine(kind, **cfg) as eng:
        serve(eng, ora, geo, calls)
        check_state(eng, ora, geo, [r for _, r in calls])


# ---------------------------------------------------------------- 7. ragged tails --------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("kind", ALL_KINDS, ids=[NAMES[k] for k in ALL_KINDS])
def test_ragged_tails(kind, path):
    """Calls whose byte length is not a multiple of 16 (the TMA body / byte-tail split) and whose last tile is partial
    (the 4-lanes-per-entry KV prefetch on a partial tile), with conflicts inside that last tile."""
    msg = wire.MSG_SIZE[kind]
    cfg = {k: v for k, v in KV_CFG.get(kind, {}).items() if k.endswith("populate")}
    geo = Geo(kind, **cfg)
    ora = make_oracle(kind, cfg)
    pool = Pool(geo, ora) if kind != LOG else None
    rng = np.random.default_rng(700 + kind)
    calls = []
    for n in (1, 2, 3, 5, 127, 129, 131, 1000):
        raw = background(kind, pool, n, rng)
        if kind != LOG and n >= 2:                 # the last min(n, 6) requests: one hot group
            k = min(n, 6)
            i = pool.pick(1, rng, set())[0]
            tail = records(kind, pool.tb[[i] * k], pool.key[[i] * k], hot_types(kind, k, rng), rng)
            raw = np.concatenate([raw[:(n - k) * msg], tail])
        calls.append((path, raw))
    assert any((n * msg) % 16 for n in (1, 2, 3, 5, 127, 129, 131, 1000))
    with Engine(kind, populate=kind in KV_CFG, **cfg) as eng:
        routes = serve(eng, ora, geo, calls)
        check_state(eng, ora, geo, [r for _, r in calls])
    if kind != LOG:
        assert all(rt[-1]["nc"] >= 2 for rt, (_, raw) in zip(routes, calls) if raw.size >= 2 * msg)


# ---------------------------------------------------------------- 8. snapshot / restore ----------------------------
def state_probe(eng, geo, raws):
    """everything check_state compares, as a value (for engine-vs-engine comparisons)"""
    kind = geo.kind
    out = []
    if kind == LOG or kind in LOG_TYPE:
        ring, appended = eng.dump_log()
        out.append((ring.tobytes(), appended))
    if kind == LOG:
        return out
    g, _ = classify(geo, np.concatenate(raws))
    rec = wire.as_records(kind, np.concatenate(raws))
    for j in np.nonzero(g >= 0)[0][:2000]:
        if kind in (LOCK2PL, FASST):
            t, k = 0, int(rec["lid"][j])
        else:
            t, k = (0 if kind == STORE else int(rec["table"][j])), int(rec["key"][j])
        if kind != STORE:
            out.append(eng.lock_state(t, int(geo.slot(t, k))))
        if kind in KV_CFG:
            out.append(eng.kv_get(t, k))
    if kind in KV_CFG:
        out += [eng.kv_count(t) for t in range(len(geo.mods) if kind != STORE else 1)]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ALL_KINDS, ids=[NAMES[k] for k in ALL_KINDS])
def test_snapshot_restore(kind):
    """snapshot, trace A, restore, trace A again: the same replies and the same final state; after another restore,
    trace B answers as an oracle fed the pre-snapshot prefix and then B."""
    cfg = {k: v for k, v in KV_CFG.get(kind, {}).items() if k.endswith("populate")}
    cfg["chunk"] = 4096
    geo = Geo(kind, **cfg)
    ora_a, ora_b = make_oracle(kind, cfg), make_oracle(kind, cfg)
    pool = Pool(geo, ora_a) if kind != LOG else None
    rng = np.random.default_rng(800 + kind)
    prefix, a, b = (background(kind, pool, n, rng) for n in (10007, 20011, 15013))
    with Engine(kind, populate=kind in KV_CFG, **cfg) as eng:
        serve(eng, ora_a, geo, [("host", prefix)])
        ora_b.process(prefix)
        snap = eng.snapshot()
        try:
            r1 = eng.submit(a)
            assert first_diff(r1, ora_a.process(a), eng.msg) is None
            s1 = state_probe(eng, geo, [prefix, a])
            eng.submit(a)                               # the state moves on ...
            eng.restore(snap)
            r2 = eng.submit(a)                          # ... and a restore brings it back
            assert first_diff(r2, r1, eng.msg) is None
            assert state_probe(eng, geo, [prefix, a]) == s1
            eng.restore(snap)
            serve(eng, ora_b, geo, [("device", b)])
            check_state(eng, ora_b, geo, [prefix, b])
        finally:
            eng.free_snapshot(snap)


def callfwd_rows(first, m, ty, rng):
    keys = np.arange(first, first + m, dtype=np.uint64) | (np.uint64(1) << np.uint64(32)) | (np.uint64(8) << np.uint64(40))
    return records(TATP, np.full(m, wire.Tatp.kCallForwarding), keys, np.full(m, ty), rng)


@pytest.mark.gpu
def test_restore_refreshes_the_kv_occupancy_mirror():
    """A call that fills a KV table past 70 % makes the next call rehash it.  Restoring a snapshot taken before that
    call restores the table's occupancy too, so the next call must NOT rehash (which would double the table and make
    the snapshot unusable); a restore after a real rehash is refused."""
    Tt = wire.Tatp
    cfg = dict(subs_populate=20, kv_capacity_log2=[0, 0, 0, 0, 11], chunk=4096)
    ora_cfg = dict(subs_populate=20)
    rng = np.random.default_rng(9)
    fill = callfwd_rows(1000, 1450, Tt.kInsertBck, rng)            # 2048 entries: 70 % is 1434
    reads = callfwd_rows(1000, 64, Tt.kRead, rng)
    with Engine(TATP, populate=True, **cfg) as eng:
        ora = O.Oracle(TATP, **ora_cfg)
        assert np.array_equal(eng.submit(reads), ora.process(reads))     # publishes the occupancy mirror
        snap = eng.snapshot()
        try:
            eng.submit(fill)
            eng.restore(snap)
            got = eng.submit(reads)
            assert first_diff(got, ora.process(reads), 55) is None
            st = eng.stats()
            assert st["kv_rebuilds"] == 0, st
            eng.restore(snap)                                            # the table was not rehashed: still restorable
            assert eng.kv_count(4) == ora.kv_count(4)
            # now fill it for real: the next call rehashes, and the snapshot no longer fits the engine
            assert first_diff(eng.submit(fill), ora.process(fill), 55) is None
            assert first_diff(eng.submit(reads), ora.process(reads), 55) is None
            assert eng.stats()["kv_rebuilds"] == 1
            with pytest.raises(DintError) as ei:
                eng.restore(snap)
            assert ei.value.code == -22
            assert eng.kv_count(4) == ora.kv_count(4)
        finally:
            eng.free_snapshot(snap)
