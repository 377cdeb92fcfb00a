"""Writes tests/golden/store_ebpf/{wb_bloom,wb,wt}.npz from the reference's eBPF store server compiled unmodified
(oracle/store_ebpf.mk -> oracle/_ref/store_ebpf_*).  One trace per variant over keys that collide in 12 buckets of the
reference's 9,000,000, so that every path of the cache tier runs: inserts into free, clean and dirty slots (every key at most once); READ hits,
bloom negatives, bloom false positives and misses with write-back; SET hits, SET misses found in the table and SETs of
absent keys; and an unknown type.  Run after `make -C oracle -f store_ebpf.mk`."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import store_ebpf_model as M  # noqa: E402


def golden_trace(seed=2023, n=3000):
    rng = np.random.default_rng(seed)
    keys = np.concatenate(M.colliding_keys(M.REF_BUCKETS, 7, 12, seed=seed))
    k = rng.choice(keys, size=n)
    t = rng.choice([0, 1, 2, 0, 1, 0, 2, 5], size=n).astype(np.uint8)    # 5: not a request type of this server
    # every key is inserted at most once and two of each bucket's seven never are: a second kvs_insert of a key would
    # leave two copies in the reference's chained table, which the engine's table does not model
    absent = set(int(x) for g in keys.reshape(12, 7) for x in g[5:])
    inserted = set()
    for i in range(n):
        if t[i] == 2:
            if int(k[i]) in inserted or int(k[i]) in absent:
                t[i] = rng.integers(0, 2)
            else:
                inserted.add(int(k[i]))
    vals = rng.integers(0, 256, size=(n, 40), dtype=np.uint8)
    vers = rng.integers(0, 4, size=n, dtype=np.uint32)
    return M.make_req(t, k, vals, vers), keys


def main():
    if not M.ref_available():
        sys.exit("oracle/_ref/store_ebpf_* missing: run make -C oracle -f store_ebpf.mk")
    req, keys = golden_trace()
    for v in M.VARIANTS:
        resp, sets, table, count = M.run_ref_store_ebpf(v, req, keys)
        out = os.path.join(ROOT, "tests", "golden", "store_ebpf", f"{v}.npz")
        np.savez_compressed(out, req=req, resp=resp, keys=keys, sets=sets, table=table.view(np.uint8).reshape(len(keys), -1),
                            kv_count=np.int64(count))
        print(out, np.bincount(resp.reshape(-1, 53)[:, 0], minlength=256)[[3, 5, 7, 8, 255]])


if __name__ == "__main__":
    main()
