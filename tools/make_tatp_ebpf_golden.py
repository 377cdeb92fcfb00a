"""Writes tests/golden/tatp_ebpf/{shard,lock}.npz from the reference's eBPF TATP shard server compiled unmodified
(oracle/tatp_ebpf.mk -> oracle/_ref/tatp_ebpf_{shard,lock}).  One trace over keys that collide in three buckets (eight keys each, the last never inserted) of every
table at the reference's sizes (S = 7,000,000), long enough that every path in tatp_ebpf_model.REQUIRED_PATHS runs:
read hits, bloom negatives (true and false), table hits and misses with clean and dirty victims, commit hits and misses
of both forms with write-backs of version 0 and n, cache-only and evicting inserts, a key inserted twice, deletes that
free their chain entry and deletes that do not, lock grants and both kinds of reject, aborts, both log types and refused
requests.  Run after `make -C oracle -f tatp_ebpf.mk`."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import tatp_ebpf_model as M  # noqa: E402

SEED, N = 2024, 8000


def golden_trace():
    groups = M.colliding_groups(M.REF_S, seed=SEED)
    req = M.random_trace(groups, N, seed=SEED)
    keys = np.array([k for g in groups for grp in g for k in grp], dtype=np.uint64)
    tables = np.array([t for t, g in enumerate(groups) for grp in g for _ in grp], dtype=np.uint8)
    return req, keys, tables


def main():
    if not M.ref_available():
        sys.exit("oracle/_ref/tatp_ebpf_* missing: run make -C oracle -f tatp_ebpf.mk")
    req, keys, tables = golden_trace()
    for v in M.VARIANTS:
        resp, sets, chains, finds, locks, log = M.run_ref_tatp_ebpf(v, req, keys, tables)
        out = os.path.join(ROOT, "tests", "golden", "tatp_ebpf", f"{v}.npz")
        np.savez_compressed(out, req=req, resp=resp, keys=keys, tables=tables, sets=sets, chains=chains.view(np.uint8),
                            finds=finds.view(np.uint8), locks=locks.view(np.uint8), log=log)
        print(out, np.bincount(resp.reshape(-1, M.MSG)[:, 1], minlength=256)[[4, 6, 7, 8, 15, 16, 20, 21, 25, 26, 28, 255]])


if __name__ == "__main__":
    main()
