"""Writes tests/golden/smallbank_ebpf/{cold,warm}.npz from the reference's eBPF SmallBank shard server compiled unmodified
(oracle/smallbank_ebpf.mk -> oracle/_ref/smallbank_ebpf).  Both traces run at the reference's sizes (A = 24,000,000
accounts, 9,000,000 buckets per table) with accounts [0, 4,000,000) populated: `cold` on an empty cache (as dint_load
leaves it), `warm` after the eBPF client's warm-up stream of shard 0 (as dint_populate leaves it).  The keys are four
buckets per table of five colliding accounts plus one colliding key the tables lack, and the traces are long enough that
together they reach every path in smallbank_ebpf_model.REQUIRED_PATHS: refused acquires of both kinds, grants, commits
and warm-up reads that hit and that miss over an invalid, a clean and a dirty victim, releases below zero, log appends
of every table byte, refused types and tables, and missing keys with and without a write-back.
Run after `make -C oracle -f smallbank_ebpf.mk`."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import smallbank_ebpf_model as M  # noqa: E402

POPULATED, N = 4_000_000, 6000
TRACES = {"cold": (False, 2024), "warm": (True, 2025)}


def golden_trace(seed):
    groups = M.colliding_groups(POPULATED, seed=seed)
    keys, tables = M.group_keys(groups)
    return M.random_trace(groups, N, seed=seed), keys, tables


def main():
    if not M.ref_available():
        sys.exit("oracle/_ref/smallbank_ebpf missing: run make -C oracle -f smallbank_ebpf.mk")
    for name, (warm, seed) in TRACES.items():
        req, keys, tables = golden_trace(seed)
        resp, sets, finds, locks, log = M.run_ref_smallbank_ebpf(req, keys, tables, populate=POPULATED, warmup=warm)
        out = os.path.join(ROOT, "tests", "golden", "smallbank_ebpf", f"{name}.npz")
        np.savez_compressed(out, req=req, resp=resp, keys=keys, tables=tables, sets=sets, finds=finds.view(np.uint8),
                            locks=locks.view(np.uint8), log=log, populated=POPULATED, warm=warm)
        print(out, np.bincount(resp.reshape(-1, M.MSG)[:, 1], minlength=256)[[7, 8, 9, 10, 11, 12, 13, 14, 15, 18, 255]])


if __name__ == "__main__":
    main()
