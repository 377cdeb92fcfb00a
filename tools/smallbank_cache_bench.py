#!/usr/bin/env python3
"""What serving SmallBank as the reference's eBPF shard server costs: the UDP-shaped smallbank engine against the eBPF
cache tier (DINT_CFG_SMALLBANK_EBPF, smallbank/ebpf/shard_kern.c).

The live SmallBank closed loop: GpuTxnClients, 2^20 clients, three full-population shard servers on one GPU
(24,000,000 accounts; the eBPF shards also serve their client's warm-up stream, as dint_populate does).  The two
configurations are alternated --repeats times in one process; each run populates fresh shards, warms up, and times at
least --min-seconds of live rounds on the host clock.

Prints one line per run and one JSON line: per configuration committed txn/s, abort rate, µs per round, requests listed
for the ordered replay per 1000 (dint_stats.conflicted), and for the tier its hit ratio (hits over hits + misses) and
table accesses and write-backs per 1000 requests; the card's name, power limit and SM clock, read right after the last
timed region.

    python tools/smallbank_cache_bench.py [--clients N] [--warmup W] [--min-seconds S] [--repeats R]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from txn_clients_bench import card  # noqa: E402

ACCOUNTS, G = 24_000_000, 3
CONFIGS = {"udp": dict(), "ebpf": dict(smallbank_ebpf=True)}


def one_run(name, clients, warmup, min_seconds):
    import torch
    from dint_b200 import GpuCluster, GpuTxnClients, wire
    per_rank = (clients + G - 1) // G
    with GpuCluster(wire.SMALLBANK, G, devices=[0] * G, max_batch=3 * per_rank, populate=True, **CONFIGS[name]) as cl:
        with GpuTxnClients(cl, clients, subscribers=ACCOUNTS) as tc:
            tc.run(warmup)
            torch.cuda.synchronize()
            s0 = tc.stats()
            e0 = [cl.engine(s).stats() for s in range(G)]
            c0 = [cl.engine(s).smallbank_cache_stats() for s in range(G)] if name != "udp" else None
            rounds, t0 = 0, time.perf_counter()
            while True:
                tc.run(10)
                rounds += 10
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
                if wall >= min_seconds:
                    break
            s1 = tc.stats()
            e1 = [cl.engine(s).stats() for s in range(G)]
            c1 = [cl.engine(s).smallbank_cache_stats() for s in range(G)] if name != "udp" else None
            after = card()
    req = max(1, s1["requests"] - s0["requests"])
    conflicted = sum(b["conflicted"] - a["conflicted"] for a, b in zip(e0, e1))
    r = {"config": name, "rounds_timed": rounds, "timed_s": round(wall, 4),
         "txn_per_s": (s1["committed"] - s0["committed"]) / wall,
         "abort_rate": 1.0 - (s1["committed"] - s0["committed"]) / max(1, s1["txns"] - s0["txns"]),
         "us_per_round": wall / rounds * 1e6, "ordered_replay_per_1000": 1000.0 * conflicted / req,
         "errors": sum(b["errors"] - a["errors"] for a, b in zip(e0, e1)), "sm_mhz_after": after.get("sm_mhz")}
    if c1 is not None:
        d = {k: sum(b[k] - a[k] for a, b in zip(c0, c1)) for k in c1[0]}
        r.update(hit_ratio=d["hits"] / max(1, d["hits"] + d["table"]), table_per_1000=1000.0 * d["table"] / req,
                 write_backs_per_1000=1000.0 * d["write_backs"] / req)
    return r, after


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--clients", type=int, default=1 << 20)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("smallbank_cache_bench: no CUDA device (there is nothing to measure without one)")
    runs, after = [], {}
    for _ in range(a.repeats):
        for name in CONFIGS:
            r, after = one_run(name, a.clients, a.warmup, a.min_seconds)
            runs.append(r)
            print(json.dumps(r), flush=True)
    mean = {n: sum(r["txn_per_s"] for r in runs if r["config"] == n) / a.repeats for n in CONFIGS}
    print(json.dumps({"clients": a.clients, "shards": G, "accounts": ACCOUNTS, "card": after,
                      "txn_per_s_mean": mean, "runs": runs}))


if __name__ == "__main__":
    main()
