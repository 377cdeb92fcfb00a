#!/usr/bin/env python3
"""What the same-key / false-sharing reject split tells a TATP deployment, and what keeping it costs.

The live TATP closed loop of README's TATP row: GpuTxnClients, 2^20 clients, three full-population shard servers on
one GPU (7,000,000 subscribers).  Run with the servers keeping holder keys (lock_holder_keys=True,
DINT_CFG_LOCK_HOLDER_KEYS) and without, alternated --repeats times in one process; each run populates fresh shards
(two clusters of full TATP shards do not fit 80 GB side by side), warms up, and times at least --min-seconds of live
rounds on the host clock (run() returns after its device work is done and checked).

Prints one JSON line:
  locks requested and the reject ratios by sharing and by same key -- the two lines tatp/caladan/client_lock.cc:403-428
  prints -- from the option-on runs; the undivided reject ratio from the option-off runs;
  committed txn/s of every run, the mean per setting, and on / off;
  the card's name, power limit and SM clock, read right after the last timed region.

    python tools/lock_sharing_bench.py [--clients N] [--warmup W] [--min-seconds S] [--repeats R]
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

SUBSCRIBERS, G = 7_000_000, 3


def one_run(option, clients, warmup, min_seconds):
    import torch
    from dint_b200 import GpuCluster, GpuTxnClients, wire
    per_rank = (clients + G - 1) // G
    with GpuCluster(wire.TATP, G, devices=[0] * G, max_batch=3 * per_rank, populate=True, lock_holder_keys=option) as cl:
        with GpuTxnClients(cl, clients, subscribers=SUBSCRIBERS) as tc:
            tc.run(warmup)
            s0 = tc.stats()
            rounds, t0 = 0, time.perf_counter()
            while True:
                tc.run(10)
                rounds += 10
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
                if wall >= min_seconds:
                    break
            s1, ls = tc.stats(), tc.lock_stats()
            after = card()
    locks = max(1, ls["locks"])
    return {"lock_holder_keys": option, "rounds_timed": rounds, "timed_s": round(wall, 4),
            "txn_per_s": (s1["committed"] - s0["committed"]) / wall,
            "requests_per_s": (s1["requests"] - s0["requests"]) / wall,
            "abort_rate": 1.0 - s1["committed"] / max(1, s1["txns"]),
            "fallback_rounds": s1["fallback_rounds"],
            "locks": ls["locks"], "reject_sharing": ls["reject_sharing"], "reject_same_key": ls["reject_same_key"],
            "reject_ratio_sharing": ls["reject_sharing"] / locks, "reject_ratio_same_key": ls["reject_same_key"] / locks,
            "sm_mhz_after": after.get("sm_mhz")}, after


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--clients", type=int, default=1 << 20)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("lock_sharing_bench: no CUDA device (there is nothing to measure without one)")
    runs, after = [], {}
    for _ in range(a.repeats):
        for option in (False, True):
            r, after = one_run(option, a.clients, a.warmup, a.min_seconds)
            runs.append(r)
            print(f"holder keys {'on ' if option else 'off'}: {r['txn_per_s'] / 1e6:.3f} M txn/s, reject ratio sharing "
                  f"{r['reject_ratio_sharing']:.4f} same key {r['reject_ratio_same_key']:.4f} ({r['locks']} locks)", flush=True)
    on = [r for r in runs if r["lock_holder_keys"]]
    off = [r for r in runs if not r["lock_holder_keys"]]
    mean = lambda rs: sum(r["txn_per_s"] for r in rs) / len(rs)   # noqa: E731
    out = {"clients": a.clients, "shards": G, "subscribers": SUBSCRIBERS, "card": after,
           "locks": on[-1]["locks"], "reject_ratio_sharing": on[-1]["reject_ratio_sharing"],
           "reject_ratio_same_key": on[-1]["reject_ratio_same_key"],
           "reject_ratio_option_off": off[-1]["reject_ratio_sharing"],
           "txn_per_s_on": mean(on), "txn_per_s_off": mean(off), "on_over_off": mean(on) / mean(off),
           "txn_per_s_off_spread": (max(r["txn_per_s"] for r in off) - min(r["txn_per_s"] for r in off)) / mean(off),
           "runs": runs}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
