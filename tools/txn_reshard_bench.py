#!/usr/bin/env python3
"""What re-sharding a live TATP or SmallBank cluster costs (GpuTxnClients.drain, GpuCluster.reshard_txn,
GpuTxnClients.rebind), all shards on one GPU.

For each workload: three populated shards and --clients GPU transaction clients run --rounds rounds; the clients drain;
the cluster is re-placed onto five shards and the clients rebound (the old cluster is then closed); --rounds more
rounds; drain; back onto three shards; rebind.  Source plus destination must fit on the one card, so the defaults are
TATP at S = 3,500,000 subscribers (half the reference's 7,000,000) and SmallBank at the reference's A = 24,000,000
accounts; the sizes run are printed.

Prints one JSON line per workload -- committed txn/s of the rounds before, between and after the re-shards (host clock
over run(), which synchronises), each drain's rounds and wall time, each re-shard's wall time (host clock), re-shard
kernel time (CUDA events) and row count plus allocation time (dint_reshard_times), the rebind's wall time and the free
device memory at the peak (both clusters resident) -- then one summary line with the card's name, power limit and SM
clock, read in the same run.

    python tools/txn_reshard_bench.py [--workloads tatp,smallbank] [--clients N] [--rounds R]
                                      [--subscribers S] [--accounts A] [--json FILE]
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


def max_batch(clients, G):
    return (clients + G - 1) // G * 3


def run_rounds(tc, rounds):
    st0 = tc.stats()
    t0 = time.perf_counter()
    tc.run(rounds)
    dt = time.perf_counter() - t0
    st1 = tc.stats()
    return {"rounds": rounds, "s": round(dt, 4), "committed_txn_per_s": round((st1["committed"] - st0["committed"]) / dt, 1)}


def measure(name, clients, rounds, keys):
    import torch
    from dint_b200 import GpuCluster, GpuTxnClients, wire
    from dint_b200.engine import reshard_times
    kind = wire.TATP if name == "tatp" else wire.SMALLBANK
    size = {"subs_sizing": keys, "subs_populate": keys} if name == "tatp" else {"accts_sizing": keys, "accts_populate": keys}
    r = {"workload": name, "keys": keys, "clients": clients, "steps": []}
    t0 = time.perf_counter()
    cl = GpuCluster(kind, 3, devices=[0] * 3, max_batch=max_batch(clients, 3), populate=True, **size)
    tc = GpuTxnClients(cl, clients, subscribers=keys)
    r["build_s"] = round(time.perf_counter() - t0, 2)
    try:
        r["steps"].append({"G": 3, **run_rounds(tc, rounds)})
        for G, G2 in ((3, 5), (5, 3)):
            t0 = time.perf_counter()
            n = tc.drain()
            drain_s = time.perf_counter() - t0
            t0 = time.perf_counter()
            new = cl.reshard_txn(G2, devices=[0] * G2, max_batch=max_batch(clients, G2))
            wall = time.perf_counter() - t0
            t = reshard_times()
            free, total = torch.cuda.mem_get_info(0)
            t0 = time.perf_counter()
            tc.rebind(new)
            rebind_s = time.perf_counter() - t0
            cl.close()
            cl = new
            r["steps"].append({"from": G, "to": G2, "drain_rounds": n, "drain_s": round(drain_s, 4),
                               "reshard_wall_s": round(wall, 4), "reshard_kernel_s": round(t["kernel_s"], 4),
                               "reshard_count_alloc_s": round(t["count_alloc_s"], 4), "rebind_s": round(rebind_s, 4),
                               "peak_free_gib": round(free / 2**30, 2), "total_gib": round(total / 2**30, 2)})
            if G2 == 5:
                r["steps"].append({"G": 5, **run_rounds(tc, rounds)})
        r["steps"].append({"G": 3, **run_rounds(tc, rounds)})
        st = tc.stats()
        r["committed"], r["rounds_served"], r["fallback_rounds"] = st["committed"], st["rounds"], st["fallback_rounds"]
    finally:
        tc.close()
        cl.close()
    return r


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--workloads", default="tatp,smallbank")
    ap.add_argument("--clients", type=int, default=1 << 20)
    ap.add_argument("--rounds", type=int, default=50)
    ap.add_argument("--subscribers", type=int, default=3_500_000, help="TATP kSubscriberNum")
    ap.add_argument("--accounts", type=int, default=24_000_000, help="SmallBank kAccountNum")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("txn_reshard_bench: no CUDA device (there is nothing to measure without one)")
    runs = []
    for name in a.workloads.split(","):
        r = measure(name, a.clients, a.rounds, a.subscribers if name == "tatp" else a.accounts)
        print(json.dumps(r), flush=True)
        runs.append(r)
    out = {"card": card(), "runs": runs}
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f)


if __name__ == "__main__":
    main()
