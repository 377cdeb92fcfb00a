#!/usr/bin/env python3
"""What re-sharding a cluster costs (dint_cluster_reshard), all shards on one GPU.

Workloads: lock_fasst at the reference's 36,000,000 lock slots after --rounds rounds of 2^20 GPU clients (REF: uniform
over 24 M ids); the store at 24 M keys (2,000,000 subscribers populated); the store with the eBPF wb_bloom cache tier,
populated through the tier.  Each starts as one shard and is re-sharded 1 -> 3 -> 8 -> 3 -> 1, the source closed after
each step (peak memory is source plus destination).

Prints one JSON line per transition -- the wall time of the call (host clock; the call synchronises), the re-shard
kernels' CUDA-event time summed over the destination shards, and the key count plus the allocation and zeroing of the
destination engines (host clock) -- then one summary line with the card's name, power limit and SM clock, read in the
same run.

    python tools/reshard_bench.py [--workloads a,b] [--rounds R] [--chain 1,3,8,3,1]
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

WORKLOADS = ["lock_fasst", "store", "store_wb_bloom"]


def build(name, rounds):
    """a one-shard cluster holding the workload's state, and the seconds it took to build"""
    import torch
    from dint_b200 import GpuCluster, GpuClusterClients, wire
    from dint_b200.workloads import REF
    t0 = time.perf_counter()
    if name == "lock_fasst":
        n = 1 << 20
        cl = GpuCluster(wire.FASST, 1, devices=[0], max_batch=n)
        with GpuClusterClients(cl, n, **REF) as cc:
            cc.run(rounds)
    else:
        cl = GpuCluster(wire.STORE, 1, devices=[0], populate=True, store_ebpf="wb_bloom" if name == "store_wb_bloom" else None)
    torch.cuda.synchronize()
    return cl, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--rounds", type=int, default=50)
    ap.add_argument("--chain", default="1,3,8,3,1", help="shard counts, the first is the starting cluster's")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("reshard_bench: no CUDA device (there is nothing to measure without one)")
    from dint_b200.engine import reshard_times
    chain = [int(x) for x in a.chain.split(",")]
    runs = []
    for name in a.workloads.split(","):
        cl, built = build(name, a.rounds)
        if chain[0] != 1:
            new = cl.reshard(chain[0], devices=[0] * chain[0])
            cl.close()
            cl = new
        keys = sum(cl.engine(s).kv_count(0) for s in range(cl.G)) if name.startswith("store") else None
        for G2 in chain[1:]:
            G = cl.G
            t0 = time.perf_counter()
            new = cl.reshard(G2, devices=[0] * G2)
            wall = time.perf_counter() - t0
            t = reshard_times()
            cl.close()
            cl = new
            r = {"workload": name, "from": G, "to": G2, "wall_s": round(wall, 4), "kernel_s": round(t["kernel_s"], 4),
                 "count_alloc_s": round(t["count_alloc_s"], 4), "build_s": round(built, 2)}
            if keys is not None:
                r["keys"] = keys
                assert sum(cl.engine(s).kv_count(0) for s in range(cl.G)) == keys, "a re-shard lost keys"
            print(json.dumps(r), flush=True)
            runs.append(r)
        cl.close()
    print(json.dumps({"card": card(), "runs": runs}))


if __name__ == "__main__":
    main()
