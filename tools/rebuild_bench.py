#!/usr/bin/env python3
"""What rebuilding a lost tatp / smallbank shard costs (dint_cluster_rebuild, dint_cluster_image_open_rebuild), all
shards on one GPU.

Workloads: three TATP shards at the reference's S = 7,000,000 subscribers and three SmallBank shards at A = 24,000,000
accounts, each fully populated and then driven by --rounds rounds of 2^20 GPU transaction clients (closed before the
rebuild).  For each: shard 1 is rebuilt in place from its replicas; then the cluster is saved as an image, opened whole,
and opened again with shard-1.img removed (rebuilt from the other two shard images).

Prints one JSON line per workload -- the rebuild's wall time (host clock; the call synchronises), the rebuild kernels'
CUDA-event time, the row count plus the new engine's allocation (host clock), the rows rebuilt, and the two opens' wall
times -- then one summary line with the card's name, power limit and SM clock, read in the same run.

    python tools/rebuild_bench.py [--workloads tatp,smallbank] [--rounds R] [--dir TMPDIR] [--no-image]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from txn_clients_bench import card  # noqa: E402

G, CLIENTS = 3, 1 << 20


def build(name, rounds):
    from dint_b200 import GpuCluster, GpuTxnClients, wire
    kind = wire.TATP if name == "tatp" else wire.SMALLBANK
    keys = 7_000_000 if name == "tatp" else 24_000_000
    t0 = time.perf_counter()
    cl = GpuCluster(kind, G, devices=[0] * G, max_batch=(CLIENTS + G - 1) // G * 3, populate=True)
    with GpuTxnClients(cl, CLIENTS, subscribers=keys) as tc:
        tc.run(rounds)
    return cl, kind, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--workloads", default="tatp,smallbank")
    ap.add_argument("--rounds", type=int, default=100)
    ap.add_argument("--dir", default=None, help="where the cluster images go (default: a temporary directory)")
    ap.add_argument("--no-image", action="store_true", help="time the live rebuild only")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("rebuild_bench: no CUDA device (there is nothing to measure without one)")
    from dint_b200 import GpuCluster
    from dint_b200.engine import rebuild_times
    runs = []
    for name in a.workloads.split(","):
        cl, kind, built = build(name, a.rounds)
        n_tables = 5 if name == "tatp" else 2
        t0 = time.perf_counter()
        cl.rebuild([1])
        wall = time.perf_counter() - t0
        t = rebuild_times()
        rows = sum(cl.engine(1).kv_count(i) for i in range(n_tables))
        r = {"workload": name, "shards": G, "rounds": a.rounds, "build_s": round(built, 2), "rebuild_wall_s": round(wall, 4),
             "rebuild_kernel_s": round(t["kernel_s"], 4), "rebuild_count_alloc_s": round(t["count_alloc_s"], 4), "rows": rows}
        base = None if a.no_image else tempfile.mkdtemp(prefix="rebuild_bench_", dir=a.dir)
        need = 24 << 30 if name == "tatp" else 8 << 30           # the three shard images, with room to spare
        if base and shutil.disk_usage(base).free < need:
            r["image"] = f"skipped: {shutil.disk_usage(base).free >> 30} GiB free, the images need about {need >> 30} GiB"
            shutil.rmtree(base, ignore_errors=True)
            base = None
        if base:
            try:
                d = os.path.join(base, "img")
                cl.save_image(d)
                cl.close()
                t0 = time.perf_counter()
                GpuCluster.open_image(d, devices=[0] * G).close()
                r["open_whole_s"] = round(time.perf_counter() - t0, 3)
                os.remove(os.path.join(d, "shard-1.img"))
                t0 = time.perf_counter()
                with GpuCluster.open_image(d, devices=[0] * G, rebuild=True) as c:
                    r["open_rebuild_s"] = round(time.perf_counter() - t0, 3)
                    t = rebuild_times()
                    r["open_rebuild_kernel_s"] = round(t["kernel_s"], 4)
                    assert c.rebuilt == [1] and sum(c.engine(1).kv_count(i) for i in range(n_tables)) == rows
            finally:
                shutil.rmtree(base, ignore_errors=True)
        cl.close()
        print(json.dumps(r), flush=True)
        runs.append(r)
    print(json.dumps({"card": card(), "runs": runs}))


if __name__ == "__main__":
    main()
