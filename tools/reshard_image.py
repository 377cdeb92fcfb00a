#!/usr/bin/env python3
"""Re-shard a saved cluster image onto another shard count, offline.

    python tools/reshard_image.py SRC_DIR DST_DIR --shards N [--device D] [--replicas]

SRC_DIR is a directory written by GpuCluster.save_image / dint_cluster_image_save (or by `dint_udp_server --image-out`
with G shards).  The tool opens it with every shard on device D, re-shards it to N shards (dint_cluster_reshard) and
saves the result to DST_DIR; `dint_udp_server --gpus N --image-in DST_DIR` then serves the same state from N GPUs, and
SRC_DIR is left as it was.  Peak device memory is the saved state twice, on the one device.

lock_2pl, lock_fasst and store clusters only: the manifest is read first, and a tatp, smallbank or log_server cluster is
refused (exit code 2) before any GPU is touched -- their shard count is the clients' replica placement or the rank
that received a record, not a layout of one server's state.

--replicas: tatp and smallbank clusters only (N = 1 or 3..8).  Every row is re-placed on its replicas under N shards,
copied from the key's old primary (dint_cluster_reshard_txn).  The image must have been saved with no lock held
(after population, or with the clients drained); one saved mid-transaction is refused by the library (exit code 1).
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dint_b200 import wire  # noqa: E402
from dint_b200.engine import read_image_header  # noqa: E402

MOVABLE = (wire.LOCK2PL, wire.FASST, wire.STORE)
REPLICATED = (wire.TATP, wire.SMALLBANK)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("src", help="cluster image directory to read")
    ap.add_argument("dst", help="directory to write the re-sharded image to")
    ap.add_argument("--shards", type=int, required=True, help="shard count of the result (1..8)")
    ap.add_argument("--device", type=int, default=0, help="CUDA device that holds both clusters while the tool runs")
    ap.add_argument("--replicas", action="store_true", help="tatp / smallbank: re-place every row on its replicas under N shards")
    a = ap.parse_args(argv)
    if not os.path.isdir(a.src):
        print(f"reshard_image: {a.src} is not a cluster image directory", file=sys.stderr)
        return 2
    try:
        hdr = read_image_header(a.src)
    except (OSError, ValueError) as e:
        print(f"reshard_image: {a.src}: cannot read the manifest: {e}", file=sys.stderr)
        return 2
    if hdr["magic"] != b"DINTCLU1":
        print(f"reshard_image: {a.src}: not a dint_b200 cluster manifest", file=sys.stderr)
        return 2
    kind = hdr["kind"]
    if a.replicas:
        if kind not in REPLICATED:
            name = wire.KIND_NAMES[kind] if 0 <= kind < len(wire.KIND_NAMES) else f"kind {kind}"
            print(f"reshard_image: --replicas re-places tatp / smallbank replicas; {a.src} holds a {name} cluster", file=sys.stderr)
            return 2
        if a.shards not in (1, 3, 4, 5, 6, 7, 8):
            print("reshard_image: --replicas --shards must be 1 or 3..8 (primary + 2 backups)", file=sys.stderr)
            return 2
    elif kind not in MOVABLE:
        name = wire.KIND_NAMES[kind] if 0 <= kind < len(wire.KIND_NAMES) else f"kind {kind}"
        why = ("a record belongs to the rank that received it" if kind == wire.LOG else
               "its shard count is the clients' replica placement (primary key % G, backups +1 and +2)")
        print(f"reshard_image: {a.src} holds a {name} cluster, which cannot be re-sharded: {why}", file=sys.stderr)
        return 2
    if not 1 <= a.shards <= 8:
        print("reshard_image: --shards must be 1..8", file=sys.stderr)
        return 2
    if os.path.abspath(a.src) == os.path.abspath(a.dst):
        print("reshard_image: DST_DIR must differ from SRC_DIR", file=sys.stderr)
        return 2
    from dint_b200 import GpuCluster
    from dint_b200.engine import DintError, reshard_times
    t0 = time.perf_counter()
    with GpuCluster.open_image(a.src, devices=[a.device] * hdr["shards"]) as src:
        t1 = time.perf_counter()
        try:
            dst = (src.reshard_txn if a.replicas else src.reshard)(a.shards, devices=[a.device] * a.shards)
        except DintError as e:
            print(f"reshard_image: {e}", file=sys.stderr)
            return 1
        with dst:
            rt = reshard_times()
            t2 = time.perf_counter()
            dst.save_image(a.dst)
            t3 = time.perf_counter()
    print(json.dumps({"src": a.src, "dst": a.dst, "kind": wire.KIND_NAMES[kind], "from_shards": hdr["shards"],
                      "to_shards": a.shards, "open_s": round(t1 - t0, 3), "reshard_s": round(t2 - t1, 3),
                      "reshard_kernel_s": round(rt["kernel_s"], 3), "save_s": round(t3 - t2, 3)}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
