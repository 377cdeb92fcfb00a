#!/usr/bin/env python3
"""What saving and opening state images costs (dint_image_save / dint_image_open, dint_cluster_image_*), against
building the same state with dint_populate.

Configurations: the store at 24 M keys (the reference's 2,000,000 subscribers), plain and with the eBPF wb_bloom cache
tier; the eBPF TATP and eBPF SmallBank servers at full size, three shards on one GPU, after --rounds rounds of 2^20 GPU
clients.  Each configuration is built once (population timed on the host clock, with a device synchronise), then saved
and opened --repeats times (default once) to a tmpfs directory and then to a directory on disk.  The state is closed before an
image is opened, so that a full-size cluster fits.

Prints one JSON line per save / open and a summary line: raw state bytes, image bytes, the wall time of the call (host
clock around the synchronising call) split into pack / unpack kernel time (CUDA events), device <-> host copy time
(CUDA events) and file time (host clock), the population time, and the card's name, power limit and SM clock.

    python tools/image_bench.py [--configs a,b] [--rounds R] [--repeats K] [--tmpfs DIR] [--disk DIR]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from txn_clients_bench import card  # noqa: E402

CONFIGS = ["store", "store_wb_bloom", "tatp_ebpf", "smallbank_ebpf"]


def build(name, rounds):
    """(handle, is_cluster, populate seconds)"""
    import torch
    from dint_b200 import Engine, GpuCluster, GpuTxnClients, wire
    t0 = time.perf_counter()
    if name.startswith("store"):
        h = Engine(wire.STORE, device=0, store_ebpf="wb_bloom" if name == "store_wb_bloom" else None)
        h.populate()
        h.sync()
        return h, False, time.perf_counter() - t0
    G, clients = 3, 1 << 20
    kind, over, subs = (wire.TATP, dict(tatp_ebpf=True), 7_000_000) if name == "tatp_ebpf" else \
        (wire.SMALLBANK, dict(smallbank_ebpf=True), 24_000_000)
    h = GpuCluster(kind, G, devices=[0] * G, max_batch=3 * ((clients + G - 1) // G), populate=True, **over)
    torch.cuda.synchronize()
    pop = time.perf_counter() - t0
    with GpuTxnClients(h, clients, subscribers=subs) as tc:
        tc.run(rounds)
    return h, True, pop


def sizes(path, cluster):
    from test_image_cpu import read_image
    files = [os.path.join(path, f) for f in sorted(os.listdir(path)) if f.endswith(".img")] if cluster else [path]
    raw = 0
    for f in files:
        hdr = read_image(f)
        raw += sum(r["bytes"] for r in hdr["regions"])
    return raw, sum(os.path.getsize(f) for f in files)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--rounds", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=1)
    ap.add_argument("--tmpfs", default="/dev/shm")
    ap.add_argument("--disk", default=tempfile.gettempdir())
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("image_bench: no CUDA device (there is nothing to measure without one)")
    from dint_b200 import Engine, GpuCluster
    from dint_b200.engine import image_times
    out = []
    for name in a.configs.split(","):
        h, cluster, pop = build(name, a.rounds)
        for rep in range(a.repeats):
            for where, base in (("tmpfs", a.tmpfs), ("disk", a.disk)):
                d = tempfile.mkdtemp(prefix="dint_image_", dir=base)
                path = d if cluster else os.path.join(d, "state.img")
                try:
                    t0 = time.perf_counter()
                    h.save_image(path)
                    save_wall = time.perf_counter() - t0
                    save = image_times()
                    raw, img = sizes(path, cluster)
                    h.close()
                    t0 = time.perf_counter()
                    h = GpuCluster.open_image(path, devices=[0] * 3, max_batch=3 * (((1 << 20) + 2) // 3)) if cluster \
                        else Engine.open_image(path)
                    torch.cuda.synchronize()
                    open_wall = time.perf_counter() - t0
                    opn = image_times()
                except Exception as e:          # e.g. a tmpfs too small for the image: reported, the next run goes on
                    r = {"config": name, "where": where, "repeat": rep, "error": str(e)}
                    print(json.dumps(r), flush=True)
                    out.append(r)
                    if getattr(h, "h", None) is None:
                        h, cluster, pop = build(name, a.rounds)
                    continue
                finally:
                    shutil.rmtree(d, ignore_errors=True)
                r = {"config": name, "where": where, "repeat": rep, "raw_bytes": raw, "image_bytes": img,
                     "ratio": img / raw, "populate_s": round(pop, 3),
                     "save_s": round(save_wall, 3), "save_pack_s": round(save["kernel_s"], 3),
                     "save_copy_s": round(save["copy_s"], 3), "save_file_s": round(save["file_s"], 3),
                     "open_s": round(open_wall, 3), "open_unpack_s": round(opn["kernel_s"], 3),
                     "open_copy_s": round(opn["copy_s"], 3), "open_file_s": round(opn["file_s"], 3)}
                print(json.dumps(r), flush=True)
                out.append(r)
        h.close()
    print(json.dumps({"card": card(), "runs": out}))


if __name__ == "__main__":
    main()
