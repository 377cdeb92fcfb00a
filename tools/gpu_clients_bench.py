#!/usr/bin/env python3
"""Live lock_2pl / store / log_server / lock_fasst closed loops on the GPU (GpuClients), one engine per workload, or
against a shard cluster (GpuClusterClients, --shards).

2^20 clients per workload at the reference's sizes:
  lock2pl_ref       lock_2pl, 24,000,000 ids uniform on 36,000,000 lock slots
  lock2pl_hot       lock_2pl, 4800 ids, Zipf 0.8
  store_parallel    store, 2,000,000 populated subscribers, no kSet
  store_contention  store, 2,000,000 populated subscribers, 50 % kSet
  log               log_server, default ring (1,000,000 entries)
  fasst_ref         lock_fasst, 24,000,000 ids uniform (the workload bench.py's gpu_clients row runs)
Per workload: warm up, then time at least --min-seconds of rounds with CUDA events on the run's stream (one call of
run(); the rounds are sized by a short calibration).  Reports committed txn/s, requests/s, microseconds per round and
the validation-abort / lock-reject / not-exist counts of the timed rounds; the card's SM clock is read again right
after.  With --check R, the first R rounds are also replayed through the host clients (Workload) and a fresh engine
fed by dint_submit; the counters must be identical.  Prints one JSON line per workload.

    python tools/gpu_clients_bench.py [--workloads a,b,...] [--clients N] [--warmup W] [--min-seconds S] [--check R]
"""
import argparse
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from txn_clients_bench import card  # noqa: E402  (the same read-only queries)

WORKLOADS = {
    # name: (kind name, engine options, client family)
    "lock2pl_ref": ("LOCK2PL", {}, dict(n_keys=24_000_000)),
    "lock2pl_hot": ("LOCK2PL", {}, dict(n_keys=4800, zipf_theta=0.8)),
    "store_parallel": ("STORE", dict(populate=True), dict(store_subscribers=2_000_000, set_pct=0)),
    "store_contention": ("STORE", dict(populate=True), dict(store_subscribers=2_000_000, set_pct=50)),
    "log": ("LOG", {}, {}),
    "fasst_ref": ("FASST", {}, dict(n_keys=24_000_000)),
}
SEED = 20230


def measure(name, clients, warmup, min_seconds):
    import torch
    from dint_b200 import Engine, GpuClients, wire
    kind_name, eng_opt, fam = WORKLOADS[name]
    kind = getattr(wire, kind_name)
    res = {"workload": name, "kind": wire.KIND_NAMES[kind], "clients": clients, "family": fam}
    with Engine(kind, **eng_opt) as eng, GpuClients(eng, clients, seed=SEED, **fam) as gc:
        stream = torch.cuda.current_stream()
        gc.run(warmup, stream.cuda_stream)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        gc.run(16, stream.cuda_stream)
        e1.record(stream)
        torch.cuda.synchronize()
        rounds = max(16, math.ceil(1.1 * min_seconds * 1e3 / (e0.elapsed_time(e1) / 16)))
        s0 = gc.stats()
        e0.record(stream)
        gc.run(rounds, stream.cuda_stream)
        e1.record(stream)
        torch.cuda.synchronize()
        s1 = gc.stats()
        res["card_after_timed"] = card()              # the SM clock while the card is still warm
        conflicted = eng.stats()["conflicted"]
    sec = e0.elapsed_time(e1) * 1e-3
    d = {k: s1[k] - s0[k] for k in s1}
    res.update(rounds_timed=rounds, timed_s=round(sec, 4), txn_per_s=d["committed"] / sec, requests_per_s=d["requests"] / sec,
               us_per_round=1e6 * sec / rounds, committed=d["committed"], validation_aborts=d["validation_aborts"],
               lock_rejects=d["lock_rejects"], not_exist=d["not_exist"], engine_conflicted_total=conflicted)
    print(f"[{name}] {rounds} rounds in {sec:.3f} s", flush=True)
    return res


def check(name, clients, rounds):
    """the first `rounds` rounds: GPU clients vs the host clients through dint_submit on a fresh engine"""
    from dint_b200 import Engine, GpuClients, wire
    from dint_b200.workloads import Workload
    kind_name, eng_opt, fam = WORKLOADS[name]
    kind = getattr(wire, kind_name)
    with Engine(kind, **eng_opt) as eng, GpuClients(eng, clients, seed=SEED, **fam) as gc:
        gc.run(rounds)
        got = gc.stats()
    with Engine(kind, **eng_opt) as eng:
        wl = Workload(kind, n_clients=clients, seed=SEED, **fam)
        for _ in range(rounds):
            wl.feed(eng.submit(wl.next()))
        want = wl.stats()
        wl.close()
    return {"check_rounds": rounds, "check_identical": got == want, "check_stats": got}


def measure_cluster(name, clients, G, devices, warmup, min_seconds):
    import torch
    from dint_b200 import GpuCluster, GpuClusterClients, wire
    kind_name, eng_opt, fam = WORKLOADS[name]
    kind = getattr(wire, kind_name)
    res = {"workload": name, "kind": wire.KIND_NAMES[kind], "clients": clients * G, "clients_per_rank": clients,
           "shards": G, "devices": devices, "family": fam}
    with GpuCluster(kind, G, devices=devices, max_batch=clients, **eng_opt) as cl, \
            GpuClusterClients(cl, clients * G, seed=SEED, **fam) as cc:
        cc.run(warmup)
        s0, m0 = cc.stats(), cc.times()
        rounds, t0 = 0, time.perf_counter()
        while True:
            cc.run(10)
            rounds += 10
            wall = time.perf_counter() - t0
            if wall >= min_seconds:
                break
        torch.cuda.synchronize()
        s1, m1 = cc.stats(), cc.times()
        res["card_after_timed"] = card()              # the SM clock while the card is still warm
    dwall, ddev = m1["wall_s"] - m0["wall_s"], m1["device_s"] - m0["device_s"]
    d = {k: s1[k] - s0[k] for k in s1}
    res.update(rounds_timed=rounds, timed_s=round(wall, 4), txn_per_s=d["committed"] / wall, requests_per_s=d["requests"] / wall,
               us_per_round=1e6 * wall / rounds, round_device_us=1e6 * ddev / rounds,
               exposed_host_us_per_round=1e6 * (dwall - ddev) / rounds, fallback_rounds=d["fallback_rounds"],
               committed=d["committed"], validation_aborts=d["validation_aborts"], lock_rejects=d["lock_rejects"],
               not_exist=d["not_exist"])
    print(f"[{name}] {G} shards: {rounds} rounds in {wall:.3f} s", flush=True)
    return res


def check_cluster(name, clients, G, devices, rounds):
    """the first `rounds` rounds: cluster clients vs GpuClients with the same clients on one engine"""
    import numpy as np
    from dint_b200 import Engine, GpuCluster, GpuClients, GpuClusterClients, wire
    kind_name, eng_opt, fam = WORKLOADS[name]
    kind = getattr(wire, kind_name)
    with GpuCluster(kind, G, devices=devices, max_batch=clients, **eng_opt) as cl, \
            GpuClusterClients(cl, clients * G, seed=SEED, **fam) as cc:
        cc.run(rounds)
        got, got_io = cc.stats(), cc.peek()
    with Engine(kind, **eng_opt) as eng, GpuClients(eng, clients * G, seed=SEED, **fam) as gc:
        gc.run(rounds)
        want, want_io = gc.stats(), gc.peek()
    same = {k: v for k, v in got.items() if k != "fallback_rounds"} == want and \
        all(np.array_equal(a, b) for a, b in zip(got_io, want_io))
    return {"check_rounds": rounds, "check_identical": same, "check_stats": got}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--clients", type=int, default=1 << 20)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--check", type=int, default=0, metavar="R")
    ap.add_argument("--shards", type=int, default=0, metavar="G")
    ap.add_argument("--devices", default=None, metavar="d0,d1,...")
    a = ap.parse_args()
    names = a.workloads.split(",")
    for n in names:
        if n not in WORKLOADS:
            ap.error(f"unknown workload {n!r}; known: {', '.join(WORKLOADS)}")
    devices = None
    if a.shards:
        devices = [int(d) for d in a.devices.split(",")] if a.devices else [0] * a.shards
        if len(devices) != a.shards:
            ap.error("--devices must name one device per shard")
    elif a.devices:
        ap.error("--devices needs --shards")
    print(json.dumps({"card": card()}), flush=True)
    ok = True
    for n in names:
        if a.shards:
            r = measure_cluster(n, a.clients, a.shards, devices, a.warmup, a.min_seconds)
            if a.check:
                r.update(check_cluster(n, a.clients, a.shards, devices, a.check))
        else:
            r = measure(n, a.clients, a.warmup, a.min_seconds)
            if a.check:
                r.update(check(n, a.clients, a.check))
        if a.check:
            ok &= r["check_identical"]
        print(f"[{n}] {r['txn_per_s'] / 1e6:.2f} M txn/s, {r['requests_per_s'] / 1e6:.1f} M req/s, {r['us_per_round']:.0f} us/round"
              + (f", {r['exposed_host_us_per_round']:.0f} us exposed host, {r['fallback_rounds']} fallback rounds" if a.shards else "")
              + (f" | check of {a.check} rounds identical: {r['check_identical']}" if a.check else ""), flush=True)
        print(json.dumps(r), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
