#!/usr/bin/env python3
"""Live TATP / SmallBank closed loops on the GPU (GpuTxnClients) against the host clients (TxnWorkload).

The setup of bench.py's txn workloads: 2^20 clients and three full-population shards on one GPU (tatp: 7,000,000
subscribers; smallbank: 24,000,000 accounts).  Per kind:
  1. GPU clients: warm up, then time at least --min-seconds of live rounds on the host clock (run() returns after
     its device work is done and checked); the card's SM clock is read again right after.  Reports txn/s
     (committed), requests/s, the abort rate, the commit rate per type, fallback_rounds, and the host time each
     round leaves exposed: wall time minus the CUDA-event time of the round's device work.
  2. Host clients, on a freshly populated cluster: the same number of rounds through TxnWorkload + GpuCluster.submit.
     Run after the first cluster is closed -- six full TATP shards do not fit 80 GB.
The final counters of the two runs must be identical.  Prints one JSON line per kind at the end.

    python tools/txn_clients_bench.py [--kind tatp|smallbank|both] [--clients N] [--warmup W] [--min-seconds S]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    """name, power limit and SM clock of device 0 (read-only queries)"""
    try:
        import pynvml as N
        N.nvmlInit()
        h = N.nvmlDeviceGetHandleByIndex(0)
        name = N.nvmlDeviceGetName(h)
        return {"name": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": N.nvmlDeviceGetPowerManagementLimit(h) / 1000.0,
                "sm_mhz": N.nvmlDeviceGetClockInfo(h, N.NVML_CLOCK_SM),
                "sm_max_mhz": N.nvmlDeviceGetMaxClockInfo(h, N.NVML_CLOCK_SM)}
    except Exception:
        pass
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"name": q[0], "power_limit_w": float(q[1]), "sm_mhz": int(q[2]), "sm_max_mhz": int(q[3])}
    except Exception as ex:
        return {"unavailable": repr(ex)[:200]}


def measure(kind_name, clients, warmup, min_seconds):
    import torch
    from dint_b200 import GpuCluster, GpuTxnClients, wire
    from dint_b200.txn_workloads import TxnWorkload
    kind = wire.TATP if kind_name == "tatp" else wire.SMALLBANK
    subscribers = 7_000_000 if kind == wire.TATP else 24_000_000
    G = 3
    per_rank = (clients + G - 1) // G
    # batch size of one rank's round: measured rounds stay below 1.6 (tatp) and 3 (smallbank) records per client
    max_batch = (3 if kind == wire.TATP else 4) * per_rank
    res = {"kind": kind_name, "clients": clients, "shards": G, "keys": subscribers}

    # ---- 1. the clients on the GPU ----
    t0 = time.perf_counter()
    with GpuCluster(kind, G, devices=[0] * G, max_batch=max_batch, populate=True) as cl:
        res["populate_s"] = round(time.perf_counter() - t0, 1)
        with GpuTxnClients(cl, clients, subscribers=subscribers) as tc:
            tc.run(warmup)
            s0, m0 = tc.stats(), tc.times()
            rounds, t0 = 0, time.perf_counter()
            while True:
                tc.run(10)
                rounds += 10
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
                if wall >= min_seconds:
                    break
            s1, m1 = tc.stats(), tc.times()
            res["card_after_timed"] = card()          # the SM clock while the card is still warm
    dwall, ddev = m1["wall_s"] - m0["wall_s"], m1["device_s"] - m0["device_s"]
    res["gpu_clients"] = {
        "rounds_timed": rounds, "timed_s": round(wall, 4),
        "txn_per_s": (s1["committed"] - s0["committed"]) / wall,
        "requests_per_s": (s1["requests"] - s0["requests"]) / wall,
        "abort_rate": 1.0 - s1["committed"] / max(1, s1["txns"]),
        "commit_rate_by_type": {k: round(v[1] / max(1, v[0]), 4) for k, v in s1["by_type"].items()},
        "fallback_rounds": s1["fallback_rounds"],
        "round_wall_us": 1e6 * dwall / rounds, "round_device_us": 1e6 * ddev / rounds,
        "exposed_host_us_per_round": 1e6 * (dwall - ddev) / rounds}
    print(f"[{kind_name}] gpu clients: {rounds} rounds in {wall:.3f} s", flush=True)

    # ---- 2. the host clients, same number of rounds, fresh shards ----
    with GpuCluster(kind, G, devices=[0] * G, max_batch=max_batch, populate=True) as cl:
        wl = TxnWorkload(kind, n_clients=clients, n_shards=G, subscribers=subscribers)
        for _ in range(warmup):
            rq, dst = wl.next()
            wl.feed(cl.submit(rq, dst))
        h0 = wl.stats()
        t0 = time.perf_counter()
        for _ in range(rounds):
            rq, dst = wl.next()
            wl.feed(cl.submit(rq, dst))
        hwall = time.perf_counter() - t0
        h1 = wl.stats()
    res["host_clients"] = {"rounds_timed": rounds, "timed_s": round(hwall, 4),
                           "txn_per_s": (h1["committed"] - h0["committed"]) / hwall,
                           "requests_per_s": (h1["requests"] - h0["requests"]) / hwall}
    res["stats_identical"] = {k: v for k, v in s1.items() if k != "fallback_rounds"} == h1
    res["final_stats"] = s1
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--kind", choices=["tatp", "smallbank", "both"], default="both")
    ap.add_argument("--clients", type=int, default=1 << 20)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    a = ap.parse_args()
    kinds = ["tatp", "smallbank"] if a.kind == "both" else [a.kind]
    print(json.dumps({"card": card()}), flush=True)
    out = [measure(k, a.clients, a.warmup, a.min_seconds) for k in kinds]
    ok = True
    for r in out:
        g, h = r["gpu_clients"], r["host_clients"]
        print(f"[{r['kind']}] GPU clients {g['txn_per_s'] / 1e6:.2f} M txn/s, {g['requests_per_s'] / 1e6:.2f} M req/s | host clients "
              f"{h['txn_per_s'] / 1e6:.3f} M txn/s | abort rate {g['abort_rate']:.4f} | round {g['round_wall_us']:.0f} us wall, "
              f"{g['round_device_us']:.0f} us device, {g['exposed_host_us_per_round']:.0f} us exposed | fallback rounds "
              f"{g['fallback_rounds']} | stats identical: {r['stats_identical']}")
        print(json.dumps(r))
        ok &= r["stats_identical"]
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
