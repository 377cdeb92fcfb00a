"""The eBPF store's cache tier under live closed loops: GpuClients of the store (the reference's REF family, 2,000,000
populated subscribers, store/caladan/client_ebpf.cc:61-63) against one engine without the tier and one per variant
(store_ebpf = wb_bloom / wb / wt), all at the reference's sizes, alternated in one process.

Workloads: parallel (GET only) and contention (set_pct = 20).  Each measurement runs `--warmup` rounds, then at least
`--seconds` of rounds timed with CUDA events, and reports committed txn/s, µs per round, the hit ratio (requests answered
from a cache set), write-backs and installs per 1000 requests, and requests that took the ordered replay per 1000.  The
card's name, power limit and SM clock are read in the same run.  Prints one JSON object.

usage: python tools/store_cache_bench.py [--clients 1048576] [--repeats 2] [--seconds 1.0] [--warmup 8]
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from txn_clients_bench import card  # noqa: E402  (read-only device queries)

VARIANTS = (None, "wb_bloom", "wb", "wt")
WORKLOADS = {"parallel": 0, "contention": 20}
SEED = 20230


def measure(eng, clients, set_pct, warmup, min_seconds):
    import torch
    from dint_b200 import GpuClients
    with GpuClients(eng, clients, seed=SEED, store_subscribers=2_000_000, set_pct=set_pct) as gc:
        stream = torch.cuda.current_stream()
        gc.run(warmup, stream.cuda_stream)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        gc.run(8, stream.cuda_stream)
        e1.record(stream)
        torch.cuda.synchronize()
        rounds = max(8, math.ceil(1.1 * min_seconds * 1e3 / (e0.elapsed_time(e1) / 8)))
        s0, c0 = gc.stats(), eng.stats()["conflicted"]
        k0 = eng.store_cache_stats() if eng.cfg.flags & 6 else None
        e0.record(stream)
        gc.run(rounds, stream.cuda_stream)
        e1.record(stream)
        torch.cuda.synchronize()
        s1, c1 = gc.stats(), eng.stats()["conflicted"]
        k1 = eng.store_cache_stats() if k0 is not None else None
    sec = e0.elapsed_time(e1) * 1e-3
    req = s1["requests"] - s0["requests"]
    out = dict(rounds_timed=rounds, timed_s=round(sec, 4), txn_per_s=(s1["committed"] - s0["committed"]) / sec,
               us_per_round=round(1e6 * sec / rounds, 1), requests=req, not_exist=s1["not_exist"] - s0["not_exist"],
               conflicted_per_1000=round(1000 * (c1 - c0) / req, 2))
    if k0 is not None:
        d = {k: k1[k] - k0[k] for k in k1}
        out.update(hit_ratio=round(d["hits"] / req, 4), write_backs_per_1000=round(1000 * d["write_backs"] / req, 2),
                   installs_per_1000=round(1000 * d["installs"] / req, 2),
                   bloom_negatives_per_1000=round(1000 * d["bloom_negatives"] / req, 2))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clients", type=int, default=1 << 20)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=8)
    a = ap.parse_args()
    from dint_b200 import Engine, wire
    engines = {}
    try:
        for v in VARIANTS:
            engines[v] = Engine(wire.STORE, device=0, populate=True, store_ebpf=v)
            print(f"[store_cache_bench] populated {v or 'off'}", file=sys.stderr, flush=True)
        res = {"clients": a.clients, "card": card(), "runs": []}
        for rep in range(a.repeats):
            for wl, set_pct in WORKLOADS.items():
                for v in VARIANTS:           # alternated: every configuration sees the same card state in turn
                    r = measure(engines[v], a.clients, set_pct, a.warmup, a.seconds)
                    r.update(repeat=rep, workload=wl, store_ebpf=v or "off")
                    res["runs"].append(r)
                    print(f"[store_cache_bench] {wl} {v or 'off'}: {r['txn_per_s'] / 1e6:.1f} M txn/s", file=sys.stderr,
                          flush=True)
        res["card_after"] = card()
    finally:
        for e in engines.values():
            e.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
