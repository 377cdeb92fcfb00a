#!/usr/bin/env python
"""A/B helper: fasst (uniform 24M ids) + store GET kernel times for the current env settings."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
from dint_b200 import Engine, wire
import trace_gen as T
from gpu_probe import probe
n = 1 << 22
tag = " ".join(f"{k}={v}" for k, v in os.environ.items() if k.startswith("DINT_"))
print("==", tag or "defaults")
# the card, its power limit and its SM clocks belong beside every time below
import subprocess
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip())
probe(wire.FASST, T.fasst_random(n, 24_000_000, seed=1, weights=(0.6, 0.15, 0.05, 0.2)), chunk=int(os.environ.get("CHUNK", 1 << 20)))
if "--store" in sys.argv:
    probe(wire.STORE, T.store_random(n, 2_000_000, seed=4, p_set=0.0, p_miss=0.0), chunk=1 << 20, populate=True)
if "--hot" in sys.argv:
    probe(wire.FASST, T.fasst_random(n, 4800, seed=1), chunk=1 << 20)
    probe(wire.LOCK2PL, T.lock2pl_random(n, 4800, seed=2), chunk=1 << 20)
if "--route" in sys.argv:   # dispatch / combine kernels alone
    # dispatch / combine kernels alone, local slabs (no NVLink): 2^20 lock_fasst records
    from dint_b200.engine import Engine as E_
    m = 1 << 20
    req = torch.from_numpy(T.fasst_random(m, 24_000_000, seed=1, weights=(0.6, 0.15, 0.05, 0.2))).cuda().view(torch.uint8).reshape(-1)
    for W in (1, 2, 8):
        eng = Engine(wire.FASST, n_shards=W, shard_id=0)
        cap = (int(m / W * 1.02) + 8 * int((m / W) ** 0.5) + 64 + 15) // 16 * 16
        slabs = torch.empty(W * cap * 9, dtype=torch.uint8, device="cuda")
        flags = torch.zeros(2, dtype=torch.int32, device="cuda")
        ptrs = E_.slab_ptrs(slabs.data_ptr(), W, cap * 9)
        out = torch.empty(m * 9, dtype=torch.uint8, device="cuda")
        state = eng.route_state(m, req.device)
        for _ in range(5):
            eng.route_dispatch(req, m, W, 0, cap, ptrs, flags, state=state); eng.route_combine(ptrs, state, m, W, cap, out)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(50): eng.route_dispatch(req, m, W, 0, cap, ptrs, flags, state=state)
        ev[1].record()
        for _ in range(50): eng.route_combine(ptrs, state, m, W, cap, out)
        ev[2].record(); torch.cuda.synchronize()
        print(f"route W={W}: dispatch {ev[0].elapsed_time(ev[1]) * 20:.1f} us  combine {ev[1].elapsed_time(ev[2]) * 20:.1f} us  roundtrip ok={bool(torch.equal(out, req))} flags={flags.tolist()}")
        eng.close()
