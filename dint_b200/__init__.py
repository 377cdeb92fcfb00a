"""dint_b200 -- GPU-resident (H100) batched implementation of DINT's per-request server hot path.

    from dint_b200 import Engine, wire
    eng = Engine(wire.FASST)            # stands in for `lock_fasst/udp/server 1`
    resp = eng.submit(requests)         # packed wire structs in, packed wire structs out
"""
from . import wire
from .engine import Engine, GpuCluster, GpuClients, GpuClusterClients, GpuTxnClients, PinnedBuffer, DintError, default_cfg, lib

__all__ = ["Engine", "GpuCluster", "GpuClients", "GpuClusterClients", "GpuTxnClients", "PinnedBuffer", "DintError", "default_cfg", "lib", "wire"]
