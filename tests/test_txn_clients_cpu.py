"""CPU: the TATP and SmallBank client state machines (dint_b200/csrc/txn_clients.cuh) are one statement shared by
the host drivers (libdint_wl.so, TxnWorkload) and the GPU clients (GpuTxnClients).  These digests of the host
request streams, destinations and final counters were recorded before the state machines moved into the shared
header; the host streams must stay bit-identical to them.  (TATP needs G >= 3 against the oracles: on one shard a
backup commit meets the primary's own lock, which the reference server refuses.)"""
import hashlib
import json

import numpy as np
import pytest

import oracle_lib as O
from dint_b200 import wire
from dint_b200.txn_workloads import Cluster, TxnWorkload

ROUNDS = 50

DIGESTS = {
    ("tatp", 3): "4b011014e52fbdfdc79c4190b8aed47b2a97cd65380df28ac328259bfc047904",
    ("tatp", 4): "83890775b7515242247709a584256048d2f2ec95dcfb918526669ca984923fd3",
    ("tatp", 5): "fe80470bd8bc5cfd9f121a90a0b4000fb691ce519254691aa7fd33352b6b480a",
    ("smallbank", 1): "7988c53c8cedaed369b621ee249974d8403645671a9c124816db89ad4c8d3a50",
    ("smallbank", 3): "ac7a488726326ef39b0918657005a0b62e980e337276a5f5b79ad5437b5d45d4",
    ("smallbank", 8): "250eb366b9775fcef48132fc754d879f44441242d93fd1efeae355ce0df18788",
}


def _digest(kind, G):
    n, clients = (3000, 1100) if kind == wire.TATP else (5000, 1300)
    cfg = dict(subs_populate=n) if kind == wire.TATP else dict(accts_populate=n)
    msg = wire.MSG_SIZE[kind]
    oras = [O.Oracle(kind, **cfg) for _ in range(G)]
    cl = Cluster([o.process for o in oras], msg)
    wl = TxnWorkload(kind, n_clients=clients, n_shards=G, subscribers=n, gid0=17)
    h = hashlib.sha256()
    for _ in range(ROUNDS):
        rq, dst = wl.next()
        h.update(np.uint64(dst.size).tobytes())
        h.update(rq.tobytes())
        h.update(dst.tobytes())
        wl.feed(cl.submit(rq, dst))
    st = wl.stats()
    h.update(json.dumps(st, sort_keys=True).encode())
    return h.hexdigest(), st


@pytest.mark.parametrize("name,G", list(DIGESTS))
def test_host_txn_streams_are_unchanged(name, G):
    kind = wire.TATP if name == "tatp" else wire.SMALLBANK
    got, st = _digest(kind, G)
    assert st["committed"] > 0 and st["rounds"] == ROUNDS
    assert got == DIGESTS[(name, G)], (name, G, got)
