"""Rebuilding lost tatp / smallbank shards, without a GPU: the source rule (dint_test_rebuild_source) against a Python
statement of it for every shard count and lost mask, and the refusals that come before any GPU work -- the argument
checks of GpuCluster.rebuild and GpuCluster.open_image(rebuild=True), a missing manifest, and missing shard images that
cannot be rebuilt."""
import os
import struct

import pytest

from dint_b200 import GpuCluster, wire
from dint_b200 import engine as E
from dint_b200.engine import DintError

EIO = -5


def source(key, G, lost):
    """the surviving replica of `key` with the lowest role: replicas (key % G + i) % G for roles i = 0, 1, 2"""
    for i in range(3):
        s = (key % G + i) % G
        if not (lost >> s) & 1:
            return s
    return -1


def leaves_a_key_without_replica(G, lost):
    """three cyclically consecutive shards lost (G >= 4), or every shard (G = 1 or 3)"""
    if G <= 3:
        return lost == (1 << G) - 1
    return any(all((lost >> ((p + i) % G)) & 1 for i in range(3)) for p in range(G))


@pytest.mark.parametrize("G", [1, 3, 4, 5, 6, 7, 8])
def test_source_rule(G):
    L = E.lib()
    keys = list(range(3 * G)) + [(1 << 32) | 5, (1 << 63) + 11, (1 << 64) - 1, 7_000_000 * 13 + 3]
    for lost in range(1 << G):
        orphaned = False
        for k in keys:
            want = source(k, G, lost)
            assert L.dint_test_rebuild_source(k, G, lost) == want, (k, G, lost)
            orphaned |= want < 0
        assert orphaned == leaves_a_key_without_replica(G, lost), (G, lost)


def _shell(kind=wire.TATP, G=5):
    cl = GpuCluster.__new__(GpuCluster)
    cl.kind, cl.msg, cl.G, cl.h = kind, wire.MSG_SIZE[kind], G, None
    return cl


@pytest.mark.parametrize("bad", [[], [5], [-1], [1, 1], [True], ["1"], [1.0]])
def test_rebuild_argument_checks(bad):
    with pytest.raises(ValueError):
        _shell().rebuild(bad)


def test_rebuild_takes_a_list():
    with pytest.raises(TypeError):
        _shell().rebuild(1)


def test_open_image_rebuild_must_be_a_bool(tmp_path):
    with pytest.raises(TypeError):
        GpuCluster.open_image(str(tmp_path), rebuild="yes")


def test_open_image_rebuild_without_a_manifest(tmp_path):
    with pytest.raises(DintError) as ei:
        GpuCluster.open_image(str(tmp_path), rebuild=True)
    assert ei.value.code == EIO and "manifest" in str(ei.value)


def _manifest(d, kind, shards, **cfg):
    c = E.default_cfg(kind, **cfg)
    raw = b"DINTCLU1" + struct.pack("<IIII", 1, kind, shards, 0) + bytes(c) + struct.pack("<I", 0)
    assert len(raw) == E.CLUSTER_MANIFEST_BYTES
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "manifest"), "wb") as f:
        f.write(raw)


@pytest.mark.parametrize("kind,G,present,cfg,why", [
    (wire.TATP, 3, [], {}, "without a replica"),
    (wire.SMALLBANK, 5, [0, 4], {}, "without a replica"),
    (wire.FASST, 3, [0, 2], {}, "keep no replicas"),
    (wire.TATP, 3, [0, 2], dict(tatp_ebpf=True), "eBPF"),
])
def test_missing_shards_that_cannot_be_rebuilt(tmp_path, kind, G, present, cfg, why):
    """judged from the files alone, before any CUDA call: DINT_EIO naming the missing shards and the reason"""
    d = str(tmp_path / "img")
    _manifest(d, kind, G, **cfg)
    for r in present:
        open(os.path.join(d, f"shard-{r}.img"), "wb").close()
    missing = sorted(set(range(G)) - set(present))
    with pytest.raises(DintError) as ei:
        GpuCluster.open_image(d, devices=[0] * G, rebuild=True)
    msg = str(ei.value)
    assert ei.value.code == EIO and "{" + ", ".join(map(str, missing)) + "}" in msg and why in msg, msg
