"""No GPU needed: tools/reshard_image.py reads the cluster manifest first and refuses the kinds that cannot be
re-sharded (tatp, smallbank, log_server) before it touches a GPU."""
import os
import struct
import subprocess
import sys

import pytest

from dint_b200 import default_cfg, wire

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "tools", "reshard_image.py")


def _manifest(d, kind, shards):
    """a manifest as dint_cluster_image_save writes it (include/dint_b200.h): magic, version, kind, shards, 0, cfg, 0"""
    os.makedirs(d, exist_ok=True)
    cfg = bytes(default_cfg(kind))
    with open(os.path.join(d, "manifest"), "wb") as f:
        f.write(b"DINTCLU1" + struct.pack("<4I", 1, kind, shards, 0) + cfg + struct.pack("<I", 0))
    assert os.path.getsize(os.path.join(d, "manifest")) == 104


def _run(*args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")        # a GPU, if any, must not be needed to refuse
    return subprocess.run([sys.executable, TOOL, *args], capture_output=True, text=True, timeout=120, env=env)


@pytest.mark.parametrize("kind", [wire.TATP, wire.SMALLBANK, wire.LOG])
def test_refuses_kinds_that_cannot_move(kind, tmp_path):
    src = str(tmp_path / "src")
    _manifest(src, kind, 3)
    r = _run(src, str(tmp_path / "dst"), "--shards", "5")
    assert r.returncode == 2, r.stdout + r.stderr
    assert wire.KIND_NAMES[kind] in r.stderr and "cannot be re-sharded" in r.stderr
    assert not os.path.exists(tmp_path / "dst")


def test_refuses_what_is_not_a_cluster_image(tmp_path):
    r = _run(str(tmp_path / "missing"), str(tmp_path / "dst"), "--shards", "2")
    assert r.returncode == 2 and "not a cluster image directory" in r.stderr
    src = str(tmp_path / "src")
    _manifest(src, wire.FASST, 3)
    r = _run(src, str(tmp_path / "dst"), "--shards", "9")
    assert r.returncode == 2 and "1..8" in r.stderr
