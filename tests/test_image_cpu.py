"""State images without a GPU: the header is checked before any CUDA call, so garbage, truncated, wrong-magic,
wrong-version, unknown-kind and unknown-flag files are refused with the right code and message on any machine, and so
are cluster directories with the wrong shard count or a missing shard file.  Also home of a small reader of the
documented layout (include/dint_b200.h, "State images"), which the GPU tests use to check checksums and to place
corruptions."""
import os
import struct

import numpy as np
import pytest

from dint_b200 import engine as E, wire

EINVAL, EIO = -22, -5
HEADER = 144
REGION_REC = 24
BLOCK = 64 << 20
LINE = 128
FH_M = np.uint64(0x880355F21E6D1965)


# ---- the layout ------------------------------------------------------------------------------------------------------
def _mix(h):
    h = h ^ (h >> np.uint64(23))
    h = h * np.uint64(0x2127599BF4325C37)
    return h ^ (h >> np.uint64(47))


def fasthash64_words(words, seeds, nbytes):
    """fasthash64 of rows of u64 words (nbytes each, no tail beyond the words), one seed per row"""
    with np.errstate(over="ignore"):
        h = np.asarray(seeds, dtype=np.uint64) ^ (np.uint64(nbytes) * FH_M)
        for j in range(words.shape[1]):
            h = (h ^ _mix(words[:, j])) * FH_M
        return _mix(h)


def block_checksum(bitmap, lines, line_index):
    """sum mod 2^64 over the bitmap words (seed 2 w) and the stored lines (128 bytes zero-padded, seed 2 i + 1)"""
    w = np.arange(bitmap.size, dtype=np.uint64)
    s = fasthash64_words(bitmap.astype(np.uint64).reshape(-1, 1), w * np.uint64(2), 4)
    total = int(s.sum(dtype=np.uint64)) if s.size else 0
    if len(line_index):
        words = lines.reshape(len(line_index), LINE).view("<u8")
        total += int(fasthash64_words(words, np.asarray(line_index, np.uint64) * np.uint64(2) + np.uint64(1), LINE).sum(dtype=np.uint64))
    return total % (1 << 64)


def lines_of(raw):
    return (raw + LINE - 1) // LINE


def words_of(raw):
    return (lines_of(raw) + 127) // 128 * 4


def read_image(path):
    """{"kind", "cfg" (bytes), "version", "kv_capacity", "regions": [{"bytes", "blocks": [...]}]}; a block is a dict with
    the file offsets of its bitmap, lines and checksum, its raw length, the stored lines' raw indices and its checksum"""
    data = open(path, "rb").read()
    magic, version, kind = data[:8], *struct.unpack_from("<II", data, 8)
    n_regions = struct.unpack_from("<I", data, 92)[0]
    kv_capacity = list(struct.unpack_from("<5Q", data, 96))
    regions, off = [], HEADER
    for r in range(n_regions):
        index, _, nbytes, nblocks = struct.unpack_from("<IIQQ", data, off)
        assert index == r and nblocks == (nbytes + BLOCK - 1) // BLOCK
        regions.append({"bytes": nbytes, "blocks": []})
        off += REGION_REC
    for reg in regions:
        for b in range((reg["bytes"] + BLOCK - 1) // BLOCK):
            raw = min(BLOCK, reg["bytes"] - b * BLOCK)
            nw = words_of(raw)
            bitmap = np.frombuffer(data, "<u4", nw, off)
            bits = np.unpackbits(bitmap.view(np.uint8), bitorder="little")
            idx = np.flatnonzero(bits)
            stored = len(idx) * LINE
            L = lines_of(raw)
            if raw % LINE and len(idx) and idx[-1] == L - 1:
                stored -= LINE - raw % LINE
            blk = {"raw": raw, "bitmap_off": off, "lines_off": off + 4 * nw, "stored": stored, "line_index": idx,
                   "sum_off": off + 4 * nw + stored}
            blk["checksum"] = struct.unpack_from("<Q", data, blk["sum_off"])[0]
            off = blk["sum_off"] + 8
            reg["blocks"].append(blk)
    assert off == len(data), "trailing bytes"
    return {"magic": magic, "version": version, "kind": kind, "cfg": data[16:92], "kv_capacity": kv_capacity,
            "regions": regions, "size": len(data)}


def recompute_checksum(path, blk):
    data = open(path, "rb").read()
    nw = (blk["lines_off"] - blk["bitmap_off"]) // 4
    bitmap = np.frombuffer(data, "<u4", nw, blk["bitmap_off"])
    n = len(blk["line_index"])
    lines = np.zeros(n * LINE, np.uint8)
    lines[:blk["stored"]] = np.frombuffer(data, np.uint8, blk["stored"], blk["lines_off"])
    return block_checksum(bitmap, lines, blk["line_index"])


def write_synthetic(path, kind=wire.FASST, version=1, flags=0, magic=b"DINTIMG1", regions=()):
    """A well-formed image of `regions` (raw byte strings), as the engine would lay one out"""
    cfg = E.default_cfg(kind)
    cfg.flags = flags
    out = bytearray(magic + struct.pack("<II", version, kind) + bytes(cfg) + struct.pack("<I", len(regions)))
    out += struct.pack("<5Q", 0, 0, 0, 0, 0) + struct.pack("<II", 0, 0)
    assert len(out) == HEADER
    for r, raw in enumerate(regions):
        out += struct.pack("<IIQQ", r, 0, len(raw), (len(raw) + BLOCK - 1) // BLOCK)
    for raw in regions:
        for b in range(0, len(raw), BLOCK):
            chunk = raw[b:b + BLOCK]
            L = lines_of(len(chunk))
            padded = np.zeros(L * LINE, np.uint8)
            padded[:len(chunk)] = np.frombuffer(chunk, np.uint8)
            nz = padded.reshape(L, LINE).any(1)
            bits = np.zeros(words_of(len(chunk)) * 32, np.uint8)
            bits[:L] = nz
            bitmap = np.packbits(bits, bitorder="little").view("<u4")
            idx = np.flatnonzero(nz)
            lines = padded.reshape(L, LINE)[idx].reshape(-1)
            stored = lines.tobytes()
            if len(chunk) % LINE and len(idx) and idx[-1] == L - 1:
                stored = stored[:len(stored) - (LINE - len(chunk) % LINE)]
            out += bitmap.tobytes() + stored + struct.pack("<Q", block_checksum(bitmap, lines, idx))
    open(path, "wb").write(bytes(out))


# ---- the tests -------------------------------------------------------------------------------------------------------
def _open(path):
    with pytest.raises(E.DintError) as ei:
        E.Engine.open_image(str(path))
    return ei.value


def test_reader_round_trips_a_synthetic_image(tmp_path):
    rng = np.random.default_rng(3)
    a = np.zeros(5000, np.uint8)
    a[rng.integers(0, 5000, 40)] = rng.integers(1, 256, 40)
    b = bytes(a[:4]) + b"\x07"           # 5 bytes: one partial line
    p = tmp_path / "x.img"
    write_synthetic(p, regions=(a.tobytes(), b"\0" * 300, b, b"\1" * 16))
    img = read_image(p)
    assert [r["bytes"] for r in img["regions"]] == [5000, 300, 5, 16]
    assert len(img["regions"][1]["blocks"][0]["line_index"]) == 0
    assert img["regions"][2]["blocks"][0]["stored"] == 5
    for reg in img["regions"]:
        for blk in reg["blocks"]:
            assert recompute_checksum(p, blk) == blk["checksum"]


def test_header_refusals_without_a_gpu(tmp_path):
    """each refusal happens before any CUDA call, so it is the same with or without a device"""
    good = tmp_path / "good.img"
    write_synthetic(good, regions=(b"\0" * 64,))
    data = good.read_bytes()

    p = tmp_path / "garbage.img"
    p.write_bytes(np.random.default_rng(1).integers(0, 256, 4096, dtype=np.uint8).tobytes())
    e = _open(p)
    assert e.code == EINVAL and "bad magic" in str(e)

    p = tmp_path / "short.img"
    p.write_bytes(data[:100])
    e = _open(p)
    assert e.code == EIO and "truncated header" in str(e)

    p = tmp_path / "magic.img"
    write_synthetic(p, magic=b"DINTIMG0", regions=(b"\0" * 64,))
    e = _open(p)
    assert e.code == EINVAL and "bad magic" in str(e)

    p = tmp_path / "version.img"
    write_synthetic(p, version=2, regions=(b"\0" * 64,))
    e = _open(p)
    assert e.code == EINVAL and "format version 2" in str(e)

    p = tmp_path / "kind.img"
    p.write_bytes(data[:12] + struct.pack("<I", 9) + data[16:])
    e = _open(p)
    assert e.code == EINVAL and "unknown kind 9" in str(e)

    p = tmp_path / "flags.img"
    write_synthetic(p, flags=1 << 7, regions=(b"\0" * 64,))
    e = _open(p)
    assert e.code == EINVAL and "unknown option flags 0x80" in str(e)

    p = tmp_path / "table.img"
    p.write_bytes(data[:HEADER + 8])
    e = _open(p)
    assert e.code == EIO and "truncated region table" in str(e)

    e = _open(tmp_path / "missing.img")
    assert e.code == EIO and "missing.img" in str(e)


def test_cluster_manifest_refusals_without_a_gpu(tmp_path):
    cfg = E.default_cfg(wire.FASST)
    d = tmp_path / "cl"
    d.mkdir()
    (d / "manifest").write_bytes(b"DINTCLU1" + struct.pack("<IIII", 1, wire.FASST, 3, 0) + bytes(cfg) + struct.pack("<I", 0))
    assert len((d / "manifest").read_bytes()) == E.CLUSTER_MANIFEST_BYTES
    assert E.read_image_header(str(d))["shards"] == 3
    with pytest.raises(E.DintError) as ei:
        E.GpuCluster.open_image(str(d), devices=[0, 0])
    assert ei.value.code == EINVAL and "3 shards, not 2" in str(ei.value)
    for r in range(2):
        write_synthetic(d / f"shard-{r}.img", regions=(b"\0" * 64,))
    with pytest.raises(E.DintError) as ei:
        E.GpuCluster.open_image(str(d), devices=[0, 0, 0])
    assert ei.value.code == EIO and "shard-2.img" in str(ei.value)
    for missing in (tmp_path / "no_such_dir", tmp_path / "empty"):
        if missing.name == "empty":
            missing.mkdir()
        with pytest.raises(E.DintError) as ei:
            E.GpuCluster.open_image(str(missing))
        assert ei.value.code == EIO and "manifest" in str(ei.value)
