"""An independent restatement (struct packing) of the saved-index manifest, <base>.hnsw.b200, that Hnsw.save writes
next to its reference-format pairs (layout: hnswlib-rs_b200/csrc/saved.cu).  Test infrastructure only: it writes
manifests for graphs built elsewhere, and reads and checks the library's, so that the format is pinned by a second
implementation.  The pairs themselves are oracle/dumpfmt.py's.  Native endian (little-endian hosts)."""
import struct

import numpy as np

MAGIC, VERSION = 0x56534248, 1
HAS_LABELS, HAS_ATTRS, HAS_DELETED = 1, 2, 4
HEAD = "=6I3Q4I4BdQQ"   # magic .. max_elements, link_mode .. batch_max, extend, keep_pruned, tie_std, columns, scale, rng, P
DTYPES = {np.dtype(np.float32): 0, np.dtype(np.uint8): 1, np.dtype(np.uint16): 2, np.dtype(np.uint32): 3,
          np.dtype(np.int32): 4}
METRICS = ("DistL1", "DistL2", "DistDot", "DistCosine", "DistHamming", "DistJaccard", "DistHellinger", "DistJeffreys",
           "DistJensenShannon")
_GOLD = np.uint64(0x9E3779B97F4A7C15)


class ManifestError(ValueError):
    pass


def _mix(z):
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def sum64(data):
    """the manifest's checksum of a byte string: mix(len + sum_i mix(w_i ^ i * golden)) mod 2^64, w_i its little-endian
    u64 words, the last zero-padded"""
    data = bytes(data)
    pad = data + b"\0" * (-len(data) % 8)
    w = np.frombuffer(pad, "<u8")
    with np.errstate(over="ignore"):
        acc = int(np.sum(_mix(w ^ (np.arange(len(w), dtype=np.uint64) * _GOLD)), dtype=np.uint64))
        return int(_mix(np.array([(acc + len(data)) % 2 ** 64], np.uint64))[0])


def file_sum(path):
    data = open(path, "rb").read()
    return len(data), sum64(data)


def pack(m):
    """the manifest bytes of a dict: dtype, metric, M, max_layer, dim, ef_c, max_elements, link_mode, visited_stages,
    batch_ratio, batch_max, extend, keep_pruned, tie_std, level_scale, rng, counts[P], pairs[P] (None for an empty
    partition, else (graph_size, graph_sum, data_size, data_sum, rank list in file order)), and labels / attrs / deleted
    (arrays by global rank, or None)"""
    cols = (HAS_LABELS if m.get("labels") is not None else 0) | (HAS_ATTRS if m.get("attrs") is not None else 0) | \
        (HAS_DELETED if m.get("deleted") is not None else 0)
    b = bytearray(struct.pack(HEAD, m.get("magic", MAGIC), m.get("version", VERSION), m["dtype"], m["metric"], m["M"],
                              m["max_layer"], m["dim"], m["ef_c"], m["max_elements"], m["link_mode"], m["visited_stages"],
                              m["batch_ratio"], m["batch_max"], int(m["extend"]), int(m["keep_pruned"]),
                              int(m["tie_std"]), cols, m["level_scale"], m["rng"], len(m["counts"])))
    b += np.asarray(m["counts"], "<u8").tobytes()
    for c, pr in zip(m["counts"], m["pairs"]):
        if c:
            b += struct.pack("=4Q", *pr[:4]) + np.asarray(pr[4], "<u8").tobytes()
    if cols & HAS_LABELS:
        b += np.asarray(m["labels"], "<u4").tobytes()
    if cols & HAS_ATTRS:
        b += np.asarray(m["attrs"], "<i8").tobytes()
    if cols & HAS_DELETED:
        b += np.packbits(np.asarray(m["deleted"], np.uint8), bitorder="little").tobytes()
    return bytes(b) + struct.pack("=Q", sum64(b))


def unpack(data):
    """pack's dict from manifest bytes; ManifestError for anything the library refuses: bad magic, bad version, a
    checksum mismatch (truncation included), a count that breaks the placement rule, a rank list that is not a
    permutation, sizes that do not add up"""
    if len(data) < 8:
        raise ManifestError("truncated")
    magic, version = struct.unpack_from("=2I", data)
    if magic != MAGIC:
        raise ManifestError("bad magic")
    if version != VERSION:
        raise ManifestError("bad version")
    if len(data) < 16 or struct.unpack_from("=Q", data, len(data) - 8)[0] != sum64(data[:-8]):
        raise ManifestError("checksum")
    body = data[:-8]
    if len(body) < struct.calcsize(HEAD):
        raise ManifestError("truncated")
    f = struct.unpack_from(HEAD, body)
    keys = ("magic", "version", "dtype", "metric", "M", "max_layer", "dim", "ef_c", "max_elements", "link_mode",
            "visited_stages", "batch_ratio", "batch_max", "extend", "keep_pruned", "tie_std", "columns", "level_scale",
            "rng", "P")
    m = dict(zip(keys, f))
    pos = struct.calcsize(HEAD)
    P = m.pop("P")
    if not 1 <= P <= 64 or len(body) < pos + 8 * P:
        raise ManifestError("partitions")
    counts = np.frombuffer(body, "<u8", P, pos).astype(np.int64).tolist()
    pos += 8 * P
    n = sum(counts)
    if n == 0 or any(c != (n + P - 1 - p) // P for p, c in enumerate(counts)):
        raise ManifestError("placement")
    pairs = []
    for c in counts:
        if not c:
            pairs.append(None)
            continue
        if len(body) < pos + 32 + 8 * c:
            raise ManifestError("truncated")
        sizes = struct.unpack_from("=4Q", body, pos)
        rank = np.frombuffer(body, "<u8", c, pos + 32).astype(np.int64)
        pos += 32 + 8 * c
        if not np.array_equal(np.sort(rank), np.arange(c)):
            raise ManifestError("not a permutation")
        pairs.append((*sizes, rank))
    cols = m.pop("columns")
    want = (4 * n if cols & HAS_LABELS else 0) + (8 * n if cols & HAS_ATTRS else 0) + \
        ((n + 7) // 8 if cols & HAS_DELETED else 0)
    if len(body) - pos != want:
        raise ManifestError("sizes")
    m["labels"] = m["attrs"] = m["deleted"] = None
    if cols & HAS_LABELS:
        m["labels"] = np.frombuffer(body, "<u4", n, pos).copy(); pos += 4 * n
    if cols & HAS_ATTRS:
        m["attrs"] = np.frombuffer(body, "<i8", n, pos).copy(); pos += 8 * n
    if cols & HAS_DELETED:
        m["deleted"] = np.unpackbits(np.frombuffer(body, np.uint8, (n + 7) // 8, pos), bitorder="little")[:n]
    m.update(counts=counts, pairs=pairs, extend=bool(m["extend"]), keep_pruned=bool(m["keep_pruned"]),
             tie_std=bool(m["tie_std"]))
    return m


def file_order(levels):
    """the insertion ranks of a pair's points in file order (layer by layer, insertion order within a layer)"""
    levels = np.asarray(levels)
    return np.concatenate([np.flatnonzero(levels == l) for l in range(16)]).astype(np.int64)


def check_pairs(dirpath, base, m):
    """ManifestError unless every pair file has the size and checksum the manifest records"""
    P = len(m["counts"])
    for p, pr in enumerate(m["pairs"]):
        if pr is None:
            continue
        pb = f"{dirpath}/{base}" + ("" if P == 1 else f"-p{p}")
        for path, (size, s) in ((pb + ".hnsw.graph", pr[0:2]), (pb + ".hnsw.data", pr[2:4])):
            if file_sum(path) != (size, s):
                raise ManifestError(f"{path}: size or checksum")
