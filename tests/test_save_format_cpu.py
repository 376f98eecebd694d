"""CPU checks of the saved-index manifest: the independent Python writer and reader (tests/savefmt.py) round-trip, and
every file the library's restore refuses before it touches a device (bad magic, bad version, truncation, a rank list
that is not a permutation, a wrong manifest or pair checksum, a missing manifest, a wrong device count) is rejected by
the Python reader too, and by the library with a message naming the file."""
import ctypes as C
import os
import struct

import numpy as np
import pytest

import savefmt


def _manifest(n=5, P=1, labels=True):
    counts = [(n + P - 1 - p) // P for p in range(P)]
    rng = np.random.default_rng(n * 7 + P)
    pairs = [(11 + p, 12, 13, 14, rng.permutation(c)) if c else None for p, c in enumerate(counts)]
    return {"dtype": 0, "metric": 1, "M": 8, "max_layer": 16, "dim": 3, "ef_c": 40, "max_elements": 100, "link_mode": 1,
            "visited_stages": 2, "batch_ratio": 4, "batch_max": 7, "extend": True, "keep_pruned": False,
            "tie_std": True, "level_scale": 1 / np.log(8) * 0.7, "rng": 0xDEADBEEF12345678, "counts": counts,
            "pairs": pairs, "labels": np.arange(n, dtype=np.uint32) if labels else None,
            "attrs": np.arange(n, dtype=np.int64) - 2 if labels else None,
            "deleted": (np.arange(n) % 3 == 0).astype(np.uint8) if labels else None}


def test_sum64_matches_a_word_loop():
    data = bytes(range(256)) * 3 + b"\x07\x01\x02"     # a partial last word
    acc, mask = 0, 2 ** 64 - 1

    def mix(z):
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & mask
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & mask
        return z ^ (z >> 31)
    pad = data + b"\0" * (-len(data) % 8)
    for i in range(len(pad) // 8):
        w = int.from_bytes(pad[8 * i:8 * i + 8], "little")
        acc = (acc + mix(w ^ ((i * 0x9E3779B97F4A7C15) & mask))) & mask
    assert savefmt.sum64(data) == mix((acc + len(data)) & mask)
    assert savefmt.sum64(data) != savefmt.sum64(data[:-1] + b"\x08")


@pytest.mark.parametrize("n,P,labels", [(5, 1, True), (5, 3, True), (2, 3, False), (17, 2, True)])
def test_manifest_round_trip(n, P, labels):
    m = _manifest(n, P, labels)
    b = savefmt.pack(m)
    assert struct.unpack_from("=2I", b) == (savefmt.MAGIC, savefmt.VERSION)
    back = savefmt.unpack(b)
    assert savefmt.pack(back) == b
    for k in ("dtype", "metric", "M", "dim", "ef_c", "max_elements", "link_mode", "visited_stages", "batch_ratio",
              "batch_max", "extend", "keep_pruned", "tie_std", "rng", "counts"):
        assert back[k] == m[k], k
    assert struct.pack("=d", back["level_scale"]) == struct.pack("=d", m["level_scale"])   # the exact double
    for p, pr in enumerate(m["pairs"]):
        assert (pr is None) == (back["pairs"][p] is None)
        if pr is not None:
            assert back["pairs"][p][:4] == pr[:4] and np.array_equal(back["pairs"][p][4], pr[4])
    for k in ("labels", "attrs", "deleted"):
        assert (m[k] is None and back[k] is None) or np.array_equal(back[k], m[k])


def _saved_set(tmp_path):
    """a 6-point f32 L2 index of two levels, as a pair written by oracle/dumpfmt.py and a manifest of its ranks"""
    import dumpfmt
    X = np.arange(18, dtype=np.float32).reshape(6, 3)
    levels = np.array([0, 1, 0, 0, 1, 0])
    nb = [[1, 2], [0, 4], [0, 3], [2, 5], [1, 3], [3, 4]]
    off = np.arange(0, 13, 2, dtype=np.uint64)
    ids = np.array(sum(nb, []), np.uint32)
    ds = np.array([float(np.sum((X[p] - X[q]) ** 2)) for p in range(6) for q in nb[p]], np.float32)
    up = np.array([0, 0, 1, 1, 1, 1, 2], np.uint64)
    layers = [(off, ids, ds), (up, np.array([4, 1], np.uint32), np.array([ds[3], ds[9]], np.float32))]
    dumpfmt.write_dump(str(tmp_path / "s"), X, np.arange(100, 106), levels, 1, layers, 8, 40, 1 / np.log(8), "DistL2")
    m = _manifest(6, 1)
    gs, gsum = savefmt.file_sum(str(tmp_path / "s.hnsw.graph"))
    dsz, dsum = savefmt.file_sum(str(tmp_path / "s.hnsw.data"))
    m["pairs"] = [(gs, gsum, dsz, dsum, savefmt.file_order(levels))]
    return m


def _restore_refusal(pkg, tmp_path, ndev=0):
    """the library's restore of tmp_path/s refuses: its message"""
    L = pkg.load_library()
    devs = (C.c_int * max(ndev, 1))()
    h = L.hnsw_b200_restore(str(tmp_path).encode(), b"s", ndev, devs)
    assert not h
    return pkg.last_error()


def test_valid_set_is_accepted_by_the_python_reader(tmp_path):
    m = _saved_set(tmp_path)
    open(tmp_path / "s.hnsw.b200", "wb").write(savefmt.pack(m))
    back = savefmt.unpack(open(tmp_path / "s.hnsw.b200", "rb").read())
    savefmt.check_pairs(str(tmp_path), "s", back)
    assert np.array_equal(back["pairs"][0][4], [0, 2, 3, 5, 1, 4])   # level 0 first: file order != rank order


def _crafted(m, kind):
    b = bytearray(savefmt.pack(m))
    if kind == "magic":
        b[0] ^= 1
    elif kind == "version":
        b[4] = 9
    elif kind == "truncated":
        b = b[:-13]
    elif kind == "checksum":
        b[60] ^= 0x40
    elif kind == "permutation":
        pr = list(m["pairs"][0])
        pr[4] = np.array([0, 2, 2, 5, 1, 4])
        b = bytearray(savefmt.pack(dict(m, pairs=[tuple(pr)])))
    elif kind == "placement":
        pairs = [(1, 2, 3, 4, np.arange(4)), (1, 2, 3, 4, np.arange(2))]
        b = bytearray(savefmt.pack(dict(m, counts=[4, 2], pairs=pairs)))
    return bytes(b)


@pytest.mark.parametrize("kind,says", [("magic", "bad magic"), ("version", "version 9"), ("truncated", "checksum"),
                                       ("checksum", "checksum"), ("permutation", "not a permutation"),
                                       ("placement", "placement rule")])
def test_crafted_manifest_is_refused_by_both(tmp_path, pkg, kind, says):
    m = _saved_set(tmp_path)
    open(tmp_path / "s.hnsw.b200", "wb").write(_crafted(m, kind))
    with pytest.raises(savefmt.ManifestError):
        savefmt.unpack(open(tmp_path / "s.hnsw.b200", "rb").read())
    e = _restore_refusal(pkg, tmp_path)
    assert "s.hnsw.b200" in e and says in e, e


@pytest.mark.parametrize("which", ["graph", "data"])
def test_changed_pair_is_refused_by_both(tmp_path, pkg, which):
    m = _saved_set(tmp_path)
    open(tmp_path / "s.hnsw.b200", "wb").write(savefmt.pack(m))
    path = tmp_path / f"s.hnsw.{which}"
    raw = bytearray(open(path, "rb").read())
    raw[-3] ^= 1
    open(path, "wb").write(bytes(raw))
    with pytest.raises(savefmt.ManifestError):
        savefmt.check_pairs(str(tmp_path), "s", savefmt.unpack(open(tmp_path / "s.hnsw.b200", "rb").read()))
    e = _restore_refusal(pkg, tmp_path)
    assert f"s.hnsw.{which}" in e and "checksum" in e, e
    open(path, "ab").write(b"\0")
    e = _restore_refusal(pkg, tmp_path)
    assert f"s.hnsw.{which}" in e and "bytes" in e, e


def test_missing_manifest_and_wrong_ndev_are_refused(tmp_path, pkg):
    m = _saved_set(tmp_path)
    e = _restore_refusal(pkg, tmp_path)
    assert "s.hnsw.b200" in e and "could not open" in e, e
    open(tmp_path / "s.hnsw.b200", "wb").write(savefmt.pack(m))
    e = _restore_refusal(pkg, tmp_path, ndev=2)
    assert "s.hnsw.b200" in e and "ndev" in e, e
    with pytest.raises(pkg.HnswError):
        pkg.Hnsw.restore(tmp_path, "nothing-here")
    assert not os.path.exists(tmp_path / "nothing-here.hnsw.b200")
