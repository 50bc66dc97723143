"""CPU-only, SURVEY §8f rank 4: the MISE restatement the CUDA kernels run (hold_b200/csrc/mise_phases.h, compiled for the
host) against the reference's own compiled Cython MISE (libmise/mise.pyx), round by round and bit for bit, on five analytic
fields.  What the reference MISE produces on those cases is stored in tests/golden/mise/mise_cases.json (per round: the number
and a SHA-256 of the sorted queried points; the dense grid's SHA-256, sign counts and a seeded sample), so the comparison runs in
every checkout.  Where $HOLD_REFERENCE names a checkout of the reference, the reference module is also built (oracle/_ref, by
oracle/build_ref_mise.py) and run alongside, and the goldens are checked against it."""
import ctypes as C
import glob
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _host():
    out = os.path.join(ROOT, "tests", "_build", "libmise_host.so")
    src = os.path.join(ROOT, "tests", "host", "mise_host.cpp")
    hdr = os.path.join(ROOT, "hold_b200", "csrc", "mise_phases.h")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    lib = C.CDLL(out)
    lib.mise_host_create.restype = C.c_void_p
    lib.mise_host_create.argtypes = [C.c_int, C.c_int, C.c_float]
    lib.mise_host_query.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    lib.mise_host_update.argtypes = [C.c_void_p, C.c_void_p]
    lib.mise_host_to_dense.argtypes = [C.c_void_p, C.c_void_p]
    lib.mise_host_destroy.argtypes = [C.c_void_p]
    return lib


def _ref_mise():
    """The reference's compiled MISE module, or None without a reference checkout."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import build_ref_mise

    so = build_ref_mise.build() or next(iter(glob.glob(os.path.join(ROOT, "oracle", "_ref", "mise*.so"))), None)
    if so is None:
        return None
    sys.path.insert(0, os.path.dirname(so))
    import mise

    return mise


def _field(seed):
    rng = np.random.default_rng(seed)
    c = rng.uniform(0.3, 0.7, size=(3, 3))
    r = rng.uniform(0.12, 0.22, size=3)

    def f(pts, R):   # union of three blobs minus a ripple, exact zeros included through quantisation
        x = pts.astype(np.float32) / np.float32(R)
        d = np.min(np.stack([np.linalg.norm(x - c[i].astype(np.float32), axis=1) - np.float32(r[i]) for i in range(3)]), 0)
        v = (d + np.float32(0.02) * np.sin(np.float32(40.0) * x[:, 0])).astype(np.float32)
        return np.round(v * 64) / 64 if seed % 2 else v     # odd seeds: many values exactly on the threshold
    return f


GOLD = os.path.join(ROOT, "tests", "golden", "mise", "mise_cases.json")
CASES = [(4, 2, 0), (4, 3, 1), (8, 2, 2), (6, 3, 3), (32, 2, 4)]


def run_mise(query, update, dense, res0, depth, seed):
    """Drive one MISE through the reference loop with the analytic field of `seed`: query() -> lattice points [n,3] (ints),
    update(points, float32 values of those points), dense() -> the value grid.  Returns the sorted point keys of every round
    and the dense grid as float64 [G,G,G]."""
    f = _field(seed)
    R = res0 << depth
    G = R + 1
    rounds = []
    while True:
        pts = np.asarray(query()).astype(np.int64)
        if pts.shape[0] == 0:
            break
        rounds.append(np.sort((pts[:, 0] * G + pts[:, 1]) * G + pts[:, 2]))
        update(pts, f(pts, R).astype(np.float32))
    return rounds, np.asarray(dense(), np.float64).reshape(G, G, G)


def digest(rounds, grid):
    """What the goldens keep of one run: exact (hashes, counts) plus a seeded sample of the grid for readable failures."""
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
    flat = grid.reshape(-1)
    idx = np.sort(np.random.default_rng(0).choice(flat.size, size=min(256, flat.size), replace=False))
    return {"rounds": [[int(k.size), sha(k.astype("<i8"))] for k in rounds], "dense_sha256": sha(flat.astype("<f8")),
            "dense_below": int((flat < 0).sum()), "dense_above": int((flat > 0).sum()),
            "dense_sample_index": idx.tolist(), "dense_sample": flat[idx].tolist()}


def assert_matches_golden(d, res0, depth, seed, what):
    g = json.load(open(GOLD))["cases"][f"{res0},{depth},{seed}"]
    assert len(d["rounds"]) == len(g["rounds"]) >= 2, f"{what}: {len(d['rounds'])} rounds vs {len(g['rounds'])}"
    for r, (a, b) in enumerate(zip(d["rounds"], g["rounds"])):
        assert a == b, f"{what}: round {r}: {a[0]} points vs {b[0]} (or a different point set)"
    assert d["dense_sample"] == g["dense_sample"] and d["dense_below"] == g["dense_below"] and d["dense_above"] == g["dense_above"], what
    assert d["dense_sha256"] == g["dense_sha256"], f"{what}: dense grid differs"


class HostMise:
    """The restatement compiled for the host, with the query / update / to_dense surface of mise.MISE."""

    def __init__(self, lib, res0, depth):
        self.lib, self.G = lib, (res0 << depth) + 1
        self.h = lib.mise_host_create(res0, depth, C.c_float(0.0))

    def query(self):
        buf = np.zeros((self.G**3, 3), np.int32)
        n = self.lib.mise_host_query(self.h, buf.ctypes.data_as(C.c_void_p), C.c_int(self.G**3))
        return buf[:n]

    def update(self, pts, vals):
        vals = np.ascontiguousarray(vals, np.float32)
        self.lib.mise_host_update(self.h, vals.ctypes.data_as(C.c_void_p))

    def to_dense(self):
        out = np.empty(self.G**3, np.float32)
        self.lib.mise_host_to_dense(self.h, out.ctypes.data_as(C.c_void_p))
        self.lib.mise_host_destroy(self.h)
        return out


@pytest.mark.parametrize("res0,depth,seed", CASES)
def test_mise_restatement_matches_reference_mise(res0, depth, seed):
    h = HostMise(_host(), res0, depth)
    d = digest(*run_mise(h.query, h.update, h.to_dense, res0, depth, seed))
    mise = _ref_mise()
    if mise is not None:   # the reference itself is at hand: the goldens must be what it produces
        ref = mise.MISE(res0, depth, 0.0)
        dr = digest(*run_mise(ref.query, lambda p, v: ref.update(p, v.astype(np.float64)), ref.to_dense, res0, depth, seed))
        assert_matches_golden(dr, res0, depth, seed, "reference MISE vs goldens")
    assert_matches_golden(d, res0, depth, seed, "restatement vs reference MISE goldens")
