"""CPU-only: the arithmetic of hold_mesh_sdf_bvh (hold_b200/csrc/mesh_bvh_phases.h) compiled for the host.  Morton codes and
Karras's links against numpy, the pruning bound against the computed tri_sqdist, and a sequential restatement of the build and
query (tests/host/mesh_bvh_host.cpp) against the brute force of k_mesh_sdf: |sdf| and face bit for bit, equal signs.  Also: the
fast winding number's error, and no floating-point or shared-memory atomic in the new kernels."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from oracle import mesh_sdf_oracle as MO
from test_cpu_decimate import latlong_sphere, meshes
from test_cpu_mesh_sdf import _lib as _brute_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAST_W_MAX_ERR = 0.05   # a 5x margin to the 0.25 trust band; measured 0.025 (noise mesh) with kBeta = 4


def _lib():
    out = os.path.join(ROOT, "tests", "_build", "libmesh_bvh_host.so")
    src = os.path.join(ROOT, "tests", "host", "mesh_bvh_host.cpp")
    hdrs = [os.path.join(ROOT, "hold_b200", "csrc", h) for h in ("mesh_bvh_phases.h", "mesh_sdf_phases.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(x) for x in [src] + hdrs):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        tmp = out + f".tmp{os.getpid()}"
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", tmp, src], check=True)
        os.replace(tmp, out)
    return C.CDLL(out)


def vp(a):
    return a.ctypes.data_as(C.c_void_p)


def bvh_meshes():
    """name -> (verts, faces): every mesh the BVH is held to, closed, open and degenerate"""
    m = dict(meshes())
    v, f = MO.star_mesh(level=3, seed=1)
    m["star"] = (v, f)
    v, f = latlong_sphere(20, 24)
    m["hemisphere"] = (v, np.ascontiguousarray(f[(v[f][:, :, 2] > -1e-6).all(1)]))   # open, unused vertices below
    m["tetrahedron"] = (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32),
                        np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32))
    m["octahedron"] = (np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32),
                       np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]], np.int32))
    v, f = MO.star_mesh(level=2, seed=3)
    extra = np.array([[0, 0, 0], [5, 5, 5], [7, 7, 7], [1, 2, 3], [4, 4, 9]], np.int32)   # zero area: one point, a collinear sliver...
    v = np.concatenate([v, [[0.3, 0.3, 0.3], [0.6, 0.6, 0.6], [0.9, 0.9, 0.9]]]).astype(np.float32)
    n = len(v)
    extra = np.concatenate([extra, [[n - 3, n - 2, n - 1], [n - 1, n - 2, n - 3]]])          # ... collinear vertices
    m["degenerate_duplicate"] = (v, np.ascontiguousarray(np.concatenate([f, f[:40], extra, f[::-7]]), np.int32))
    return {k: (np.ascontiguousarray(v, np.float32), np.ascontiguousarray(f, np.int32)) for k, (v, f) in m.items()}


def query_points(v, n, seed):
    """uniform in the mesh's box (enlarged), points on vertices, edges and faces, far points, NaN and inf"""
    rng = np.random.default_rng(seed)
    lo, hi = v.min(0), v.max(0)
    c, e = (lo + hi) / 2, (hi - lo) / 2 * 1.3 + 1e-3
    pts = c + rng.uniform(-1, 1, size=(n, 3)) * e
    k = n // 10
    pts[:k] = v[rng.integers(0, len(v), k)]
    a, b = v[rng.integers(0, len(v), k)], v[rng.integers(0, len(v), k)]
    pts[k:2 * k] = a + rng.uniform(0, 1, (k, 1)) * (b - a)
    pts[2 * k:2 * k + 4] = [[np.nan, 0, 0], [0, np.inf, 0], [-np.inf, np.inf, np.nan], [30.0, -40.0, 50.0]]
    return np.ascontiguousarray(pts, np.float32)


def brute(v, f, pts):
    sdf, fi = np.empty(len(pts), np.float32), np.empty(len(pts), np.int32)
    assert _brute_lib().mesh_sdf_host(len(pts), len(v), len(f), vp(pts), vp(v), vp(f), vp(sdf), vp(fi)) == 0
    return sdf, fi


def bvh(v, f, pts, want_w=False):
    P = len(pts)
    sdf, fi, band = np.empty(P, np.float32), np.empty(P, np.int32), np.empty(P, np.int32)
    wf, we = (np.empty(P, np.float32), np.empty(P, np.float32)) if want_w else (None, None)
    assert _lib().bvh_sdf_host(P, len(v), len(f), vp(pts), vp(v), vp(f), vp(sdf), vp(fi), vp(band),
                               vp(wf) if want_w else None, vp(we) if want_w else None) == 0
    return sdf, fi, band.astype(bool), wf, we


# ---------------------------------------------------------------- codes and links

def _np_expand(x):
    out = np.zeros_like(x, dtype=np.int64)
    for bit in range(10):
        out |= ((x >> bit) & 1) << (3 * bit)
    return out


def test_morton_codes_against_numpy():
    rng = np.random.default_rng(1)
    F = 5000
    tris = rng.uniform(-2, 3, size=(F, 9)).astype(np.float32)
    tris[:7] = 0.5                                             # equal centroids
    lo = np.array([-2, -2, -2], np.float32)
    inv = np.array([1 / 5, 1 / 5, 0], np.float32)             # a flat axis
    codes = np.empty(F, np.int32)
    assert _lib().bvh_morton_host(F, vp(tris), vp(lo), vp(inv), vp(codes)) == 0
    cen = ((tris[:, 0:3] + tris[:, 3:6] + tris[:, 6:9]) * np.float32(1 / 3)).astype(np.float32)
    q = np.clip((cen - lo) * inv * np.float32(1024), 0, 1023).astype(np.int64)
    want = (_np_expand(q[:, 0]) << 2) | (_np_expand(q[:, 1]) << 1) | _np_expand(q[:, 2])
    assert np.array_equal(codes.astype(np.int64), want)
    assert (codes >= 0).all() and codes.max() < (1 << 30)


def _check_links(codes):
    """Karras's links against a top-down split of the 64-bit keys (code, position); every leaf reached once; depth bound"""
    F = len(codes)
    left, right = np.empty(max(F - 1, 0), np.int32), np.empty(max(F - 1, 0), np.int32)
    assert _lib().bvh_karras_host(F, vp(codes), vp(left), vp(right)) == 0
    keys = [(int(c) << 32) | i for i, c in enumerate(codes)]
    seen, max_depth = np.zeros(F, np.int64), 0
    stack = [(0, 0, F - 1, 0)]                                 # node, range, depth
    while stack:
        n, lo, hi, depth = stack.pop()
        max_depth = max(max_depth, depth)
        if n >= F - 1:
            assert lo == hi == n - (F - 1)
            seen[lo] += 1
            continue
        common = 64 - (keys[lo] ^ keys[hi]).bit_length()
        s = max(i for i in range(lo, hi) if 64 - (keys[lo] ^ keys[i]).bit_length() > common)
        l, r = int(left[n]), int(right[n])
        stack.append((l, lo, s, depth + 1))
        stack.append((r, s + 1, hi, depth + 1))
        assert (l >= F - 1) == (s == lo) and (r >= F - 1) == (s + 1 == hi)
    assert (seen == 1).all()
    assert max_depth <= 30 + math.ceil(math.log2(F)) if F > 1 else max_depth == 0
    return max_depth


@pytest.mark.parametrize("case", ["random", "all_equal", "runs", "one", "two"])
def test_karras_links(case):
    rng = np.random.default_rng(2)
    F = {"one": 1, "two": 2}.get(case, 3000)
    if case == "random":
        codes = rng.integers(0, 1 << 30, F)
    elif case == "all_equal":
        codes = np.full(F, 12345)
    else:
        codes = rng.integers(0, 40, F) << 20 if case == "runs" else rng.integers(0, 1 << 30, F)
    codes = np.ascontiguousarray(np.sort(codes), np.int32)
    depth = _check_links(codes)
    if case == "all_equal":
        assert depth == math.ceil(math.log2(F))               # the index bits alone: a balanced tree


# ---------------------------------------------------------------- the pruning bound

def test_box_lower_bound_never_exceeds_tri_sqdist():
    rng = np.random.default_rng(3)
    N = 400_000
    groups = []
    for scale in (1.0, 1e3):                                   # near the origin, far from it
        c = rng.uniform(-scale, scale, (N, 1, 3))
        size = 10.0 ** rng.uniform(-6, 0, (N, 1, 1)) * max(1.0, scale * 1e-3)
        tris = (c + rng.normal(size=(N, 3, 3)) * size).astype(np.float32)
        w = rng.dirichlet([1, 1, 1], N)
        kind = rng.integers(0, 5, N)
        on = np.einsum("nk,nkc->nc", w, tris)                          # on the face
        edge = tris[:, 0] + rng.uniform(0, 1, (N, 1)) * (tris[:, 1] - tris[:, 0])
        vert = tris[np.arange(N), rng.integers(0, 3, N)]
        base = np.where((kind == 0)[:, None], on, np.where((kind == 1)[:, None], edge, vert))
        off = rng.normal(size=(N, 3)) * size[:, 0] * 10.0 ** rng.uniform(-7, 1, (N, 1))   # tiny to large distances
        pts = np.where((kind == 4)[:, None], c[:, 0] + rng.normal(size=(N, 3)) * size[:, 0] * 5, base + off)
        groups.append((tris.reshape(N, 9), pts))
    # slivers: nearly collinear vertices
    t = rng.uniform(-1, 1, (N, 3, 3))
    t[:, 2] = t[:, 0] + rng.uniform(0, 1, (N, 1)) * (t[:, 1] - t[:, 0]) + rng.normal(size=(N, 3)) * 1e-6
    groups.append((t.reshape(N, 9), t[:, 0] + rng.normal(size=(N, 3)) * 1e-3))
    total = 0
    for tris, pts in groups:
        tris, pts = np.ascontiguousarray(tris, np.float32), np.ascontiguousarray(pts, np.float32)
        n = len(tris)
        scale = np.maximum(np.abs(tris).max(1), np.abs(pts).max(1)).astype(np.float32)
        lower, d = np.empty(n, np.float32), np.empty(n, np.float32)
        assert _lib().bvh_bound_host(n, vp(tris), vp(pts), vp(scale), vp(lower), vp(d)) == 0
        ok = np.isfinite(d)
        bad = ok & (lower > d)
        assert not bad.any(), (tris[bad][:3], pts[bad][:3], lower[bad][:3], d[bad][:3])
        total += int(ok.sum())
    assert total >= 1_000_000


# ---------------------------------------------------------------- build and query against the brute force

def _same(a, b):
    (s0, f0), (s1, f1) = a, b
    return (np.array_equal(np.abs(s0).view(np.int32), np.abs(s1).view(np.int32)) and np.array_equal(np.signbit(s0), np.signbit(s1))
            and np.array_equal(f0, f1))


@pytest.mark.parametrize("name", list(bvh_meshes()))
def test_host_restatement_equals_brute_force(name):
    v, f = bvh_meshes()[name]
    pts = query_points(v, 3000, seed=len(name))
    s0, f0 = brute(v, f, pts)
    s1, f1, band, _, _ = bvh(v, f, pts)
    assert _same((s1, f1), (s0, f0)), np.nonzero((s0 != s1) | (f0 != f1))[0][:10]
    fin = np.isfinite(pts).all(1)
    assert (f1[~fin] == -1).all() and (s1[~fin] == np.sqrt(np.float32(3e38))).all() and band[~fin].all()
    print(f"{name}: F {len(f)}, band {band[fin].mean():.4f}")


def test_bad_mesh_coordinates():
    """NaN and inf vertices: the NaN faces are never nearest, every point sums exactly"""
    v, f = MO.star_mesh(level=2, seed=5)
    v = v.copy()
    v[3] = np.nan
    v[7] = [np.inf, 0, 0]
    pts = query_points(v[np.isfinite(v).all(1)], 500, seed=9)
    s0, f0 = brute(v, f, pts)
    s1, f1, band, _, _ = bvh(v, f, pts)
    assert _same((s1, f1), (s0, f0)) and band.all()


def test_fast_winding_number_error():
    worst = {}
    for name, (v, f) in bvh_meshes().items():
        pts = query_points(v, 2000, seed=7)
        pts = pts[np.isfinite(pts).all(1)]
        _, _, _, wf, we = bvh(v, f, np.ascontiguousarray(pts), want_w=True)
        worst[name] = float(np.abs(wf - we).max())
    print("max |w_fast - w_exact|:", {k: f"{e:.2e}" for k, e in worst.items()})
    assert max(worst.values()) <= FAST_W_MAX_ERR, worst


# ---------------------------------------------------------------- no float or shared atomics

BVH_KERNELS = ("k_bvh_bounds", "k_bvh_codes", "k_bvh_link", "k_bvh_refit", "k_bvh_query", "k_bvh_band")


def test_bvh_kernels_have_no_float_or_shared_atomics(built):
    from hold_b200 import capi
    from test_cpu_repro_bwd_sass import _unordered_adds
    from test_cpu_wgrad_sass import _sass_by_function

    funcs = _sass_by_function(capi.LIB_PATH)
    for w in BVH_KERNELS:
        names = [k for k in funcs if w in k]
        assert names, f"no kernel named {w}"
        for k in names:
            assert not _unordered_adds(funcs[k]), (k, _unordered_adds(funcs[k]))
            assert not [op for op in funcs[k] if op.startswith(("ATOMS", "RED.", "REDG")) and "F32" in op], k
