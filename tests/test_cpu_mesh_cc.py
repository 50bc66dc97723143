"""CPU-only: the largest-component selection as hold_largest_component runs it (hold_b200/csrc/mesh_cc_phases.h, restated
sequentially in tests/host/mesh_cc_host.cpp, compiled with -ffp-contract=off) against hold_b200.meshing.largest_component, the
scipy / numpy selection the reference's trimesh.split + argmax performs: labels, face areas, per-component sums, the chosen
component and the re-indexed output, bit for bit.  Meshes: multi-blob marching-cubes meshes, random triangle soups with isolated
and unused vertices, duplicate and zero-area faces, a component with more faces but less area, exact ties, all areas zero with
vertex 0 isolated, a single face.  Joining the edges in reversed and shuffled face order gives the same labels.  The new
kernels hold no floating-point atomic."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_cpu_wgrad_sass import FLOAT_GLOBAL_ADD, _sass_by_function

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    out = os.path.join(ROOT, "tests", "_build", "libmesh_cc_host.so")
    src = os.path.join(ROOT, "tests", "host", "mesh_cc_host.cpp")
    hdr = os.path.join(ROOT, "hold_b200", "csrc", "mesh_cc_phases.h")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        tmp = out + f".tmp{os.getpid()}"
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", tmp, src], check=True)
        os.replace(tmp, out)
    lib = C.CDLL(out)
    lib.cc_largest_host.restype = C.c_int
    lib.cc_before_host.restype = C.c_int
    lib.cc_before_host.argtypes = [C.c_double, C.c_int, C.c_double, C.c_int]
    return lib


_p = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None


def host_largest(verts, faces, face_order=None):
    """hold_largest_component on the host -> (verts, faces, labels, area, sums, best)"""
    v = np.ascontiguousarray(verts, np.float32).reshape(-1, 3)
    f = np.ascontiguousarray(faces, np.int32).reshape(-1, 3)
    order = None if face_order is None else np.ascontiguousarray(face_order, np.int32)
    V, F = v.shape[0], f.shape[0]
    vo, fo = np.zeros_like(v), np.zeros_like(f)
    labels, area, sums = np.zeros(V, np.int32), np.zeros(F, np.float32), np.zeros(V, np.float64)
    nv, nf = C.c_int(0), C.c_int(0)
    best = _lib().cc_largest_host(V, _p(v), F, _p(f), _p(order), _p(vo), _p(fo), C.byref(nv), C.byref(nf), _p(labels), _p(area),
                                  _p(sums))
    return vo[: nv.value], fo[: nf.value], labels, area, sums, best


def host_labels(V, faces, face_order=None):
    f = np.ascontiguousarray(faces, np.int32)
    labels = np.zeros(V, np.int32)
    _lib().cc_labels_host(V, f.shape[0], _p(f), _p(None if face_order is None else np.ascontiguousarray(face_order, np.int32)),
                          _p(labels))
    return labels


# ---------------------------------------------------------------- meshes

def blobs(n=40, seed=0):
    """marching-cubes mesh of several spheres of different radii (oracle/marching_cubes.py), in world units"""
    from oracle.marching_cubes import marching_cubes

    rng = np.random.default_rng(seed)
    a = np.linspace(-1.0, 1.0, n, dtype=np.float32)
    x, y, z = np.meshgrid(a, a, a, indexing="ij")
    field = np.full(x.shape, 10.0, np.float32)
    for c, r in zip(rng.uniform(-0.6, 0.6, (5, 3)), rng.uniform(0.08, 0.3, 5)):
        field = np.minimum(field, np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2) - r)
    v, f = marching_cubes(field, 0.0)
    return (v * (2.0 / (n - 1)) - 1.0).astype(np.float32), f.astype(np.int32)


def soup(seed, V=300, F=400):
    """random triangles over a vertex pool with unused vertices, duplicate faces and zero-area faces"""
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((V, 3)).astype(np.float32) * rng.uniform(0.01, 10)
    used = rng.choice(V, V * 2 // 3, replace=False)            # a third of the vertices are never used
    f = used[rng.integers(0, used.shape[0], (F, 3))]
    f[:20] = f[20:40]                                          # duplicates
    f[40:50, 2] = f[40:50, 1]                                  # two equal corners: zero area
    v[f[50:60, 2]] = v[f[50:60, 0]]                            # coincident corners
    return v, f.astype(np.int32)


def strip(n, offset):
    """a connected strip of 2 n unit right triangles on the integer grid: area 0.5 each, exact; 2 n + 2 vertices"""
    v = np.array([[offset + i, j, 0] for i in range(n + 1) for j in (0, 1)], np.float32)
    f = [[2 * i, 2 * i + 2, 2 * i + 1] for i in range(n)] + [[2 * i + 1, 2 * i + 2, 2 * i + 3] for i in range(n)]
    return v, np.array(f, np.int32)


def cases():
    out = {}
    for s in range(3):
        out[f"blobs{s}"] = blobs(36 + 4 * s, s)
    for s in range(6):
        out[f"soup{s}"] = soup(s)
    # more faces, less area: 50 tiny triangles (vertex ids first) against one large one
    va, fa = strip(25, 0)
    va *= 0.01
    vb = np.array([[10, 0, 0], [20, 0, 0], [10, 10, 0]], np.float32)
    out["many_small"] = (np.concatenate([va, vb]), np.concatenate([fa, [[52, 53, 54]]]).astype(np.int32))
    # exact ties: translated integer copies of one mesh; the copy listed first in the faces has the larger vertex ids
    v1, f1 = strip(4, 0)
    v2, _ = strip(4, 100)
    v3, _ = strip(4, -50)
    out["tie"] = (np.concatenate([v1, v2, v3]), np.concatenate([f1 + 20, f1 + 10, f1]).astype(np.int32))
    out["tie_reversed"] = (np.concatenate([v1, v2]), np.concatenate([f1 + 10, f1]).astype(np.int32)[::-1].copy())
    # every area zero, vertex 0 isolated: the component of vertex 0 is chosen, and it has no face
    vz = np.zeros((6, 3), np.float32)
    vz[:, 0] = np.arange(6)
    out["zero_area"] = (vz, np.array([[1, 2, 3], [3, 4, 5]], np.int32))
    out["zero_area_v0_used"] = (vz, np.array([[1, 2, 3], [3, 4, 0]], np.int32))
    out["single"] = (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32), np.array([[0, 1, 2]], np.int32))
    out["single_unused"] = (np.array([[5, 5, 5], [0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32), np.array([[3, 1, 2]], np.int32))
    return out


# ---------------------------------------------------------------- numpy / scipy side

def reference_parts(v, f):
    """what meshing.largest_component computes on the way: scipy labels, float32 face areas, bincount sums"""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components

    f64 = f.astype(np.int64)
    nv = v.shape[0]
    e = np.concatenate([f64[:, [0, 1]], f64[:, [1, 2]], f64[:, [2, 0]]], 0)
    g = sp.coo_matrix((np.ones(e.shape[0], np.int8), (e[:, 0], e[:, 1])), shape=(nv, nv))
    _, label = connected_components(g, directed=False)
    tri = v[f64]
    area = 0.5 * np.linalg.norm(np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), axis=1)
    per = np.bincount(label[f64[:, 0]], weights=area)
    return label, area, per


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


@pytest.fixture(scope="module")
def all_cases():
    return cases()


NAMES = ["blobs0", "blobs1", "blobs2", "soup0", "soup1", "soup2", "soup3", "soup4", "soup5", "many_small", "tie", "tie_reversed",
         "zero_area", "zero_area_v0_used", "single", "single_unused"]


def test_case_names(all_cases):
    assert sorted(NAMES) == sorted(all_cases)


@pytest.mark.parametrize("name", NAMES)
def test_equals_host_selection(all_cases, name):
    from hold_b200.meshing import largest_component

    v, f = all_cases[name]
    ref_v, ref_f = largest_component(v, f.astype(np.int64))
    hv, hf, labels, area, sums, best = host_largest(v, f)
    assert hv.dtype == ref_v.dtype == np.float32
    assert hv.shape == ref_v.shape and hf.shape == ref_f.shape
    assert np.array_equal(bits(hv), bits(ref_v)) and np.array_equal(hf, ref_f), name
    label, ref_area, per = reference_parts(v, f)
    # labels: the smallest vertex of each scipy component, and scipy numbers the components in that order
    mins = np.full(label.max() + 1, v.shape[0])
    np.minimum.at(mins, label, np.arange(v.shape[0]))
    assert np.array_equal(labels, mins[label]) and np.all(np.diff(mins) > 0)
    assert ref_area.dtype == np.float32 and np.array_equal(bits(area), bits(ref_area))
    assert np.array_equal(bits(sums[mins[: per.shape[0]]]), bits(per))
    assert best == mins[int(np.argmax(per))]
    print(f"{name}: V {v.shape[0]} F {f.shape[0]}, {label.max() + 1} components -> V {hv.shape[0]} F {hf.shape[0]}")


def test_cases_cover_what_they_claim(all_cases):
    from hold_b200.meshing import largest_component

    v, f = all_cases["many_small"]
    _, hf, *_ = host_largest(v, f)
    assert hf.shape[0] == 1                                          # the single large face wins over 50 small ones
    v, f = all_cases["tie"]
    _, area, per = reference_parts(v, f)
    assert per[0] == per[1] == per[2]                                # three exact ties ...
    _, hf, _, _, _, best = host_largest(v, f)
    assert best == 0 and hf.shape[0] == 8 and np.array_equal(np.unique(hf), np.arange(10))   # ... the smallest label wins
    assert (largest_component(v, f)[1] == hf).all()
    v, f = all_cases["zero_area"]
    hv, hf, *_ = host_largest(v, f)
    assert hv.shape[0] == 0 and hf.shape[0] == 0
    for s in range(6):
        v, f = all_cases[f"soup{s}"]
        label, area, _ = reference_parts(v, f)
        assert (area == 0).any() and np.setdiff1d(np.arange(v.shape[0]), f).size > 0
        assert np.unique(np.sort(f, 1), axis=0).shape[0] < f.shape[0]
    assert max(reference_parts(*all_cases["blobs0"])[0]) >= 3         # several blobs


@pytest.mark.parametrize("name", ["blobs0", "blobs2", "soup0", "soup3", "tie"])
def test_labels_do_not_depend_on_the_join_order(all_cases, name):
    v, f = all_cases[name]
    V, F = v.shape[0], f.shape[0]
    ref = host_labels(V, f)
    assert np.array_equal(host_labels(V, f, np.arange(F)[::-1]), ref)
    rng = np.random.default_rng(7)
    for _ in range(5):
        assert np.array_equal(host_labels(V, f, rng.permutation(F)), ref)
    full = host_largest(v, f, rng.permutation(F))
    base = host_largest(v, f)
    assert all(np.array_equal(bits(a), bits(b)) for a, b in zip(full[:5], base[:5])) and full[5] == base[5]


def test_area_order_of_the_norm():
    """numpy's norm over three float32 components is (x0^2 + x1^2) + x2^2: the kernels' order, on 200 000 random rows"""
    rng = np.random.default_rng(3)
    v = (rng.standard_normal((200000, 3, 3)) * 10.0 ** rng.uniform(-3, 3, (200000, 1, 1))).astype(np.float32)
    f = np.arange(600000, dtype=np.int32).reshape(-1, 3)
    area = np.zeros(200000, np.float32)
    _lib().cc_areas_host(_p(np.ascontiguousarray(v.reshape(-1, 3))), 200000, _p(f), _p(area))
    tri = v
    ref = 0.5 * np.linalg.norm(np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), axis=1)
    assert np.array_equal(bits(area), bits(ref))


def test_argmax_order():
    lib = _lib()
    nan = float("nan")
    assert lib.cc_before_host(2.0, 5, 1.0, 0) and not lib.cc_before_host(1.0, 0, 2.0, 5)
    assert lib.cc_before_host(1.0, 3, 1.0, 4) and not lib.cc_before_host(1.0, 4, 1.0, 3)      # ties: the smaller label
    assert lib.cc_before_host(nan, 9, float("inf"), 0) and not lib.cc_before_host(float("inf"), 0, nan, 9)   # the first NaN
    assert lib.cc_before_host(nan, 2, nan, 3) and not lib.cc_before_host(nan, 3, nan, 2)
    per = np.array([1.0, nan, 3.0, nan])
    assert int(np.argmax(per)) == 1


def test_new_kernels_have_no_float_atomics(built):
    from hold_b200 import capi

    funcs = _sass_by_function(capi.LIB_PATH)
    names = [k for k in funcs if "k_cc_" in k]
    assert len(names) == 9, names
    for k in names:
        bad = [op for op in funcs[k] if FLOAT_GLOBAL_ADD.match(op) or (op.startswith(("ATOM", "RED")) and ".F" in op)]
        print(f"{k}: {len(funcs[k])} SASS instructions, {len(bad)} floating-point atomics")
        assert not bad, (k, sorted(set(bad)))
