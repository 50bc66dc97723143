"""CPU-only: the point-cloud evaluation steps as the CUDA kernels run them (hold_b200/csrc/pointcloud_phases.h compiled for the
host) against the oracle (oracle/pointcloud_oracle.py): top-K in (distance, index) order with duplicates and K > P, the ICP
correspondence bound, the 3x3 SVD and Umeyama (random, rank-deficient and reflected correspondences, with and without scaling,
against numpy), the ICP bookkeeping; the oracle's chamfer / F-score reductions against torch on CPU tensors; the argument
checks of hold_b200.pointcloud."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import pointcloud_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    out = os.path.join(ROOT, "tests", "_build", "libpointcloud_host.so")
    src = os.path.join(ROOT, "tests", "host", "pointcloud_host.cpp")
    hdrs = [os.path.join(ROOT, "hold_b200", "csrc", h) for h in ("pointcloud_phases.h", "knn_phases.h")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(p) for p in [src] + hdrs):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", out, src], check=True)
    lib = C.CDLL(out)
    lib.corr_host.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p]
    lib.fitness_rmse_host.argtypes = [C.c_double, C.c_double, C.c_double, C.c_void_p]
    lib.converged_host.argtypes = [C.c_double] * 6
    return lib


_p = lambda a: a.ctypes.data_as(C.c_void_p)


def _svd(lib, A):
    A = np.ascontiguousarray(A, np.float64)
    U, s, V = np.zeros(9), np.zeros(3), np.zeros(9)
    lib.svd3_host(_p(A), _p(U), _p(s), _p(V))
    return U.reshape(3, 3), s, V.reshape(3, 3)


def _umeyama(lib, src, dst, scaling):
    src, dst = np.ascontiguousarray(src, np.float64), np.ascontiguousarray(dst, np.float64)
    T = np.zeros(12)
    lib.umeyama_host(len(src), _p(src), _p(dst), int(scaling), _p(T))
    return np.vstack([T.reshape(3, 4), [0, 0, 0, 1]])


@pytest.mark.parametrize("K", [1, 3, 15, 32])
def test_topk_duplicates_and_k_beyond_p(K):
    lib = _lib()
    rng = np.random.default_rng(K)
    for P in (5, 40, 300):
        p = rng.normal(size=(P, 3)).astype(np.float32)
        p[P // 2] = p[1]                      # duplicates: exact ties, resolved by index
        p[P - 1] = p[1]
        q = rng.normal(size=(200, 3)).astype(np.float32)
        q[0] = p[1]                           # a query on a triplicated point
        q[1] = q[2]
        d, i = np.zeros((200, K), np.float32), np.zeros((200, K), np.int32)
        assert lib.topk_host(200, P, _p(q), _p(p), K, _p(d), _p(i)) == 0
        rd, ri = O.knn_brute(q, p, K)
        k = min(K, P)
        assert np.array_equal(i[:, :k], ri[:, :k]) and np.array_equal(d[:, :k], rd[:, :k])
        assert (i[:, k:] == 2**31 - 1).all() and np.isinf(d[:, k:]).all()   # empty slots (the kernel writes them as padding)
        assert i[0, 0] == 1 and d[0, 0] == 0.0
        if K >= 3 and P >= 3:
            assert list(i[0, :3]) == [1, P // 2, P - 1]


def test_correspondence_bound_is_strict():
    lib = _lib()
    rng = np.random.default_rng(0)
    p = rng.normal(size=(50, 3))
    q = rng.normal(size=(64, 3))
    full, fi = O.knn_brute(q, p, 1)
    max_d2 = float(np.sort(full[:, 0])[32])   # one query's nearest distance equals the bound exactly: not a correspondence
    d, i = np.zeros(64), np.zeros(64, np.int32)
    lib.corr_host(64, 50, _p(q), _p(p), max_d2, _p(d), _p(i))
    ok = full[:, 0] < max_d2
    assert (full[:, 0] == max_d2).sum() >= 1
    assert np.array_equal(i >= 0, ok) and np.array_equal(i[ok], fi[ok, 0]) and np.array_equal(d[ok], full[ok, 0])
    idx, d2, _, _ = O.correspondences(q, p, np.sqrt(max_d2))
    assert np.array_equal(idx >= 0, (full[:, 0] < np.sqrt(max_d2) ** 2))


def _check_svd(lib, A, tol=1e-12):
    U, s, V = _svd(lib, A)
    sr = np.linalg.svd(A, compute_uv=False)
    scale = max(sr[0], 1e-300)
    assert np.all(np.diff(s) <= 0) and np.all(s >= 0)
    assert np.abs(s - sr).max() <= tol * scale, (s, sr)
    assert np.abs(U.T @ U - np.eye(3)).max() <= tol and np.abs(V.T @ V - np.eye(3)).max() <= tol
    assert np.abs(U @ np.diag(s) @ V.T - A).max() <= tol * scale


def test_svd3():
    lib = _lib()
    rng = np.random.default_rng(1)
    for _ in range(300):
        _check_svd(lib, rng.normal(size=(3, 3)) * 10.0 ** rng.uniform(-4, 4))
    a, b, c = rng.normal(size=(3, 3))
    _check_svd(lib, np.outer(a, b))                           # rank 1
    _check_svd(lib, np.outer(a, b) + np.outer(c, a))          # rank 2
    _check_svd(lib, np.diag([3.0, 3.0, 1.0]))                 # repeated singular values
    _check_svd(lib, np.diag([1.0, -2.0, 0.5]))
    _check_svd(lib, np.zeros((3, 3)))


def _rot(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


@pytest.mark.parametrize("scaling", [False, True])
def test_umeyama(scaling):
    lib = _lib()
    rng = np.random.default_rng(2 + scaling)
    for case in range(60):
        m = int(rng.integers(3, 200))
        src = rng.normal(size=(m, 3))
        R, t, c = _rot(rng), rng.normal(size=3), rng.uniform(0.5, 2.0)
        dst = c * src @ R.T + t + rng.normal(size=(m, 3)) * 0.1 * (case % 3)
        if case % 5 == 4:
            dst[:, 0] = -dst[:, 0]                            # a reflection: det U det V < 0
        if case % 7 == 6:
            src[:, 2] = 0.3                                   # coplanar source: rank 2
        T, Tr = _umeyama(lib, src, dst, scaling), O.umeyama(src, dst, scaling)
        assert np.abs(T - Tr).max() <= 1e-12 * max(1.0, np.abs(Tr).max()), (case, T, Tr)
        Rn = T[:3, :3] / np.cbrt(np.linalg.det(T[:3, :3]))
        assert np.abs(Rn @ Rn.T - np.eye(3)).max() <= 1e-12 and np.linalg.det(T[:3, :3]) > 0


@pytest.mark.parametrize("scaling", [False, True])
def test_umeyama_collinear(scaling):
    """Rank 1: the rotation about the line is not unique, so R is held to being a rotation and the moved points to numpy's."""
    lib = _lib()
    rng = np.random.default_rng(9)
    w = rng.normal(size=3)
    src = rng.normal(size=(40, 1)) * w + rng.normal(size=3)
    dst = 1.5 * src @ _rot(rng).T + rng.normal(size=3)
    T, Tr = _umeyama(lib, src, dst, scaling), O.umeyama(src, dst, scaling)
    Rn = T[:3, :3] / np.cbrt(np.linalg.det(T[:3, :3]))
    assert np.abs(Rn @ Rn.T - np.eye(3)).max() <= 1e-12 and np.linalg.det(T[:3, :3]) > 0
    assert np.abs(O.transform(T, src) - O.transform(Tr, src)).max() <= 1e-12 * np.abs(dst).max()
    assert np.abs(np.linalg.det(T[:3, :3]) - np.linalg.det(Tr[:3, :3])) <= 1e-12


def test_umeyama_empty_and_degenerate():
    lib = _lib()
    assert np.array_equal(_umeyama(lib, np.zeros((0, 3)), np.zeros((0, 3)), False), np.eye(4))
    s = np.array([[1.0, 2.0, 3.0]])
    T = _umeyama(lib, s, s + [0.5, -1.0, 2.0], False)   # one correspondence: a pure translation
    assert np.array_equal(T[:3, :3], np.eye(3)) and np.allclose(T[:3, 3], [0.5, -1.0, 2.0], atol=1e-15)


def test_compose_and_apply():
    lib = _lib()
    rng = np.random.default_rng(4)
    T = np.eye(4)
    T[:3] = rng.normal(size=(3, 4))
    U = np.ascontiguousarray(rng.normal(size=(3, 4)))
    Tc = T.reshape(-1).copy()
    lib.compose_host(_p(U), _p(Tc))
    assert np.abs(Tc.reshape(4, 4) - np.vstack([U, [0, 0, 0, 1]]) @ T).max() <= 1e-14
    x = np.ascontiguousarray(rng.normal(size=3))
    y = x.copy()
    lib.apply_host(_p(U), _p(y))
    assert np.abs(y - (U[:, :3] @ x + U[:, 3])).max() <= 1e-14


def test_icp_bookkeeping():
    lib = _lib()
    out = np.zeros(2)
    lib.fitness_rmse_host(0.0, 0.0, 10.0, _p(out))
    assert list(out) == [0.0, 0.0]
    lib.fitness_rmse_host(3.0, 12.0, 4.0, _p(out))
    assert list(out) == [0.75, 2.0]
    assert lib.converged_host(0.5, 0.1, 0.5, 0.1, 1e-6, 1e-6) == 1
    assert lib.converged_host(0.5, 0.1, 0.5 + 2e-6, 0.1, 1e-6, 1e-6) == 0
    assert lib.converged_host(0.5, 0.1, 0.5, 0.1 - 2e-6, 1e-6, 1e-6) == 0
    assert lib.converged_host(0.5, 0.25, 0.5, 0.5, 1e-6, 0.25) == 0       # |d rmse| == the threshold: strict
    # the oracle's loop: a shifted copy converges with fitness 1 and rmse 0
    rng = np.random.default_rng(5)
    src = rng.normal(size=(100, 3))
    T, fit, rmse, it = O.icp(src, src + [0.01, 0.0, -0.02], 0.5)
    assert fit == 1.0 and rmse < 1e-12 and np.allclose(T[:3, 3], [0.01, 0.0, -0.02], atol=1e-12) and 1 <= it < 30
    T, fit, rmse, it = O.icp(src, src + 10.0, 0.5)                         # nothing in range: the identity
    assert np.array_equal(T, np.eye(4)) and fit == 0.0 and rmse == 0.0


def _torch_cham(x, y, xl, yl):
    from hold_b200 import fitting

    out = []
    for n in range(x.shape[0]):
        a, b = x[n:n + 1, :xl[n]], y[n:n + 1, :yl[n]]
        cx = fitting.knn_points(a, b, 1).dists[0, :, 0] if xl[n] and yl[n] else torch.zeros(xl[n], dtype=x.dtype)
        cy = fitting.knn_points(b, a, 1).dists[0, :, 0] if xl[n] and yl[n] else torch.zeros(yl[n], dtype=x.dtype)
        out.append((cx, cy))
    return out


@pytest.mark.parametrize("batch_reduction", [None, "sum", "mean"])
@pytest.mark.parametrize("point_reduction", ["sum", "mean"])
def test_oracle_chamfer_reductions(batch_reduction, point_reduction):
    g = torch.Generator().manual_seed(6)
    x, y = torch.randn(3, 40, 3, generator=g, dtype=torch.float64), torch.randn(3, 30, 3, generator=g, dtype=torch.float64)
    xl, yl = [40, 17, 0], [30, 30, 5]
    per = _torch_cham(x, y, xl, yl)
    cx = torch.stack([c.sum() for c, _ in per])
    cy = torch.stack([c.sum() for _, c in per])
    if point_reduction == "mean":
        cx, cy = cx / torch.tensor(xl).clamp(min=1), cy / torch.tensor(yl).clamp(min=1)
    if batch_reduction is not None:
        cx, cy = cx.sum(), cy.sum()
        if batch_reduction == "mean":
            cx, cy = cx / 3, cy / 3
    ref = (cx + cy).numpy()
    got = O.chamfer_distance(x.numpy(), y.numpy(), xl, yl, batch_reduction, point_reduction)
    assert np.allclose(got, ref, rtol=1e-12, atol=0)


def test_oracle_fscore():
    g = torch.Generator().manual_seed(7)
    x, y = torch.randn(2, 50, 3, generator=g, dtype=torch.float64), torch.randn(2, 60, 3, generator=g, dtype=torch.float64)
    xl, yl = [50, 20], [60, 0]
    tau = [0.1, 0.3, 1.0]
    f, p, r = O.fscore(x.numpy(), y.numpy(), tau, xl, yl)
    d = torch.cdist(x[0], y[0])
    for k, t in enumerate(tau):
        pk, rk = (d.min(1).values < t).double().mean().item(), (d.min(0).values < t).double().mean().item()
        assert p[0, k] == pytest.approx(pk, abs=1e-15) and r[0, k] == pytest.approx(rk, abs=1e-15)
        assert f[0, k] == pytest.approx(0.0 if pk + rk == 0 else 2 * pk * rk / (pk + rk), abs=1e-15)
    assert (p[1] == 0).all() and (r[1] == 0).all() and (f[1] == 0).all()   # an empty gt


def test_python_argument_checks():
    from hold_b200 import pointcloud as PC

    x, y = torch.zeros(2, 5, 3), torch.zeros(2, 4, 3)
    with pytest.raises(ValueError):
        PC.chamfer_distance(None, x, y, x_normals=x)
    with pytest.raises(ValueError):
        PC.chamfer_distance(None, x, y, norm=1)
    with pytest.raises(ValueError):
        PC.chamfer_distance(None, x, y, single_directional=True)
    with pytest.raises(ValueError):
        PC.chamfer_distance(None, x, y, batch_reduction="max")
    with pytest.raises(ValueError):
        PC.knn_points(None, x, y, K=33)
    with pytest.raises(ValueError):
        PC.knn_points(None, x, y, lengths1=torch.tensor([6, 1]))
    with pytest.raises(ValueError):
        PC.knn_points(None, x, torch.zeros(3, 4, 3))
    with pytest.raises(ValueError):
        PC.knn_points(None, torch.zeros(2, 5, 2), torch.zeros(2, 4, 2))


class _Saved:
    """stand-in for the autograd context of KnnPointsFn.backward"""

    def __init__(self, *saved):
        self.saved_tensors, self.dtypes = saved, (torch.float32, torch.float32)


def test_knn_backward_reads_only_valid_slots():
    """pytorch3d's backward over the valid slots only: inf / NaN padding rows and an empty second cloud give finite (zero)
    gradients, and no index of an empty cloud is read."""
    from hold_b200.pointcloud import KnnPointsFn

    g = torch.Generator().manual_seed(8)
    a = torch.randn(2, 4, 3, generator=g)
    b = torch.randn(2, 5, 3, generator=g)
    a[0, 3] = float("inf")                      # padding row of p1
    b[1, 2:] = float("nan")                     # padding of p2
    l1, l2 = torch.tensor([3, 4], dtype=torch.int32), torch.tensor([5, 2], dtype=torch.int32)
    K = 3
    idx = torch.zeros(2, 4, K, dtype=torch.int32)
    for n in range(2):
        for i in range(int(l1[n])):
            d = ((a[n, i] - b[n, :int(l2[n])]) ** 2).sum(-1)
            o = torch.argsort(d, stable=True)[:K]
            idx[n, i, :len(o)] = o.int()
    gd = torch.randn(2, 4, K, generator=g)
    gd[0, 3] = float("nan")                     # an upstream gradient in a padding slot is ignored too
    g1, g2, *_ = KnnPointsFn.backward(_Saved(a, b, l1, l2, idx), gd, None)
    assert torch.isfinite(g1).all() and torch.isfinite(g2).all()
    r1, r2 = torch.zeros_like(a), torch.zeros_like(b)
    for n in range(2):
        for i in range(int(l1[n])):
            for k in range(min(K, int(l2[n]))):
                j = int(idx[n, i, k])
                dd = 2.0 * (a[n, i] - b[n, j]) * gd[n, i, k]
                r1[n, i] += dd
                r2[n, j] -= dd
    assert torch.allclose(g1, r1, rtol=1e-6, atol=1e-6) and torch.allclose(g2, r2, rtol=1e-6, atol=1e-6)
    # an empty second cloud: zero gradients, nothing gathered
    e = torch.empty(2, 0, 3)
    g1, g2, *_ = KnnPointsFn.backward(_Saved(a, e, l1, torch.zeros(2, dtype=torch.int32), idx), gd, None)
    assert g2.shape == (2, 0, 3) and torch.equal(g1, torch.zeros_like(a))


def test_lengths_checked_together():
    from hold_b200.pointcloud import _check_lengths, check_lengths

    l1, l2 = _check_lengths(((torch.tensor([3, 0]), 4, "a"), (None, 6, "b")), 2, "cpu")
    assert l1.dtype == torch.int32 and l1.tolist() == [3, 0] and l2.tolist() == [6, 6]
    with pytest.raises(ValueError, match="b span"):
        _check_lengths(((torch.tensor([3, 0]), 4, "a"), (torch.tensor([7, 1]), 6, "b")), 2, "cpu")
    with pytest.raises(ValueError, match="must be"):
        check_lengths(torch.tensor([1, 2, 3]), 2, 4, "cpu")
