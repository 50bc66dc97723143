"""CPU restatement of the point-cloud evaluation: pytorch3d v0.7.4's knn_points / chamfer_distance rules, an F-score at
distance thresholds, and open3d's point-to-point ICP (registration_icp + TransformationEstimationPointToPoint, Eigen::umeyama).
Neither library is available to pin these, so they are restated here, unpinned.  The rules live in exactly two places, this
file and hold_b200/csrc/pointcloud_phases.h, which change together (DESIGN.md row 4d).

The KNN computes the squared distance as ((dx*dx + dy*dy) + dz*dz) in the inputs' dtype (numpy never contracts to FMA) and
orders by (distance, index); ICP runs it in float64.  Umeyama uses numpy.linalg.svd.
"""
from __future__ import annotations

import numpy as np


def sq_dist(q, p):
    """[Q,P] squared distances ((dx*dx + dy*dy) + dz*dz) in the common dtype of q [Q,3] and p [P,3]."""
    d = q[:, None, :] - p[None, :, :]
    s = d * d
    return (s[..., 0] + s[..., 1]) + s[..., 2]


def knn_brute(q, p, K, chunk=512):
    """Exact K nearest (dists [Q,K], idx [Q,K]) of q [Q,3] in p [P,3], (distance, index) order; K > P leaves -1 / inf."""
    Q, P = q.shape[0], p.shape[0]
    k = min(K, P)
    dists = np.full((Q, K), np.inf, dtype=np.result_type(q, p))
    idx = np.full((Q, K), -1, dtype=np.int64)
    for a in range(0, Q, chunk):
        d = sq_dist(q[a:a + chunk], p)
        if k == 1:   # argmin returns the first of equal minima: the lower index
            o = np.argmin(d, axis=-1)[:, None]
        else:
            o = np.lexsort((np.broadcast_to(np.arange(P), d.shape), d), axis=-1)[:, :k]
        idx[a:a + chunk, :k] = o
        dists[a:a + chunk, :k] = np.take_along_axis(d, o, -1)
    return dists, idx


def knn_kdtree(q, p, K):
    """cKDTree path for large clouds: (float64 squared dists [Q,K], idx [Q,K]).  Ties are not ordered by index."""
    from scipy.spatial import cKDTree

    d, i = cKDTree(np.asarray(p, np.float64)).query(np.asarray(q, np.float64), k=K)
    d, i = np.asarray(d).reshape(len(q), K), np.asarray(i).reshape(len(q), K)
    return d * d, i


def knn_points(p1, p2, lengths1=None, lengths2=None, K=1):
    """knn_points over a batch: p1 [N,P1,3], p2 [N,P2,3] -> dists [N,P1,K], idx [N,P1,K] int64, padding slots 0."""
    N, P1, P2 = p1.shape[0], p1.shape[1], p2.shape[1]
    l1 = np.full(N, P1) if lengths1 is None else np.asarray(lengths1)
    l2 = np.full(N, P2) if lengths2 is None else np.asarray(lengths2)
    dists = np.zeros((N, P1, K), dtype=np.result_type(p1, p2))
    idx = np.zeros((N, P1, K), dtype=np.int64)
    for n in range(N):
        a, b = int(l1[n]), int(l2[n])
        if a == 0 or b == 0:
            continue
        d, i = knn_brute(p1[n, :a], p2[n, :b], K)
        k = min(K, b)
        dists[n, :a, :k], idx[n, :a, :k] = d[:, :k], i[:, :k]
    return dists, idx


def chamfer_distance(x, y, x_lengths=None, y_lengths=None, batch_reduction="mean", point_reduction="mean"):
    """pytorch3d v0.7.4 chamfer_distance (no normals / weights, norm 2), float64."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    N, P1, P2 = x.shape[0], x.shape[1], y.shape[1]
    xl = np.full(N, P1) if x_lengths is None else np.asarray(x_lengths)
    yl = np.full(N, P2) if y_lengths is None else np.asarray(y_lengths)
    cx, _ = knn_points(x, y, xl, yl, 1)
    cy, _ = knn_points(y, x, yl, xl, 1)
    cx, cy = cx[..., 0].sum(1), cy[..., 0].sum(1)
    if point_reduction == "mean":
        cx, cy = cx / np.maximum(xl, 1), cy / np.maximum(yl, 1)
    if batch_reduction is not None:
        cx, cy = cx.sum(), cy.sum()
        if batch_reduction == "mean":
            cx, cy = cx / max(N, 1), cy / max(N, 1)
    return cx + cy


def fscore(pred, gt, thresholds, pred_lengths=None, gt_lengths=None):
    """(f, precision, recall) [N,T] float64: precision = share of valid pred points with sqrt(d^2) < tau, recall the same for gt;
    f = 2pr/(p+r), 0 when p + r = 0; a point has no neighbour in an empty cloud, an empty cloud's share is 0."""
    pred, gt = np.asarray(pred), np.asarray(gt)   # distances in the clouds' dtype, their square roots compared in float64
    tau = np.asarray(thresholds, np.float64).reshape(-1)
    N, P1, P2 = pred.shape[0], pred.shape[1], gt.shape[1]
    pl = np.full(N, P1) if pred_lengths is None else np.asarray(pred_lengths)
    gl = np.full(N, P2) if gt_lengths is None else np.asarray(gt_lengths)

    def share(a, b, la, lb):
        out = np.zeros((N, len(tau)))
        for n in range(N):
            if la[n] == 0 or lb[n] == 0:
                continue
            d, _ = knn_brute(a[n, :la[n]], b[n, :lb[n]], 1)
            out[n] = (np.sqrt(d[:, 0].astype(np.float64))[:, None] < tau[None]).sum(0) / la[n]
        return out

    p, r = share(pred, gt, pl, gl), share(gt, pred, gl, pl)
    s = p + r
    f = np.where(s > 0, 2 * p * r / np.where(s > 0, s, 1.0), 0.0)
    return f, p, r


def umeyama(src, dst, with_scaling=False):
    """Eigen::umeyama(src [m,3], dst [m,3]) -> 4x4 [cR | t].  m = 0: the identity."""
    T = np.eye(4)
    m = src.shape[0]
    if m == 0:
        return T
    inv = 1.0 / m
    mu_s, mu_d = src.sum(0) * inv, dst.sum(0) * inv
    ds, dd = src - mu_s, dst - mu_d
    var_s = (ds * ds).sum() * inv
    sigma = (dd.T @ ds) * inv
    U, sv, Vt = np.linalg.svd(sigma)
    S = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1.0
    R = U @ np.diag(S) @ Vt
    c = (sv @ S) / var_s if with_scaling else 1.0
    T[:3, :3] = c * R
    T[:3, 3] = mu_d - c * (R @ mu_s)
    return T


def transform(T, x):
    return x @ T[:3, :3].T + T[:3, 3]


def correspondences(xs, tgt, max_d):
    """open3d's GetRegistrationResultAndCorrespondences: the nearest target point (ties to the lower index) of each source
    point, kept when d^2 < max_d^2 (strict); -> (idx [Ps] or -1, d2 [Ps], fitness, inlier_rmse)."""
    Ps = xs.shape[0]
    idx = np.full(Ps, -1, np.int64)
    d2 = np.zeros(Ps)
    if max_d > 0 and Ps > 0 and tgt.shape[0] > 0:
        d, i = knn_brute(xs, tgt, 1)
        ok = d[:, 0] < max_d * max_d
        idx[ok], d2[ok] = i[ok, 0], d[ok, 0]
    n = int((idx >= 0).sum())
    if n == 0:
        return idx, d2, 0.0, 0.0
    return idx, d2, n / Ps, float(np.sqrt(d2[idx >= 0].sum() / n))


def icp(source, target, max_correspondence_distance, init=None, with_scaling=False, relative_fitness=1e-6, relative_rmse=1e-6,
        max_iteration=30):
    """open3d registration_icp (point to point) for one pair: -> (T 4x4, fitness, inlier_rmse, iterations run)."""
    src, tgt = np.asarray(source, np.float64), np.asarray(target, np.float64)
    T = np.eye(4) if init is None else np.asarray(init, np.float64).copy()
    xs = src if init is None else transform(T, src)
    idx, _, fit, rmse = correspondences(xs, tgt, max_correspondence_distance)
    it = 0
    for i in range(max_iteration):
        ok = idx >= 0
        upd = umeyama(xs[ok], tgt[idx[ok]], with_scaling)
        T = upd @ T
        xs = transform(upd, xs)
        fit0, rmse0 = fit, rmse
        idx, _, fit, rmse = correspondences(xs, tgt, max_correspondence_distance)
        it = i + 1
        if abs(fit0 - fit) < relative_fitness and abs(rmse0 - rmse) < relative_rmse:
            break
    return T, fit, rmse, it
