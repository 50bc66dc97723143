"""The point-cloud metrics of the reference's evaluate.py (utils/eval_modules.py) without pytorch3d or open3d: exact K-nearest
neighbours (hold_knn_points), pytorch3d's chamfer_distance on top of them, an F-score at distance thresholds, and open3d's
point-to-point ICP (hold_icp), all on the library's sm_90a kernels.

The rules are pytorch3d v0.7.4's and open3d's, restated and unpinned (hold_b200/csrc/pointcloud_phases.h and
oracle/pointcloud_oracle.py, DESIGN.md row 4d).  The evaluation protocol itself (which frames, alignment variants, units) is
the caller's.
"""
from __future__ import annotations

import collections

import torch

from .capi import KNN_MAX_K, IcpCfg, check, lib, ptr, stream_ptr
from .fitting import KNN

ICPResult = collections.namedtuple("ICPResult", ["transformation", "fitness", "inlier_rmse", "iterations"])


def _cloud(p, name):
    if p.dim() != 3 or p.shape[2] != 3:
        raise ValueError(f"{name} must be [N,P,3], got {tuple(p.shape)}")
    return p


def check_lengths(lengths, N, P, device, name="lengths"):
    """lengths as contiguous int32 [N] on `device`, every entry in [0, P] (None: all P).  One min / max read by the host: this
    synchronises the stream once when lengths are given."""
    return _check_lengths(((lengths, P, name),), N, device)[0]


def _check_lengths(specs, N, device):
    """check_lengths for several (lengths, P, name) at once, with a single host read for all the given ones."""
    out, given = [], []
    for lengths, P, name in specs:
        if lengths is None:
            out.append(torch.full((N,), P, dtype=torch.int32, device=device))
            continue
        l = torch.as_tensor(lengths).to(device=device, dtype=torch.int32).contiguous()
        if l.shape != (N,):
            raise ValueError(f"{name} must be [{N}], got {tuple(l.shape)}")
        out.append(l)
        given.append((l, P, name))
    if given and N > 0:
        spans = torch.stack([torch.stack(tuple(torch.aminmax(l))) for l, _, _ in given]).tolist()   # the one synchronisation
        for (lo, hi), (_, P, name) in zip(spans, given):
            if lo < 0 or hi > P:
                raise ValueError(f"{name} span [{lo}, {hi}], outside [0, {P}]")
    return out


def _valid(l1, l2, P1, K):
    """[N,P1,K] mask of the slots that hold a neighbour: row < lengths1[n] and k < lengths2[n]."""
    dev = l1.device
    return (torch.arange(P1, device=dev)[None, :, None] < l1[:, None, None]) & (torch.arange(K, device=dev)[None, None, :] < l2[:, None, None])


class KnnPointsFn(torch.autograd.Function):
    """dists [N,P1,K] (squared, differentiable in p1 and p2) and idx [N,P1,K] int32 of hold_knn_points, and with return_nn
    knn [N,P1,K,3] = p2[idx] in p2's dtype, zero in the slots k >= lengths2 (pytorch3d's knn_gather, differentiable in p2).
    The backward is pytorch3d's on hold_knn_points_bwd: g_p1 += 2 (p1 - p2[idx]) g, g_p2[idx] -= the same over the valid
    slots, plus knn's gradient at idx; every sum in a fixed order (bitwise reproducible), accumulated in fp32."""

    @staticmethod
    def forward(fctx, p1, p2, l1, l2, K, ctx, return_nn=False):
        a, b = p1.detach().float().contiguous(), p2.detach().float().contiguous()
        N, P1, _ = a.shape
        P2 = b.shape[1]
        dists = torch.empty(N, P1, K, device=a.device)
        idx = torch.empty(N, P1, K, dtype=torch.int32, device=a.device)
        check(lib().hold_knn_points(ctx.h, N, P1, ptr(a), ptr(l1), P2, ptr(b), ptr(l2), K, ptr(dists), ptr(idx), stream_ptr()))
        fctx.save_for_backward(a, b, l1, l2, idx)
        fctx.mark_non_differentiable(idx)
        fctx.dtypes, fctx.ctx, fctx.return_nn = (p1.dtype, p2.dtype), ctx, return_nn
        if not return_nn:
            return dists, idx
        if P2 == 0:
            knn = p2.new_zeros(N, P1, K, 3)
        else:
            knn = torch.gather(p2.detach(), 1, idx.long().reshape(N, P1 * K, 1).expand(-1, -1, 3)).reshape(N, P1, K, 3)
            knn = knn * (torch.arange(K, device=p1.device)[None, None, :] < l2[:, None, None])[..., None]
        return dists, idx, knn

    @staticmethod
    def backward(fctx, g_dists, _g_idx, g_knn=None):
        a, b, l1, l2, idx = fctx.saved_tensors
        N, P1, K = idx.shape
        P2 = b.shape[1]
        gd = g_dists.float().contiguous()
        gk = g_knn.float().contiguous() if g_knn is not None and P2 > 0 else None
        if a.is_cuda:
            g1 = torch.empty(N, P1, 3, device=a.device)
            g2 = torch.empty(N, P2, 3, device=b.device)
            # only the valid slots contribute: padding rows of p1 and padding slots (which hold index 0, or address an empty p2)
            # are selected away on the device, so whatever they hold (inf, NaN) does not reach the gradients
            check(lib().hold_knn_points_bwd(fctx.ctx.h, N, P1, ptr(a), ptr(l1), P2, ptr(b), ptr(l2), K, ptr(idx), ptr(gd), ptr(gk),
                                            ptr(g1), ptr(g2), stream_ptr()))
        else:
            g1, g2 = _knn_backward_host(a, b, l1, l2, idx, gd, gk)
        return g1.to(fctx.dtypes[0]), g2.to(fctx.dtypes[1]), None, None, None, None, None


def _knn_backward_host(a, b, l1, l2, idx, gd, gk):
    """hold_knn_points_bwd's rules in torch ops for host tensors, whose index_add_ adds in index order."""
    N, P1, K = idx.shape
    P2 = b.shape[1]
    g1, g2 = torch.zeros(N, P1, 3), torch.zeros(N * P2, 3)
    if P1 > 0 and P2 > 0:
        ok = _valid(l1, l2, P1, K)[..., None]
        il = idx.long()
        nn = torch.gather(b, 1, il.reshape(N, P1 * K, 1).expand(-1, -1, 3)).reshape(N, P1, K, 3)
        diff = torch.where(ok, 2.0 * (a[:, :, None, :] - nn) * gd[..., None], torch.zeros(()))
        g1 = diff.sum(2)
        flat = (il + (torch.arange(N) * P2)[:, None, None]).reshape(-1)
        g2.index_add_(0, flat, -diff.reshape(-1, 3))
        if gk is not None:
            kmask = (torch.arange(K)[None, None, :] < l2[:, None, None])[..., None]
            g2.index_add_(0, flat, torch.where(kmask, gk, torch.zeros(())).reshape(-1, 3))
    return g1, g2.reshape(N, P2, 3)


def _knn(ctx, p1, p2, l1, l2, K, return_nn=False):
    """(dists, idx int64[, knn]) of KnnPointsFn for lengths that _check_lengths has already checked."""
    out = KnnPointsFn.apply(p1, p2, l1, l2, K, ctx, return_nn)
    return (out[0], out[1].long()) + tuple(out[2:])


def knn_points(ctx, p1, p2, lengths1=None, lengths2=None, K=1, return_nn=False):
    """pytorch3d.ops.knn_points (v0.7.4 rules, D = 3) on hold_knn_points: p1 [N,P1,3], p2 [N,P2,3] -> KNN(dists [N,P1,K]
    squared and ascending, idx [N,P1,K] int64, knn [N,P1,K,3] or None).  Ties go to the lower index; padding slots (row >=
    lengths1[n] or k >= lengths2[n]) hold 0.  dists is float32 whatever the inputs' dtype: the kernel computes in fp32 (its
    gradients come back in the inputs' dtypes).  dists is differentiable in p1 and p2, knn in p2; the backward is bitwise
    reproducible (hold_knn_points_bwd).  Checks
    the lengths on the host first (one stream synchronisation when lengths are given)."""
    _cloud(p1, "p1"), _cloud(p2, "p2")
    if p1.shape[0] != p2.shape[0]:
        raise ValueError(f"p1 and p2 batch sizes differ: {p1.shape[0]} vs {p2.shape[0]}")
    if not 1 <= K <= KNN_MAX_K:
        raise ValueError(f"K {K} outside [1, {KNN_MAX_K}]")
    N, P1, P2 = p1.shape[0], p1.shape[1], p2.shape[1]
    l1, l2 = _check_lengths(((lengths1, P1, "lengths1"), (lengths2, P2, "lengths2")), N, p1.device)
    if return_nn:   # pytorch3d's knn_gather (zeros in the slots k >= lengths2), its gradient in the same fixed-order sum
        return KNN(*_knn(ctx, p1, p2, l1, l2, K, True))
    dists, idx = _knn(ctx, p1, p2, l1, l2, K)
    return KNN(dists, idx, None)


def chamfer_distance(ctx, x, y, x_lengths=None, y_lengths=None, x_normals=None, y_normals=None, weights=None,
                     batch_reduction="mean", point_reduction="mean", norm=2, single_directional=False):
    """pytorch3d.loss.chamfer_distance (v0.7.4 rules) for x [N,P1,3], y [N,P2,3] -> (loss, None).  cham_x[n,i] = the squared
    distance from x[n,i] to its nearest y (0 for i >= x_lengths[n]); "sum" sums over the points, "mean" divides that by
    x_lengths clamped to >= 1; batch_reduction None gives [N], "sum" sums over N, "mean" divides the sum by max(N, 1); the
    loss is cham_x + cham_y.  Differentiable in x and y.  Normals, weights, norm = 1 and single_directional are not
    supported (the evaluation does not use them) and raise ValueError."""
    if x_normals is not None or y_normals is not None or weights is not None or norm != 2 or single_directional:
        raise ValueError("chamfer_distance supports neither normals, weights, norm=1 nor single_directional")
    if batch_reduction not in (None, "mean", "sum"):
        raise ValueError('batch_reduction must be one of ["mean", "sum"] or None')
    if point_reduction not in ("mean", "sum"):
        raise ValueError('point_reduction must be one of ["mean", "sum"]')
    _cloud(x, "x"), _cloud(y, "y")
    N, P1, P2 = x.shape[0], x.shape[1], y.shape[1]
    if y.shape[0] != N:
        raise ValueError("y does not have the same batch size as x")
    xl, yl = _check_lengths(((x_lengths, P1, "x_lengths"), (y_lengths, P2, "y_lengths")), N, x.device)
    cham_x = _knn(ctx, x, y, xl, yl, 1)[0][..., 0]
    cham_y = _knn(ctx, y, x, yl, xl, 1)[0][..., 0]
    cham_x = cham_x.masked_fill(torch.arange(P1, device=x.device)[None] >= xl[:, None], 0.0)
    cham_y = cham_y.masked_fill(torch.arange(P2, device=x.device)[None] >= yl[:, None], 0.0)
    cham_x, cham_y = cham_x.sum(1), cham_y.sum(1)
    if point_reduction == "mean":
        cham_x = cham_x / xl.clamp(min=1)
        cham_y = cham_y / yl.clamp(min=1)
    if batch_reduction is not None:
        cham_x, cham_y = cham_x.sum(), cham_y.sum()
        if batch_reduction == "mean":
            cham_x, cham_y = cham_x / max(N, 1), cham_y / max(N, 1)
    return cham_x + cham_y, None


def fscore(ctx, pred, gt, thresholds, pred_lengths=None, gt_lengths=None):
    """F-score of pred [N,P1,3] against gt [N,P2,3] at each distance threshold tau of `thresholds` [T] -> (f, precision,
    recall), each [N,T] float64.  precision = the share of the valid pred points whose nearest-gt distance sqrt(d^2) < tau
    (compared in float64), recall = the same for the gt points; f = 2 p r / (p + r), 0 when p + r = 0.  A point has no
    neighbour when the other cloud is empty; an empty cloud's share is 0."""
    _cloud(pred, "pred"), _cloud(gt, "gt")
    N, P1, P2 = pred.shape[0], pred.shape[1], gt.shape[1]
    if gt.shape[0] != N:
        raise ValueError("gt does not have the same batch size as pred")
    tau = torch.as_tensor(thresholds, dtype=torch.float64, device=pred.device).reshape(-1)
    pl, gl = _check_lengths(((pred_lengths, P1, "pred_lengths"), (gt_lengths, P2, "gt_lengths")), N, pred.device)
    with torch.no_grad():

        def share(a, b, la, lb, P):
            d = _knn(ctx, a, b, la, lb, 1)[0][..., 0].double().sqrt()
            ok = (torch.arange(P, device=a.device)[None] < la[:, None]) & (lb[:, None] > 0)
            hit = (d[:, :, None] < tau[None, None]) & ok[:, :, None]
            return hit.sum(1).double() / la.clamp(min=1)[:, None].double()

        p = share(pred, gt, pl, gl, P1)
        r = share(gt, pred, gl, pl, P2)
        s = p + r
        f = torch.where(s > 0, 2.0 * p * r / torch.where(s > 0, s, torch.ones_like(s)), torch.zeros_like(s))
    return f, p, r


def icp(ctx, source, target, max_correspondence_distance, init=None, with_scaling=False, relative_fitness=1e-6,
        relative_rmse=1e-6, max_iteration=30, source_lengths=None, target_lengths=None):
    """open3d's registration_icp with TransformationEstimationPointToPoint(with_scaling) on hold_icp, for N independent pairs
    source [N,Ps,3], target [N,Pt,3] (or one pair [Ps,3], [Pt,3]) -> ICPResult(transformation [N,4,4], fitness [N],
    inlier_rmse [N] float64, iterations [N] int32), without a batch dimension for one unbatched pair.  init [N,4,4] or [4,4]
    (default: identity).  Points are held in double; no host synchronisation beyond the length check."""
    single = source.dim() == 2
    if single:
        source, target = source[None], target[None]
        if init is not None:
            init = torch.as_tensor(init)
            if init.dim() == 2:
                init = init[None]
    _cloud(source, "source"), _cloud(target, "target")
    N, Ps, Pt = source.shape[0], source.shape[1], target.shape[1]
    if target.shape[0] != N:
        raise ValueError("source and target batch sizes differ")
    if max_iteration < 0:
        raise ValueError(f"max_iteration {max_iteration} < 0")
    dev = source.device
    sl, tl = _check_lengths(((source_lengths, Ps, "source_lengths"), (target_lengths, Pt, "target_lengths")), N, dev)
    s = source.detach().float().contiguous()
    t = target.detach().to(device=dev, dtype=torch.float32).contiguous()
    ini = None
    if init is not None:
        ini = torch.as_tensor(init).to(device=dev, dtype=torch.float64).expand(N, 4, 4).contiguous()
    cfg = IcpCfg(float(max_correspondence_distance), float(relative_fitness), float(relative_rmse), int(max_iteration), int(bool(with_scaling)))
    T = torch.empty(N, 4, 4, dtype=torch.float64, device=dev)
    fit = torch.empty(N, dtype=torch.float64, device=dev)
    rmse = torch.empty(N, dtype=torch.float64, device=dev)
    iters = torch.empty(N, dtype=torch.int32, device=dev)
    check(lib().hold_icp(ctx.h, N, Ps, ptr(s), ptr(sl), Pt, ptr(t), ptr(tl), ptr(ini), cfg, ptr(T), ptr(fit), ptr(rmse), ptr(iters),
                         stream_ptr()))
    if single:
        return ICPResult(T[0], fit[0], rmse[0], iters[0])
    return ICPResult(T, fit, rmse, iters)
