"""hold_knn_points / hold_icp and hold_b200.pointcloud (pytorch3d's knn_points and chamfer_distance, an F-score, open3d's
point-to-point ICP) against the oracle (oracle/pointcloud_oracle.py): exact neighbours and fp32 distances, padding and length
rules, a 2^17 x 2^15 cloud, argument rejection, the gradient, every chamfer reduction, exact F-score counts, ICP against the
oracle's loop, batch independence, reproducibility, CUDA-graph capture, and an evaluation end to end.  New kernels: each case
runs in a fresh interpreter (`isolated`)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pointcloud_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _raw_knn(c, p1, p2, K, l1=None, l2=None):
    from hold_b200.capi import lib, ptr, stream_ptr

    N, P1, P2 = p1.shape[0], p1.shape[1], p2.shape[1]
    d = torch.full((N, P1, max(K, 1)), float("nan"), device=DEV)   # a K outside [1, 32] is refused before any write
    i = torch.full((N, P1, max(K, 1)), -7, dtype=torch.int32, device=DEV)
    rc = lib().hold_knn_points(c.h, N, P1, ptr(p1), ptr(l1), P2, ptr(p2), ptr(l2), K, ptr(d), ptr(i), stream_ptr())
    return rc, d, i


def _fp32_dist_at(p1, p2, idx):
    """the no-FMA fp32 expression at the given indices: [N,P1,K]"""
    a, b = p1.cpu().numpy(), p2.cpu().numpy()
    ii = idx.cpu().numpy()
    out = np.zeros(ii.shape, np.float32)
    for n in range(a.shape[0]):
        nb = b[n][ii[n]]                                   # [P1,K,3]
        dd = a[n][:, None, :] - nb
        s = dd * dd
        out[n] = (s[..., 0] + s[..., 1]) + s[..., 2]
    return out


def impl_knn(c):
    from hold_b200 import pointcloud as PC

    g = torch.Generator().manual_seed(0)
    for K in (1, 4, 15, 32):
        N, P1, P2 = 3, 517, 700
        p1 = torch.randn(N, P1, 3, generator=g)
        p2 = torch.randn(N, P2, 3, generator=g)
        p2[:, 100] = p2[:, 3]                              # duplicates: exact ties
        p2[:, 650] = p2[:, 3]
        p1[:, 7] = p2[:, 3]                                # queries on the triplicated point
        p1[:, 8] = p1[:, 9]
        l1, l2 = torch.tensor([517, 300, 0]), torch.tensor([700, 9, 600])   # K > lengths2 in frame 1, no query in frame 2
        for lens in ((None, None), (l1, l2)):
            r = PC.knn_points(c, p1.to(DEV), p2.to(DEV), *(None if x is None else x.to(DEV) for x in lens), K=K)
            c.check()
            rd, ri = O.knn_points(p1.numpy(), p2.numpy(), *(None if x is None else x.numpy() for x in lens), K=K)
            d, i = r.dists.cpu().numpy(), r.idx.cpu().numpy()
            assert r.idx.dtype == torch.int64 and r.dists.dtype == torch.float32
            same = i == ri
            assert np.array_equal(d[~same], rd[~same]), "an index differs without an exact distance tie"
            print(f"K={K} lengths={lens[0] is not None}: {int((~same).sum())} slots differ by ties of {i.size}")
            assert same.mean() == 1.0   # the kernel keeps (distance, index) order: even ties agree
            assert np.array_equal(d, rd)
            L1, L2 = (np.full(N, P1), np.full(N, P2)) if lens[0] is None else (l1.numpy(), l2.numpy())
            valid = (np.arange(P1)[None, :, None] < L1[:, None, None]) & (np.arange(K)[None, None, :] < L2[:, None, None])
            assert np.array_equal(d[valid], _fp32_dist_at(p1, p2, r.idx)[valid])   # bit for bit the no-FMA fp32 expression
            if lens[0] is not None:
                assert (d[1, 300:] == 0).all() and (i[1, 300:] == 0).all() and (d[2] == 0).all() and (i[2] == 0).all()
                assert (d[1, :300, 9:] == 0).all() and (i[1, :300, 9:] == 0).all()
            if K >= 3:
                assert list(i[0, 7, :3]) == [3, 100, 650] and (d[0, 7, :3] == 0).all()
        # return_nn: pytorch3d's knn_gather
        r = PC.knn_points(c, p1.to(DEV), p2.to(DEV), l1.to(DEV), l2.to(DEV), K=K, return_nn=True)
        ref = torch.gather(p2, 1, r.idx.cpu().reshape(N, -1, 1).expand(-1, -1, 3)).reshape(N, P1, K, 3)
        ref = ref * (torch.arange(K)[None, None, :] < l2[:, None, None])[..., None]
        assert torch.equal(r.knn.cpu(), ref)
    # P2 = 0 and K beyond P2
    rc, d, i = _raw_knn(c, torch.randn(2, 5, 3, device=DEV), torch.randn(2, 3, 3, device=DEV), 8)
    assert rc == 0
    c.check()
    assert (d[..., 3:] == 0).all() and (i[..., 3:] == 0).all() and (i[..., :3] >= 0).all()
    rc, d, i = _raw_knn(c, torch.randn(2, 5, 3, device=DEV), torch.empty(2, 0, 3, device=DEV), 2)
    assert rc == 0 and (d == 0).all() and (i == 0).all()


def impl_knn_large(c):
    from hold_b200 import pointcloud as PC

    g = torch.Generator().manual_seed(1)
    p1 = torch.rand(1, 2**17, 3, generator=g)
    p2 = torch.rand(1, 2**15, 3, generator=g) * 0.9 + 0.05
    r = PC.knn_points(c, p1.to(DEV), p2.to(DEV), K=1)
    c.check()
    sub = np.sort(np.random.default_rng(2).choice(2**17, 4096, replace=False))
    d = r.dists[0, sub, 0].cpu().numpy()
    i = r.idx[0, sub, 0].cpu().numpy()
    td, ti = O.knn_kdtree(p1[0, sub].numpy(), p2[0].numpy(), 1)
    q, p = p1[0, sub].numpy(), p2[0].numpy()
    assert np.array_equal(d, _fp32_dist_at(p1[:, sub], p2, r.idx[:, sub].cpu())[0, :, 0])
    ex, _ = O.knn_brute(q, p, 1, chunk=128)               # exact fp32 brute force on the subset
    assert np.array_equal(d, ex[:, 0])
    agree = i == ti[:, 0]
    p64 = p.astype(np.float64)
    dk = ((q.astype(np.float64) - p64[i]) ** 2).sum(1)
    assert np.all(dk[~agree] <= td[~agree, 0] * (1 + 1e-6) + 1e-12), "a differing index must be a near tie"
    print(f"large: {agree.mean():.5f} of the subset equal cKDTree's index; max |d - d_tree| {np.abs(d - td[:, 0]).max():.2e}")
    assert agree.mean() > 0.999
    assert np.abs(d - td[:, 0]).max() <= 1e-6


def impl_knn_errors(c):
    from hold_b200.capi import HoldError, lib, ptr, stream_ptr

    p1, p2 = torch.randn(2, 20, 3, device=DEV), torch.randn(2, 30, 3, device=DEV)
    for K in (0, 33, -1):
        assert _raw_knn(c, p1, p2, K)[0] == -1
    d = torch.empty(2, 20, 1, device=DEV)
    i = torch.empty(2, 20, 1, dtype=torch.int32, device=DEV)
    assert lib().hold_knn_points(c.h, -1, 20, ptr(p1), None, 30, ptr(p2), None, 1, ptr(d), ptr(i), stream_ptr()) == -1
    assert lib().hold_knn_points(c.h, 2, 20, None, None, 30, ptr(p2), None, 1, ptr(d), ptr(i), stream_ptr()) == -1
    # a bad length: clamped by the kernel, reported by hold_ctx_check
    for l1, l2, want1, want2 in (([25, 5], None, [20, 5], [30, 30]), (None, [-3, 31], [20, 20], [0, 30])):
        t1 = None if l1 is None else torch.tensor(l1, dtype=torch.int32, device=DEV)
        t2 = None if l2 is None else torch.tensor(l2, dtype=torch.int32, device=DEV)
        rc, d, i = _raw_knn(c, p1, p2, 2, t1, t2)
        assert rc == 0
        with pytest.raises(HoldError, match="length"):
            c.check()
        c.check()   # the error word is cleared
        rc, dc, ic = _raw_knn(c, p1, p2, 2, torch.tensor(want1, dtype=torch.int32, device=DEV), torch.tensor(want2, dtype=torch.int32, device=DEV))
        c.check()
        assert torch.equal(d, dc) and torch.equal(i, ic)


def impl_knn_grad(c):
    from hold_b200 import fitting
    from hold_b200 import pointcloud as PC

    g = torch.Generator().manual_seed(3)
    N, P1, P2, K = 2, 300, 400, 5
    a, b = torch.randn(N, P1, 3, generator=g), torch.randn(N, P2, 3, generator=g)
    w = torch.randn(N, P1, K, generator=g)
    l1, l2 = torch.tensor([300, 120]), torch.tensor([400, 3])
    for lens in ((None, None), (l1, l2)):
        p1, p2 = a.to(DEV).requires_grad_(True), b.to(DEV).requires_grad_(True)
        r = PC.knn_points(c, p1, p2, *(None if x is None else x.to(DEV) for x in lens), K=K)
        (r.dists * w.to(DEV)).sum().backward()
        # float64 reference: fitting.knn_points' expression at the kernel's indices, masked to the valid slots
        a64, b64 = a.double().requires_grad_(True), b.double().requires_grad_(True)
        idx = r.idx.cpu()
        nn = torch.gather(b64, 1, idx.reshape(N, -1, 1).expand(-1, -1, 3)).reshape(N, P1, K, 3)
        dref = ((a64[:, :, None, :] - nn) ** 2).sum(-1)
        if lens[0] is not None:
            dref = dref * ((torch.arange(P1)[None, :, None] < l1[:, None, None]) & (torch.arange(K)[None, None, :] < l2[:, None, None]))
        (dref * w.double()).sum().backward()
        for got, ref in ((p1.grad, a64.grad), (p2.grad, b64.grad)):
            err = (got.cpu().double() - ref).abs().max().item()
            assert err <= 1e-5 * ref.abs().max().item(), err
        if lens[0] is None:   # and fitting.knn_points itself, where it picks the same neighbours
            assert torch.equal(fitting.knn_points(a, b, K).idx, idx)
            if not torch.equal(fitting.knn_points(a.double(), b.double(), K).idx, idx):
                print("float64 picks other neighbours (a near tie): its autograd is not comparable")
                continue
            a2, b2 = a.double().requires_grad_(True), b.double().requires_grad_(True)
            (fitting.knn_points(a2, b2, K).dists * w.double()).sum().backward()
            assert (p1.grad.cpu().double() - a2.grad).abs().max() <= 1e-5 * a2.grad.abs().max()
            assert (p2.grad.cpu().double() - b2.grad).abs().max() <= 1e-5 * b2.grad.abs().max()


def impl_chamfer_fscore(c):
    from hold_b200 import pointcloud as PC

    g = torch.Generator().manual_seed(4)
    x, y = torch.randn(3, 600, 3, generator=g), torch.randn(3, 450, 3, generator=g) * 1.1
    xl, yl = torch.tensor([600, 250, 0]), torch.tensor([450, 450, 17])
    for lens in ((None, None), (xl, yl)):
        for br in (None, "sum", "mean"):
            for pr in ("sum", "mean"):
                xd, yd = x.to(DEV).requires_grad_(True), y.to(DEV)
                loss, nrm = PC.chamfer_distance(c, xd, yd, *(None if t is None else t.to(DEV) for t in lens), batch_reduction=br, point_reduction=pr)
                assert nrm is None
                ref = O.chamfer_distance(x.numpy(), y.numpy(), *(None if t is None else t.numpy() for t in lens), br, pr)
                got = loss.detach().cpu().double().numpy()
                assert got.shape == np.shape(ref)
                assert np.all(np.abs(got - ref) <= 1e-6 * np.maximum(np.abs(ref), 1e-30)), (br, pr, got, ref)
                loss.sum().backward()
                assert torch.isfinite(xd.grad).all()
        f, p, r = PC.fscore(c, x.to(DEV), y.to(DEV), [0.05, 0.1, 0.3], *(None if t is None else t.to(DEV) for t in lens))
        fr, prr, rr = O.fscore(x.numpy(), y.numpy(), [0.05, 0.1, 0.3], *(None if t is None else t.numpy() for t in lens))
        ln = (np.array([600, 600, 600]) if lens[0] is None else xl.numpy())[:, None]
        lg = (np.array([450, 450, 450]) if lens[0] is None else yl.numpy())[:, None]
        assert p.dtype == torch.float64
        assert np.array_equal(np.round(p.cpu().numpy() * ln), np.round(prr * ln))   # exact counts
        assert np.array_equal(np.round(r.cpu().numpy() * lg), np.round(rr * lg))
        assert np.allclose(f.cpu().numpy(), fr, rtol=1e-12, atol=0)


def _rt(rng, ang=0.1, tr=0.05):
    from oracle.hold_oracle import axis_angle_to_matrix

    T = np.eye(4)
    T[:3, :3] = axis_angle_to_matrix(torch.from_numpy(rng.normal(size=(1, 3)) * ang))[0].numpy()
    T[:3, 3] = rng.normal(size=3) * tr
    return T


def _icp(c, s, t, md, **kw):
    from hold_b200 import pointcloud as PC

    r = PC.icp(c, s.to(DEV), t.to(DEV), md, **kw)
    c.check()
    return [x.cpu() for x in r]


def impl_icp_rigid(c):
    rng = np.random.default_rng(5)
    src = rng.uniform(-1, 1, size=(3000, 3)).astype(np.float32)
    for scaling, scale in ((False, 1.0), (True, 1.08)):
        T0 = _rt(rng, 0.04, 0.02)
        T0[:3, :3] *= scale
        tgt = O.transform(T0, src.astype(np.float64)).astype(np.float32)
        T, fit, rmse, it = _icp(c, torch.from_numpy(src), torch.from_numpy(tgt), 0.2, with_scaling=scaling, relative_fitness=1e-9,
                                relative_rmse=1e-12, max_iteration=60)
        # the targets are T0's images rounded to fp32: the known transform of the data is the least-squares fit over the true
        # correspondences, which is T0 to the rounding of the targets
        Tls = O.umeyama(src.astype(np.float64), tgt.astype(np.float64), scaling)
        err, err0 = np.abs(T.numpy() - Tls).max(), np.abs(T.numpy() - T0).max()
        print(f"rigid scaling={scaling}: |T - T_ls| {err:.2e}, |T - T0| {err0:.2e}, fitness {fit.item()}, rmse {rmse.item():.2e}, "
              f"iterations {it.item()}")
        assert err <= 1e-9 and err0 <= 1e-6 and fit.item() == 1.0
        Tr, fr, rr, ir = O.icp(src, tgt, 0.2, None, scaling, 1e-9, 1e-12, 60)
        assert np.abs(T.numpy() - Tr).max() <= 1e-9 and it.item() == ir


def _partial_pair(rng, n=2500, noise=0.005):
    base = rng.uniform(-1, 1, size=(n, 3))
    s = base[rng.random(n) < 0.8]
    t = base[rng.random(n) < 0.7]
    T0 = _rt(rng, 0.06, 0.03)
    t = O.transform(T0, t) + rng.normal(size=t.shape) * noise
    return s.astype(np.float32), t.astype(np.float32)


def impl_icp_oracle(c):
    rng = np.random.default_rng(6)
    for scaling in (False, True):
        for k in range(3):
            s, t = _partial_pair(rng)
            init = _rt(rng, 0.01, 0.01) if k == 2 else None
            kw = dict(with_scaling=scaling)
            if init is not None:
                kw["init"] = torch.from_numpy(init)
            T, fit, rmse, it = _icp(c, torch.from_numpy(s), torch.from_numpy(t), 0.15, **kw)
            Tr, fr, rr, ir = O.icp(s, t, 0.15, init, scaling)
            print(f"oracle scaling={scaling} case {k}: iterations {it.item()} / {ir}, |T - T_oracle| {np.abs(T.numpy() - Tr).max():.2e}, "
                  f"fitness {fit.item():.4f} / {fr:.4f}, rmse {rmse.item():.6f} / {rr:.6f}")
            assert it.item() == ir
            assert np.abs(T.numpy() - Tr).max() <= 1e-9
            assert fit.item() == fr and abs(rmse.item() - rr) <= 1e-9


def impl_icp_edges(c):
    rng = np.random.default_rng(7)
    s, t = _partial_pair(rng, 800)
    # nothing within range: the identity, fitness 0, rmse 0
    T, fit, rmse, it = _icp(c, torch.from_numpy(s), torch.from_numpy(t + 50.0), 0.5)
    assert torch.equal(T, torch.eye(4, dtype=torch.float64)) and fit.item() == 0.0 and rmse.item() == 0.0
    assert it.item() == O.icp(s, t + 50.0, 0.5)[3]
    for md in (0.0, -1.0):   # open3d: no correspondence unless max_correspondence_distance > 0
        T, fit, rmse, it = _icp(c, torch.from_numpy(s), torch.from_numpy(t), md)
        assert torch.equal(T, torch.eye(4, dtype=torch.float64)) and fit.item() == 0.0
    # init is honoured: max_iteration = 0 returns init and its correspondences
    init = _rt(rng)
    T, fit, rmse, it = _icp(c, torch.from_numpy(s), torch.from_numpy(t), 0.15, init=torch.from_numpy(init), max_iteration=0)
    _, _, fr, rr = O.correspondences(O.transform(init, s.astype(np.float64)), t.astype(np.float64), 0.15)
    assert torch.equal(T, torch.from_numpy(init)) and it.item() == 0
    assert fit.item() == fr and abs(rmse.item() - rr) <= 1e-12
    # lengths: a pair with padding equals the same pair without it
    sp = np.concatenate([s, np.full((100, 3), 7.0, np.float32)])
    tp = np.concatenate([t, np.full((50, 3), -7.0, np.float32)])
    from hold_b200 import pointcloud as PC

    a = PC.icp(c, torch.from_numpy(s)[None].to(DEV), torch.from_numpy(t)[None].to(DEV), 0.15)
    b = PC.icp(c, torch.from_numpy(sp)[None].to(DEV), torch.from_numpy(tp)[None].to(DEV), 0.15,
               source_lengths=torch.tensor([len(s)], device=DEV), target_lengths=torch.tensor([len(t)], device=DEV))
    c.check()
    assert torch.allclose(a.transformation, b.transformation, rtol=0, atol=1e-12) and torch.equal(a.iterations, b.iterations)
    assert torch.equal(a.fitness, b.fitness)


def impl_icp_batch(c):
    from hold_b200 import pointcloud as PC

    rng = np.random.default_rng(8)
    pairs = [_partial_pair(rng, 1500) for _ in range(8)]
    Ps, Pt = max(len(s) for s, _ in pairs), max(len(t) for _, t in pairs)
    S = torch.zeros(8, Ps, 3)
    Tg = torch.zeros(8, Pt, 3)
    for k, (s, t) in enumerate(pairs):
        S[k, :len(s)], Tg[k, :len(t)] = torch.from_numpy(s), torch.from_numpy(t)
    ls = torch.tensor([len(s) for s, _ in pairs], device=DEV)
    lt = torch.tensor([len(t) for _, t in pairs], device=DEV)
    S, Tg = S.to(DEV), Tg.to(DEV)
    r1 = PC.icp(c, S, Tg, 0.15, source_lengths=ls, target_lengths=lt)
    r2 = PC.icp(c, S, Tg, 0.15, source_lengths=ls, target_lengths=lt)
    c.check()
    for a, b in zip(r1, r2):
        assert torch.equal(a, b), "two runs differ"
    assert len(set(r1.iterations.tolist())) > 1, "the pairs should converge at different iterations"
    for k in (0, 5):
        rk = PC.icp(c, S[k:k + 1].contiguous(), Tg[k:k + 1].contiguous(), 0.15, source_lengths=ls[k:k + 1], target_lengths=lt[k:k + 1])
        for a, b in zip(r1, rk):
            assert torch.equal(a[k:k + 1], b), f"pair {k} alone differs from pair {k} in the batch"
    # CUDA-graph capture of the whole call (the workspace exists from the calls above)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        PC.icp(c, S, Tg, 0.15)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        rg = PC.icp(c, S, Tg, 0.15)
    graph.replay()
    torch.cuda.synchronize()
    rd = PC.icp(c, S, Tg, 0.15)
    c.check()
    for a, b in zip(rg, rd):
        assert torch.equal(a, b), "graph replay differs"


def impl_e2e(c):
    """Evaluation of a reconstructed star mesh: its vertices moved by a known pose plus noise, aligned back with ICP, then
    Chamfer distance and F-scores at two thresholds, against the oracle's pipeline."""
    from hold_b200 import pointcloud as PC
    from oracle.mesh_sdf_oracle import star_mesh

    rng = np.random.default_rng(9)
    gt, _ = star_mesh(level=4, seed=1)
    T0 = _rt(rng, 0.03, 0.02)
    pred = (O.transform(T0, gt.astype(np.float64)) + rng.normal(size=gt.shape) * 0.003).astype(np.float32)
    r = PC.icp(c, torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV), 0.1)
    aligned = (O.transform(r.transformation.cpu().numpy(), pred.astype(np.float64))).astype(np.float32)
    cd, _ = PC.chamfer_distance(c, torch.from_numpy(aligned)[None].to(DEV), torch.from_numpy(gt)[None].to(DEV))
    f, p, rc = PC.fscore(c, torch.from_numpy(aligned)[None].to(DEV), torch.from_numpy(gt)[None].to(DEV), [0.005, 0.01])
    c.check()
    Tr, fr, rr, ir = O.icp(pred, gt, 0.1)
    al_r = O.transform(Tr, pred.astype(np.float64)).astype(np.float32)
    cd_r = O.chamfer_distance(al_r[None], gt[None])
    f_r, _, _ = O.fscore(al_r[None], gt[None], [0.005, 0.01])
    print(f"e2e: iterations {r.iterations.item()} / {ir}, CD {cd.item():.6e} / {cd_r:.6e}, F5 {f[0, 0].item():.4f} / {f_r[0, 0]:.4f}, "
          f"F10 {f[0, 1].item():.4f} / {f_r[0, 1]:.4f}")
    assert r.iterations.item() == ir and np.abs(r.transformation.cpu().numpy() - Tr).max() <= 1e-9
    assert np.abs(np.linalg.inv(Tr) - T0).max() < 0.002                 # the pose is recovered
    assert abs(cd.item() - cd_r) <= 1e-6 * cd_r
    assert np.abs(f.cpu().numpy() - f_r).max() <= 1.0 / len(gt)          # at most one point across a threshold


def impl_grad_padding(c):
    """The backward reads only valid slots: an empty second cloud (an empty reconstruction) and inf-padded rows give finite
    gradients; chamfer_distance against an empty cloud back-propagates zeros."""
    from hold_b200 import pointcloud as PC

    g = torch.Generator().manual_seed(10)
    x = torch.randn(2, 50, 3, generator=g).to(DEV).requires_grad_(True)
    empty = torch.empty(2, 0, 3, device=DEV, requires_grad=True)
    r = PC.knn_points(c, x, empty, K=4, return_nn=True)
    (r.dists.sum() + r.knn.sum()).backward()
    c.check()
    assert (r.dists == 0).all() and (r.idx == 0).all() and torch.equal(x.grad, torch.zeros_like(x))
    x.grad = None
    loss, _ = PC.chamfer_distance(c, x, empty)
    loss.sum().backward()
    c.check()
    assert torch.equal(x.grad, torch.zeros_like(x)) and empty.grad.shape == (2, 0, 3)
    # inf padding rows in both clouds, excluded by the lengths
    a, b = torch.randn(2, 40, 3, generator=g), torch.randn(2, 30, 3, generator=g)
    a[:, 35:] = float("inf")
    b[:, 25:] = float("nan")
    p1, p2 = a.to(DEV).requires_grad_(True), b.to(DEV).requires_grad_(True)
    lx, ly = torch.tensor([35, 20], device=DEV), torch.tensor([25, 25], device=DEV)
    loss, _ = PC.chamfer_distance(c, p1, p2, lx, ly, batch_reduction="sum")
    loss.backward()
    c.check()
    assert torch.isfinite(loss) and torch.isfinite(p1.grad).all() and torch.isfinite(p2.grad).all()
    assert (p1.grad[0, 35:] == 0).all() and (p1.grad[1, 20:] == 0).all() and (p2.grad[:, 25:] == 0).all()
    # the same clouds without padding give the same gradients on the valid points
    q1 = a[0:1, :35].to(DEV).requires_grad_(True)
    q2 = b[0:1, :25].to(DEV).requires_grad_(True)
    ref, _ = PC.chamfer_distance(c, q1, q2, batch_reduction="sum")
    ref.backward()
    assert torch.allclose(p1.grad[0, :35], q1.grad[0], rtol=1e-6, atol=1e-7)
    assert torch.allclose(p2.grad[0, :25], q2.grad[0], rtol=1e-6, atol=1e-7)
    # one unbatched ICP pair with a numpy init
    s = torch.rand(300, 3, generator=g)
    init = np.eye(4)
    init[:3, 3] = [0.01, 0.0, -0.01]
    res = PC.icp(c, s.to(DEV), (s + torch.tensor([0.01, 0.0, -0.01])).to(DEV), 0.1, init=init, max_iteration=0)
    c.check()
    assert res.transformation.shape == (4, 4) and np.array_equal(res.transformation.cpu().numpy(), init)


@pytest.mark.parametrize("case", ["impl_knn", "impl_grad_padding", "impl_knn_large", "impl_knn_errors", "impl_knn_grad", "impl_chamfer_fscore",
                                  "impl_icp_rigid", "impl_icp_oracle", "impl_icp_edges", "impl_icp_batch", "impl_e2e"])
def test_pointcloud(isolated, case):
    isolated("tests/test_gpu_pointcloud.py", case, timeout=900)
