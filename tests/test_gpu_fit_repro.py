"""Bitwise-reproducible pose refinement on one GPU.  The soft-silhouette backward (hold_raster_silhouette_bwd) and the K-NN backward
(hold_knn_points_bwd) add in a fixed order: repeated calls, a frame alone or inside a batch, and replays of a captured graph give
the same bits, within the float64 bounds of test_gpu_raster.py and test_gpu_pointcloud.py.  A refinement in the style of
optimize_ckpt.py -- the synthetic MANO rig and an object, an L1 silhouette loss and a fingertip contact term -- run twice gives
identical losses, poses, gradients and Adam moments, eager and graph-replayed, with no torch op flagged by the deterministic-
algorithms mode; tools/dump_fit_steps.py twice gives identical dumps.  New kernels: each case runs in a fresh interpreter."""
import ctypes as C
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
STEPS = 50


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, path))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _bwd(c, v, f, H, W, cfg, g):
    from hold_b200.capi import check, lib, ptr, stream_ptr

    B, V, _ = v.shape
    gv = torch.full((B, V, 3), float("nan"), device=DEV)
    check(lib().hold_raster_silhouette_bwd(c.h, B, V, ptr(v), f.shape[0], ptr(f), H, W, C.byref(cfg), ptr(g), ptr(gv), stream_ptr()))
    return gv


def _sil_repro(c, v, f, H, W, cfg, label):
    """ten calls, each frame alone, and graph replays: all bit-identical"""
    g = torch.randn(v.shape[0], H, W, generator=torch.Generator().manual_seed(5)).to(DEV)
    ref = _bwd(c, v, f, H, W, cfg, g)
    assert torch.isfinite(ref).all() and ref[..., :2].abs().max() > 0, label
    for _ in range(9):
        assert torch.equal(_bwd(c, v, f, H, W, cfg, g), ref), label
    for b in range(v.shape[0]):
        assert torch.equal(_bwd(c, v[b:b + 1].contiguous(), f, H, W, cfg, g[b:b + 1].contiguous())[0], ref[b]), (label, b)
    out = torch.empty_like(ref)
    from hold_b200.capi import check, lib, ptr, stream_ptr

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        check(lib().hold_raster_silhouette_bwd(c.h, v.shape[0], v.shape[1], ptr(v), f.shape[0], ptr(f), H, W, C.byref(cfg), ptr(g),
                                               ptr(out), stream_ptr()))
    for _ in range(3):
        out.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, ref), label
    c.check()
    print(f"{label}: bitwise over 10 calls, {v.shape[0]} single frames and 3 replays; max|g| {ref.abs().max().item():.3e}")


def impl_silhouette_bwd(c):
    from hold_b200 import fitting

    bench = _load("tools/bench_silhouette.py", "bench_silhouette")
    R = _load("tests/test_gpu_raster.py", "test_gpu_raster")
    cfg = fitting._cfg(100, None, 1e-4, True, None, False)
    for name in ("scene", "quads"):
        v, f = getattr(bench, name)(8)
        _sil_repro(c, v.to(DEV).contiguous(), f.to(DEV).contiguous(), 512, 512, cfg, f"{name} 8x512x512 K100")
    v, f = R._star_ndc(3, 48, 80, [2.5, 3.5, 6.0], seed=2)
    _sil_repro(c, v.to(DEV), f.to(DEV), 48, 80, fitting._cfg(8, None, 1e-4, True, None, False), "star 48x80 K8")
    v, f = R._random_tris(2, 96, seed=3)
    _sil_repro(c, v.to(DEV), f.to(DEV), 80, 48, fitting._cfg(8, None, 1e-3, True, None, False), "random 80x48 K8")
    # the float64 oracle at the bounds of test_gpu_raster.py
    v, f = R._star_ndc(2, 64, 64, [2.6, 4.0])
    R._check_case(c, v, f, 64, 64, 100, label="star 64x64 K100")
    v, f = R._quad_stack()
    R._check_case(c, v, f, 48, 80, 100, sigma=1e-4, label="quads 48x80 K100")


def _knn_grads(c, p1, p2, l1, l2, K, w, wk):
    from hold_b200 import pointcloud as PC

    a, b = p1.clone().requires_grad_(True), p2.clone().requires_grad_(True)
    r = PC.knn_points(c, a, b, l1, l2, K=K, return_nn=True)
    ((r.dists * w).sum() + (r.knn * wk).sum()).backward()
    return a.grad, b.grad, r.idx


def impl_knn_bwd(c):
    from hold_b200.capi import check, lib, ptr, stream_ptr

    g = torch.Generator().manual_seed(7)
    cases = []
    N, P1, P2 = 3, 517, 700
    p1, p2 = torch.randn(N, P1, 3, generator=g), torch.randn(N, P2, 3, generator=g)
    p2[:, 100] = p2[:, 3]                                   # duplicates
    p2[:, 650] = p2[:, 3]
    p1[:, 7] = p2[:, 3]
    cases.append(("ragged", p1, p2, torch.tensor([517, 300, 0]), torch.tensor([700, 9, 600])))
    cases.append(("full", p1, p2, None, None))
    q = torch.rand(1, 2**17, 3, generator=g) * 0.01          # every query's nearest neighbour is target 5
    t = torch.rand(1, 64, 3, generator=g) + 1.0
    t[0, 5] = 0.005
    cases.append(("one target", q, t, None, None))
    for name, p1, p2, l1, l2 in cases:
        for K in (1, 15, 32):
            if name == "one target" and K > 1:
                continue
            N, P1, P2 = p1.shape[0], p1.shape[1], p2.shape[1]
            w, wk = torch.randn(N, P1, K, generator=g).to(DEV), torch.randn(N, P1, K, 3, generator=g).to(DEV)
            d1, d2 = p1.to(DEV), p2.to(DEV)
            L1, L2 = (None if l is None else l.to(DEV) for l in (l1, l2))
            ga, gb, idx = _knn_grads(c, d1, d2, L1, L2, K, w, wk)
            if name == "one target":
                assert (idx == 5).all()
            for _ in range(9):
                a2, b2, _ = _knn_grads(c, d1, d2, L1, L2, K, w, wk)
                assert torch.equal(a2, ga) and torch.equal(b2, gb), (name, K)
            # float64 autograd at the kernel's indices, masked as pytorch3d does: dists over the valid slots, knn where k < lengths2
            a64, b64 = p1.double().requires_grad_(True), p2.double().requires_grad_(True)
            ii = idx.cpu()
            nn = torch.gather(b64, 1, ii.reshape(N, -1, 1).expand(-1, -1, 3)).reshape(N, P1, K, 3)
            dref = ((a64[:, :, None, :] - nn) ** 2).sum(-1)
            kmask = torch.ones(N, 1, K, dtype=torch.bool) if l2 is None else (torch.arange(K)[None, None, :] < l2[:, None, None])
            if l1 is not None:
                dref = dref * ((torch.arange(P1)[None, :, None] < l1[:, None, None]) & kmask)
            ((dref * w.cpu().double()).sum() + (nn * kmask[..., None] * wk.cpu().double()).sum()).backward()
            for got, ref in ((ga, a64.grad), (gb, b64.grad)):
                err = (got.cpu().double() - ref).abs().max().item()
                # one target: 2^17 fp32 terms in one sum, whose rounding grows with the count
                assert err <= (1e-4 if name == "one target" else 1e-5) * max(ref.abs().max().item(), 1e-30), (name, K, err)
            # the raw export captured in a graph
            gd, gk = w.contiguous(), wk.contiguous()
            i32 = idx.int().contiguous()
            l1t = torch.full((N,), P1, dtype=torch.int32, device=DEV) if L1 is None else L1.int()
            l2t = torch.full((N,), P2, dtype=torch.int32, device=DEV) if L2 is None else L2.int()
            o1, o2 = torch.empty(N, P1, 3, device=DEV), torch.empty(N, P2, 3, device=DEV)
            call = lambda: check(lib().hold_knn_points_bwd(c.h, N, P1, ptr(d1), ptr(l1t), P2, ptr(d2), ptr(l2t), K, ptr(i32), ptr(gd), ptr(gk),
                                                           ptr(o1), ptr(o2), stream_ptr()))
            call()
            assert torch.equal(o1, ga) and torch.equal(o2, gb), (name, K)
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=s):
                call()
            for _ in range(3):
                o1.fill_(float("nan")), o2.fill_(float("nan"))
                graph.replay()
                torch.cuda.synchronize()
                assert torch.equal(o1, ga) and torch.equal(o2, gb), (name, K)
            c.check()
            print(f"knn {name} K={K}: bitwise over 10 calls and 3 replays")


# ------------------------------------------------------------------------------------------------ refinement scene

def refine_scene(ctx, B=2, H=96, W=96):
    """optimize_ckpt.py's refinement on synthetic data: the synthetic MANO rig (hold_mano_lbs / _bwd) with convex-hull faces, the
    star mesh as the object (hold_object_tf / _bwd, obj_scale frozen), drawn together as one mesh.  The target silhouette is
    rendered at the true poses; the leaves start from perturbed ones.  Returns (leaves, loss_fn)."""
    from scipy.spatial import ConvexHull

    from hold_b200 import fitting, synth
    from hold_b200 import pointcloud as PC
    from hold_b200.model import MANOServer, ObjectServer
    from oracle.mesh_sdf_oracle import star_mesh

    dev = torch.device("cuda", ctx.device)
    g = torch.Generator().manual_seed(21)
    m = synth.make_mano_struct(2)
    hand = MANOServer(ctx, m, 0.3 * torch.randn(10, generator=g))
    hf = torch.as_tensor(ConvexHull(hand.verts_c[0].detach().cpu().double().numpy()).simplices.astype("int32"))
    vs, fs = star_mesh(level=3, seed=1)
    obj = ObjectServer(ctx, torch.from_numpy(vs).float() * 0.05, obj_scale=1.0)
    faces = fitting.check_faces(torch.cat([hf, torch.from_numpy(fs.astype(np.int32)) + 778]), 778 + vs.shape[0], dev)
    tips = m["tip_ids"].long().to(dev)
    Kc = torch.tensor([[130.0, 0, W / 2], [0, 130.0, H / 2], [0, 0, 1]], device=dev)
    cfg = fitting._cfg(50, None, 1e-3, True, None, False)
    ones = torch.ones(B, device=dev)
    truth = {"h_rot": 0.3 * torch.randn(B, 3, generator=g), "h_pose": 0.2 * torch.randn(B, 45, generator=g),
             "h_transl": torch.tensor([[-0.02, -0.05, 0.5]]).repeat(B, 1), "o_rot": torch.randn(B, 3, generator=g),
             "o_transl": torch.tensor([[0.05, 0.02, 0.55]]).repeat(B, 1)}
    truth = {k: v.to(dev) for k, v in truth.items()}

    def verts(p):
        hv = hand.forward(ones, p["h_transl"], torch.cat([p["h_rot"], p["h_pose"]], 1), hand.betas)["verts"]
        ov = obj.forward(ones, p["o_transl"], p["o_rot"])["verts"]
        return hv, ov

    def silhouette(hv, ov):
        return fitting.SoftSilhouetteFn.apply(fitting.project_ndc(torch.cat([hv, ov], 1), Kc, H, W), faces, ctx, H, W, cfg)

    with torch.no_grad():
        target = silhouette(*verts(truth))
    leaves = {k: (v + 0.04 * torch.randn(v.shape, generator=g).to(dev)).requires_grad_(True) for k, v in truth.items()}

    def loss_fn():
        hv, ov = verts(leaves)
        sil = (silhouette(hv, ov) - target).abs().mean()
        r = PC.knn_points(ctx, hv[:, tips], ov, K=4, return_nn=True)
        contact = r.dists.mean() + 0.1 * (hv[:, tips, None] - r.knn).abs().mean()
        return sil + contact

    return leaves, loss_fn


def refine_snapshot(leaves, opt, loss):
    snap = {"loss": loss.detach().clone()}
    for k, p in leaves.items():
        snap[f"pose.{k}"] = p.detach().clone()
        snap[f"grad.{k}"] = p.grad.clone()
        for s, v in opt.state.get(p, {}).items():
            snap[f"adam_{s}.{k}"] = v.clone()
    return snap


def refine_run(ctx, steps, graph=False):
    """`steps` Adam steps (capturable Adam) of refine_scene, eager or as replays of one captured step (after 3 eager warm-up
    steps on a side stream) -> a snapshot per step."""
    leaves, loss_fn = refine_scene(ctx)
    opt = torch.optim.Adam(list(leaves.values()), lr=2e-3, capturable=True)

    def step():
        opt.zero_grad(set_to_none=False)
        loss = loss_fn()
        loss.backward()
        opt.step()
        return loss

    snaps = []
    if not graph:
        for _ in range(steps):
            snaps.append(refine_snapshot(leaves, opt, step()))
    else:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(3):
                step()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            static_loss = step()
        for _ in range(steps):
            g.replay()
            snaps.append(refine_snapshot(leaves, opt, static_loss))
    torch.cuda.synchronize()
    ctx.check()
    return snaps


def _assert_equal_runs(a, b):
    assert len(a) == len(b)
    for i, (sa, sb) in enumerate(zip(a, b)):
        assert sa.keys() == sb.keys()
        diff = [k for k in sa if not torch.equal(sa[k], sb[k])]
        assert not diff, f"step {i}: {len(diff)} of {len(sa)} tensors differ, e.g. {diff[:6]}"
    assert any(k.startswith("adam_exp_avg_sq.") for k in a[-1])


def impl_refine_bitwise(c):
    for graph in (False, True):
        a = refine_run(c, STEPS, graph)
        b = refine_run(c, STEPS, graph)
        losses = [s["loss"].item() for s in a]
        print(f"refine graph={graph}: loss {losses[0]:.5f} -> {losses[-1]:.5f}")
        assert losses[-1] < losses[0]
        _assert_equal_runs(a, b)


def audit_refine_ops(c):
    """every op of the refinement steps, eager and captured, under torch.use_deterministic_algorithms(True, warn_only=True)"""
    import warnings

    torch.use_deterministic_algorithms(True, warn_only=True)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        refine_run(c, 3)
        refine_run(c, 3, graph=True)
        found = sorted({str(w.message).splitlines()[0] for w in rec if "determinis" in str(w.message)})
    for f in found:
        print("nondeterministic:", f)
    assert not found, found


@pytest.mark.parametrize("case", ["impl_silhouette_bwd", "impl_knn_bwd", "impl_refine_bitwise", "audit_refine_ops"])
def test_fit_repro(isolated, case):
    isolated("tests/test_gpu_fit_repro.py", case, timeout=1200, env={"CUBLAS_WORKSPACE_CONFIG": ":4096:8"})


def test_dump_fit_steps_twice_identical(built, tmp_path):
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    tool = os.path.join(ROOT, "tools", "dump_fit_steps.py")
    for mode in ([], ["--graph"]):
        dirs = []
        for run in ("a", "b"):
            d = str(tmp_path / ("graph" if mode else "eager") / run)
            r = subprocess.run([sys.executable, tool, d, "--steps", "5"] + mode, cwd=ROOT, capture_output=True, text=True, timeout=600)
            assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
            dirs.append(d)
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "compare_dumps.py"), *dirs], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        rep = json.loads(r.stdout.strip().splitlines()[-1])
        names = sorted(rep["arrays"])
        assert not rep["mismatched"] and "step004.loss" in names and any(".grad." in k for k in names)
        assert any(".adam_exp_avg_sq." in k for k in names)
        diff = [k for k, v in rep["arrays"].items() if not v["identical"]]
        assert not diff, (mode, diff[:8])
