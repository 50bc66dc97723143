"""hold_mesh_sdf_bvh against hold_mesh_sdf bit for bit (sdf and face_idx): every mesh of test_cpu_mesh_bvh.py, the 491 148-face
canonical object mesh with 125 440 points, B in {1, 3, 10} with shared and batched vertices, P not a multiple of the block,
points on the surface, NaN and inf points; repeated calls and CUDA-graph replays; argument checks; and forward_train's loss
targets with the object mesh and a hand mesh attached against the brute force on the same canonical points."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_cpu_mesh_bvh import bvh_meshes, query_points
from test_gpu_decimate import object_mesh  # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def run(ctx, fn, pts, v, f, batched):
    """pts [B,P,3], v [B,V,3] or [V,3] on the device -> (sdf, face_idx)"""
    from hold_b200.capi import check, lib, stream_ptr

    B, P, _ = pts.shape
    sdf = torch.full((B, P), 7.0, device="cuda")
    fi = torch.full((B, P), -7, dtype=torch.int32, device="cuda")
    check(getattr(lib(), fn)(ctx.h, B, P, _p(pts), v.shape[-2], _p(v), int(batched), f.shape[0], _p(f), _p(sdf), _p(fi), stream_ptr()))
    return sdf, fi


def same(a, b):
    return torch.equal(a[0].view(torch.int32), b[0].view(torch.int32)) and torch.equal(a[1], b[1])


def both(ctx, pts, v, f, batched):
    ref = run(ctx, "hold_mesh_sdf", pts, v, f, batched)
    got = run(ctx, "hold_mesh_sdf_bvh", pts, v, f, batched)
    ctx.check()
    return ref, got


@pytest.mark.parametrize("B", [1, 3, 10])
def test_equals_brute_force_on_every_mesh(ctx, B):
    for name, (v, f) in bvh_meshes().items():
        P = 1000 + 37                                                # not a multiple of the block
        pts = np.stack([query_points(v * (1 + 0.05 * b), P, seed=b) for b in range(B)])
        pts_d = torch.from_numpy(pts).cuda()
        fd = torch.from_numpy(f).cuda()
        vb = torch.from_numpy(np.stack([v * (1 + 0.05 * b) for b in range(B)]).astype(np.float32)).cuda()
        ref, got = both(ctx, pts_d, vb, fd, True)                    # a mesh per frame
        assert same(ref, got), (name, B, "batched", int((ref[0] != got[0]).sum()), int((ref[1] != got[1]).sum()))
        ref, got = both(ctx, pts_d, vb[0].contiguous(), fd, False)   # one shared mesh
        assert same(ref, got), (name, B, "shared")
        if B > 1:                                                    # shared == batched copies
            rep = run(ctx, "hold_mesh_sdf_bvh", pts_d, vb[0].expand(B, -1, -1).contiguous(), fd, True)
            assert same(rep, got)
        fin = torch.isfinite(pts_d).all(-1)
        assert (got[1][~fin] == -1).all() and (got[0][~fin] == float(np.sqrt(np.float32(3e38)))).all()


def test_object_mesh_125440_points(ctx, object_mesh):  # noqa: F811
    v, f = object_mesh
    assert f.shape[0] == 491148, f.shape
    g = torch.Generator(device="cuda").manual_seed(0)
    vd, fd = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    lo, hi = vd.min(0).values, vd.max(0).values
    n = 125440
    pts = lo + torch.rand(n, 3, device="cuda", generator=g) * (hi - lo) * 1.1 - 0.05 * (hi - lo)
    k = n // 4                                                       # near and on the surface
    pts[:k] = vd[torch.randint(0, v.shape[0], (k,), device="cuda", generator=g)] + torch.randn(k, 3, device="cuda", generator=g) * 1e-3
    pts[k:k + 1000] = vd[:1000]
    pts[k + 1000] = float("nan")
    ref, got = both(ctx, pts[None].contiguous(), vd, fd, False)
    assert same(ref, got), (int((ref[0] != got[0]).sum()), int((ref[1] != got[1]).sum()))
    ref3, got3 = both(ctx, pts.reshape(2, -1, 3).contiguous(), vd, fd, False)
    assert same((ref3[0].reshape(1, -1), ref3[1].reshape(1, -1)), ref) and same(ref3, got3)


def test_repeats_and_graph_replays(ctx):
    v, f = bvh_meshes()["noise"]
    B, P = 3, 5000
    pts = torch.from_numpy(np.stack([query_points(v, P, seed=b) for b in range(B)])).cuda()
    vb = torch.from_numpy(np.stack([v, v * 0.9, v * 1.1]).astype(np.float32)).cuda()
    fd = torch.from_numpy(f).cuda()
    ref = run(ctx, "hold_mesh_sdf", pts, vb, fd, True)
    first = run(ctx, "hold_mesh_sdf_bvh", pts, vb, fd, True)        # the eager call sizes the workspace
    assert same(ref, first)
    for _ in range(5):
        assert same(run(ctx, "hold_mesh_sdf_bvh", pts, vb, fd, True), first)
    from hold_b200.capi import check, lib

    sdf, fi = torch.empty(B, P, device="cuda"), torch.empty(B, P, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            check(lib().hold_mesh_sdf_bvh(ctx.h, B, P, _p(pts), v.shape[0], _p(vb), 1, f.shape[0], _p(fd), _p(sdf), _p(fi),
                                          C.c_void_p(s.cuda_stream)))
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(3):
        sdf.fill_(5.0), fi.fill_(-5)
        graph.replay()
        torch.cuda.synchronize()
        assert same((sdf, fi), first)
    ctx.check()


def test_argument_checks(ctx):
    from hold_b200.capi import HoldError, lib, stream_ptr

    v, f = bvh_meshes()["tetrahedron"]
    vd, fd = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    pts = torch.zeros(1, 10, 3, device="cuda")
    sdf, fi = torch.empty(1, 10, device="cuda"), torch.empty(1, 10, dtype=torch.int32, device="cuda")
    L = lib()
    call = lambda fn, V, F, fp=fd, pp=pts, vp=vd, sp=sdf: getattr(L, fn)(ctx.h, 1, 10, _p(pp), V, _p(vp), 0, F, _p(fp), _p(sp), _p(fi), stream_ptr())
    for fn in ("hold_mesh_sdf", "hold_mesh_sdf_bvh"):
        assert call(fn, 4, 0) != 0 and call(fn, 0, 4) != 0           # F = 0, V = 0: rejected alike
        assert call(fn, 4, 4, pp=None) != 0 and call(fn, 4, 4, vp=None) != 0 and call(fn, 4, 4, fp=None) != 0 and call(fn, 4, 4, sp=None) != 0
    assert L.hold_mesh_sdf_bvh(None, 1, 10, _p(pts), 4, _p(vd), 0, 4, _p(fd), _p(sdf), _p(fi), stream_ptr()) != 0
    assert call("hold_mesh_sdf_bvh", 4, (1 << 24) + 1) != 0          # over 2^24 faces, rejected before any read
    ctx.check()
    bad = fd.clone()
    bad[2, 1] = 4                                                    # == V
    assert call("hold_mesh_sdf_bvh", 4, 4, fp=bad) == 0
    with pytest.raises(HoldError, match="hold_mesh_sdf_bvh"):
        ctx.check()
    assert torch.isnan(sdf).all() and (fi == -1).all()
    bad[2, 1] = -1
    assert call("hold_mesh_sdf_bvh", 4, 4, fp=bad) == 0
    with pytest.raises(HoldError):
        ctx.check()
    assert call("hold_mesh_sdf_bvh", 4, 4) == 0                      # a good call after a bad one
    ctx.check()
    assert torch.isfinite(sdf).all() and (fi >= 0).all()


def test_forward_train_targets_with_object_and_hand_meshes(ctx, object_mesh):  # noqa: F811
    """the loss targets that forward_train computes through hold_mesh_sdf_bvh equal hold_mesh_sdf + hold_off_in_surface on the same
    canonical points, with the 491 148-face object mesh and a closed hand-sized mesh attached; Loss(...).backward() runs"""
    from hold_b200 import capi, ops, scene_io, synth, train
    from hold_b200.model import HOLDNet
    from test_cpu_decimate import meshes

    sc = synth.make_scene(H=8, W=8, S=32, nodes=("right", "object"), B=2, seed=11)
    dev = torch.device("cuda", 0)
    net = scene_io.build_net(sc, ctx, capi.MLP_TC)
    full = HOLDNet(ctx, dict(net.nodes), background=None)
    right, obj = full.nodes["right"], full.nodes["object"]
    hv, hf = meshes()["noise"]                                       # closed, 7 160 faces, moved onto the hand's canonical box
    vc = right.server.verts_c[0].detach()
    lo, hi = vc.min(0).values, vc.max(0).values
    hv = torch.from_numpy(hv).to(dev)
    right.mesh_v_cano_div = ((hv - hv.min(0).values) / (hv.max(0).values - hv.min(0).values) * (hi - lo) + lo).contiguous()
    right.mesh_f_cano_div = torch.from_numpy(hf).to(dev)
    obj.mesh_vo_cano, obj.mesh_fo_cano = torch.from_numpy(object_mesh[0]).to(dev), torch.from_numpy(object_mesh[1]).to(dev)
    calls, orig = [], ops.compute_mano_cano_sdf

    def spy(ctx_, v, f, x):
        out = orig(ctx_, v, f, x)
        calls.append((v.detach().clone(), f.detach().clone(), x.detach().clone(), out.clone()))
        return out

    ops.compute_mano_cano_sdf = spy
    try:
        inp = scene_io.scene_input(sc, dev)
        B, P = inp["uv"].shape[:2]
        out = train.forward_train(full, {**inp, "current_epoch": 30, "global_step": 12000}, generator=torch.Generator(device=dev).manual_seed(0))
    finally:
        ops.compute_mano_cano_sdf = orig
    ctx.check()
    assert len(calls) == 3                                           # hand: pts2mano_sdf_cano, off-surface; object: off-surface
    for v, f, x, got in calls:
        batched = v.dim() == 3
        ref = run(ctx, "hold_mesh_sdf", x.float().contiguous(), v, f.int().contiguous(), batched)[0]
        assert torch.equal(ref.view(torch.int32), got.view(torch.int32))
    assert torch.equal(out["right.pts2mano_sdf_cano"], calls[0][3])
    for (v, f, x, _), nid, thr in ((calls[1], "right", 0.01), (calls[2], "object", 0.05)):
        ref = run(ctx, "hold_mesh_sdf", x.float().contiguous(), v, f.int().contiguous(), v.dim() == 3)[0].reshape(B * P, -1).contiguous()
        off = torch.empty(B * P, dtype=torch.uint8, device=dev)
        capi.check(capi.lib().hold_off_in_surface(ctx.h, B * P, ref.shape[1], _p(ref), C.c_float(thr), _p(off), None, capi.stream_ptr()))
        assert torch.equal(out[f"{nid}.index_off_surface"], off.bool()), nid
    assert calls[2][0].shape == (object_mesh[0].shape[0], 3)          # one shared mesh, one tree
    g = torch.Generator(device=dev).manual_seed(1)
    batch = {"idx": inp["idx"], "gt.rgb": torch.rand(B, P, 3, device=dev, generator=g),
             "gt.mask": torch.tensor([0, 50, 150], device=dev)[torch.randint(0, 3, (B, P), device=dev, generator=g)]}
    full.zero_grad(set_to_none=True)
    ld = train.Loss()(batch, out)
    ld["loss"].backward()
    assert torch.isfinite(ld["loss"]).item()
