"""BASELINE configs[4] in miniature — a joint SDF + LBS backward for pose refinement through the kernels:
L = sum_p c_p * sdf(x_c(p; pose))  ->  d sdf/d x_c (hold_sdf_eval) -> d/d tfs (hold_inverse_warp_bwd) -> d/d pose, betas, transl,
scale (hold_mano_lbs_bwd), against torch.autograd over the oracle's whole chain.  The pieces' arithmetic runs on the host
already (tests/test_cpu_{warp,pose}_bwd.py); the GPU run is kept isolated."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def impl_pose_gradient_through_sdf(ctx):
    import ctypes as C

    from hold_b200 import capi, ops, scene_io, synth
    from hold_b200.capi import NodePose, check, lib, ptr, stream_ptr
    from oracle import hold_oracle as O

    dev = torch.device("cuda", 0)
    sc = synth.make_scene(H=4, W=4, S=32, nodes=("right",), B=1, seed=3)
    net = scene_io.build_net(sc, ctx, capi.MLP_FP32)
    node = net.nodes["right"]
    m, p = sc.mano["right"], sc.params["right"]
    betas = sc.betas["right"][None]
    full_pose = torch.cat([p["global_orient"], p["pose"]], 1)
    scale = torch.full((1,), float(sc.scene_scale))
    _, tci = O.mano_canonical(m, betas[0])
    g = torch.Generator().manual_seed(0)
    # ---- oracle: autograd through server -> inverse warp (detached weights) -> SDF net
    leaves = [t.clone().requires_grad_() for t in (betas, full_pose, p["transl"], scale)]
    out = O.mano_server(m, leaves[3], leaves[2], leaves[1], leaves[0], tci)
    verts0 = out["verts"][0].detach()
    P = 256
    x = (verts0[torch.randint(0, 778, (P,), generator=g)] + 0.03 * torch.randn(P, 3, generator=g)).contiguous()
    coef = torch.randn(P, generator=g)
    w, _, idx = O.skin_weights_query(x, verts0, m["lbs_weights"])
    T = torch.einsum("pn,nij->pij", w.detach(), out["tfs"][0])
    xc = torch.einsum("pij,pj->pi", T.inverse(), torch.nn.functional.pad(x, (0, 1), value=1.0))[:, :3]
    cond = (full_pose[:, 3:] / torch.pi).expand(P, -1)
    sdf = O.sdf_mlp(xc, sc.sdf_state["right"], cond)[:, 0]
    ref = torch.autograd.grad((coef * sdf).sum(), leaves)
    # ---- kernels
    srv = node.server
    lv = [t.clone().to(dev).requires_grad_() for t in (betas, full_pose, p["transl"], scale)]
    o = srv.forward(lv[3], lv[2], lv[1], lv[0])
    pose = NodePose()
    tfs_d, verts_d = o["tfs"].detach().contiguous(), o["verts"].detach().contiguous()
    cond_d = (full_pose[:, 3:] / torch.pi).float().to(dev).contiguous()
    beta_d = torch.tensor([0.1], device=dev)
    pose.tfs, pose.posed_verts, pose.pose_cond, pose.beta_param = tfs_d.data_ptr(), verts_d.data_ptr(), cond_d.data_ptr(), beta_d.data_ptr()
    xd = x.to(dev)[None].contiguous()
    xc_d, idx_d, _ = ops.inverse_warp(node, xd, pose, want_idx=True)
    sdf_d, grad_d, feat_d = torch.empty(P, device=dev), torch.empty(P, 3, device=dev), torch.empty(P, 256, device=dev)
    check(lib().hold_sdf_eval(ctx.h, node.slot, P, ptr(xc_d.reshape(P, 3).contiguous()), None, ptr(sdf_d), ptr(grad_d), ptr(feat_d), stream_ptr()))
    g_xc = (coef.to(dev)[:, None] * grad_d)[None].contiguous()
    g_tfs, _ = ops.inverse_warp_bwd(node, xd, pose, idx_d, g_xc)
    got = torch.autograd.grad(o["tfs"], lv, grad_outputs=g_tfs)
    ctx.check()
    assert torch.equal(idx_d.cpu().long().reshape(P, 15), idx)
    for name, a, b in zip(("betas", "pose", "transl", "scale"), got, ref):
        err = (a.cpu() - b).abs().max().item() / max(1.0, b.abs().max().item())
        assert err < 2e-4, f"{name}: {err:.2e}"


def test_pose_gradient_through_sdf(isolated):
    isolated("tests/test_gpu_warp_bwd.py", "impl_pose_gradient_through_sdf")
