"""SURVEY §8f rank 4: the pose servers under autograd (optimize_ckpt.py's `server.forward_param` + backward).
hold_mano_lbs_bwd / hold_object_tf_bwd against torch.autograd over the oracle (pinned to the reference's own autograd in
oracle/ref_harness.py check_pose_grads).  The kernels' phase code is already exercised on the CPU
(tests/test_cpu_pose_bwd.py)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def impl_mano_server_backward(ctx):
    from hold_b200 import synth
    from hold_b200.model import MANOServer
    from oracle import hold_oracle as O

    dev = torch.device("cuda", 0)
    m = synth.make_mano_struct(1)
    g = torch.Generator().manual_seed(13)
    B = 3
    betas = 0.5 * torch.randn(1, 10, generator=g)
    pose, transl, scale = 0.4 * torch.randn(B, 48, generator=g), torch.randn(B, 3, generator=g), 1.0 + 0.3 * torch.rand(B, generator=g)
    gv, gj, gt = torch.randn(B, 778, 3, generator=g), torch.randn(B, 21, 3, generator=g), torch.randn(B, 16, 4, 4, generator=g)
    srv = MANOServer(ctx, m, betas[0])
    _, tci = O.mano_canonical(m, betas[0])
    leaves_ref = [t.clone().requires_grad_() for t in (betas, pose, transl, scale)]
    out = O.mano_server(m, leaves_ref[3], leaves_ref[2], leaves_ref[1], leaves_ref[0].expand(B, 10), tci)
    ref = torch.autograd.grad((out["verts"] * gv).sum() + (out["jnts"] * gj).sum() + (out["tfs"] * gt).sum(), leaves_ref)
    leaves = [t.clone().to(dev).requires_grad_() for t in (betas, pose, transl, scale)]
    o = srv.forward(leaves[3], leaves[2], leaves[1], leaves[0])
    loss = (o["verts"] * gv.to(dev)).sum() + (o["jnts"] * gj.to(dev)).sum() + (o["tfs"] * gt.to(dev)).sum()
    got = torch.autograd.grad(loss, leaves)
    ctx.check()
    for name, a, b in zip(("betas", "pose", "transl", "scale"), got, ref):
        err = (a.cpu() - b).abs().max().item() / max(1.0, b.abs().max().item())
        assert err < 1e-4, f"{name}: {err:.2e}"


def impl_object_server_backward(ctx):
    from hold_b200.model import ObjectServer
    from oracle import hold_oracle as O

    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(17)
    B, Nv = 3, 500
    rot, trans, ss = 0.8 * torch.randn(B, 3, generator=g), torch.randn(B, 3, generator=g), 1.0 + 0.3 * torch.rand(B, generator=g)
    pts = torch.randn(Nv, 3, generator=g)
    gv = torch.randn(B, Nv, 3, generator=g)
    srv = ObjectServer(ctx, pts, obj_scale=1.0)
    srv.obj_scale = torch.tensor(1.7, device=dev, requires_grad=True)   # fitting/model.py:113
    lr = [t.clone().requires_grad_() for t in (rot, trans, ss)]
    osc = torch.tensor(1.7, requires_grad=True)
    _, v = O.object_server(lr[0], lr[1], lr[2], osc, torch.eye(4), pts)
    ref = torch.autograd.grad((v * gv).sum(), lr + [osc])
    lg = [t.clone().to(dev).requires_grad_() for t in (rot, trans, ss)]
    o = srv.forward(lg[2], lg[1], lg[0])
    got = torch.autograd.grad((o["verts"] * gv.to(dev)).sum(), lg + [srv.obj_scale])
    ctx.check()
    for name, a, b in zip(("rot", "trans", "scene_scale", "obj_scale"), got, ref):
        err = (a.cpu() - b).abs().max().item() / max(1.0, b.abs().max().item())
        assert err < 1e-4, f"{name}: {err:.2e}"


def test_mano_server_backward(isolated):
    isolated("tests/test_gpu_pose_bwd.py", "impl_mano_server_backward")


def test_object_server_backward(isolated):
    isolated("tests/test_gpu_pose_bwd.py", "impl_object_server_backward")
