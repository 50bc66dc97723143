"""The reverse-mode tensor-core MLP kernel (sdf, 256-d feature and d sdf / d x_c: k_mlp_tc<3>) across tiles.

test_gpu_stages.py's sdf tests run up to 1 500 points, at most one 128-row tile per CTA.  Here P = 2 * 132 * 128 + 77 points: on a
132-SM H100 every persistent CTA walks two or three tiles and the last tile is partial, so the state a CTA carries from one tile to
the next (the per-row head and gradient sums, the stash of softplus', the skip layer's embedding columns) has to be reset or
rewritten per tile.  Both node nets, with and without BARF embedding weights; lin0's and lin4's embedding columns are trained away
from the geometric initialisation's zeros so that both d sdf / d embed chains carry gradient."""
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = 1e-4                      # test_gpu_stages.py's TOL for the same outputs
P = 2 * 132 * 128 + 77


def close(a, b, name):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    scale = max(1.0, b.abs().max().item())
    d = (a - b).abs().max().item()
    assert d <= TOL * scale, f"{name}: max|d| {d:.3e} > {TOL:.0e} * {scale:.3e}"


@pytest.fixture(scope="module")
def net(ctx):
    from hold_b200 import capi, scene_io, synth

    sc = synth.make_scene(H=8, W=8, S=32, nodes=("right", "object"), seed=11)
    return sc, scene_io.build_net(sc, ctx, capi.MLP_TC)


@pytest.mark.parametrize("barf", [False, True], ids=["plain", "barf"])
@pytest.mark.parametrize("nid", ["right", "object"])
def test_sdf_eval_multi_tile(net, ctx, nid, barf):
    from oracle import hold_oracle as O

    sc, hnet = net
    node = hnet.nodes[nid]
    g = torch.Generator().manual_seed(21)
    x = (torch.rand(1, P, 3, generator=g) - 0.5) * 1.6
    perm = torch.randperm(P, generator=g)
    w = O.barf_weights(2.6) if barf else None
    sd0 = {k: v.clone() for k, v in sc.sdf_state[nid].items()}
    sd = {k: v.clone() for k, v in sd0.items()}
    sd["lin0.weight_v"][:, 3:39] += 0.05 * torch.randn(sd["lin0.weight_v"][:, 3:39].shape, generator=g)
    sd["lin4.weight_v"][:, 217 + 3:] += 0.05 * torch.randn(sd["lin4.weight_v"][:, 217 + 3:].shape, generator=g)
    node.implicit_network.load_state_dict(sd, strict=True)
    node.sync_weights()
    node.barf_weights = w.to(torch.device("cuda", 0)).contiguous() if barf else None
    try:
        xd = x.to(torch.device("cuda", 0))
        out = node.implicit_network(xd, None).clone()
        grad = node.implicit_network.last_gradient.clone()
        out_p = node.implicit_network(xd[:, perm].contiguous(), None).clone()
        grad_p = node.implicit_network.last_gradient.clone()
        ctx.check()
    finally:
        node.barf_weights = None
        node.implicit_network.load_state_dict(sd0, strict=True)
        node.sync_weights()
    # a point's outputs do not depend on its row, tile or CTA: bit for bit
    assert torch.equal(out_p, out[:, perm]), "sdf / feature depend on the point's position in the launch"
    assert torch.equal(grad_p, grad[:, perm]), "gradient depends on the point's position in the launch"
    xg = x[0].clone().requires_grad_(True)
    cond = torch.zeros(P, 45) if nid != "object" else None
    ref = O.sdf_mlp(xg, sd, cond, w)
    gref = torch.autograd.grad(ref[:, 0].sum(), xg)[0]
    close(out[0, :, 0], ref[:, 0], f"{nid}.sdf")
    close(out[0, :, 1:], ref[:, 1:], f"{nid}.feat")
    close(grad[0], gref, f"{nid}.grad")
    assert (gref - torch.autograd.grad(O.sdf_mlp(xg, sd0, cond, w)[:, 0].sum(), xg)[0]).abs().max().item() > 1e-3, \
        "the embedding columns must carry gradient for this to test the d sdf / d embed chains"
