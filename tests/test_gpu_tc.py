"""Tensor-core (wgmma, fp16 hi/lo split x3) MLP kernels against the exact-fp32 CUDA-core kernels and the oracle."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nets(ctx):
    from hold_b200 import capi, scene_io, synth

    sc = synth.make_scene(H=8, W=8, S=32, nodes=("right", "object"), seed=4)
    dev = torch.device("cuda", 0)
    n32 = scene_io.build_net(sc, ctx, capi.MLP_FP32)
    out = {}
    g = torch.Generator().manual_seed(9)
    x = ((torch.rand(1, 5000, 3, generator=g) - 0.5) * 1.6).to(dev)
    for nid in sc.node_ids:
        o = n32.nodes[nid].implicit_network(x, None)
        out[nid] = (o.clone(), n32.nodes[nid].implicit_network.last_gradient.clone())
    torch.cuda.synchronize()
    ntc = scene_io.build_net(sc, ctx, capi.MLP_TC)   # same ctx slots, re-configured for the tensor-core mode
    return dict(sc=sc, x=x, ref=out, ntc=ntc, dev=dev)


def rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1.0)).item()


def test_tc_sdf_eval(nets, ctx):
    for nid in nets["sc"].node_ids:
        node = nets["ntc"].nodes[nid]
        o = node.implicit_network(nets["x"], None)
        g = node.implicit_network.last_gradient
        ctx.check()
        ro, rg = nets["ref"][nid]
        e_sdf, e_feat, e_grad = rel(o[..., 0], ro[..., 0]), rel(o[..., 1:], ro[..., 1:]), rel(g, rg)
        print(f"{nid}: tc vs fp32  sdf {e_sdf:.2e} feat {e_feat:.2e} grad {e_grad:.2e}")
        assert e_sdf < 1e-4 and e_feat < 1e-4 and e_grad < 1e-4


def test_tc_sdf_only(nets, ctx):
    """The sampler-round launch shape (sdf head only, 128 points per tile)."""
    import ctypes as C
    from hold_b200 import capi

    x = nets["x"][0].contiguous()
    for nid in nets["sc"].node_ids:
        node = nets["ntc"].nodes[nid]
        sdf = torch.empty(x.shape[0], device=x.device)
        capi.check(capi.lib().hold_sdf_eval(ctx.h, node.slot, x.shape[0], capi.ptr(x), None, capi.ptr(sdf), None, None, capi.stream_ptr()))
        ctx.check()
        e = rel(sdf, nets["ref"][nid][0][0, :, 0])
        print(f"{nid}: tc sdf-only vs fp32 {e:.2e}")
        assert e < 1e-4


def test_tc_full_render(nets, ctx):
    from hold_b200 import capi, scene_io
    from oracle import hold_oracle as O

    sc = nets["sc"]
    out = nets["ntc"].forward_fg(scene_io.scene_input(sc, nets["dev"]))
    ctx.check()
    ref, _ = O.render_scene(sc, stable_ties=True)
    for k, nid in enumerate(sc.node_ids):
        for key in ("fg_rgb", "depth", "normal", "mask_prob"):
            a, b = out[f"{nid}.{key}"].cpu().reshape(ref[0]["render"][k][key].shape), ref[0]["render"][k][key]
            d = (a - b).abs()
            frac = (d <= 1e-4 * max(1.0, b.abs().max().item())).float().mean().item()
            print(f"{nid}.{key}: max {d.max().item():.2e} within-1e-4 {frac:.3f}")
            assert frac >= 0.95 and d.max().item() < 1e-2  # 64 pixels: one pixel is 1.6 %
