"""Stage-wise parity of the CUDA path (through the C ABI) against the CPU oracle: each stage gets the SAME
inputs as the oracle's stage, so the tolerance is the north-star 1e-4 relative (indices exact)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = 1e-4


def close(a, b, tol=TOL, name="", frac=1.0):
    """max-abs relative to the tensor's scale; frac < 1 allows that share of entries to differ (used where the
    reference itself has a discrete, last-bit-sensitive choice upstream: the 15th nearest vertex)."""
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    assert a.shape == b.shape, f"{name}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    scale = max(1.0, b.abs().max().item())
    d = (a - b).abs()
    ok = (d <= tol * scale).float().mean().item()
    assert ok >= frac, f"{name}: only {ok:.5f} within {tol:.0e} * {scale:.3e} (max|d| {d.max().item():.3e})"
    return d.max().item()


@pytest.fixture(scope="module")
def scene():
    from hold_b200 import synth
    from oracle import hold_oracle as O

    sc = synth.make_scene(H=16, W=16, S=128, nodes=("right", "left", "object"), B=2, seed=3)
    for nid in sc.node_ids:
        sc.beta[nid] = torch.tensor(0.05)
    # The reference's up-sampling PDF is (exp(E) - 1) * T + add_tiny with add_tiny = 1e-6: where E is tiny,
    # exp(E) - 1 is a multiple of 2^-23 decided by the last bit of exp(), i.e. by the libm (tools/noise_floor.py:
    # a +-1 ulp exp moves 11-24 % of the reference's own z_vals).  test_sampler (whole loop, all rounds chained) therefore
    # raises add_tiny (a config constant, confs/general.yaml:78) so that the sampler LOGIC is compared above that noise; the
    # DEFAULT constant is held round by round, teacher-forced, in tests/test_gpu_sampler_rounds.py, and end to end in
    # test_gpu_e2e.py.
    sc.sampler["add_tiny"] = 1e-3
    return dict(sc=sc, art=O.scene_articulation(sc), O=O)


@pytest.fixture(scope="module", params=["fp32", "tc"])
def setup(ctx, scene, request):
    """Every stage test runs in both arithmetic modes of the MLPs: exact fp32 on CUDA cores (HOLD_MLP_FP32) and the tensor-core
    split-precision path (HOLD_MLP_TC) that bench.py and smoke() use — both are held to the ORACLE at the same tolerance."""
    from hold_b200 import capi, scene_io

    sc = scene["sc"]
    net = scene_io.build_net(sc, ctx, capi.MLP_TC if request.param == "tc" else capi.MLP_FP32)
    dev = torch.device("cuda", 0)
    inp = scene_io.scene_input(sc, dev)
    return dict(sc=sc, net=net, inp=inp, art=scene["art"], dev=dev, O=scene["O"], mode=request.param)


def test_mano_server(setup, ctx):
    s = setup
    for nid in ("right", "left"):
        node = s["net"].nodes[nid]
        _, _, out, _ = node.articulate(s["inp"])
        a = s["art"][nid]
        close(out["verts"], a["verts"], 1e-5, f"{nid}.verts")
        close(out["jnts"], a["jnts"], 1e-5, f"{nid}.jnts")
        close(out["tfs"], a["tfs"], 1e-5, f"{nid}.tfs")
        close(out["v_posed"], a["v_posed"], 1e-5, f"{nid}.v_posed")
        close(node.server.verts_c[0], a["cano_verts"], 1e-5, f"{nid}.verts_c")
        close(node.server.tfs_c_inv, a["tfs_c_inv"], 1e-4, f"{nid}.tfs_c_inv")
    ctx.check()


def test_object_server(setup, ctx):
    s = setup
    node = s["net"].nodes["object"]
    _, _, out, tfs = node.articulate(s["inp"])
    close(tfs, s["art"]["object"]["tfs"], 1e-5, "obj_tfs")
    close(out["verts"], s["art"]["object"]["verts"], 1e-5, "obj_verts")


def test_object_server_with_object_model_buffers(setup, ctx):
    """obj_scale != 1 and a non-identity norm_mat (real sequences: data.npy entities.object, model/obj/object_model.py:23-27),
    set the way checkpoint.load_reference_state_dict sets them (from `nodes.object.server.object_model.*`)."""
    from hold_b200 import checkpoint

    s, O = setup, setup["O"]
    sc = s["sc"]
    node = s["net"].nodes["object"]
    g = torch.Generator().manual_seed(12)
    nm = torch.eye(4)
    nm[:3, :3] = torch.linalg.qr(torch.randn(3, 3, generator=g))[0] * 1.7
    nm[:3, 3] = torch.tensor([0.11, -0.07, 0.23])
    sd = {"model.nodes.object.server.object_model.obj_scale": torch.tensor([0.83]),
          "model.nodes.object.server.object_model.norm_mat": nm,
          "model.nodes.object.server.object_model.denorm_mat": torch.linalg.inv(nm),
          "model.nodes.object.server.object_model.v3d_cano": node.server.v3d_cano.cpu().clone()}
    bufs = checkpoint.object_model_buffers(sd)["object"]
    old = (node.server.obj_scale, node.server.norm_mat.clone())
    node.server.set_object_model(**bufs)
    try:
        _, _, out, tfs = node.articulate(s["inp"])
        ctx.check()
    finally:
        node.server.set_object_model(obj_scale=old[0], norm_mat=old[1])
    p = sc.params["object"]
    scale = torch.full((sc.B,), float(sc.scene_scale))
    tf, v = O.object_server(p["global_orient"], p["transl"], scale, 0.83, torch.linalg.inv(nm), sc.obj_pts_cano)
    close(tfs, tf, 1e-5, "obj_tfs (obj_scale 0.83, norm_mat)")
    close(out["verts"], v, 1e-5, "obj_verts (obj_scale 0.83, norm_mat)")
    assert (tf - s["art"]["object"]["tfs"]).abs().max().item() > 1e-2, "the buffers must change the transform"


def test_camera_rays(setup, ctx):
    from hold_b200 import ops

    s, O = setup, setup["O"]
    sc = s["sc"]
    d, c = ops.camera_rays(ctx, s["inp"]["uv"], s["inp"]["extrinsics"], s["inp"]["intrinsics"])
    do, co = O.camera_rays(sc.uv, sc.extrinsics, sc.intrinsics)
    close(d, do.reshape(-1, 3), 1e-6, "ray_dirs")
    close(c, co[:, None].expand(-1, sc.uv.shape[1], -1).reshape(-1, 3), 1e-6, "cam_loc")


def test_inverse_warp(setup, ctx):
    from hold_b200 import ops

    s, O = setup, setup["O"]
    g = torch.Generator().manual_seed(5)
    x = (torch.rand(2, 3000, 3, generator=g) - 0.5) * 2.4
    for nid in s["sc"].node_ids:
        node = s["net"].nodes[nid]
        pose, keep, _, _ = node.articulate(s["inp"])
        xc, idx, mask = ops.inverse_warp(node, x.to(s["dev"]), pose, want_idx=True)
        a = s["art"][nid]
        for b in range(2):
            if a["kind"] == "hand":
                xo, out_o, idx_o = O.hand_inverse_warp(x[b], a["verts"][b], a["skin_W"], a["tfs"][b])
                same = (idx[b].cpu().long() == idx_o).all(1)
                assert same.float().mean().item() > 0.999, f"{nid} knn indices differ on {(~same).sum().item()} points"
                close(xc[b].cpu()[same], xo[same], TOL, f"{nid}.x_c")
                assert (mask[b].cpu().bool() == out_o)[same].all()
            else:
                close(xc[b], O.rigid_inverse_warp(x[b], a["tfs"][b]), TOL, f"{nid}.x_c")
    ctx.check()


def test_sdf_eval(setup, ctx):
    s, O = setup, setup["O"]
    g = torch.Generator().manual_seed(6)
    x = (torch.rand(1, 1111, 3, generator=g) - 0.5) * 1.6
    for nid in s["sc"].node_ids:
        node = s["net"].nodes[nid]
        out = node.implicit_network(x.to(s["dev"]), None)
        grad = node.implicit_network.last_gradient
        xg = x[0].clone().requires_grad_(True)
        cond = torch.zeros(x.shape[1], 45) if nid != "object" else None
        ref = O.sdf_mlp(xg, s["sc"].sdf_state[nid], cond)
        gref = torch.autograd.grad(ref[:, 0].sum(), xg)[0]
        close(out[0, :, 0], ref[:, 0], TOL, f"{nid}.sdf")
        close(out[0, :, 1:], ref[:, 1:], TOL, f"{nid}.feat")
        close(grad[0], gref, TOL, f"{nid}.grad")


def test_sdf_eval_barf_weights(setup, ctx):
    """BarfEmbedder.embed (engine/embedders.py:92-122): the object's Fourier embedding times the coarse-to-fine mask
    barf_weights(alpha) — mid-training (alpha = 2.6: frequencies 0,1 fully on, 2 partially, 3.. off), sdf, feature and the
    gradient (which chains through the weighted embedding) against the oracle.  The geometric initialisation zeroes lin0's
    weights on the Fourier columns (shape_net.py:57-60), so the test trains them away from zero first (+ N(0, 0.05^2))."""
    s, O = setup, setup["O"]
    g = torch.Generator().manual_seed(8)
    x = (torch.rand(1, 1500, 3, generator=g) - 0.5) * 1.6
    node = s["net"].nodes["object"]
    w = O.barf_weights(2.6)
    assert w.shape == (39,) and 0.0 < w[3 + 6 * 2].item() < 1.0 and w[-1].item() == 0.0, "the mask must be non-trivial"
    sd0 = {k: v.clone() for k, v in s["sc"].sdf_state["object"].items()}
    sd = {k: v.clone() for k, v in sd0.items()}
    sd["lin0.weight_v"][:, 3:] += 0.05 * torch.randn(sd["lin0.weight_v"][:, 3:].shape, generator=g)
    sd["lin4.weight_v"][:, 217 + 3:] += 0.05 * torch.randn(sd["lin4.weight_v"][:, 217 + 3:].shape, generator=g)
    node.implicit_network.load_state_dict(sd, strict=True)
    node.sync_weights()
    node.barf_weights = w.to(s["dev"]).contiguous()
    try:
        out = node.implicit_network(x.to(s["dev"]), None)
        grad = node.implicit_network.last_gradient
        ctx.check()
    finally:
        node.barf_weights = None
        node.implicit_network.load_state_dict(sd0, strict=True)
        node.sync_weights()
    xg = x[0].clone().requires_grad_(True)
    ref = O.sdf_mlp(xg, sd, None, w)
    gref = torch.autograd.grad(ref[:, 0].sum(), xg)[0]
    plain = O.sdf_mlp(x[0], sd, None, None)
    assert (plain[:, 0] - ref[:, 0]).abs().max().item() > 1e-3, "the mask must change the result for this to test anything"
    close(out[0, :, 0], ref[:, 0], TOL, "object.sdf (BARF)")
    close(out[0, :, 1:], ref[:, 1:], TOL, "object.feat (BARF)")
    close(grad[0], gref, TOL, "object.grad (BARF)")


def _oracle_node(s, nid, ray_ids=None):
    O, sc, a = s["O"], s["sc"], s["art"][nid]
    dirs, cam = O.camera_rays(sc.uv, sc.extrinsics, sc.intrinsics)
    P = dirs.shape[1]
    dirs = dirs.reshape(-1, 3)
    cam = cam.unsqueeze(1).repeat(1, P, 1).reshape(-1, 3)
    frame = torch.arange(sc.B).repeat_interleave(P)
    return O.node_forward(a["kind"], O.CLASS_ID[nid], dirs, cam, frame, sc.sdf_state[nid], sc.rgb_state[nid], sc.beta[nid],
                          sc.sampler, sc.bounding_sphere, a["tfs"], posed_verts=a.get("verts") if a["kind"] == "hand" else None,
                          cano_verts=a.get("cano_verts"), skin_W=a.get("skin_W"), pose_cond=a.get("pose_cond"),
                          time_code=sc.time_code if a["kind"] == "object" else None), dirs, cam


@pytest.fixture(scope="module")
def oracle_nodes(scene):
    return {nid: _oracle_node(scene, nid) for nid in scene["sc"].node_ids}


def test_sampler(setup, oracle_nodes, ctx):
    """z_vals after all rounds (add_tiny = 1e-3, see the fixture).  The final draw uses pdf = w + 1e-5 with
    w = (1 - exp(-fe)) * T, again last-bit sensitive where w ~ 0, so ~2 % of the samples may snap to a
    neighbouring bin edge: >= 95 % within 1e-4 * R_s, weight-carrying samples within 3e-3 * R_s."""
    from hold_b200.model import ErrorBoundSampler

    s = setup
    for nid in s["sc"].node_ids:
        f, dirs, cam = oracle_nodes[nid]
        node = s["net"].nodes[nid]
        pose, keep, _, _ = node.articulate(s["inp"])
        z, iters = ErrorBoundSampler(node).get_z_vals(dirs.to(s["dev"]), cam.to(s["dev"]), pose, s["sc"].B)
        ctx.check()
        assert int(iters.item()) == f["iters"], f"{nid}: rounds {int(iters.item())} vs oracle {f['iters']}"
        z = z.cpu()
        assert (z[:, 1:] >= z[:, :-1]).all(), "z_vals not sorted"
        d = (z - f["z_vals"]).abs()
        frac = (d <= 1e-4 * 8.0).float().mean().item()
        from oracle import hold_oracle as O
        w, _ = O.density2weight(f["density"][:, :, 0], f["z_vals"], f["z_vals"][:, -1])
        assert frac >= 0.95, f"{nid}: only {frac:.4f} of z_vals within tolerance"
        assert (d * (w > 1e-4)).max().item() < 3e-3 * 8.0


def test_shade_given_z(setup, oracle_nodes, ctx):
    from hold_b200 import ops

    s = setup
    for nid in s["sc"].node_ids:
        f, dirs, cam = oracle_nodes[nid]
        node = s["net"].nodes[nid]
        pose, keep, _, _ = node.articulate(s["inp"])
        t = ops.shade(node, dirs.to(s["dev"]), cam.to(s["dev"]), pose, f["z_vals"].to(s["dev"]), s["sc"].B)
        ctx.check()
        fr = 0.9995 if nid != "object" else 1.0
        close(t["canonical_pts"], f["canonical_pts"], TOL, f"{nid}.x_c", fr)
        close(t["sdf"], f["sdf"], TOL, f"{nid}.sdf", fr)
        close(t["normal"], f["normal"], 2e-4, f"{nid}.normal", fr)
        close(t["color"], f["color"], TOL, f"{nid}.color", fr)
        close(t["density"], f["density"][:, :, 0], TOL, f"{nid}.density", fr)


@pytest.mark.parametrize("beta", [0.1, 0.03, 0.01])
def test_density_given_z_beta_sweep(setup, oracle_nodes, ctx, beta):
    """LaplaceDensity (engine/density.py:21-30) amplifies an sdf error by exp(-|s|/beta) / (2 beta^2): the smaller beta (it
    anneals down during training; bench.py runs beta = 0.03), the tighter the sdf has to be.  Same oracle z_vals, sdf from the
    kernels under test, density against the oracle's sdf pushed through the reference formula, relative to max|density| = 1/beta."""
    from hold_b200 import ops

    s, O = setup, setup["O"]
    worst = 0.0
    for nid in s["sc"].node_ids:
        f, dirs, cam = oracle_nodes[nid]
        node = s["net"].nodes[nid]
        old = node.density.beta.data.clone()
        node.density.beta.data.fill_(beta)
        try:
            pose, keep, _, _ = node.articulate(s["inp"])
            t = ops.shade(node, dirs.to(s["dev"]), cam.to(s["dev"]), pose, f["z_vals"].to(s["dev"]), s["sc"].B)
            ctx.check()
        finally:
            node.density.beta.data.copy_(old)
        ref = O.laplace_density(f["sdf"], O.density_beta(torch.tensor(beta)))
        d = (t["density"].cpu() - ref).abs()
        ds = (t["sdf"].cpu() - f["sdf"]).abs()
        fr = 0.9995 if nid != "object" else 1.0   # the hand's 15th-nearest-vertex choice is last-bit sensitive upstream
        k = max(1, int(round((1.0 - fr) * d.numel())))
        dk = d.flatten().topk(k).values[-1].item() if fr < 1.0 else d.max().item()
        rel = dk * beta   # relative to max|density| = 1 / beta
        worst = max(worst, rel)
        print(f"[{s['mode']}] beta {beta}: {nid} density rel err {rel:.2e} (abs {dk:.2e}), sdf max err {ds.max().item():.2e}")
        close(t["density"], ref, TOL, f"{nid}.density(beta={beta})", fr)


def test_color_net_given_oracle_inputs(setup, oracle_nodes, ctx):
    """RenderingNet (networks/texture_net.py:46-101) in isolation: the colour net of the mode under test is fed the ORACLE's
    canonical points / normals / features through hold_shade's own inputs being reproduced — i.e. colour is compared at the
    oracle's z_vals, and additionally the colour error is bounded where the upstream normal agrees to 1e-5, so that what is
    measured is the colour net's arithmetic (k_mlp_tc<MLP_COLOR> in tensor-core mode), not the normal's."""
    from hold_b200 import ops

    s = setup
    for nid in s["sc"].node_ids:
        f, dirs, cam = oracle_nodes[nid]
        node = s["net"].nodes[nid]
        pose, keep, _, _ = node.articulate(s["inp"])
        t = ops.shade(node, dirs.to(s["dev"]), cam.to(s["dev"]), pose, f["z_vals"].to(s["dev"]), s["sc"].B)
        ctx.check()
        same_n = ((t["normal"].cpu() - f["normal"]).abs().amax(-1) <= 1e-5)
        d = (t["color"].cpu() - f["color"]).abs().amax(-1)
        print(f"[{s['mode']}] {nid}: colour max err {d.max().item():.2e}; where normals agree to 1e-5 ({same_n.float().mean().item():.3f} of samples): {d[same_n].max().item():.2e}")
        assert d[same_n].max().item() <= TOL, f"{nid}: colour net error {d[same_n].max().item():.2e} with matching inputs"


def test_composite_given_factors(setup, oracle_nodes, ctx):
    from hold_b200 import ops

    s, O = setup, setup["O"]
    ids = s["sc"].node_ids
    fl = [oracle_nodes[nid][0] for nid in ids]
    ref = O.composite(fl, stable=True)  # canonical tie order, see oracle.merge_factors
    dev = s["dev"]
    facs = [dict(color=f["color"].to(dev), normal=f["normal"].to(dev), density=f["density"][:, :, 0].to(dev), z_vals=f["z_vals"].to(dev)) for f in fl]
    comp, per = ops.composite(ctx, facs, [O.CLASS_ID[n] for n in ids])
    for k in ("fg_rgb", "mask_prob", "normal", "depth", "fg_semantics", "bg_weights", "fg_weights"):
        close(comp[k].reshape(ref["comp"][k].shape), ref["comp"][k], 1e-5, f"comp.{k}")
        for i in range(len(ids)):
            close(per[i][k].reshape(ref[i][k].shape), ref[i][k], 1e-5, f"{ids[i]}.{k}")
