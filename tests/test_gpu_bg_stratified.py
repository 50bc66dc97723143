"""Training-mode (stratified) sampling: hold_bg_encode / hold_bg_integrate(_bwd) of the background leg against the oracle, and
forward_train / TrainStep with stratified=True (the reference's training-mode ErrorBoundSampler and inverse_sample,
engine/ray_sampler.py:54-85,292,328)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel(a, r):
    a, r = a.detach().double().cpu(), r.detach().double().cpu()
    return ((a - r).abs().max() / r.abs().max().clamp_min(1e-30)).item()


def _scene(ctx, seed=8, H=12):
    from hold_b200 import capi, scene_io, synth
    from oracle import hold_oracle as O

    sc = synth.make_scene(H=H, W=H, S=32, nodes=("right", "object"), B=2, seed=seed)
    sc.intrinsics[:, 0, 2] += 0.37   # keep every ray off the sphere centre (0/0 in the reference's depth2pts_outside)
    sc.intrinsics[:, 1, 2] -= 0.21
    net = scene_io.build_net(sc, ctx, capi.MLP_TC)
    bg, sdf_sd, rgb_sd = scene_io.build_background(sc, ctx, mlp_mode=capi.MLP_TC)
    dirs, cam = O.camera_rays(sc.uv, sc.extrinsics, sc.intrinsics)
    P = dirs.shape[1]
    dirs, cam = dirs.reshape(-1, 3).contiguous(), cam.unsqueeze(1).repeat(1, P, 1).reshape(-1, 3).contiguous()
    return sc, net, bg, sdf_sd, rgb_sd, dirs, cam


def test_bg_encode(ctx):
    """jitter = None: hold_background's depths bit for bit (and the torch expression forward_train used before); PE rows against
    the oracle in float64.  With jitter: the oracle's depths, each inside its stratum."""
    from hold_b200 import capi, train
    from hold_b200.capi import check, lib, ptr, stream_ptr
    from oracle import hold_oracle as O

    sc, net, bg, _, _, dirs, cam = _scene(ctx)
    dev = torch.device("cuda", 0)
    R, R_s = dirs.shape[0], sc.bounding_sphere
    dg, cg = dirs.to(dev), cam.to(dev)
    z, pe, pv = train.bg_encode(ctx, dg, cg, sc.B)
    ctx.check()
    ref_z = torch.empty(R, 32, device=dev)
    fc = torch.zeros(sc.B, 32, device=dev)
    check(lib().hold_background(ctx.h, R, sc.B, ptr(cg), ptr(dg), ptr(fc), ptr(torch.rand(R, device=dev)), None, None, None,
                                ptr(ref_z), stream_ptr()))
    ctx.check()
    assert torch.equal(z, ref_z)
    assert torch.equal(z, (torch.linspace(0.0, 1.0, 32, device=dev) * (1.0 / R_s))[None].expand(R, 32))
    # PE rows, flipped sample order: the 4-d point against float64, the embedding of it exactly as the oracle's embed_n
    zf = torch.flip(z.cpu().double(), dims=[-1])
    p4 = O.depth2pts_outside(cam.double()[:, None].expand(R, 32, 3), dirs.double()[:, None].expand(R, 32, 3), zf, R_s).reshape(-1, 4)
    e_pts = (pe[:, :4].cpu().double() - p4).abs().max().item()
    # sin / cos(2^k x) amplify the float32 rounding of x by 2^k (up to 512): the sines are checked on the kernel's own x
    e_emb = (pe.cpu().double() - O.embed_n(pe[:, :4].cpu().double(), 10)).abs().max().item()
    e_view = (pv.cpu().double() - O.embed_n(dirs.double().repeat_interleave(32, 0), 4)).abs().max().item()
    print(f"encode: point {e_pts:.2e}, PE-10 {e_emb:.2e}, view PE-4 {e_view:.2e}")
    assert e_pts <= 1e-5 and e_emb <= 1e-5 and e_view <= 1e-5
    # jittered depths
    g = torch.Generator().manual_seed(2)
    jitter = torch.rand(R, 32, generator=g)
    zj, pej, _ = train.bg_encode(ctx, dg, cg, sc.B, jitter.to(dev))
    lo = train.bg_encode(ctx, dg[:1], cg[:1], 1, torch.zeros(1, 32, device=dev))[0].cpu()
    hi = train.bg_encode(ctx, dg[:1], cg[:1], 1, torch.ones(1, 32, device=dev))[0].cpu()
    ctx.check()
    zj = zj.cpu()
    assert (zj >= lo).all() and (zj <= hi).all()
    ref = O.uniform_z(0.0, torch.ones(R, 1), 32, jitter) * (1.0 / R_s)
    # the device fuses lower + (upper - lower) * u into one fma; torch rounds the product first: at most one float32 ulp apart
    e = (zj - ref).abs().max().item()
    print(f"jittered depths vs oracle: {e:.2e}")
    assert e <= 2.0 ** -23 * ref.abs().max().item()
    p4j = O.depth2pts_outside(cam.double()[:, None].expand(R, 32, 3), dirs.double()[:, None].expand(R, 32, 3),
                              torch.flip(zj.double(), dims=[-1]), R_s).reshape(-1, 4)
    assert (pej[:, :4].cpu().double() - p4j).abs().max().item() <= 1e-5


def _background(bg_weights, ray_dirs, cam_loc, frame_code, frame_of_ray, bg_sdf_sd, bg_rgb_sd, R_s, jitter=None):
    """The oracle's `background` (hold_net.py:91-118, background.py:35-165) with training-mode inverse_sample depths: the same
    steps on the oracle's own pieces, the depths from its uniform_z(..., jitter) (ray_sampler.py:70-78)."""
    from oracle import hold_oracle as O

    R, n = ray_dirs.shape[0], 32
    z_bg = O.uniform_z(0.0, torch.ones(R, 1), n, jitter) * (1.0 / R_s)
    zf = torch.flip(z_bg, dims=[-1])
    dirs = ray_dirs.unsqueeze(1).repeat(1, n, 1)
    locs = cam_loc.unsqueeze(1).repeat(1, n, 1)
    p4 = O.depth2pts_outside(locs, dirs, zf, R_s).reshape(-1, 4)
    fc = frame_code[frame_of_ray].repeat_interleave(n, 0)
    o = O.bg_sdf_mlp(p4, fc, bg_sdf_sd)
    sdf, feat = o[:, :1], o[:, 1:]
    rgb = O.bg_rgb_mlp(dirs.reshape(-1, 3), fc, feat, bg_rgb_sd).reshape(R, n, 3)
    fe = torch.cat([zf[:, :-1] - zf[:, 1:], torch.full((R, 1), 1e10)], -1) * sdf.abs().reshape(R, n)
    w = (1 - torch.exp(-fe)) * torch.exp(-torch.cumsum(torch.cat([torch.zeros(R, 1), fe[:, :-1]], -1), -1))
    only = (w.unsqueeze(-1) * rgb).sum(1)
    sem = torch.zeros(R, 4)
    sem[:, 0] = 1.0
    return bg_weights.unsqueeze(-1) * only, only, bg_weights.unsqueeze(-1) * sem, z_bg


def test_background_training_jittered(ctx):
    """The background leg with jittered depths against float64 autograd over the oracle's background leg with the same draw
    (_background, which equals the oracle's `background` without jitter): outputs and the gradients w.r.t. both nets, the frame
    codes and bg_weights (bounds of test_background_training)."""
    from hold_b200 import train
    from oracle import hold_oracle as O

    sc, _, bg, sdf_sd, rgb_sd, dirs, cam = _scene(ctx)
    dev = torch.device("cuda", 0)
    R = dirs.shape[0]
    P = R // sc.B
    g = torch.Generator().manual_seed(3)
    bgw = torch.rand(R, generator=g)
    d_rgb, d_only, d_sem = torch.randn(R, 3, generator=g), torch.randn(R, 3, generator=g), torch.randn(R, 4, generator=g)
    jitter = torch.rand(R, 32, generator=g)
    frame = torch.arange(sc.B).repeat_interleave(P)
    idx = torch.as_tensor(sc.frame_idx)

    emb = bg.frame_latent_encoder.weight.detach().cpu().double().requires_grad_(True)
    s64 = {k: v.double().requires_grad_(True) for k, v in sdf_sd.items()}
    r64 = {k: v.double().requires_grad_(True) for k, v in rgb_sd.items()}
    bgw64 = bgw.double().requires_grad_(True)
    with torch.no_grad():   # the restatement is the oracle's background leg when the depths are not jittered
        a = _background(bgw.double(), dirs.double(), cam.double(), emb[idx], frame, s64, r64, sc.bounding_sphere)
        b = O.background(bgw.double(), dirs.double(), cam.double(), emb[idx], frame, s64, r64, sc.bounding_sphere)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
    o = _background(bgw64, dirs.double(), cam.double(), emb[idx], frame, s64, r64, sc.bounding_sphere, jitter=jitter.double())
    (o[0] * d_rgb.double()).sum().add((o[1] * d_only.double()).sum()).add((o[2] * d_sem.double()).sum()).backward()

    bg.zero_grad(set_to_none=True)
    bgw_d = bgw.to(dev).requires_grad_(True)
    out = train.background_forward_train(bg, bgw_d, dirs.to(dev), cam.to(dev), idx.to(dev), sc.B, sc.bounding_sphere, jitter=jitter.to(dev))
    ctx.check()
    assert (out["bg_z_vals"].cpu().double() - o[3]).abs().max().item() <= 1e-7
    for name, a, r in (("bg_rgb", out["bg_rgb"], o[0]), ("bg_rgb_only", out["bg_rgb_only"], o[1]), ("bg_semantics", out["bg_semantics"], o[2])):
        err = (a.detach().cpu().double() - r.detach()).abs().max().item()
        print(f"jittered background: forward {name} {err:.2e}")
        assert err <= 1e-4, f"{name}: {err:.2e}"
    ((out["bg_rgb"] * d_rgb.to(dev)).sum() + (out["bg_rgb_only"] * d_only.to(dev)).sum() + (out["bg_semantics"] * d_sem.to(dev)).sum()).backward()
    ctx.check()
    checks = [("bg_weights", bgw_d.grad, bgw64.grad), ("frame codes", bg.frame_latent_encoder.weight.grad, emb.grad)]
    for l in range(9):
        lin = getattr(bg.bg_implicit_network, f"lin{l}")
        checks += [(f"sdf.lin{l}.weight", lin.weight.grad, s64[f"lin{l}.weight"].grad), (f"sdf.lin{l}.bias", lin.bias.grad, s64[f"lin{l}.bias"].grad)]
    for l in range(2):
        lin = getattr(bg.bg_rendering_network, f"lin{l}")
        checks += [(f"rgb.lin{l}.weight", lin.weight.grad, r64[f"lin{l}.weight"].grad), (f"rgb.lin{l}.bias", lin.bias.grad, r64[f"lin{l}.bias"].grad)]
    for name, a, r in checks:
        assert a is not None, f"no gradient for {name}"
        e = rel(a, r)
        print(f"jittered background: grad {name} {e:.2e}")
        assert e <= 2e-4, f"grad {name}: rel {e:.2e}"


def _full(ctx, seed=11):
    from hold_b200 import capi, scene_io, synth
    from hold_b200.model import HOLDNet

    sc = synth.make_scene(H=8, W=8, S=32, nodes=("right", "object"), B=2, seed=seed)
    sc.intrinsics[:, 0, 2] += 0.37
    net = scene_io.build_net(sc, ctx, capi.MLP_TC)
    bg, _, _ = scene_io.build_background(sc, ctx, mlp_mode=capi.MLP_TC)
    return sc, HOLDNet(ctx, dict(net.nodes), background=bg)


def test_forward_train_stratified(ctx):
    """Same generator seed -> identical outputs; another seed -> other foreground and background depths.  The stratified
    foreground samples (the sampler_rand draw forward_train makes per node) are sorted and inside [0, far]."""
    from hold_b200 import ops, scene_io, train
    from hold_b200.model import ErrorBoundSampler, sampler_rand

    sc, full = _full(ctx)
    dev = torch.device("cuda", 0)
    inp = {**scene_io.scene_input(sc, dev), "current_epoch": 30, "global_step": 100}
    gen = lambda s: torch.Generator(device=dev).manual_seed(s)
    with torch.no_grad():
        a = train.forward_train(full, inp, gen(1), stratified=True)
        b = train.forward_train(full, inp, gen(1), stratified=True)
        c = train.forward_train(full, inp, gen(2), stratified=True)
        plain = train.forward_train(full, inp, gen(1))
    ctx.check()
    for k in ("rgb", "bg_z_vals", "right.depth", "object.depth", "bg_rgb_only"):
        assert torch.equal(a[k], b[k]), k
    R = a["rgb"].shape[0]
    assert not torch.equal(a["bg_z_vals"], c["bg_z_vals"]) and not torch.equal(a["right.depth"], c["right.depth"])
    assert torch.equal(plain["bg_z_vals"], (torch.linspace(0.0, 1.0, 32, device=dev) * (1.0 / sc.bounding_sphere))[None].expand(R, 32))
    assert not torch.equal(a["bg_z_vals"], plain["bg_z_vals"])
    # the foreground samples
    B, P = inp["uv"].shape[:2]
    dirs, cam = ops.camera_rays(full.ctx, inp["uv"], inp["extrinsics"], inp["intrinsics"])
    b_ = (dirs * cam).sum(-1)
    far = torch.sqrt(b_ ** 2 - ((cam ** 2).sum(-1) - sc.bounding_sphere ** 2)) - b_
    zs = {}
    for s in (1, 2):
        for node in full.nodes.values():
            with torch.no_grad():
                pose, _, _, _ = node.articulate(inp)
                z, _ = ErrorBoundSampler(node).get_z_vals(dirs, cam, pose, B, rand=sampler_rand(B * P, node.sampler_cfg, dev, gen(s)))
            ctx.check()
            zs[(s, node.node_id)] = z
            assert (z[:, 1:] >= z[:, :-1]).all(), node.node_id
            assert (z >= 0).all() and (z <= far[:, None] * (1 + 1e-6)).all(), node.node_id
    for node in full.nodes.values():
        assert not torch.equal(zs[(1, node.node_id)], zs[(2, node.node_id)])


def test_train_step_stratified(ctx):
    """A stratified TrainStep.step: finite loss, finite gradient for every parameter; graph capture of it is refused."""
    from hold_b200 import scene_io, train

    sc, full = _full(ctx, seed=5)
    dev = torch.device("cuda", 0)
    inp = scene_io.scene_input(sc, dev)
    R = sc.B * sc.uv.shape[1]
    g = torch.Generator(device=dev).manual_seed(0)
    gt_rgb, gt_mask = torch.rand(R, 3, device=dev, generator=g), torch.zeros(R, 4, device=dev)
    gt_mask[:, 0] = 1.0
    ts = train.TrainStep(full, lr=1e-4, n_eik=64, stratified=True)
    loss, parts = ts.step(inp, gt_rgb, gt_mask, generator=torch.Generator(device=dev).manual_seed(1))
    ctx.check()
    assert torch.isfinite(loss).item(), parts
    missing = [n for n, p in full.named_parameters() if p.requires_grad and (p.grad is None or not torch.isfinite(p.grad).all())]
    assert not missing, f"parameters without a finite gradient: {missing[:8]}"
    assert max(p.grad.abs().max().item() for p in full.background.parameters()) > 0
    with pytest.raises(ValueError, match="stratified"):
        train.TrainStep(full, capturable=True, stratified=True)
