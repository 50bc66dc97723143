"""The skinning warps on the device at the sizes the product runs them (references, generators and error measures:
tests/test_cpu_skin_warps.py, which runs them on the CPU first).

1. The hot path's ray-walk KNN (k_inverse_warp_hand_rays, reached through hold_shade) gives the full scan's canonical points
   (k_inverse_warp<true,false>, through hold_inverse_warp) bit for bit, at every walk length launch_inverse_warp picks (32, 16, 8
   and 4 samples per thread), a full 512 x 512 frame at S = 128, the training batch at S = 98 (a partial last walk), S = 33, ray
   counts that are not a multiple of 128, both hands and several frames with their own poses per launch.
2. hold_inverse_warp / hold_forward_warp: neighbours and outlier mask exactly the float32 brute force's; x_c / x_d against float64 on
   the same neighbours, within 4x of float32 torch's worst point (floor 2^-20) and never above 1e-4.
3. hold_inverse_warp_bwd at the training batch (10 frames x 12 544 points = 98 full 128-point blocks per frame, or a partial block)
   against float64 autograd: g_tfs entries relative to the sum of |terms| they add up, g_x like x_c; the constant row's gradient is
   0, g_x = NULL leaves g_tfs bitwise unchanged, repeated calls are bitwise equal; empty sizes and error codes.
The MLPs run inside hold_shade only to reach the hot warp; their outputs are not asserted here.

The hand path has no non-finite check on a singular blended transform (only the object path reports HOLD_E_NONFINITE); the cases
here keep every blended transform well conditioned."""
import ctypes as C

import pytest
import torch

import test_cpu_skin_warps as T

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def net(ctx):
    from hold_b200 import capi, scene_io, synth

    sc = synth.make_scene(H=4, W=4, S=32, nodes=("right", "left", "object"), B=1, seed=0)
    return scene_io.build_net(sc, ctx, capi.MLP_TC)


@pytest.fixture(scope="module")
def pix():
    return T.pixel_dirs()


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def node_pose(tfs, verts=None):
    """NodePose of caller-given transforms (and posed vertices): pose_cond zeros, beta 0.1, a time code for the object."""
    from hold_b200.capi import NodePose

    B = tfs.shape[0]
    keep = [tfs.to(DEV).contiguous(), torch.zeros(B, 45, device=DEV), torch.full((1,), 0.1, device=DEV), torch.zeros(B, 32, device=DEV)]
    p = NodePose()
    p.tfs, p.pose_cond, p.beta_param, p.time_code = (t.data_ptr() for t in keep)
    if verts is not None:
        keep.append(verts.to(DEV).contiguous())
        p.posed_verts = keep[-1].data_ptr()
    return p, keep


def skin_w(net, nid):
    return net.nodes[nid].server.m["lbs_weights"]


# ------------------------------------------------------------------------------------------------ 1. ray walk == full scan
WALK_CASES = [
    # id, node, frames, samples per ray, walk length (None: rays per frame given), rays per frame
    ("frame512_S128", "right", 1, 128, 32, 512 * 512),
    ("train_B10_S98", "right", 10, 98, 4, 128),
    ("B10_S98_L32", "left", 10, 98, 32, None),
    ("B10_S98_L16", "right", 10, 98, 16, None),
    ("B10_S98_L8", "left", 10, 98, 8, None),
    ("B2_S128_L16", "left", 2, 128, 16, None),
    ("B3_S128_L8", "right", 3, 128, 8, None),
    ("B2_S128_L4", "left", 2, 128, 4, 1001),
    ("B3_S33_L8", "left", 3, 33, 8, None),
    ("B4_S33_L4", "right", 4, 33, 4, 389),
]


def _mismatch_report(net, nid, x, got, full, verts, tfs, P):
    """Tells different neighbours (errors of a skin weight's size) from the same neighbours a few ulp apart."""
    bad = (got != full).any(-1)
    lines = [f"{int(bad.sum())} of {bad.numel()} points differ"]
    for b in range(x.shape[0]):
        i = bad[b].nonzero()[:, 0][:2048]
        if i.numel() == 0:
            continue
        xs = x[b, i]
        _, idx = T.brute_knn(xs, verts[b])
        r64 = T.hand_warp_ref(xs, idx, verts[b], skin_w(net, nid), tfs[b], torch.float64)
        eh = (got[b, i].double() - r64).abs().max().item()
        ef = (full[b, i].double() - r64).abs().max().item()
        lines.append(f"frame {b}: max |hot - f64| {eh:.3e}, max |full scan - f64| {ef:.3e} (first point {i[0].item() % P})")
    return "\n".join(lines)


@pytest.mark.parametrize("case", WALK_CASES, ids=[c[0] for c in WALK_CASES])
def test_ray_walk_is_the_full_scan(net, ctx, pix, case):
    from hold_b200 import ops

    name, nid, B, S, L, rpf = case
    sm = sm_count()
    if rpf is None:
        rpf = T.rays_for_seg_len(L, B, S, sm)
    seg = T.expected_seg_len(B, rpf, S, sm)
    print(f"{name}: {sm} SMs, {B} x {rpf} rays x {S} samples -> walk length {seg}")
    assert seg == L, f"{name}: walk length {seg}, wanted {L}"
    verts, tfs, ties = T.posed_hand(nid, B, seed=WALK_CASES.index(case))
    cams, dirs, zs, nspecial = [], [], [], 0
    for b in range(B):
        c, d, z, ns = T.frame_rays(verts[b], ties[b], rpf, S, seed=b, pix=pix, dev=DEV)
        cams.append(c), dirs.append(d), zs.append(z)
        nspecial += ns
    cam, dr, z = torch.cat(cams), torch.cat(dirs), torch.cat(zs)
    vd, td = verts.to(DEV), tfs.to(DEV)
    node = net.nodes[nid]
    pose, keep = node_pose(td, vd)
    t = ops.shade(node, dr, cam, pose, z, B)
    x = T.ray_points(cam, dr, z).reshape(B, rpf * S, 3)
    full, _, _ = ops.inverse_warp(node, x, pose)
    torch.cuda.synchronize()
    ctx.check()
    got = t["canonical_pts"].reshape(B, rpf * S, 3)
    if not torch.equal(got, full):
        pytest.fail(f"{name}: hot path != full scan\n" + _mismatch_report(net, nid, x, got, full, vd, td, rpf * S))
    # the constructed edges are present: ties straddling the 15th / 16th cut on duplicates
    assert sum(T.straddles(T.ray_points(cams[b][:16], dirs[b][:16], zs[b][:16]).reshape(-1, 3), vd[b]) for b in range(min(B, 2))) > 0
    assert nspecial == B * T.N_SPECIAL


# ------------------------------------------------------------------------------------------------ 2. warps against float64
def hand_points(v, P, seed):
    """Edge points first (every vertex exactly, far points where every confidence clamps, points along the tie and duplicate
    rays), then points within ~1 cm of the hand and some farther out.  Returns (x [P,3] on DEV, number of edge points)."""
    g = torch.Generator().manual_seed(seed)
    vc = v.cpu()
    c = vc.mean(0)
    far = c + 4.0 * torch.nn.functional.normalize(torch.randn(32, 3, generator=g), dim=1)
    edge = [vc, far]
    edge = torch.cat(edge)[:P]
    n = P - edge.shape[0]
    near = vc[torch.randint(0, vc.shape[0], (n,), generator=g)] + 0.01 * torch.randn(n, 3, generator=g)
    near[::9] += 0.1 * torch.randn(near[::9].shape, generator=g)
    x = torch.cat([edge, near]) if n > 0 else edge
    return x.to(DEV).contiguous(), edge.shape[0]


def _check_warp(label, got, x, idx, v, W, tf, forward, n_edge, stride):
    sub = torch.cat([torch.arange(n_edge, device=DEV), torch.arange(n_edge, x.shape[0], stride, device=DEV)])
    xs, ids = x[sub], idx[sub]
    r64 = T.hand_warp_ref(xs, ids, v, W, tf, torch.float64, forward)
    r32 = T.hand_warp_ref(xs, ids, v, W, tf, torch.float32, forward)
    wk, w32 = T.worst(got[sub], r64), T.worst(r32, r64)
    print(f"{label}: {sub.numel()} points vs float64: kernel {wk:.2e}, float32 torch {w32:.2e}")
    assert wk <= T.F32_FACTOR * max(w32, T.F32_FLOOR), f"{label}: {wk:.2e} > {T.F32_FACTOR} x float32 torch's {w32:.2e}"
    assert wk <= T.REL_TOL, f"{label}: {wk:.2e}"


@pytest.mark.parametrize("nid,B,P,stride", [("right", 1, 4 * 1024 * 1024 + 1, 4), ("left", 10, 12545, 1), ("right", 10, 1, 1)])
def test_hand_inverse_warp_against_float64(net, ctx, nid, B, P, stride):
    from hold_b200 import ops

    verts, tfs, ties = T.posed_hand(nid, B, seed=P % 97)
    vd, td = verts.to(DEV), tfs.to(DEV)
    W = skin_w(net, nid)
    xs, n_edge = [], 0
    for b in range(B):
        xb, n_edge = hand_points(verts[b], P, seed=b)
        if P > 1000:   # points along the tie rays and through the duplicates
            c, d, z, _ = T.frame_rays(verts[b], ties[b], T.N_SPECIAL, 64, seed=b, dev=DEV)
            e = T.ray_points(c, d, z).reshape(-1, 3)
            xb = torch.cat([xb[:n_edge], e, xb[n_edge + e.shape[0]:]])
            n_edge += e.shape[0]
        xs.append(xb)
    x = torch.stack(xs).contiguous()
    pose, keep = node_pose(td, vd)
    xc, idx, mask = ops.inverse_warp(net.nodes[nid], x, pose, want_idx=True)
    torch.cuda.synchronize()
    ctx.check()
    for b in range(B):
        d, ib = T.brute_knn(x[b], vd[b])
        assert torch.equal(idx[b].long(), ib), f"{nid} frame {b}: knn_idx differs on {(idx[b].long() != ib).any(1).sum().item()} points"
        assert torch.equal(mask[b].bool(), torch.sqrt(d[:, 0].clamp(max=4.0)) > 0.1), f"{nid} frame {b}: outlier mask"
        _check_warp(f"{nid} inverse B={B} P={P} frame {b}", xc[b], x[b], ib, vd[b], W, td[b], False, min(n_edge, P), stride)
    if P > 1000:
        assert mask.bool().any() and not mask.bool().all()


@pytest.mark.parametrize("nid,B,P,stride", [("left", 1, 4 * 1024 * 1024 + 1, 4), ("right", 10, 12545, 1)])
def test_hand_forward_warp_against_float64(net, ctx, nid, B, P, stride):
    from hold_b200.capi import check, lib, ptr, stream_ptr

    node = net.nodes[nid]
    cano = node.server.verts_c[0].contiguous()
    _, tfs, _ = T.posed_hand(nid, B, seed=3)
    td = tfs.to(DEV)
    W = skin_w(net, nid)
    pts = [hand_points(cano, P, seed=10 + b) for b in range(B)]
    x, n_edge = torch.stack([p[0] for p in pts]).contiguous(), pts[0][1]
    pose, keep = node_pose(td, None)
    xd = torch.full((B, P, 3), float("nan"), device=DEV)
    idx = torch.full((B, P, 15), -1, dtype=torch.int32, device=DEV)
    mask = torch.full((B, P), 7, dtype=torch.uint8, device=DEV)
    check(lib().hold_forward_warp(ctx.h, node.slot, B, P, ptr(x), C.byref(pose), ptr(xd), ptr(idx), ptr(mask), stream_ptr()))
    torch.cuda.synchronize()
    ctx.check()
    d, ib = T.brute_knn(x.reshape(-1, 3), cano)
    d, ib = d.reshape(B, P, 15), ib.reshape(B, P, 15)
    assert torch.equal(idx.long(), ib)
    assert torch.equal(mask.bool(), torch.sqrt(d[..., 0].clamp(max=4.0)) > 0.1)
    for b in range(B):
        _check_warp(f"{nid} forward B={B} P={P} frame {b}", xd[b], x[b], ib[b], cano, W, td[b], True, n_edge, stride)


def object_points(tf, P, seed, forward):
    """Canonical points (forward) or their images under tf (inverse), plus the origin and points 10x farther out."""
    g = torch.Generator().manual_seed(seed)
    p = 0.5 * torch.randn(P, 3, generator=g)
    p[:8] *= 10.0
    p[8:9] = 0.0
    if not forward:
        y = torch.nn.functional.pad(p.double(), (0, 1), value=1.0) @ tf.double().T
        p = (y[:, :3] / y[:, 3:]).float()
        p[9:10] = 0.0
    return p


@pytest.mark.parametrize("B,P,stride", [(10, 12545, 1), (5, 4 * 1024 * 1024 + 1, 4)])
def test_object_warps_against_float64(net, ctx, B, P, stride):
    from hold_b200.capi import check, lib, ptr, stream_ptr

    node = net.nodes["object"]
    tfs = T.object_tfs(B, seed=B)
    td = tfs.to(DEV)
    pose, keep = node_pose(td)
    for forward in (False, True):
        x = torch.stack([object_points(tfs[b], P, b, forward) for b in range(B)]).to(DEV).contiguous()
        out = torch.full((B, P, 3), float("nan"), device=DEV)
        fn = lib().hold_forward_warp if forward else lib().hold_inverse_warp
        check(fn(ctx.h, node.slot, B, P, ptr(x), C.byref(pose), ptr(out), None, None, stream_ptr()))
        torch.cuda.synchronize()
        ctx.check()
        sub = torch.cat([torch.arange(16, device=DEV), torch.arange(16, P, stride, device=DEV)])
        for b in range(B):
            r64 = T.rigid_ref(x[b, sub], td[b], torch.float64, forward)
            r32 = T.rigid_ref(x[b, sub], td[b], torch.float32, forward)
            wk, w32 = T.worst(out[b, sub], r64), T.worst(r32, r64)
            label = f"object {'forward' if forward else 'inverse'} frame {b} (scale {td[b, :3, :3].det().abs().item() ** (1 / 3):.3g}, s {td[b, 3, 3].item()})"
            print(f"{label}: kernel {wk:.2e}, float32 torch {w32:.2e}")
            assert wk <= T.F32_FACTOR * max(w32, T.F32_FLOOR), f"{label}: {wk:.2e} > {T.F32_FACTOR} x float32 torch's {w32:.2e}"
            assert wk <= T.REL_TOL, label


# ------------------------------------------------------------------------------------------------ 3. backward
def _bwd(ctx, node, x, pose, idx, g, want_gx, B=None, P=None):
    from hold_b200.capi import lib, ptr, stream_ptr

    B = x.shape[0] if B is None else B
    P = x.shape[1] if P is None else P
    hand = node.kind == "hand"
    g_tfs = torch.full((max(B, 1), 16, 4, 4) if hand else (max(B, 1), 4, 4), float("nan"), device=DEV)
    g_x = torch.full((max(B, 1), max(P, 1), 3), float("nan"), device=DEV) if want_gx else None
    p = lambda t: ptr(t) if t is not None and t.numel() > 0 else None
    rc = lib().hold_inverse_warp_bwd(ctx.h, node.slot, B, P, p(x), C.byref(pose), p(idx), p(g), ptr(g_tfs), ptr(g_x), stream_ptr())
    torch.cuda.synchronize()
    return rc, g_tfs, g_x


@pytest.mark.parametrize("P", [12544, 12545, 1])
@pytest.mark.parametrize("nid", ["right", "left", "object"])
def test_inverse_warp_bwd_against_float64(net, ctx, nid, P):
    from hold_b200 import ops

    B = 10
    node = net.nodes[nid]
    g = torch.Generator().manual_seed(P)
    if nid == "object":
        tfs = T.object_tfs(B, seed=P)
        verts = None
        x = torch.stack([object_points(tfs[b], P, b, False) for b in range(B)]).to(DEV).contiguous()
        idx = None
    else:
        verts, tfs, ties = T.posed_hand(nid, B, seed=P)
        # points on and near the hand's own vertices: the 16 vertices moved into the tie construction blend bones posed far
        # apart into a nearly singular transform (measured: g_x 5e-6 against float32 autograd's 6e-7 at such points, with the
        # kernel's adjugate inverse against torch's pivoted LU); the forward tests cover those points
        x = torch.stack([hand_points(verts[b][verts[b][:, 0] < ties[b][0] - 1.0], P, seed=b)[0] for b in range(B)]).contiguous()
    td = tfs.to(DEV)
    vd = verts.to(DEV) if verts is not None else None
    pose, keep = node_pose(td, vd)
    if nid != "object":
        _, idx, _ = ops.inverse_warp(node, x, pose, want_idx=True)
    gxc = torch.randn(B, P, 3, generator=g).to(DEV)
    rc, g_tfs, g_x = _bwd(ctx, node, x, pose, idx, gxc, True)
    assert rc == 0
    rc2, g_tfs2, _ = _bwd(ctx, node, x, pose, idx, gxc, False)
    rc3, g_tfs3, _ = _bwd(ctx, node, x, pose, idx, gxc, True)
    ctx.check()
    assert rc2 == 0 and rc3 == 0
    assert torch.equal(g_tfs, g_tfs2), "g_x = NULL changed g_tfs"
    assert torch.equal(g_tfs, g_tfs3), "two identical calls differ"
    assert (g_tfs[..., 3, :3] == 0).all(), "the constant row's gradient must be 0"
    wk = w32 = wm = xk = x32 = 0.0
    for b in range(B):
        w = None
        if nid != "object":
            w64, _ = T.skin_weights(x[b], idx[b].long(), vd[b], skin_w(net, nid), torch.float64)
            w32_, _ = T.skin_weights(x[b], idx[b].long(), vd[b], skin_w(net, nid), torch.float32)
            w = w64
        t64, gx64 = T.bwd_ref(x[b], gxc[b], td[b], w, torch.float64)
        t32, gx32 = T.bwd_ref(x[b], gxc[b], td[b], None if w is None else w32_, torch.float32)
        terms = T.bwd_terms(x[b], gxc[b], td[b], w)
        wk, w32 = max(wk, T.worst_entry(g_tfs[b], t64, terms)), max(w32, T.worst_entry(t32, t64, terms))
        wm = max(wm, T.worst_entry(g_tfs[b], t64, T.bwd_terms(x[b], gxc[b], td[b], w, magnitude=True)))
        xk, x32 = max(xk, T.worst(g_x[b], gx64)), max(x32, T.worst(gx32, gx64))
    print(f"{nid} B={B} P={P}: g_tfs vs sum|terms|: kernel {wk:.2e}, float32 autograd {w32:.2e}; vs the terms' magnitudes {wm:.2e}; "
          f"g_x: kernel {xk:.2e}, float32 {x32:.2e}")
    assert wk <= T.F32_FACTOR * max(w32, T.F32_FLOOR), f"g_tfs: {wk:.2e} > {T.F32_FACTOR} x float32 autograd's {w32:.2e}"
    # 1e-5 of the terms' magnitudes rather than of sum |term|: at P = 1 there is no sum and the one term is itself a difference
    # (measured on a point on a vertex: the kernel 3.3e-5 and float32 autograd 9.0e-4 of |term|)
    assert wm <= T.BWD_TOL, f"g_tfs: {wm:.2e}"
    assert xk <= T.F32_FACTOR * max(x32, T.F32_FLOOR), f"g_x: {xk:.2e} > {T.F32_FACTOR} x float32 autograd's {x32:.2e}"
    assert xk <= T.REL_TOL, f"g_x: {xk:.2e}"


@pytest.mark.parametrize("nid", ["right", "object"])
def test_inverse_warp_bwd_empty_sizes(net, ctx, nid):
    node = net.nodes[nid]
    if nid == "object":
        tfs, verts = T.object_tfs(3, 0), None
    else:
        verts, tfs, _ = T.posed_hand(nid, 3, 0)
    pose, keep = node_pose(tfs.to(DEV), None if verts is None else verts.to(DEV))
    empty = torch.empty(3, 0, 3, device=DEV)
    rc, g_tfs, _ = _bwd(ctx, node, empty, pose, None, empty, False)
    assert rc == 0 and (g_tfs == 0).all(), "P = 0 writes an all-zero g_tfs"
    rc, g_tfs, g_x = _bwd(ctx, node, empty, pose, None, empty, True, B=0, P=5)
    assert rc == 0 and g_tfs.isnan().all() and g_x.isnan().all(), "B = 0 is a no-op"
    ctx.check()


def test_warp_error_codes(net, ctx):
    from hold_b200 import capi
    from hold_b200.capi import NodeCfg, check, lib, ptr, stream_ptr

    HOLD_E_BADARG, HOLD_E_STATE = -1, -6
    verts, tfs, _ = T.posed_hand("right", 2, 0)
    pose, keep = node_pose(tfs.to(DEV), verts.to(DEV))
    x = torch.zeros(2, 5, 3, device=DEV)
    out = torch.empty(2, 5, 3, device=DEV)
    gt = torch.empty(2, 16, 4, 4, device=DEV)
    idx = torch.zeros(2, 5, 15, dtype=torch.int32, device=DEV)
    node = net.nodes["right"]
    assert lib().hold_inverse_warp_bwd(ctx.h, node.slot, 2, 5, ptr(x), C.byref(pose), None, ptr(x), ptr(gt), None, stream_ptr()) == HOLD_E_BADARG
    # a hand node that is configured but has no rig: a fresh context, so that no earlier rig is left in the slot
    c2 = capi.Context(0)
    try:
        cfg, s = NodeCfg(), node.sampler_cfg
        cfg.kind, cfg.class_id = capi.KIND_HAND, node.class_id
        cfg.n_samples_eval, cfg.n_samples, cfg.n_samples_extra = s["N_samples_eval"], s["N_samples"], s["N_samples_extra"]
        cfg.beta_iters, cfg.max_total_iters, cfg.mlp_mode = s["beta_iters"], s["max_total_iters"], capi.MLP_FP32
        cfg.eps, cfg.add_tiny, cfg.near, cfg.bounding_sphere, cfg.beta_min = s["eps"], s["add_tiny"], s["near"], 6.0, 1e-4
        check(lib().hold_node_configure(c2.h, 0, C.byref(cfg)))
        assert lib().hold_inverse_warp(c2.h, 0, 2, 5, ptr(x), C.byref(pose), ptr(out), None, None, stream_ptr()) == HOLD_E_STATE
        assert lib().hold_forward_warp(c2.h, 0, 2, 5, ptr(x), C.byref(pose), ptr(out), None, None, stream_ptr()) == HOLD_E_STATE
        assert lib().hold_inverse_warp_bwd(c2.h, 0, 2, 5, ptr(x), C.byref(pose), ptr(idx), ptr(x), ptr(gt), None, stream_ptr()) == HOLD_E_STATE
        assert lib().hold_inverse_warp_bwd(c2.h, 0, 2, 0, None, C.byref(pose), None, None, ptr(gt), None, stream_ptr()) == HOLD_E_STATE
        torch.cuda.synchronize()
        c2.check()
    finally:
        c2.close()
    ctx.check()
