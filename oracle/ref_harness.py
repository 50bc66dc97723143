"""Pin the oracle against the reference's OWN modules (needs a checkout of the reference, named by $HOLD_REFERENCE).

Imports `$HOLD_REFERENCE/code/src/...` unmodified behind harness-side shims (SURVEY §8c):
  * `torch.Tensor.cuda` / `nn.Module.cuda` -> identity (the reference hard-codes `.cuda()`, SURVEY D5)
  * stub modules `kaolin`, `trimesh`, `easydict`, `cv2`-free paths, `pytorch3d.ops.knn_points`
    stand-in (squared L2 + topk, the documented contract of pytorch3d 35badc08)
  * synthetic MANO-shaped struct fed to the vendored `lbs()` directly (MANO pickles are licensed)

Usage:
    python oracle/ref_harness.py check      # compare oracle vs reference, print max errors
    python oracle/ref_harness.py golden     # (re)write tests/golden/*.pt from the REFERENCE modules

Nothing at test or benchmark run time needs the reference checkout; only this script, oracle/build_ref_mise.py and the tests
that pin the oracle to it (skipped without $HOLD_REFERENCE) read it.
"""
from __future__ import annotations

import math
import os
import sys
import types

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("HOLD_REFERENCE", "")
sys.path.insert(0, REPO)


def install_shims():
    if not os.path.isdir(REF):
        raise RuntimeError("reference tree not present: set $HOLD_REFERENCE to a checkout of the reference")
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    class EasyDict(dict):
        def __init__(self, d=None, **kw):
            super().__init__()
            for k, v in {**(d or {}), **kw}.items():
                self[k] = v

        __getattr__ = dict.__getitem__
        __setattr__ = dict.__setitem__

    mod("easydict", EasyDict=EasyDict)
    k = mod("kaolin")
    k.ops = mod("kaolin.ops")
    k.ops.mesh = mod("kaolin.ops.mesh", index_vertices_by_faces=lambda *a, **kw: None)
    k.metrics = mod("kaolin.metrics")
    k.metrics.trianglemesh = mod("kaolin.metrics.trianglemesh")
    mod("trimesh")

    def knn_points(p1, p2, K=1, return_nn=False, **kw):
        d2 = ((p1[:, :, None, :] - p2[:, None, :, :]) ** 2).sum(-1)
        d, i = torch.topk(d2, K, dim=2, largest=False, sorted=True)
        nn = torch.gather(p2[:, None].expand(-1, p1.shape[1], -1, -1), 2, i[..., None].expand(-1, -1, -1, 3))
        return d, i, nn

    p3d = mod("pytorch3d")
    p3d.ops = mod("pytorch3d.ops", knn_points=knn_points)
    if "cv2" not in sys.modules:
        try:
            import cv2  # noqa: F401
        except Exception:
            mod("cv2")
    sys.path.insert(0, os.path.join(REF, "code"))
    sys.path.insert(0, REF)


def ns(**kw):
    return types.SimpleNamespace(**kw)


def build_ref_node(sc, nid):
    """Reference ImplicitNet / RenderingNet / density / sampler / deformer for one node of a SynthScene."""
    from src.engine.density import LaplaceDensity
    from src.engine.embedders import BarfEmbedder
    from src.engine.ray_sampler import ErrorBoundSampler
    from src.networks.shape_net import ImplicitNet
    from src.networks.texture_net import RenderingNet

    hand = nid in ("right", "left")
    specs = ns(pose_dim=45 if hand else 0, embedding="fourier")
    args = ns(barf_s=0, barf_e=10, no_barf=False)
    iopt = ns(d_in=3, d_out=1, feature_vector_size=256, dims=[256] * 8, init="geometry", bias=0.6,
              skip_in=[4], weight_norm=True, multires=6, cond="pose")
    ropt = ns(feature_vector_size=256, mode="pose", d_in=14 + (0 if hand else 32), d_out=3,
              dims=[256] * 4, weight_norm=True, multires_view=-1)
    inet = ImplicitNet(iopt, args, specs)
    rnet = RenderingNet(ropt, args, specs)
    if not hand:  # object nodes embed with BARF (obj/specs.py:10); eval() => plain Fourier (render.py:43-47)
        inet.embedder_obj = BarfEmbedder(3, 6, start=0, end=10, dev=torch.device("cpu"))
        inet.embedder_obj.eval()
    inet.load_state_dict(sc.sdf_state[nid], strict=False)  # embedder_obj.alpha_* buffers keep their init
    rsd = dict(sc.rgb_state[nid])
    if not hand:
        rsd["lin_pose.weight"] = rnet.lin_pose.weight.data
    rnet.load_state_dict(rsd, strict=True)
    dens = LaplaceDensity(params_init={"beta": float(sc.beta[nid])}, beta_min=1e-4)
    sampler = ErrorBoundSampler(sc.bounding_sphere, inverse_sphere_bg=True, N_samples_inverse_sphere=32, **sc.sampler)
    inet.eval(), rnet.eval()
    return inet, rnet, dens, sampler


class _FakeServer:
    pass


def build_ref_deformer(sc, nid, art):
    if nid in ("right", "left"):
        from src.model.mano.deformer import KNNDeformer

        d = KNNDeformer.__new__(KNNDeformer)
        d.max_dist, d.K = 0.1, 15
        d.verts = art[nid]["cano_verts"][None]
        d.skin_weights = art[nid]["skin_W"][None]
        return d
    from src.model.obj.deformer import ObjectDeformer

    return ObjectDeformer()


def ref_servers(sc):
    """Articulation from the reference's vendored lbs() / ObjectModel.forward."""
    from src.utils.external.lbs import lbs
    from src.model.obj.object_model import ObjectModel

    art = {}
    B = sc.B
    scale = torch.full((B,), float(sc.scene_scale))
    for nid in sc.node_ids:
        p = sc.params[nid]
        if nid in ("right", "left"):
            m = sc.mano[nid]
            pose_mean = torch.cat([torch.zeros(3), m["hands_mean"]])

            def server(scene_scale, transl, thetas, betas, tfs_c_inv=None):
                # GenericServer.forward (mano/server.py:62-99) with MANO.forward's pose_mean add
                verts, joints, T_w, W, T, v_posed = lbs(betas, thetas + pose_mean, m["v_template"], m["shapedirs"],
                                                        m["posedirs"], m["J_regressor"], m["parents"], m["lbs_weights"])
                joints = torch.cat([joints, verts[:, m["tip_ids"]]], 1)
                s = scene_scale.view(-1, 1, 1)
                t = transl.view(-1, 1, 3)
                out = {"verts": verts * s + t * s, "jnts": joints * s + t * s}
                tf = T.clone()
                tf[:, :, :3, :] = tf[:, :, :3, :] * s.view(-1, 1, 1, 1)
                tf[:, :, :3, 3] = tf[:, :, :3, 3] + t * s
                if tfs_c_inv is not None:
                    tf = torch.einsum("bnij,njk->bnik", tf, tfs_c_inv)
                out["tfs"], out["v_posed"] = tf, v_posed
                return out

            cano = server(torch.ones(1), torch.zeros(1, 3), torch.cat([torch.zeros(3), -m["hands_mean"]])[None],
                          sc.betas[nid][None])
            tfs_c_inv = cano["tfs"][0].inverse()
            full_pose = torch.cat([p["global_orient"], p["pose"]], 1)
            out = server(scale, p["transl"], full_pose, sc.betas[nid][None].repeat(B, 1), tfs_c_inv)
            art[nid] = dict(kind="hand", tfs=out["tfs"], verts=out["verts"], jnts=out["jnts"], v_posed=out["v_posed"],
                            cano_verts=cano["verts"][0], skin_W=m["lbs_weights"], pose_cond=full_pose[:, 3:] / math.pi)
        else:
            om = ObjectModel.__new__(ObjectModel)
            torch.nn.Module.__init__(om)
            om.register_buffer("obj_scale", torch.FloatTensor([1.0]))
            om.register_buffer("v3d_cano", sc.obj_pts_cano)
            om.register_buffer("norm_mat", torch.eye(4))
            om.register_buffer("denorm_mat", torch.eye(4))
            o = om.forward(p["global_orient"], p["transl"], scale)
            art[nid] = dict(kind="object", tfs=o["T"], verts=o["vertices"])
    return art


def ref_render_scene(sc, ray_ids=None, chunk=None):
    """The reference's own code path: get_camera_params -> ErrorBoundSampler.get_z_vals(sdf_func_with_deformer)
    -> sdf_func_with_deformer -> render_color -> density -> merge_factors -> volumetric_render."""
    import src.engine.volsdf_utils as vu
    from src.datasets.utils import get_camera_params
    from src.engine.rendering import render_color
    from src.hold.hold_utils import merge_factors, volumetric_render

    CLASS_ID = {"object": 1, "right": 2, "left": 3}
    art = ref_servers(sc)
    dirs, cam = get_camera_params(sc.uv, sc.extrinsics, sc.intrinsics)
    P = dirs.shape[1]
    dirs = dirs.reshape(-1, 3)
    cam = cam.unsqueeze(1).repeat(1, P, 1).reshape(-1, 3)
    assert sc.B == 1 or ray_ids is None, "harness renders whole frames when B > 1"
    if ray_ids is None:
        ray_ids = torch.arange(dirs.shape[0])
    chunk = chunk or ray_ids.numel()
    nets = {nid: build_ref_node(sc, nid) for nid in sc.node_ids}
    defs = {nid: build_ref_deformer(sc, nid, art) for nid in sc.node_ids}
    outs = []
    for s in range(0, ray_ids.numel(), chunk):
        ids = ray_ids[s:s + chunk]
        fl = []
        for nid in sc.node_ids:
            inet, rnet, dens, sampler = nets[nid]
            a = art[nid]
            hand = a["kind"] == "hand"
            cond = {"pose": a["pose_cond"]} if hand else {"pose": torch.zeros(sc.B, 0)}
            info = {"cond": cond, "tfs": a["tfs"]}
            if hand:
                info["verts"] = a["verts"]
            d, c = dirs[ids], cam[ids]
            z = sampler.get_z_vals(vu.sdf_func_with_deformer, defs[nid], inet, d, c, dens, False, info)
            inet.eval()
            S = z.shape[1]
            pts = c.unsqueeze(1) + z.unsqueeze(2) * d.unsqueeze(1)
            sdf, x_c, feat = vu.sdf_func_with_deformer(defs[nid], inet, False, pts.reshape(-1, 3), info)
            tfs4 = a["tfs"] if hand else a["tfs"][:, None]
            color, normal, sem = render_color(defs[nid], inet, rnet, d, cond, tfs4 if hand else a["tfs"][:, None],
                                              x_c, feat, False, S, CLASS_ID[nid],
                                              None if hand else sc.time_code)
            density = dens(sdf).view(-1, S, 1)
            fl.append({"color": color.detach(), "normal": normal.detach(), "density": density.detach(),
                       "semantics": sem, "z_vals": z, "sdf": sdf.detach().reshape(-1, S),
                       "canonical_pts": x_c.detach().reshape(-1, S, 3)})
        core = [{k: f[k] for k in ("color", "normal", "density", "semantics", "z_vals")} for f in fl]
        comp = merge_factors(core, check=True)
        r = {"comp": dict(volumetric_render(comp, False))}
        r["comp"]["z_vals"] = comp["z_vals"]
        for k, f in enumerate(core):
            f = dict(f)
            f["z_max"] = f["z_vals"][:, -1]
            r[k] = dict(volumetric_render(f, False))
        outs.append(dict(nodes=fl, render=r))
    return outs, art


def _cmp(name, a, b, tol, w=None, tol_max=None):
    """Comparison relative to the tensor's scale.

    The pipeline is ill-conditioned *end to end*: the sampler's inverse-CDF has a flat PDF behind the
    surface and a discontinuous `denom < 1e-5` branch (ray_sampler.py:304-305), so a 1e-6 change of one SDF
    value (e.g. a different GEMM summation order) moves a few samples by ~1e-3 and a few pixels by ~3e-4.
    End-to-end tensors are therefore held to: >= 97 % of entries within `tol`, and every entry (every entry with
    reference weight > 1e-4 for per-sample tensors) within `tol_max` (default 30 tol).  Stage-wise parity
    (same inputs per stage) is what is held to `tol` everywhere -- see tests/."""
    a, b = a.detach().float(), b.detach().float()
    d = (a - b).abs()
    scale = max(b.abs().max().item(), 1.0)
    tol_max = tol_max or 30 * tol
    frac = (d <= tol * scale).float().mean().item()
    if w is not None:
        m = (w > 1e-4)
        while m.dim() < d.dim():
            m = m.unsqueeze(-1)
        d = d * m
    err = d.max().item()
    ok = err <= tol_max * scale and frac >= 0.97
    print(f"  {name:28s} max|d| {err:.3e}  within-tol {frac:.4f}  (scale {scale:.3e})  {'ok' if ok else 'MISMATCH'}")
    return ok


def check():
    from hold_b200 import synth
    from oracle import hold_oracle as O

    ok = True
    for cfgname, kw, beta in [("n2 beta.1", dict(H=12, W=12, S=128, nodes=("right", "object")), 0.1),
                              ("n3 beta.03 S32", dict(H=8, W=8, S=32, nodes=("right", "left", "object")), 0.03),
                              ("n2 B2", dict(H=6, W=6, S=128, nodes=("right", "object"), B=2), 0.05)]:
        sc = synth.make_scene(**kw)
        for nid in sc.node_ids:
            sc.beta[nid] = torch.tensor(beta)
        print(f"[{cfgname}]")
        ro, ra = ref_render_scene(sc)
        oo, oa = O.render_scene(sc)
        for nid in sc.node_ids:
            for k in ("tfs", "verts"):
                ok &= _cmp(f"{nid}.{k}", oa[nid][k], ra[nid][k], 1e-5)
            if nid != "object":
                ok &= _cmp(f"{nid}.jnts", oa[nid]["jnts"], ra[nid]["jnts"], 1e-5)
        for k, nid in enumerate(sc.node_ids):
            wref = ro[0]["render"][k]["fg_weights"]
            for key in ("z_vals", "sdf", "canonical_pts", "normal", "color", "density"):
                ok &= _cmp(f"{nid}.{key}", oo[0]["nodes"][k][key], ro[0]["nodes"][k][key], 1e-4, wref)
            for key in ("fg_rgb", "mask_prob", "depth", "normal", "bg_weights"):
                ok &= _cmp(f"{nid}.render.{key}", oo[0]["render"][k][key], ro[0]["render"][k][key], 1e-4)
        for key in ("fg_rgb", "mask_prob", "depth", "normal", "fg_semantics", "bg_weights"):
            ok &= _cmp(f"comp.{key}", oo[0]["render"]["comp"][key], ro[0]["render"]["comp"][key], 1e-4)
    ok &= check_background()
    ok &= check_pose_grads()
    print("ORACLE == REFERENCE" if ok else "ORACLE != REFERENCE")
    return ok


def check_pose_grads():
    """Gradients of the pose servers: torch.autograd through the REFERENCE's lbs() / ObjectModel.forward against
    torch.autograd through the oracle's restatement (the oracle for hold_mano_lbs_bwd / hold_object_tf_bwd)."""
    from hold_b200 import synth
    from oracle import hold_oracle as O
    from src.model.obj.object_model import ObjectModel
    from src.utils.external.lbs import lbs

    sc = synth.make_scene(H=4, W=4, S=32, nodes=("right", "object"), B=2, seed=11)
    m = sc.mano["right"]
    p = sc.params["right"]
    g = torch.Generator().manual_seed(1)
    gv, gj = torch.randn(2, 778, 3, generator=g), torch.randn(2, 16, 3, generator=g)
    pose_mean = torch.cat([torch.zeros(3), m["hands_mean"]])
    leaves = lambda: [t.clone().requires_grad_() for t in (sc.betas["right"][None].repeat(2, 1), torch.cat([p["global_orient"], p["pose"]], 1), p["transl"])]
    be, th, tr = leaves()
    verts, joints, *_ = lbs(be, th + pose_mean, m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["parents"], m["lbs_weights"])
    s = float(sc.scene_scale)
    ref = torch.autograd.grad((((verts + tr[:, None]) * s) * gv).sum() + (((joints + tr[:, None]) * s) * gj).sum(), (be, th, tr))
    be, th, tr = leaves()
    out = O.mano_server(m, torch.full((2,), s), tr, th, be)
    got = torch.autograd.grad((out["verts"] * gv).sum() + (out["jnts"][:, :16] * gj).sum(), (be, th, tr))
    print("[pose-server gradients]")
    ok = True
    for name, a, b in zip(("hand.g_betas", "hand.g_pose", "hand.g_transl"), got, ref):
        ok &= _cmp(name, a, b, 1e-5)
    po = sc.params["object"]
    om = ObjectModel.__new__(ObjectModel)
    torch.nn.Module.__init__(om)
    om.register_buffer("obj_scale", torch.FloatTensor([1.0]))
    om.register_buffer("v3d_cano", sc.obj_pts_cano)
    om.register_buffer("norm_mat", torch.eye(4))
    om.register_buffer("denorm_mat", torch.eye(4))
    gvo = torch.randn(2, sc.obj_pts_cano.shape[0], 3, generator=g)
    r1, t1, s1 = po["global_orient"].clone().requires_grad_(), po["transl"].clone().requires_grad_(), torch.full((2,), s).requires_grad_()
    o = om.forward(r1, t1, s1)
    ref = torch.autograd.grad((o["vertices"] * gvo).sum(), (r1, t1, s1))
    r2, t2, s2 = po["global_orient"].clone().requires_grad_(), po["transl"].clone().requires_grad_(), torch.full((2,), s).requires_grad_()
    _, v = O.object_server(r2, t2, s2, 1.0, torch.eye(4), sc.obj_pts_cano)
    got = torch.autograd.grad((v * gvo).sum(), (r2, t2, s2))
    for name, a, b in zip(("object.g_rot", "object.g_trans", "object.g_scene_scale"), got, ref):
        ok &= _cmp(name, a, b, 1e-5)
    return ok


def _bg_case():
    """A background case: seeded inputs + the REFERENCE Background class's outputs (model/renderables/background.py)."""
    from hold_b200 import synth
    from oracle.hold_oracle import camera_rays
    from src.model.renderables.background import Background

    opt = ns(bg_implicit_network=ns(feature_vector_size=256, d_in=4, d_out=1, dims=[256] * 8, init="none", bias=0.0, skip_in=[4],
                                    weight_norm=False, multires=10, cond="frame", dim_frame_encoding=32),
             bg_rendering_network=ns(feature_vector_size=256, mode="nerf_frame_encoding", d_in=3, d_out=3, dims=[128],
                                     weight_norm=False, multires_view=4, dim_frame_encoding=32))
    bg = Background(opt, ns(barf_s=0, barf_e=10, no_barf=False), 3, 6.0)
    sdf_sd, rgb_sd = synth.make_bg_state(0)
    bg.bg_implicit_network.load_state_dict(sdf_sd, strict=False)
    bg.bg_rendering_network.load_state_dict(rgb_sd, strict=False)
    bg.eval()
    sc = synth.make_scene(H=8, W=8, S=32, B=2)
    sc.intrinsics[:, 0, 2] += 0.37   # a ray through the sphere centre is a 0/0 in depth2pts_outside (background.py:118-119)
    sc.intrinsics[:, 1, 2] -= 0.21
    dirs, cam = camera_rays(sc.uv, sc.extrinsics, sc.intrinsics)
    P = dirs.shape[1]
    dirs, cam = dirs.reshape(-1, 3), cam.unsqueeze(1).repeat(1, P, 1).reshape(-1, 3)
    bgw = torch.rand(dirs.shape[0], generator=torch.Generator().manual_seed(0))
    idx = torch.tensor([2, 0])
    zbg = bg.inverse_sphere_sampler.inverse_sample(dirs, cam, False, 6.0)
    with torch.no_grad():
        ref = bg(bgw, dirs, cam, zbg, idx)
    inp = dict(bg_weights=bgw, ray_dirs=dirs, cam_loc=cam, frame_code=bg.frame_latent_encoder.weight.data[idx].clone(),
               frame_of_ray=torch.arange(2).repeat_interleave(P), r_sphere=6.0, bg_state_seed=0)
    out = dict(bg_rgb=ref["bg_rgb"], bg_rgb_only=ref["bg_rgb_only"], bg_semantics=ref["bg_semantics"], bg_z_vals=zbg)
    return inp, out, (sdf_sd, rgb_sd)


def check_background():
    """oracle.background vs the reference's Background class."""
    from oracle import hold_oracle as O

    inp, ref, (sdf_sd, rgb_sd) = _bg_case()
    o = O.background(inp["bg_weights"], inp["ray_dirs"], inp["cam_loc"], inp["frame_code"], inp["frame_of_ray"], sdf_sd, rgb_sd, 6.0)
    print("[background]")
    ok = _cmp("bg_rgb", o[0], ref["bg_rgb"], 1e-6) & _cmp("bg_rgb_only", o[1], ref["bg_rgb_only"], 1e-6)
    ok &= _cmp("bg_semantics", o[2], ref["bg_semantics"], 1e-6) & _cmp("bg_z_vals", o[3], ref["bg_z_vals"], 1e-7)
    return ok


def golden_background():
    """tests/golden/background/*.pt: inputs + the reference Background class's outputs."""
    inp, ref, _ = _bg_case()
    d = os.path.join(REPO, "tests", "golden", "background")
    os.makedirs(d, exist_ok=True)
    path = os.path.join(d, "bg_8x8_B2.pt")
    torch.save({"in": {k: (v.clone() if torch.is_tensor(v) else v) for k, v in inp.items()},
                "out": {k: v.detach().clone() for k, v in ref.items()}}, path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


def _loss_case(seed, step, with_targets):
    """A synthetic training output dict + batch for hold/loss.py (the keys HOLDNet.forward writes in training mode)."""
    g = torch.Generator().manual_seed(seed)
    B, P = 2, 24
    R = B * P
    r = lambda *sh: torch.rand(*sh, generator=g)
    mo = {"rgb": r(R, 3), "semantics": r(R, 4), "step": step, "epoch": 3}
    mask = torch.tensor([0, 50, 150, 250, 24, 99, 101, 201])[torch.randint(0, 8, (R,), generator=g)]
    batch = {"idx": torch.arange(B), "gt.rgb": r(B, P, 3), "gt.mask": mask.reshape(B, P), "im_path": [["unused"]]}
    for nid in ("right", "object"):
        mo[f"{nid}.mask_prob"] = r(R, 1)
        if with_targets:
            mo[f"{nid}.index_off_surface"] = r(R) > 0.6
            mo[f"{nid}.grad_theta"] = torch.randn(B, 307, 3, generator=g) * (12.0 if nid == "right" else 1.0)
    if with_targets:
        mo["right.pts2mano_sdf_cano"] = torch.randn(B, 307, generator=g) * 0.02
        mo["right.pred_sdf"] = torch.randn(B, 307, generator=g) * 0.02
    return batch, mo


def golden_loss():
    """tests/golden/loss/*.pt: synthetic training outputs + the loss dict of the REFERENCE's hold/loss.py Loss module."""
    from src.hold.loss import Loss
    from common.xdict import xdict

    d = os.path.join(REPO, "tests", "golden", "loss")
    os.makedirs(d, exist_ok=True)
    for name, (seed, step, wt) in {"early_no_targets": (1, 0, False), "mid_targets": (2, 12000, True), "late_targets": (3, 45000, True)}.items():
        batch, mo = _loss_case(seed, step, wt)
        L = Loss(ns())
        L.im_w, L.im_h = 64, 64            # skips the PIL read of the frame's image file
        ld = L(batch, xdict(mo))
        path = os.path.join(d, name + ".pt")
        torch.save({"batch": batch, "outputs": mo, "loss": {k: torch.as_tensor(v).detach().clone() for k, v in ld.items()}}, path)
        print("wrote", path, {k: float(v) for k, v in ld.items()})


def golden_barf():
    """tests/golden/barf/barf_weights.pt: BARF weights of the REFERENCE's BarfEmbedder (engine/embedders.py:53-126) along its schedule."""
    from src.engine.embedders import BarfEmbedder

    rec = {}
    for start, end in ((5, 25), (1000, 10000)):
        e = BarfEmbedder(3, 6, start, end, "cpu")
        its = sorted({0, start, start + 1, (start + end) // 2, end - 2, end - 1, end + 50})
        w = {}
        for it in range(max(its) + 1):
            if it in its:
                w[it] = e.barf_weights.clone()
            e.step()
        rec[(start, end)] = w
    path = os.path.join(REPO, "tests", "golden", "barf", "barf_weights.pt")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    torch.save(rec, path)
    print("wrote", path)


def golden():
    """tests/golden/*.pt: inputs are regenerated from the seed; outputs come from the REFERENCE modules."""
    from hold_b200 import synth

    os.makedirs(os.path.join(REPO, "tests", "golden"), exist_ok=True)
    cases = {
        "c1_64x64_S32_n2": (dict(H=64, W=64, S=32, nodes=("right", "object"), seed=0), 0.1, 256),
        "s128_n2_beta03": (dict(H=64, W=64, S=128, nodes=("right", "object"), seed=1), 0.03, 128),
        "s128_n3_beta05": (dict(H=64, W=64, S=128, nodes=("right", "left", "object"), seed=2), 0.05, 96),
    }
    for name, (kw, beta, nrays) in cases.items():
        sc = synth.make_scene(**kw)
        for nid in sc.node_ids:
            sc.beta[nid] = torch.tensor(beta)
        g = torch.Generator().manual_seed(7)
        ids = torch.sort(torch.randperm(kw["H"] * kw["W"], generator=g)[:nrays]).values
        ro, ra = ref_render_scene(sc, ray_ids=ids)
        rec = {"scene_kwargs": kw, "beta": beta, "ray_ids": ids, "nodes": {}, "render": {}, "art": {}}
        for k, nid in enumerate(sc.node_ids):
            n = ro[0]["nodes"][k]
            rec["nodes"][nid] = {key: n[key].to(torch.float32).clone() for key in
                                 ("z_vals", "sdf", "canonical_pts", "normal", "color", "density")}
            rec["render"][nid] = {key: ro[0]["render"][k][key].clone() for key in
                                  ("fg_rgb", "mask_prob", "depth", "normal", "bg_weights")}
            rec["art"][nid] = {key: ra[nid][key].clone() for key in ("tfs", "verts")}
            if nid != "object":
                rec["art"][nid]["jnts"] = ra[nid]["jnts"].clone()
        rec["render"]["comp"] = {key: ro[0]["render"]["comp"][key].clone() for key in
                                 ("fg_rgb", "mask_prob", "depth", "normal", "fg_semantics", "bg_weights", "z_vals")}
        path = os.path.join(REPO, "tests", "golden", name + ".pt")
        torch.save(rec, path)
        print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    install_shims()
    torch.manual_seed(0)
    cmd = sys.argv[1] if len(sys.argv) > 1 else "check"
    if cmd == "check":
        sys.exit(0 if check() else 1)
    elif cmd == "golden":
        golden()
    elif cmd == "golden_background":
        golden_background()
    elif cmd == "golden_loss":
        golden_loss()
    elif cmd == "golden_barf":
        golden_barf()
