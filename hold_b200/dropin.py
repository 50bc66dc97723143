"""Reference-signature adaptors (SURVEY.md §8b, "Python surface to preserve"): classes whose methods take exactly the
arguments the reference's call sites pass, so that `hold_net.py:64-67`, `mano_node.py:100-109`, `node.py:57-67` and
`volsdf_utils.py:150-169` can call into libhold_b200.so without being edited beyond the constructor that builds them.

    reference call site                                                        adaptor here
    ray_sampler.get_z_vals(sdf_fn, deformer, implicit_network, ray_dirs,        ErrorBoundSampler.get_z_vals  (same 8 arguments)
        cam_loc, density_fn, is_training, deform_info)   ray_sampler.py:128-138
    deformer.forward(x, tfs, return_weights, inverse, verts)  mano/deformer.py:34   MANODeformer.forward / ObjectDeformer.forward
    deformer.forward_skinning(xc, cond, tfs)            mano/deformer.py:70      .forward_skinning
    implicit_network(x, cond)                           shape_net.py:84          hold_b200.model.ImplicitNet.forward(input, cond, current_epoch=None)
    rendering_network(points, normals, view_dirs, body_pose, feature_vectors)    RenderingNetAdaptor.forward
                                                        texture_net.py:46-53
    sdf_func_with_deformer(deformer, sdf_fn, training, x, deform_info)           sdf_func_with_deformer (module function)
                                                        volsdf_utils.py:150-169

Each adaptor is bound to a hold_b200.model.Node (the ctx slot that holds the packed weights and the rig); the objects the
reference passes along (sdf_fn, deformer, density_fn) are accepted and used only for what cannot be known otherwise (beta from
density_fn).  tests/test_cpu_dropin.py compares these signatures with `inspect.signature` of the reference's classes (where
$HOLD_REFERENCE names a checkout of the reference); tests/test_gpu_dropin.py runs them against the oracle."""
from __future__ import annotations

import ctypes as C

import torch

from . import capi
from .capi import NodePose, check, lib, ptr, stream_ptr
from .model import sampler_rand


def _node_of(obj):
    node = getattr(obj, "_node", None) or getattr(obj, "node", None)
    if node is None:
        raise TypeError("this object is not bound to a hold_b200 Node (expected the mirror's ImplicitNet / an adaptor)")
    return node


def _pose_from_deform_info(node, deform_info, density_fn=None):
    """hold_node_pose from the reference's deform_info dict {"cond", "tfs", "verts"} (mano_node.py:94-98 / object_node.py:78-82)."""
    pose, keep = NodePose(), []
    tfs = deform_info["tfs"].detach().float()
    if node.kind == "hand":
        tfs = tfs.reshape(-1, 16, 4, 4).contiguous()
        verts = deform_info["verts"].detach().float().contiguous()
        pose.tfs, pose.posed_verts = tfs.data_ptr(), verts.data_ptr()
        cond = deform_info.get("cond", {})
        pc = cond.get("pose") if isinstance(cond, dict) else None
        if pc is not None:
            pc = pc.detach().float().contiguous()
            pose.pose_cond = pc.data_ptr()
            keep.append(pc)
        keep += [tfs, verts]
    else:
        tfs = tfs.reshape(-1, 4, 4).contiguous()
        pose.tfs = tfs.data_ptr()
        keep.append(tfs)
        tc = deform_info.get("time_code")
        if tc is not None:
            tc = tc.detach().float().contiguous()
            pose.time_code = tc.data_ptr()
            keep.append(tc)
    if node.barf_weights is not None:
        pose.embed_w = node.barf_weights.data_ptr()
    beta_src = density_fn if density_fn is not None else node.density
    beta = beta_src.beta.detach().float().reshape(1).contiguous()
    pose.beta_param = beta.data_ptr()
    keep.append(beta)
    return pose, keep, tfs.shape[0]


class UniformInverseSphereSampler:
    """UniformSampler(1.0, 0.0, 32, False, far=1.0).inverse_sample (engine/ray_sampler.py:82-85) — the `inverse_sphere_sampler`
    attribute HOLDNet.forward_fg reads (hold_net.py:91-96).  32 fixed numbers; hold_background recomputes them on the device."""

    def __init__(self, n=32):
        self.N_samples = n

    def inverse_sample(self, ray_dirs, cam_loc, is_training, sdf_bounding_sphere):
        z = torch.linspace(0.0, 1.0, self.N_samples, device=ray_dirs.device).unsqueeze(0).repeat(ray_dirs.shape[0], 1)
        assert not is_training, "training-mode background samples: hold_b200.train.background_forward_train(..., jitter=...)"
        return z * (1.0 / sdf_bounding_sphere)


class ErrorBoundSampler:
    """engine/ray_sampler.py:88-352, same constructor and get_z_vals signature."""

    def __init__(self, scene_bounding_sphere, near, N_samples, N_samples_eval, N_samples_extra, eps, beta_iters, max_total_iters,
                 inverse_sphere_bg=False, N_samples_inverse_sphere=0, add_tiny=0.0):
        self.scene_bounding_sphere, self.near = scene_bounding_sphere, near
        self.N_samples, self.N_samples_eval, self.N_samples_extra = N_samples, N_samples_eval, N_samples_extra
        self.eps, self.beta_iters, self.max_total_iters, self.add_tiny = eps, beta_iters, max_total_iters, add_tiny
        self.inverse_sphere_bg = inverse_sphere_bg
        if inverse_sphere_bg:
            self.inverse_sphere_sampler = UniformInverseSphereSampler(32)

    def cfg(self):
        return dict(N_samples=self.N_samples, N_samples_eval=self.N_samples_eval, N_samples_extra=self.N_samples_extra, eps=self.eps,
                    beta_iters=self.beta_iters, max_total_iters=self.max_total_iters, add_tiny=self.add_tiny, near=self.near)

    def get_z_vals(self, sdf_fn, deformer, implicit_network, ray_dirs, cam_loc, density_fn, is_training, deform_info):
        node = _node_of(implicit_network)
        mine, theirs = self.cfg(), {k: node.sampler_cfg[k] for k in self.cfg()}
        if mine != theirs or abs(node.bounding_sphere - self.scene_bounding_sphere) > 0:
            node.sampler_cfg.update(mine)
            node.bounding_sphere = self.scene_bounding_sphere
            node.configure()   # hold_node_configure with this sampler's constants
            node.S = self.N_samples + self.N_samples_extra + 2
        pose, keep, B = _pose_from_deform_info(node, deform_info, density_fn)
        ray_dirs, cam_loc = ray_dirs.detach().float().contiguous(), cam_loc.detach().float().contiguous()
        R = ray_dirs.shape[0]
        z = torch.empty(R, node.S, device=ray_dirs.device)
        rnd = None
        if is_training:   # randomness is an input of the library: generated here with torch, as the reference does (:70-78,:292,:328)
            draw = sampler_rand(R, mine, ray_dirs.device)
            rnd = capi.SamplerRand()
            rnd.jitter, rnd.u, rnd.extra_idx = draw["jitter"].data_ptr(), draw["u"].data_ptr(), draw["extra_idx"].data_ptr()
            keep += list(draw.values())
        self.last_iters = torch.zeros(1, dtype=torch.int32, device=ray_dirs.device)
        check(lib().hold_sample(node.ctx.h, node.slot, R, B, ptr(cam_loc), ptr(ray_dirs), C.byref(pose),
                                C.byref(rnd) if rnd is not None else None, ptr(z), ptr(self.last_iters), stream_ptr()))
        return z


class _Deformer:
    def __init__(self, node):
        self.node = node

    def _pose(self, tfs, verts=None):
        info = {"tfs": tfs, "cond": {}}
        if verts is not None:
            info["verts"] = verts
        elif self.node.kind == "hand":
            info["verts"] = self.node.server.verts_c.expand(tfs.shape[0], -1, -1)
        return _pose_from_deform_info(self.node, info)

    def forward(self, x, tfs, return_weights=True, inverse=False, verts=None):
        """model/mano/deformer.py:34-68 / model/obj/deformer.py:10-38: x [B,P,3] -> (x_transformed, outlier_mask).
        `return_weights=True` (the reference's query_weights path) is not part of the hot path and is not served."""
        assert x.dim() == 3, "x is [num_images, num_points, 3]"
        if return_weights:
            raise NotImplementedError("skinning-weight queries are not on the rendering path (deformer.py:62-63)")
        if x.shape[0] == 0:
            return x
        node = self.node
        B, P, _ = x.shape
        pose, keep, _ = self._pose(tfs, verts)
        xi = x.detach().float().contiguous()
        out = torch.empty(B, P, 3, device=x.device)
        mask = torch.zeros(B, P, dtype=torch.uint8, device=x.device)
        hand = node.kind == "hand"
        fn = lib().hold_inverse_warp if inverse else lib().hold_forward_warp
        check(fn(node.ctx.h, node.slot, B, P, ptr(xi), C.byref(pose), ptr(out), None, ptr(mask) if hand else None, stream_ptr()))
        return out, mask.bool()

    def forward_skinning(self, xc, cond, tfs):
        """model/mano/deformer.py:70-82 / model/obj/deformer.py:40-46: canonical -> deformed."""
        return self.forward(xc, tfs, return_weights=False, inverse=False, verts=None)[0]


class MANODeformer(_Deformer):
    """model/mano/deformer.py:108-142 (KNNDeformer with K=15 over the node's MANO rig)."""


class ObjectDeformer(_Deformer):
    """model/obj/deformer.py:5-46: rigid transform; the reference ignores `return_weights` here (default None) and returns
    outlier_mask None unless deformed-space vertices are passed (K = 1 KNN, test-time only, not on the rendering path)."""

    def forward(self, x, tfs, return_weights=None, inverse=False, verts=None):
        if verts is not None and inverse:
            raise NotImplementedError("the K=1 outlier test against object vertices is not on the rendering path (obj/deformer.py:33-38)")
        x_tf, _ = super().forward(x, tfs.view(-1, 4, 4), return_weights=False, inverse=inverse, verts=None)
        return x_tf, None


class RenderingNetAdaptor:
    """rendering_network(points, normals, view_dirs, body_pose, feature_vectors) -> [P,3] (texture_net.py:46-101, mode 'pose')."""

    def __init__(self, node):
        self.node = node

    def forward(self, points, normals, view_dirs, body_pose, feature_vectors, frame_latent_code=None):
        node = self.node
        P = points.reshape(-1, 3).shape[0]
        dev = points.device
        f = lambda t: t.detach().float().contiguous()
        feat = feature_vectors.reshape(P, -1)
        if node.kind == "hand":
            B = body_pose.shape[0]
            pc, tc = f(body_pose), None
        else:
            # the reference concatenates the per-frame time code to every point's features (volsdf_utils.py:133-141)
            assert feat.shape[1] == 256 + 32, "object features are [feature(256) | time_code(32)]"
            B = max(1, int(body_pose.shape[0])) if body_pose is not None else 1
            tc = f(feat.view(B, P // B, -1)[:, 0, 256:])
            pc = None
        rgb = torch.empty(P, 3, device=dev)
        check(lib().hold_rgb_eval(node.ctx.h, node.slot, B, P, ptr(f(points.reshape(P, 3))), ptr(f(normals.reshape(P, 3))), ptr(pc),
                                  ptr(f(feat[:, :256])), ptr(tc), ptr(rgb), stream_ptr()))
        return rgb

    __call__ = forward


def sdf_func_with_deformer(deformer, sdf_fn, training, x, deform_info):
    """engine/volsdf_utils.py:150-169: -> (sdf [B,P,1], x_c [B,P,3], feature [B,P,256])."""
    tfs = deform_info["tfs"]
    num_images = tfs.shape[0]
    x = x.view(num_images, -1, 3)
    x_c, _ = deformer.forward(x, tfs, return_weights=False, inverse=True, verts=deform_info.get("verts"))
    out = sdf_fn(x_c, deform_info["cond"])
    return out[:, :, 0:1], x_c, out[:, :, 1:]


# ------------------------------------------------------------------------------------------------ constructors with the reference's signatures
# The reference builds its scene from (args, opt): `opt` is the `model:` block of confs/general.yaml, `args` the parsed command line
# (args.n_images, args.case).  The classes below take exactly those positional arguments and hand back hold_b200.model objects.
# What the reference reads from disk inside its constructors (the MANO model file, data/<case>/build/data.npy) is passed as
# keyword-only extras, because the library reads no files: `mano` (dict of MANO arrays, see hold_b200.synth.make_mano / the keys
# MANOServer.m uses), `obj_pts` / `obj_scale` / `norm_mat` (entities.object of data.npy).
_SUPPORTED = {
    "implicit_network": dict(feature_vector_size=256, d_in=3, d_out=1, dims=[256] * 8, skip_in=[4], weight_norm=True, multires=6),
    "rendering_network": dict(feature_vector_size=256, mode="pose", d_out=3, dims=[256] * 4, weight_norm=True, multires_view=-1),
    "bg_implicit_network": dict(feature_vector_size=256, d_in=4, d_out=1, dims=[256] * 8, skip_in=[4], weight_norm=False, multires=10,
                                dim_frame_encoding=32),
    "bg_rendering_network": dict(feature_vector_size=256, mode="nerf_frame_encoding", d_in=3, d_out=3, dims=[128], weight_norm=False,
                                 multires_view=4, dim_frame_encoding=32),
}


def _get(o, k):
    return o[k] if isinstance(o, dict) else getattr(o, k)


def _check_opt(opt, block):
    """The kernels are specialised to the architecture of confs/general.yaml; anything else must fail here, loudly."""
    o = _get(opt, block)
    for k, want in _SUPPORTED[block].items():
        have = _get(o, k)
        have = list(have) if isinstance(want, list) else have
        if have != want:
            raise ValueError(f"hold_b200 kernels are built for model.{block}.{k} = {want!r} (confs/general.yaml), got {have!r}")


def _sampler_cfg(opt):
    rs = _get(opt, "ray_sampler")
    return {k: _get(rs, k) for k in ("N_samples", "N_samples_eval", "N_samples_extra", "eps", "beta_iters", "max_total_iters", "add_tiny", "near")}


def _default_ctx(ctx):
    if ctx is not None:
        return ctx
    return capi.Context(torch.cuda.current_device())


class MANONode:
    """MANONode(args, opt, betas, sdf_bounding_sphere, node_id) (model/renderables/mano_node.py:18-60) -> hold_b200.model.Node."""

    def __new__(cls, args, opt, betas, sdf_bounding_sphere, node_id, *, ctx=None, slot=None, mano=None, mlp_mode=capi.MLP_TC):
        from .model import Node

        assert node_id in ("right", "left")
        _check_opt(opt, "implicit_network")
        _check_opt(opt, "rendering_network")
        if mano is None:
            raise ValueError("pass mano=<dict of MANO model arrays>: the library reads no model files (the reference's MANOServer loads them from disk)")
        d = _get(opt, "density")
        return Node(_default_ctx(ctx), {"right": 0, "left": 1}[node_id] if slot is None else slot, node_id, _sampler_cfg(opt), sdf_bounding_sphere,
                    n_frames=_get(args, "n_images"), mano=mano, betas=betas, mlp_mode=mlp_mode, beta=_get(_get(d, "params_init"), "beta"))


class ObjectNode:
    """ObjectNode(args, opt, sdf_bounding_sphere, node_id) (model/renderables/object_node.py:17-52) -> hold_b200.model.Node.
    (The reference adds the 32-d time code to opt.rendering_network.d_in in place, :19; so does this.)"""

    def __new__(cls, args, opt, sdf_bounding_sphere, node_id, *, ctx=None, slot=None, obj_pts=None, obj_scale=1.0, norm_mat=None, mlp_mode=capi.MLP_TC):
        from .model import Node

        _check_opt(opt, "implicit_network")
        _check_opt(opt, "rendering_network")
        rn = _get(opt, "rendering_network")
        if isinstance(rn, dict):
            rn["d_in"] = rn["d_in"] + 32
        else:
            rn.d_in = rn.d_in + 32
        if obj_pts is None:
            raise ValueError("pass obj_pts=<canonical object points [N,3]> (data.npy entities.object.pts.cano): the library reads no files")
        d = _get(opt, "density")
        return Node(_default_ctx(ctx), 2 if slot is None else slot, node_id, _sampler_cfg(opt), sdf_bounding_sphere, n_frames=_get(args, "n_images"),
                    obj_pts=obj_pts, obj_scale=obj_scale, norm_mat=norm_mat, mlp_mode=mlp_mode, beta=_get(_get(d, "params_init"), "beta"))


class Background:
    """Background(opt, args, num_frames, sdf_bounding_sphere) (model/renderables/background.py:9-33) -> hold_b200.model.Background."""

    def __new__(cls, opt, args, num_frames, sdf_bounding_sphere, *, ctx=None, mlp_mode=capi.MLP_TC):
        from .model import Background as _Background

        _check_opt(opt, "bg_implicit_network")
        _check_opt(opt, "bg_rendering_network")
        bg = _Background(_default_ctx(ctx), num_frames, mlp_mode)
        bg.sdf_bounding_sphere = sdf_bounding_sphere
        return bg


class HOLDNet:
    """HOLDNet(opt, betas_r, betas_l, num_frames, args) (hold/hold_net.py:24-51) -> hold_b200.model.HOLDNet with nodes
    {right?, left?, object} in the reference's order and the background."""

    def __new__(cls, opt, betas_r, betas_l, num_frames, args, *, ctx=None, mano_r=None, mano_l=None, obj_pts=None, obj_scale=1.0, norm_mat=None,
                mlp_mode=capi.MLP_TC):
        from .model import HOLDNet as _HOLDNet

        ctx = _default_ctx(ctx)
        R = _get(opt, "scene_bounding_sphere")
        nodes, slot = {}, 0
        if betas_r is not None:
            nodes["right"] = MANONode(args, opt, betas_r, R, "right", ctx=ctx, slot=slot, mano=mano_r, mlp_mode=mlp_mode)
            slot += 1
        if betas_l is not None:
            nodes["left"] = MANONode(args, opt, betas_l, R, "left", ctx=ctx, slot=slot, mano=mano_l, mlp_mode=mlp_mode)
            slot += 1
        nodes["object"] = ObjectNode(args, opt, R, "object", ctx=ctx, slot=slot, obj_pts=obj_pts, obj_scale=obj_scale, norm_mat=norm_mat, mlp_mode=mlp_mode)
        bg = Background(opt, args, num_frames, R, ctx=ctx, mlp_mode=mlp_mode)
        net = _HOLDNet(ctx, nodes, background=bg)
        net.sdf_bounding_sphere, net.threshold = R, 0.05
        return net
