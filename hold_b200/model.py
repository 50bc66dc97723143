"""Host-side mirror of the reference's call surface for the hot path (SURVEY.md §8b).

Same class names, argument meaning and state_dict keys as the reference (file:line cited per class,
relative to the reference's code/src), so `load_state_dict`, `--load_pose`, `--shape_init` style key
filters keep working; every `forward` body is a call into libhold_b200.so.  Inference (eval-mode)
semantics; the backward kernels are SURVEY §8f rank 2.

The modules own parameters only.  Packed device copies of the weights are refreshed by
`Node.sync_weights()` (call after an optimiser step / load_state_dict).
"""
from __future__ import annotations

import ctypes as C
import math

import torch
import torch.nn as nn

from . import capi
from .capi import Factors, ManoModel, NodeCfg, NodePose, RenderOut, check, lib, ptr, stream_ptr

CLASS_ID = {"object": 1, "right": 2, "left": 3}  # engine/rendering.py:59-61 via mano_node.py:20-25, object_node.py:22


def _wn_linear(i, o):
    return nn.utils.weight_norm(nn.Linear(i, o))


class LaplaceDensity(nn.Module):
    """engine/density.py:16-30 (parameter `beta`, floor beta_min)."""

    def __init__(self, beta=0.1, beta_min=1e-4):
        super().__init__()
        self.beta = nn.Parameter(torch.tensor(float(beta)))
        self.beta_min = beta_min

    def get_beta(self):
        return self.beta.abs() + self.beta_min


class ImplicitNet(nn.Module):
    """networks/shape_net.py:8-130: 9 weight-normed layers, skip at 4, Softplus(beta=100);
    keys `lin<k>.{weight_g,weight_v,bias}`.  forward(x [B,P,3], cond) -> [B,P,257]."""

    def __init__(self, kind: str):
        super().__init__()
        self.kind = kind
        d0 = 39 + (45 if kind == "hand" else 0)
        dims = [d0] + [256] * 8 + [257]
        for l in range(9):
            out = dims[l + 1] - 39 if l + 1 == 4 else dims[l + 1]
            setattr(self, f"lin{l}", _wn_linear(dims[l] if l > 0 else d0, out))
        object.__setattr__(self, "_node", None)

    def forward(self, input, cond, current_epoch=None):
        """Same signature as networks/shape_net.py:84.  `cond` is accepted and unused: the hand's pose condition is multiplied
        by zero in the reference (shape_net.py:104-106) and the object has none."""
        x = input
        if x.ndim == 2:
            x = x.unsqueeze(0)
        Bn, P, _ = x.shape
        node = self._node
        pts = x.reshape(-1, 3).contiguous().float()
        n = pts.shape[0]
        sdf = torch.empty(n, device=pts.device)
        grad = torch.empty(n, 3, device=pts.device)
        feat = torch.empty(n, 256, device=pts.device)
        check(lib().hold_sdf_eval(node.ctx.h, node.slot, n, ptr(pts), ptr(node.embed_w()), ptr(sdf), ptr(grad), ptr(feat), stream_ptr()))
        self.last_gradient = grad.view(Bn, P, 3)
        return torch.cat([sdf[:, None], feat], 1).view(Bn, P, 257)


class RenderingNet(nn.Module):
    """networks/texture_net.py:7-101, mode 'pose': lin0..lin4 weight-normed + lin_pose (45 -> 8)."""

    def __init__(self, kind: str):
        super().__init__()
        d0 = 270 if kind == "hand" else 302
        dims = [d0, 256, 256, 256, 256, 3]
        for l in range(5):
            setattr(self, f"lin{l}", _wn_linear(dims[l], dims[l + 1]))
        self.lin_pose = nn.Linear(45 if kind == "hand" else 0, 8)


class _ManoLbsFn(torch.autograd.Function):
    """GenericServer.forward under autograd (fitting/model.py:117): forward = hold_mano_lbs, backward = hold_mano_lbs_bwd."""

    @staticmethod
    def forward(fctx, server, absolute, scene_scale, transl, thetas, betas):
        out = server._forward_nograd(scene_scale, transl, thetas, betas, absolute)
        fctx.server, fctx.absolute = server, absolute
        fctx.save_for_backward(scene_scale.detach(), transl.detach(), thetas.detach(), betas.detach())
        fctx.mark_non_differentiable(out["v_posed"])
        return out["verts"], out["jnts"], out["tfs"], out["v_posed"]

    @staticmethod
    def backward(fctx, g_verts, g_jnts, g_tfs, _g_vposed):
        srv = fctx.server
        scene_scale, transl, thetas, betas = fctx.saved_tensors
        B = thetas.shape[0]
        dev = thetas.device
        f = lambda t, shape: t.detach().float().reshape(shape).contiguous()
        scene_scale, transl, thetas, betas = f(scene_scale, (B,)), f(transl, (B, 3)), f(thetas, (B, 48)), f(betas.expand(B, 10), (B, 10))
        gc = lambda g: None if g is None else g.float().contiguous()
        g_verts, g_jnts, g_tfs = gc(g_verts), gc(g_jnts), gc(g_tfs)
        gb, gp, gt, gs = (torch.empty(B, 10, device=dev), torch.empty(B, 48, device=dev), torch.empty(B, 3, device=dev),
                          torch.empty(B, device=dev))
        m = srv._model()
        tci = None if (fctx.absolute or srv.tfs_c_inv is None) else srv.tfs_c_inv
        check(lib().hold_mano_lbs_bwd(srv.ctx.h, C.byref(m), B, ptr(betas), ptr(thetas), ptr(transl), ptr(scene_scale), ptr(tci),
                                      ptr(g_verts), ptr(g_jnts), ptr(g_tfs), ptr(gb), ptr(gp), ptr(gt), ptr(gs), stream_ptr()))
        return None, None, gs, gt, gp, gb


class _ObjectTfFn(torch.autograd.Function):
    """ObjectModel.forward under autograd: forward = hold_object_tf, backward = hold_object_tf_bwd."""

    @staticmethod
    def forward(fctx, server, scene_scale, transl, thetas, obj_scale, obj_scale_host=None):
        # obj_scale_host: the scale as a Python float when it is not being optimised (no device->host read: capturable as a CUDA graph)
        val = float(obj_scale) if obj_scale_host is None else obj_scale_host
        out = server._forward_nograd(scene_scale, transl, thetas, val)
        fctx.server, fctx.obj_scale_val = server, val
        fctx.save_for_backward(scene_scale.detach(), transl.detach(), thetas.detach(), obj_scale.detach())
        return out["verts"], out["obj_tfs"]

    @staticmethod
    def backward(fctx, g_verts, g_tfs):
        srv = fctx.server
        scene_scale, transl, thetas, obj_scale = fctx.saved_tensors
        B = thetas.shape[0]
        dev = srv.v3d_cano.device
        f = lambda t, shape: t.detach().float().reshape(shape).contiguous()
        gc = lambda g, shape: None if g is None else g.float().reshape(shape).contiguous()
        Nv = srv.v3d_cano.shape[0]
        gr, gt, gs, go = torch.empty(B, 3, device=dev), torch.empty(B, 3, device=dev), torch.empty(B, device=dev), torch.empty(B, device=dev)
        check(lib().hold_object_tf_bwd(srv.ctx.h, B, ptr(f(thetas, (B, 3))), ptr(f(transl, (B, 3))), ptr(f(scene_scale, (B,))),
                                       fctx.obj_scale_val, ptr(srv.denorm_mat), ptr(srv.v3d_cano), Nv, ptr(gc(g_verts, (B, Nv, 3))),
                                       ptr(gc(g_tfs, (B, 4, 4))), ptr(gr), ptr(gt), ptr(gs), ptr(go), stream_ptr()))
        return None, gs.reshape(scene_scale.shape), gt.reshape(transl.shape), gr.reshape(thetas.shape), go.sum().reshape(obj_scale.shape), None


class MANOServer(nn.Module):
    """model/mano/server.py:20-133 (GenericServer + MANOServer) over a MANO model struct
    (dict with v_template, shapedirs, posedirs, J_regressor, lbs_weights, hands_mean, parents, tip_ids)."""

    def __init__(self, ctx, mano: dict, betas):
        super().__init__()
        self.ctx = ctx
        dev = torch.device("cuda", ctx.device)
        self.m = {k: (v.to(dev).contiguous() if torch.is_tensor(v) and v.dtype.is_floating_point else v) for k, v in mano.items()}
        par = mano["parents"].to(torch.int32).tolist()
        par[0] = -1
        self._parents = (C.c_int32 * 16)(*par)
        self._tips = (C.c_int32 * 5)(*mano["tip_ids"].to(torch.int32).tolist())
        self.betas = torch.as_tensor(betas, dtype=torch.float32, device=dev).view(1, 10)
        self.tfs_c_inv = None
        # canonical pose = flat hand: pose = -hands_mean, scale 1, transl 0 (server.py:11-17)
        cano_pose = torch.cat([torch.zeros(3, device=dev), -self.m["hands_mean"]])[None]
        out = self.forward(torch.ones(1, device=dev), torch.zeros(1, 3, device=dev), cano_pose, self.betas, absolute=True)
        self.verts_c, self.joints_c = out["verts"], out["jnts"]
        self.tfs_c_inv = torch.linalg.inv(out["tfs"][0]).contiguous()  # one-off 16 4x4 inverses at construction

    def _model(self):
        m = ManoModel()
        for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights", "hands_mean"):
            setattr(m, k, self.m[k].data_ptr())
        m.parents_host = C.cast(self._parents, C.POINTER(C.c_int32))
        m.tip_ids_host = C.cast(self._tips, C.POINTER(C.c_int32))
        return m

    def forward(self, scene_scale, transl, thetas, betas, absolute=False):
        """Differentiable w.r.t. scene_scale / transl / thetas / betas when any of them requires grad (the pose refinement
        of optimize_ckpt.py); otherwise the plain forward."""
        if torch.is_grad_enabled() and any(t.requires_grad for t in (scene_scale, transl, thetas, betas)):
            B = thetas.shape[0]
            verts, jnts, tfs, v_posed = _ManoLbsFn.apply(self, absolute, scene_scale.reshape(B), transl.reshape(B, 3),
                                                         thetas.reshape(B, 48), betas.expand(B, 10))
            return {"verts": verts, "jnts": jnts, "tfs": tfs, "v_posed": v_posed,
                    "skin_weights": self.m["lbs_weights"][None].expand(B, -1, -1)}
        return self._forward_nograd(scene_scale, transl, thetas, betas, absolute)

    def _forward_nograd(self, scene_scale, transl, thetas, betas, absolute=False):
        B = thetas.shape[0]
        dev = thetas.device
        f = lambda t, shape: t.detach().float().reshape(shape).contiguous()
        scene_scale, transl, thetas, betas = f(scene_scale, (B,)), f(transl, (B, 3)), f(thetas, (B, 48)), f(betas.expand(B, 10), (B, 10))
        verts = torch.empty(B, 778, 3, device=dev)
        jnts = torch.empty(B, 21, 3, device=dev)
        tfs = torch.empty(B, 16, 4, 4, device=dev)
        v_posed = torch.empty(B, 778, 3, device=dev)
        m = self._model()
        tci = None if (absolute or self.tfs_c_inv is None) else self.tfs_c_inv
        check(lib().hold_mano_lbs(self.ctx.h, C.byref(m), B, ptr(betas), ptr(thetas), ptr(transl), ptr(scene_scale), ptr(tci),
                                  ptr(verts), ptr(jnts), ptr(tfs), ptr(v_posed), stream_ptr()))
        return {"verts": verts, "jnts": jnts, "tfs": tfs, "v_posed": v_posed,
                "skin_weights": self.m["lbs_weights"][None].expand(B, -1, -1)}

    def forward_param(self, param_dict):
        """server.py:101-113 (optimize_ckpt.py's only hot-path call, fitting/model.py:117)."""
        get = lambda k: next(v for kk, v in param_dict.items() if k in kk)
        full_pose = torch.cat((get("global_orient"), get("pose")), dim=1)
        B = full_pose.shape[0]
        return self.forward(get("scene_scale").view(-1).repeat(B), get("transl"), full_pose, get("betas").repeat(B, 1))


class ObjectServer(nn.Module):
    """model/obj/server.py:19-56 + object_model.py:12-70."""

    def __init__(self, ctx, pts_cano, obj_scale=1.0, norm_mat=None):
        super().__init__()
        self.ctx = ctx
        dev = torch.device("cuda", ctx.device)
        self.v3d_cano = pts_cano.to(dev).float().contiguous()
        self.set_object_model(obj_scale=obj_scale, norm_mat=norm_mat)

    def set_object_model(self, obj_scale=None, norm_mat=None, v3d_cano=None):
        """The registered buffers of the reference's ObjectModel (model/obj/object_model.py:23-27): `obj_scale`, `norm_mat`
        (-> `denorm_mat` = its inverse), `v3d_cano`.  Real sequences carry non-trivial values (data.npy); a reference checkpoint
        stores them under `nodes.object.server.object_model.*` (checkpoint.load_reference_state_dict feeds them here)."""
        dev = torch.device("cuda", self.ctx.device)
        if v3d_cano is not None:
            self.v3d_cano = v3d_cano.to(dev).float().contiguous()
        if obj_scale is not None:
            self.obj_scale = obj_scale if (torch.is_tensor(obj_scale) and obj_scale.requires_grad) else float(torch.as_tensor(obj_scale).reshape(-1)[0])
        if norm_mat is not None or not hasattr(self, "norm_mat"):
            nm = torch.eye(4) if norm_mat is None else norm_mat.detach().float().cpu().reshape(4, 4)
            self.norm_mat = nm.to(dev).contiguous()
            self.denorm_mat = torch.linalg.inv(nm.double()).float().to(dev).contiguous()
        self.verts_c = self.v3d_cano[None]

    def forward(self, scene_scale, transl, thetas, absolute=False):
        """Differentiable w.r.t. scene_scale / transl / thetas / obj_scale (when `self.obj_scale` is a tensor, as
        fitting/model.py:113 sets it) if any of them requires grad; otherwise the plain forward."""
        osc = self.obj_scale
        needs = torch.is_grad_enabled() and any(torch.is_tensor(t) and t.requires_grad for t in (scene_scale, transl, thetas, osc))
        if needs:
            # torch.full = a fill kernel; torch.tensor(float, device=cuda) would be a pageable host->device copy (not capturable)
            osc_t = osc if torch.is_tensor(osc) else torch.full((), float(osc), device=self.v3d_cano.device)
            verts, tfs = _ObjectTfFn.apply(self, scene_scale, transl, thetas, osc_t, None if torch.is_tensor(osc) else float(osc))
            return {"verts": verts, "obj_tfs": tfs}
        return self._forward_nograd(scene_scale, transl, thetas, float(osc))

    def _forward_nograd(self, scene_scale, transl, thetas, obj_scale):
        B = thetas.shape[0]
        dev = self.v3d_cano.device
        f = lambda t, shape: t.detach().float().reshape(shape).contiguous()
        tfs = torch.empty(B, 4, 4, device=dev)
        verts = torch.empty(B, self.v3d_cano.shape[0], 3, device=dev)
        check(lib().hold_object_tf(self.ctx.h, B, ptr(f(thetas, (B, 3))), ptr(f(transl, (B, 3))), ptr(f(scene_scale, (B,))),
                                   float(obj_scale), ptr(self.denorm_mat), ptr(self.v3d_cano), self.v3d_cano.shape[0],
                                   ptr(tfs), ptr(verts), stream_ptr()))
        return {"verts": verts, "obj_tfs": tfs[:, None]}

    def forward_param(self, param_dict):
        get = lambda k: next(v for kk, v in param_dict.items() if k in kk)
        go = get("global_orient")
        return self.forward(get("scene_scale").view(-1).repeat(go.shape[0]), get("transl"), go)


class Node(nn.Module):
    """model/renderables/node.py:14-109 (+ mano_node.py / object_node.py): one entity of the scene.
    state_dict keys: implicit_network.lin*, rendering_network.lin*, rendering_network.lin_pose.*,
    density.beta, frame_latent_encoder.weight (object)."""

    def __init__(self, ctx, slot, node_id, sampler_cfg, bounding_sphere, n_frames=1, mano=None, betas=None, obj_pts=None,
                 mlp_mode=capi.MLP_FP32, beta=0.1, obj_scale=1.0, norm_mat=None):
        super().__init__()
        self.ctx, self.slot, self.node_id = ctx, slot, node_id
        self.kind = "hand" if node_id in ("right", "left") else "object"
        self.class_id = CLASS_ID[node_id]
        self.implicit_network = ImplicitNet(self.kind)
        object.__setattr__(self.implicit_network, "_node", self)  # back-reference, not a submodule
        self.rendering_network = RenderingNet(self.kind)
        self.density = LaplaceDensity(beta)
        self.sampler_cfg = dict(sampler_cfg)
        self.bounding_sphere = bounding_sphere
        self.barf_weights = None  # [39] BARF mask of the object's embedder (eval(): None == all ones, render.py:43-47)
        if self.kind == "hand":
            self.server = MANOServer(ctx, mano, betas)
        else:
            self.server = ObjectServer(ctx, obj_pts, obj_scale=obj_scale, norm_mat=norm_mat)   # data.npy: entities.object.{obj_scale,norm_mat}
            self.frame_latent_encoder = nn.Embedding(n_frames, 32)
        # per-frame pose parameters, same module names as the reference (model/generic/params.py) so that a reference
        # checkpoint loads (hold_b200/checkpoint.py); used when the input dict carries only frame ids
        from .checkpoint import HAND_PARAMS, OBJECT_PARAMS, GenericParams
        self.params = GenericParams(n_frames, HAND_PARAMS if self.kind == "hand" else OBJECT_PARAMS, node_id)
        self.mlp_mode = mlp_mode
        self.configure()
        self.S = sampler_cfg["N_samples"] + sampler_cfg["N_samples_extra"] + 2

    def configure(self):
        c, s = NodeCfg(), self.sampler_cfg
        c.kind = capi.KIND_HAND if self.kind == "hand" else capi.KIND_OBJECT
        c.class_id = self.class_id
        c.n_samples_eval, c.n_samples, c.n_samples_extra = s["N_samples_eval"], s["N_samples"], s["N_samples_extra"]
        c.beta_iters, c.max_total_iters, c.mlp_mode = s["beta_iters"], s["max_total_iters"], self.mlp_mode
        c.eps, c.add_tiny, c.near = s["eps"], s["add_tiny"], s["near"]
        c.bounding_sphere, c.beta_min = self.bounding_sphere, self.density.beta_min
        check(lib().hold_node_configure(self.ctx.h, self.slot, C.byref(c)))
        if self.kind == "hand":
            check(lib().hold_node_set_rig(self.ctx.h, self.slot, ptr(self.server.verts_c[0].contiguous()),
                                          ptr(self.server.m["lbs_weights"]), stream_ptr()))

    def embed_w(self):
        return self.barf_weights

    def start_barf(self, start=1000, end=10000):
        """Training-mode coarse-to-fine mask of the object's embedder (engine/embedders.py:53-126, BarfEmbedder; parser.py:32-33
        barf_s / barf_e): frequency k of the 6 is weighted clamp(alpha - k, 0, 1) with a cosine ramp inside (0, 1), alpha follows
        [0]*start + linspace(0, 6, end - start) and advances once per training forward (step_embedding).  Hands and the background
        use the plain Fourier embedder (model/*/specs.py), whose step() does nothing."""
        assert self.kind == "object", "only the object's ImplicitNet uses the BARF embedder (model/obj/specs.py:10)"
        dev = self.density.beta.device
        sched = BarfSchedule(6, 3, start, end)
        # the whole schedule as a device table + a device-side counter; the weights the kernels read live in ONE persistent buffer
        # that step_embedding refreshes in place: no host->device copy per step, and a step captured as a CUDA graph
        # (TrainStep.capture) keeps advancing the schedule on replay
        self._barf_table = sched.table().to(dev)
        self._barf_it = torch.zeros((), dtype=torch.int64, device=dev)
        self._barf = sched
        self.barf_weights = self._barf_table[0].clone()

    def step_embedding(self):
        """Node.step_embedding (node.py:108-109)."""
        if getattr(self, "_barf", None) is not None and self.barf_weights is not None:
            self._barf.step()      # host mirror of the counter (bookkeeping only)
            self._barf_it.add_(1).clamp_(max=self._barf_table.shape[0] - 1)
            self.barf_weights.copy_(self._barf_table.index_select(0, self._barf_it.reshape(1))[0])

    def eval(self):
        """BarfEmbedder.eval(): no_barf = True -> all frequencies pass (embedders.py:124-125, render.py:43-47)."""
        if getattr(self, "_barf", None) is not None:
            self.barf_weights = None
        return super().eval()

    def sync_weights(self):
        """Re-pack the (possibly updated) parameters into the library (hold_node_set_weights)."""
        isd = {k: v for k, v in self.implicit_network.state_dict().items()}
        rsd = {k: v for k, v in self.rendering_network.state_dict().items()}
        wi, k1 = capi.mlp_weights(isd, 9)
        wr, k2 = capi.mlp_weights(rsd, 5)
        lp_w = rsd["lin_pose.weight"].float().contiguous() if self.kind == "hand" else None
        lp_b = rsd["lin_pose.bias"].float().contiguous() if self.kind == "hand" else None
        check(lib().hold_node_set_weights(self.ctx.h, self.slot, C.byref(wi), C.byref(wr), ptr(lp_w), ptr(lp_b), stream_ptr()))
        # no host sync: the packing kernels run on the current stream, and the caching allocator hands the temporaries (k1, k2)
        # back only to later work of that same stream (a sync here stalled every training step three times and made the step
        # uncapturable as a CUDA graph)

    def meshing_cano(self, res_init=32, res_up=3):
        """The node's canonical mesh from its current SDF, as HOLD.meshing_cano builds it (hold.py:139-167) -> (verts [n,3]
        float32, faces [m,3] int32) on the device (meshing.extract_mesh).  The weights are re-packed first, as every training
        step does, and the SDF is queried as ImplicitNet.forward does, with the current BARF mask of the object's embedder.
        The bounding box is the server's canonical vertices.  The object node keeps the mesh as mesh_vo_cano / mesh_fo_cano,
        the loss targets' mesh (train.prepare_loss_targets); a hand's targets use the MANO mesh, so a hand only returns it."""
        from . import meshing

        self.sync_weights()
        f = meshing.node_sdf_func(self.ctx, self, embed_w=self.embed_w())
        v, fc = meshing.extract_mesh(self.ctx, f, self.server.verts_c[0], res_init=res_init, res_up=res_up)
        if self.kind == "object":
            self.mesh_vo_cano, self.mesh_fo_cano = v, fc
        return v, fc

    # -- articulation ---------------------------------------------------------------------------------
    def articulate(self, input):
        """The server call at the top of sample_points (mano_node.py:72-79 / object_node.py:58-62) -> NodePose."""
        nid = self.node_id
        if f"{nid}.transl" not in input:   # only frame ids given: the node's own per-frame parameters (hold.py: params(idx))
            input = {**input, **self.params(input["idx"])}
            if self.kind == "hand":
                input[f"{nid}.full_pose"] = torch.cat([input[f"{nid}.global_orient"], input[f"{nid}.pose"]], 1)
        scale = input[f"{nid}.params"][:, 0]
        pose = NodePose()
        keep = []
        if self.kind == "hand":
            full_pose = input[f"{nid}.full_pose"]
            out = self.server(scale, input[f"{nid}.transl"], full_pose, input[f"{nid}.betas"])
            cond = (full_pose[:, 3:] / math.pi).float().contiguous()  # mano_node.py:81 (eval: never zeroed)
            keep += [out["tfs"], out["verts"], cond]
            pose.tfs, pose.posed_verts, pose.pose_cond = out["tfs"].data_ptr(), out["verts"].data_ptr(), cond.data_ptr()
            tfs = out["tfs"]
        else:
            out = self.server(scale, input[f"{nid}.transl"], input[f"{nid}.global_orient"])
            tfs = out["obj_tfs"][:, 0].contiguous()
            tc = self.frame_latent_encoder(input["idx"]).detach().float().contiguous()  # object_node.py:52-55
            keep += [tfs, tc]
            pose.tfs, pose.time_code = tfs.data_ptr(), tc.data_ptr()
        if self.barf_weights is not None:
            pose.embed_w = self.barf_weights.data_ptr()
        beta = self.density.beta.detach().float().reshape(1).contiguous()
        keep.append(beta)
        pose.beta_param = beta.data_ptr()
        return pose, keep, out, tfs


def sampler_rand(R, cfg, device, generator=None):
    """The training-mode randomness of ErrorBoundSampler.get_z_vals for R rays (the library takes it as an input,
    hold_sampler_rand), drawn with torch as the reference draws it: stratified jitter [R, N_samples_eval] (ray_sampler.py:70-78),
    inverse-CDF uniforms u [R, N_samples] (:292) and, for every possible final buffer size n = (j + 1) * N_samples_eval, the
    extras permutation randperm(n)[:N_samples_extra] (:328) as one int32 row of extra_idx [max_total_iters, N_samples_extra].
    cfg: the sampler's N_samples, N_samples_eval, N_samples_extra, max_total_iters."""
    ne = cfg["N_samples_eval"]
    jitter = torch.rand(R, ne, device=device, generator=generator)
    u = torch.rand(R, cfg["N_samples"], device=device, generator=generator)
    extra = torch.stack([torch.randperm((j + 1) * ne, device=device, generator=generator)[: cfg["N_samples_extra"]]
                         for j in range(cfg["max_total_iters"])]).int().contiguous()
    return dict(jitter=jitter, u=u, extra_idx=extra)


class ErrorBoundSampler:
    """engine/ray_sampler.py:88-352 behind hold_sample; bound to a Node's ctx slot."""

    def __init__(self, node: Node):
        self.node = node

    def get_z_vals(self, ray_dirs, cam_loc, pose: NodePose, B: int, rand=None):
        n = self.node
        ray_dirs, cam_loc = ray_dirs.float().contiguous(), cam_loc.float().contiguous()
        R = ray_dirs.shape[0]
        z = torch.empty(R, n.S, device=ray_dirs.device)
        iters = torch.zeros(1, dtype=torch.int32, device=ray_dirs.device)
        rnd = None
        if rand is not None:
            rnd = capi.SamplerRand()
            ex = rand["extra_idx"].to(torch.int32)
            if ex.dim() == 1:   # one draw for every round count (valid when it indexes below N_samples_eval)
                ex = ex[None].repeat(n.sampler_cfg["max_total_iters"], 1)
            ex = ex.contiguous()
            self._keep = ex
            rnd.jitter, rnd.u, rnd.extra_idx = rand["jitter"].data_ptr(), rand["u"].data_ptr(), ex.data_ptr()
        check(lib().hold_sample(n.ctx.h, n.slot, R, B, ptr(cam_loc), ptr(ray_dirs), C.byref(pose),
                                C.byref(rnd) if rnd is not None else None, ptr(z), ptr(iters), stream_ptr()))
        return z, iters


class Background(nn.Module):
    """model/renderables/background.py:9-165 — the NeRF++ inverted-sphere background (SURVEY §8f rank 1).
    state_dict keys: bg_implicit_network.lin<k>.{weight,bias}, bg_rendering_network.lin<k>.{weight,bias},
    frame_latent_encoder.weight (the reference's `background.*` keys)."""

    def __init__(self, ctx, num_frames, mlp_mode=capi.MLP_FP32):
        super().__init__()
        self.ctx = ctx
        self.mlp_mode = mlp_mode   # arithmetic of both background nets (HOLD_MLP_FP32 exact fp32, HOLD_MLP_TC tensor-core split precision)
        dims = [84] + [256] * 8 + [257]
        self.bg_implicit_network = nn.Module()
        for l in range(9):
            out = dims[l + 1] - 84 if l + 1 == 4 else dims[l + 1]
            setattr(self.bg_implicit_network, f"lin{l}", nn.Linear(dims[l] + (32 if l == 0 else 0), out))
        self.bg_rendering_network = nn.Module()
        self.bg_rendering_network.lin0 = nn.Linear(315, 128)
        self.bg_rendering_network.lin1 = nn.Linear(128, 3)
        self.frame_latent_encoder = nn.Embedding(num_frames, 32)

    def sync_weights(self):
        isd = dict(self.bg_implicit_network.state_dict())
        rsd = dict(self.bg_rendering_network.state_dict())
        wi, k1 = capi.mlp_weights(isd, 9)
        wr, k2 = capi.mlp_weights(rsd, 2)
        check(lib().hold_bg_set_weights(self.ctx.h, C.byref(wi), C.byref(wr), self.mlp_mode, stream_ptr()))   # stream-ordered, no host sync

    @torch.no_grad()
    def forward(self, bg_weights, ray_dirs, cam_loc, idx, B):
        """Background.forward + inverse_sample -> dict(bg_rgb, bg_rgb_only, bg_semantics, bg_z_vals)."""
        R = ray_dirs.shape[0]
        dev = ray_dirs.device
        fc = self.frame_latent_encoder(idx).detach().float().contiguous()
        out = dict(bg_rgb=torch.empty(R, 3, device=dev), bg_rgb_only=torch.empty(R, 3, device=dev),
                   bg_semantics=torch.empty(R, 4, device=dev), bg_z_vals=torch.empty(R, 32, device=dev))
        check(lib().hold_background(self.ctx.h, R, B, ptr(cam_loc.float().contiguous()), ptr(ray_dirs.float().contiguous()), ptr(fc),
                                    ptr(bg_weights.float().contiguous()), ptr(out["bg_rgb"]), ptr(out["bg_rgb_only"]),
                                    ptr(out["bg_semantics"]), ptr(out["bg_z_vals"]), stream_ptr()))
        return out


class BarfSchedule:
    """alpha schedule + weights of engine/embedders.py:53-106 (BarfEmbedder.__init__, compute_barf_weights, step)."""

    def __init__(self, num_freq, input_dims, start, end):
        self.L, self.D = num_freq, input_dims
        self.alphas = torch.cat((torch.zeros(start), torch.linspace(0, num_freq, end - start)), 0)
        self.alpha_iter = 0

    def step(self):
        self.alpha_iter = min(self.alpha_iter + 1, len(self.alphas) - 1)

    def table(self):
        """[len(alphas), D + 2 L D]: the weights of every iteration."""
        keep = self.alpha_iter
        rows = []
        for it in range(len(self.alphas)):
            self.alpha_iter = it
            rows.append(self.weights())
        self.alpha_iter = keep
        return torch.stack(rows)

    def weights(self):
        ak = self.alphas[self.alpha_iter] - torch.arange(self.L, dtype=torch.float32)
        w = torch.clamp(ak, 0, 1)
        ramp = torch.logical_and(0 <= ak, ak < 1)
        w[ramp] = ((1 - torch.cos(ak * math.pi)) / 2)[ramp]
        w = w[:, None].repeat(1, self.D * 2).view(-1)       # sin and cos of every coordinate share the frequency's weight
        return torch.cat((torch.ones(self.D), w), 0).contiguous()


class HOLDNet(nn.Module):
    """hold/hold_net.py:23-134, foreground: nodes{right,left,object}; forward_fg(input) -> out dict with the
    reference's keys (fg_rgb, mask_prob, normal, depth, fg_semantics, fg_weights, bg_weights, <node>.*, ray_dirs, cam_loc)."""

    def __init__(self, ctx, nodes: dict, background=None):
        super().__init__()
        self.ctx = ctx
        self.nodes = nn.ModuleDict(nodes)
        self.background = background

    def step_embedding(self):
        """hold_net.py:104-108 (the background's Fourier embedders have nothing to step)."""
        for n in self.nodes.values():
            n.step_embedding()

    def sync_weights(self):
        for n in self.nodes.values():
            n.sync_weights()
        if self.background is not None:
            self.background.sync_weights()

    @torch.no_grad()
    def forward(self, input, chunk=None):
        """HOLDNet.forward + composite (hold/hold_net.py:110-134), eval: rgb = fg_rgb + bg_rgb, semantics,
        bg_rgb_only, instance_map = argmax(semantics).  chunk: see forward_fg."""
        out = self.forward_fg(input, return_factors=False, chunk=chunk)
        B = input["uv"].shape[0]
        bg = self.background(out["bg_weights"], out["ray_dirs"], out["cam_loc"], input["idx"], B)
        out["bg_z_vals"] = bg["bg_z_vals"]
        out["rgb"] = out["fg_rgb"] + bg["bg_rgb"]
        out["semantics"] = out["fg_semantics"] + bg["bg_semantics"]
        out["bg_rgb_only"] = bg["bg_rgb_only"]
        out["instance_map"] = torch.argmax(out["semantics"], dim=1)
        return out

    @torch.no_grad()
    def forward_fg(self, input, return_factors=True, want_weights=True, chunk=None):
        """chunk: rays per call.  The sampler's convergence flag `beta.max() > beta0` is global over the rays of ONE call
        (engine/ray_sampler.py:244); the reference's render path issues 512-pixel calls (datasets/eval_datasets.py:13,
        hold.py:190-192), so `chunk=512` reproduces its per-chunk round counts, while `chunk=None` renders the whole frame in
        one call (all rays run as many rounds as the slowest ray of the frame needs)."""
        if chunk is not None and input["uv"].shape[1] > chunk:
            assert input["uv"].shape[0] == 1, "chunked rendering follows the reference's eval path: one frame per call"
            outs = []
            for s0 in range(0, input["uv"].shape[1], chunk):
                sub = dict(input)
                sub["uv"] = input["uv"][:, s0:s0 + chunk].contiguous()
                outs.append(self.forward_fg(sub, return_factors=return_factors, want_weights=want_weights, chunk=None))
            out = {}
            for k, v in outs[0].items():
                if k == "sampler_iters":
                    out[k] = torch.stack([o[k] for o in outs]).amax(0)
                    out["sampler_iters_per_chunk"] = torch.stack([o[k] for o in outs])
                elif k == "factors":
                    out[k] = {nid: {kk: torch.cat([o[k][nid][kk] for o in outs]) for kk in v[nid]} for nid in v}
                elif torch.is_tensor(v) and v.dim() >= 1 and v.shape[0] == outs[0]["ray_dirs"].shape[0]:
                    out[k] = torch.cat([o[k] for o in outs])
                else:
                    out[k] = v
            return out
        uv, ext, intr = input["uv"].float().contiguous(), input["extrinsics"].float().contiguous(), input["intrinsics"].float().contiguous()
        B, P, _ = uv.shape
        dev = uv.device
        R = B * P
        dirs = torch.empty(R, 3, device=dev)
        cam = torch.empty(R, 3, device=dev)
        check(lib().hold_camera_rays(self.ctx.h, B, P, ptr(uv), ptr(ext), ptr(intr), ptr(dirs), ptr(cam), stream_ptr()))
        nodes = list(self.nodes.values())
        n = len(nodes)
        S = nodes[0].S
        poses = (NodePose * n)()
        facs = (Factors * n)()
        keep, fac_t, arts = [], [], {}
        for k, node in enumerate(nodes):
            pose, kp, art, _ = node.articulate(input)
            poses[k] = pose
            keep += kp
            arts[node.node_id] = art
            t = dict(color=torch.empty(R, S, 3, device=dev), normal=torch.empty(R, S, 3, device=dev),
                     density=torch.empty(R, S, device=dev), z_vals=torch.empty(R, S, device=dev),
                     sdf=torch.empty(R, S, device=dev), canonical_pts=torch.empty(R, S, 3, device=dev))
            fac_t.append(t)
            for kk, v in t.items():
                setattr(facs[k], kk, v.data_ptr())
        M = n * S - 2 * n + 1

        def render_out(m):
            t = dict(fg_rgb=torch.empty(R, 3, device=dev), mask_prob=torch.empty(R, device=dev), normal=torch.empty(R, 3, device=dev),
                     depth=torch.empty(R, device=dev), fg_semantics=torch.empty(R, 4, device=dev), bg_weights=torch.empty(R, device=dev))
            if want_weights:
                t["fg_weights"] = torch.empty(R, m, device=dev)
            ro = RenderOut()
            for kk, v in t.items():
                setattr(ro, kk, v.data_ptr())
            return ro, t

        comp, comp_t = render_out(M)
        per = (RenderOut * n)()
        per_t = []
        for k in range(n):
            per[k], t = render_out(S)
            per_t.append(t)
        iters = torch.zeros(n, dtype=torch.int32, device=dev)
        ids = (C.c_int32 * n)(*[nd.slot for nd in nodes])
        check(lib().hold_render_fg(self.ctx.h, n, ids, R, B, ptr(cam), ptr(dirs), poses, facs, C.byref(comp), per, ptr(iters), stream_ptr()))
        out = {k: (v[:, None] if v.dim() == 1 else v) for k, v in comp_t.items()}
        out["bg_weights"] = comp_t["bg_weights"]
        out["fg_rgb.vis"] = comp_t["fg_rgb"] + comp_t["bg_weights"][:, None]  # hold_utils.py:268-270
        for k, node in enumerate(nodes):
            for kk, v in per_t[k].items():
                out[f"{node.node_id}.{kk}"] = v[:, None] if (v.dim() == 1 and kk != "bg_weights") else v
        out["ray_dirs"], out["cam_loc"], out["index"] = dirs, cam, input.get("idx")
        out["sampler_iters"] = iters
        if return_factors:
            out["factors"] = {node.node_id: fac_t[k] for k, node in enumerate(nodes)}
            out["articulation"] = arts
        return out
