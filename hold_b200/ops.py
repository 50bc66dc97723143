"""Stage-level entry points (thin wrappers over the C ABI) used by tests and by callers that drive the
stages themselves: shade (Node.forward after sampling) and composite (merge_factors + volumetric_render)."""
from __future__ import annotations

import ctypes as C

import torch

from .capi import Factors, NodePose, RenderOut, check, lib, ptr, stream_ptr


def camera_rays(ctx, uv, pose, intrinsics):
    B, P, _ = uv.shape
    dirs = torch.empty(B * P, 3, device=uv.device)
    cam = torch.empty(B * P, 3, device=uv.device)
    check(lib().hold_camera_rays(ctx.h, B, P, ptr(uv.float().contiguous()), ptr(pose.float().contiguous()),
                                 ptr(intrinsics.float().contiguous()), ptr(dirs), ptr(cam), stream_ptr()))
    return dirs, cam


def shade(node, ray_dirs, cam_loc, pose: NodePose, z_vals, B: int):
    R, S = z_vals.shape
    dev = z_vals.device
    ray_dirs, cam_loc = ray_dirs.float().contiguous(), cam_loc.float().contiguous()
    t = dict(color=torch.empty(R, S, 3, device=dev), normal=torch.empty(R, S, 3, device=dev), density=torch.empty(R, S, device=dev),
             z_vals=z_vals.contiguous(), sdf=torch.empty(R, S, device=dev), canonical_pts=torch.empty(R, S, 3, device=dev))
    f = Factors()
    for k, v in t.items():
        setattr(f, k, v.data_ptr())
    check(lib().hold_shade(node.ctx.h, node.slot, R, B, S, ptr(cam_loc), ptr(ray_dirs), C.byref(pose), C.byref(f), stream_ptr()))
    return t


def composite(ctx, factors: list, class_ids: list, want_weights=True):
    n = len(factors)
    R, S = factors[0]["z_vals"].shape
    dev = factors[0]["z_vals"].device
    facs = (Factors * n)()
    keep = []
    for k, f in enumerate(factors):
        for kk in ("color", "normal", "density", "z_vals"):
            v = f[kk].float().contiguous()
            keep.append(v)
            setattr(facs[k], kk, v.data_ptr())

    def mk(m):
        t = dict(fg_rgb=torch.empty(R, 3, device=dev), mask_prob=torch.empty(R, device=dev), normal=torch.empty(R, 3, device=dev),
                 depth=torch.empty(R, device=dev), fg_semantics=torch.empty(R, 4, device=dev), bg_weights=torch.empty(R, device=dev))
        if want_weights:
            t["fg_weights"] = torch.empty(R, m, device=dev)
        ro = RenderOut()
        for kk, v in t.items():
            setattr(ro, kk, v.data_ptr())
        return ro, t

    comp, comp_t = mk(n * S - 2 * n + 1)
    per = (RenderOut * n)()
    per_t = []
    for k in range(n):
        per[k], t = mk(S)
        per_t.append(t)
    cls = (C.c_int32 * n)(*class_ids)
    check(lib().hold_composite(ctx.h, n, R, S, facs, cls, C.byref(comp), per, stream_ptr()))
    return comp_t, per_t


def inverse_warp(node, x, pose: NodePose, want_idx=False):
    B, P, _ = x.shape
    xc = torch.empty(B, P, 3, device=x.device)
    idx = torch.empty(B, P, 15, dtype=torch.int32, device=x.device) if want_idx else None
    mask = torch.empty(B, P, dtype=torch.uint8, device=x.device) if want_idx else None
    check(lib().hold_inverse_warp(node.ctx.h, node.slot, B, P, ptr(x.float().contiguous()), C.byref(pose), ptr(xc), ptr(idx), ptr(mask), stream_ptr()))
    return xc, idx, mask


def inverse_warp_bwd(node, x, pose: NodePose, knn_idx, g_xc, want_gx=False):
    """Reverse mode of `inverse_warp` w.r.t. the transforms: g_xc [B,P,3] -> g_tfs ([B,16,4,4] hand / [B,4,4] object), g_x."""
    B, P, _ = x.shape
    hand = node.kind == "hand"
    g_tfs = torch.empty((B, 16, 4, 4) if hand else (B, 4, 4), device=x.device)
    g_x = torch.empty(B, P, 3, device=x.device) if want_gx else None
    check(lib().hold_inverse_warp_bwd(node.ctx.h, node.slot, B, P, ptr(x.float().contiguous()), C.byref(pose),
                                      ptr(knn_idx) if knn_idx is not None else None, ptr(g_xc.float().contiguous()), ptr(g_tfs), ptr(g_x),
                                      stream_ptr()))
    return g_tfs, g_x


def compute_mano_cano_sdf(ctx, mesh_v_cano, mesh_f_cano, x_cano):
    """engine/volsdf_utils.py:172-186 without kaolin: signed distance [B,P] of x_cano [B,P,3] to the closed mesh
    (mesh_v_cano [B,V,3] or [V,3]; mesh_f_cano [F,3] integer)."""
    x = x_cano.detach().float().contiguous()
    B, P, _ = x.shape
    v = mesh_v_cano.detach().float().contiguous()
    batched = v.dim() == 3 and v.shape[0] == B and B > 1
    if v.dim() == 3 and not batched:
        v = v[0].contiguous()
    f = mesh_f_cano.to(torch.int32).contiguous()
    out = torch.empty(B, P, device=x.device)
    check(lib().hold_mesh_sdf_bvh(ctx.h, B, P, ptr(x), v.shape[-2], ptr(v), int(batched), f.shape[0], ptr(f), ptr(out), None, stream_ptr()))
    return out


def check_off_in_surface_points_cano_mesh(ctx, mesh_v_cano, mesh_f_cano, x_cano, num_pixels_total, threshold=0.05):
    """engine/volsdf_utils.py:189-217: (index_off_surface, index_in_surface), bool [num_pixels_total]."""
    sd = compute_mano_cano_sdf(ctx, mesh_v_cano, mesh_f_cano, x_cano).reshape(num_pixels_total, -1).contiguous()
    off = torch.empty(num_pixels_total, dtype=torch.uint8, device=sd.device)
    inn = torch.empty_like(off)
    check(lib().hold_off_in_surface(ctx.h, num_pixels_total, sd.shape[1], ptr(sd), float(threshold), ptr(off), ptr(inn), stream_ptr()))
    return off.bool(), inn.bool()


def sampler_round(node, it: int, z_new, sdf_new, beta_in, far, z_old=None, sdf_old=None):
    """One while-loop iteration of ErrorBoundSampler.get_z_vals (engine/ray_sampler.py:160-311) on caller-supplied state
    (hold_sampler_round).  Returns dict(z, sdf [merged], beta, samples, upsample)."""
    R, Ne = z_new.shape
    dev = z_new.device
    n = (it + 1) * Ne
    S = node.S
    f = lambda t: None if t is None else t.float().contiguous()
    z_new, sdf_new, beta_in, far, z_old, sdf_old = f(z_new), f(sdf_new), f(beta_in), f(far.reshape(-1)), f(z_old), f(sdf_old)
    zm, sm = torch.empty(R, n, device=dev), torch.empty(R, n, device=dev)
    beta_out = torch.empty(R, device=dev)
    samples = torch.empty(R, max(Ne, S), device=dev)
    up = C.c_int32(0)
    beta_param = node.density.beta.detach().float().reshape(1).contiguous()
    check(lib().hold_sampler_round(node.ctx.h, node.slot, R, it, ptr(z_old), ptr(sdf_old), ptr(z_new), ptr(sdf_new), ptr(beta_in),
                                   ptr(far), ptr(beta_param), ptr(zm), ptr(sm), ptr(beta_out), ptr(samples), C.byref(up), stream_ptr()))
    ncol = Ne if up.value else S
    return dict(z=zm, sdf=sm, beta=beta_out, samples=samples.reshape(-1)[: R * ncol].reshape(R, ncol), upsample=bool(up.value))
