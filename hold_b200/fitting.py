"""The pytorch3d pieces of optimize_ckpt.py's pose refinement (fitting/utils.py:101-118, fitting/loss.py:90,131,134), without
pytorch3d: a perspective projection to pytorch3d NDC, the soft-silhouette renderer (MeshRasterizer + SoftSilhouetteShader on
the library's sm_90a kernels, hold_raster_silhouette / _bwd) and knn_points for the contact term.

The rasteriser's rules are pytorch3d v0.7.4's, restated and unpinned (hold_b200/csrc/raster_phases.h, DESIGN.md row 4c).
"""
from __future__ import annotations

import collections
import math

import torch
from torch import nn

from .capi import RASTER_MAX_K, RasterCfg, check, lib, ptr, stream_ptr


def default_blur_radius(sigma=1e-4):
    """pytorch3d's soft-silhouette recipe: blur_radius = ln(1 / 1e-4 - 1) * sigma (compared with the squared distance)."""
    return math.log(1.0 / 1e-4 - 1.0) * sigma


def project_ndc(verts_cam, K, H, W):
    """OpenCV camera coordinates verts_cam [B,V,3] and intrinsics K ([B,3,3], [3,3] or the 4x4 forms) -> pytorch3d NDC
    [B,V,3]: x = (W/2 - (fx X/Z + cx)) 2/s, y = (H/2 - (fy Y/Z + cy)) 2/s, z = Z, s = min(H, W).  This is pytorch3d's
    cameras_from_opencv_projection + transform_points_ndc, restated (unpinned).  Plain torch ops, differentiable."""
    K = K if K.dim() == 3 else K[None]
    fx, fy, cx, cy = (K[:, r, c][:, None] for r, c in ((0, 0), (1, 1), (0, 2), (1, 2)))
    X, Y, Z = verts_cam.unbind(-1)
    s = min(H, W)
    x = (W / 2 - (fx * X / Z + cx)) * (2.0 / s)
    y = (H / 2 - (fy * Y / Z + cy)) * (2.0 / s)
    return torch.stack([x, y, Z], -1)


def _cfg(faces_per_pixel, blur_radius, sigma, perspective_correct, clip_barycentric_coords, cull_backfaces):
    if blur_radius is None:
        blur_radius = default_blur_radius(sigma)
    if clip_barycentric_coords is None:
        clip_barycentric_coords = blur_radius > 0
    return RasterCfg(int(faces_per_pixel), int(bool(perspective_correct)), int(bool(clip_barycentric_coords)),
                     int(bool(cull_backfaces)), float(blur_radius), float(sigma))


def check_faces(faces, V, device):
    """faces as contiguous int32 [F,3] on `device`, every index in [0, V).  One min / max over F x 3 ints, read by the host:
    this synchronises the stream once per call."""
    if faces.dim() != 2 or faces.shape[1] != 3 or faces.shape[0] == 0:
        raise ValueError(f"faces must be [F,3] with F >= 1, got {tuple(faces.shape)}")
    f = faces.to(device=device, dtype=torch.int32).contiguous()
    lo, hi = torch.aminmax(f)
    lo, hi = int(lo), int(hi)
    if lo < 0 or hi >= V:
        raise ValueError(f"face indices span [{lo}, {hi}], outside [0, {V})")
    return f


class SoftSilhouetteFn(torch.autograd.Function):
    """silhouette [B,H,W] of verts_ndc [B,V,3] (differentiable in x and y) over faces [F,3] int32 (already checked):
    forward = hold_raster_silhouette, backward = hold_raster_silhouette_bwd."""

    @staticmethod
    def forward(fctx, verts_ndc, faces, ctx, H, W, cfg):
        v = verts_ndc.detach().float().contiguous()
        B, V, _ = v.shape
        sil = torch.empty(B, H, W, device=v.device)
        check(lib().hold_raster_silhouette(ctx.h, B, V, ptr(v), faces.shape[0], ptr(faces), H, W, cfg, ptr(sil), None, None, None,
                                           stream_ptr()))
        fctx.ctx, fctx.H, fctx.W, fctx.cfg = ctx, H, W, cfg
        fctx.save_for_backward(v, faces)
        return sil

    @staticmethod
    def backward(fctx, g_sil):
        v, faces = fctx.saved_tensors
        B, V, _ = v.shape
        g = torch.empty(B, V, 3, device=v.device)
        check(lib().hold_raster_silhouette_bwd(fctx.ctx.h, B, V, ptr(v), faces.shape[0], ptr(faces), fctx.H, fctx.W, fctx.cfg,
                                               ptr(g_sil.float().contiguous()), ptr(g), stream_ptr()))
        return g, None, None, None, None, None


def soft_silhouette(ctx, verts_ndc, faces, image_size, faces_per_pixel=100, blur_radius=None, sigma=1e-4, perspective_correct=True,
                    clip_barycentric_coords=None, cull_backfaces=False):
    """Soft silhouette [B,H,W] of the meshes (verts_ndc [B,V,3] in pytorch3d NDC with view-space z, faces [F,3] shared by the
    frames).  Defaults follow pytorch3d's soft-silhouette recipe: blur_radius = ln(1/1e-4 - 1) sigma, clipping on exactly
    when blur_radius > 0.  Checks faces against V on the host first (one stream synchronisation)."""
    H, W = (image_size, image_size) if isinstance(image_size, int) else tuple(image_size)
    if not 1 <= faces_per_pixel <= RASTER_MAX_K:
        raise ValueError(f"faces_per_pixel {faces_per_pixel} outside [1, {RASTER_MAX_K}]")
    f = check_faces(faces, verts_ndc.shape[1], verts_ndc.device)
    cfg = _cfg(faces_per_pixel, blur_radius, sigma, perspective_correct, clip_barycentric_coords, cull_backfaces)
    return SoftSilhouetteFn.apply(verts_ndc, f, ctx, H, W, cfg)


class SilhouetteRenderer(nn.Module):
    """MeshRenderer(MeshRasterizer, SoftSilhouetteShader): forward(verts_ndc, faces) -> [B,H,W,4], rgb = 1 and alpha = the
    soft silhouette."""

    def __init__(self, ctx, image_size, blur_radius=None, faces_per_pixel=100, perspective_correct=True,
                 clip_barycentric_coords=None, cull_backfaces=False, sigma=1e-4):
        super().__init__()
        self.ctx, self.image_size = ctx, image_size
        self.kw = dict(faces_per_pixel=faces_per_pixel, blur_radius=blur_radius, sigma=sigma, perspective_correct=perspective_correct,
                       clip_barycentric_coords=clip_barycentric_coords, cull_backfaces=cull_backfaces)

    def forward(self, verts_ndc, faces):
        sil = soft_silhouette(self.ctx, verts_ndc, faces, self.image_size, **self.kw)
        return torch.cat([torch.ones(sil.shape + (3,), device=sil.device, dtype=sil.dtype), sil[..., None]], -1)


KNN = collections.namedtuple("KNN", ["dists", "idx", "knn"])


def knn_points(p1, p2, K=1):
    """pytorch3d.ops.knn_points for equal-length batches: p1 [N,P1,D], p2 [N,P2,D] -> dists [N,P1,K] (squared, ascending),
    idx [N,P1,K] int64, knn [N,P1,K,D].  Differentiable through dists (and knn).  Brute force in torch: the contact term
    compares fingertips with object vertices, a few thousand pairs."""
    d = ((p1[:, :, None, :] - p2[:, None, :, :]) ** 2).sum(-1)
    dists, idx = torch.topk(d, K, dim=-1, largest=False, sorted=True)
    knn = torch.gather(p2[:, None].expand(-1, p1.shape[1], -1, -1), 2, idx[..., None].expand(-1, -1, -1, p2.shape[-1]))
    return KNN(dists, idx, knn)
