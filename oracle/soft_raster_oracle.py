"""Float64 restatement of the soft-silhouette rasteriser: pytorch3d v0.7.4's MeshRasterizer (rasterize_meshes) and
SoftSilhouetteShader (sigmoid_alpha_blend), as hold_b200/csrc/raster_phases.h states them.  pytorch3d is not available to pin
this; the two files encode the same rules and change together (DESIGN.md row 4c).

The selection loops over the faces in index order with an explicit K-slot queue, as pytorch3d's naive kernel does, so it does
not share the threshold selection of the CUDA kernel.  `silhouette_from_selection` recomputes the kept faces' distances from
the vertices, so torch.autograd in float64 gives the reference gradient for a given selection.
"""
from __future__ import annotations

import math

import torch

EPS = 1e-8


def default_blur_radius(sigma=1e-4):
    """pytorch3d's soft-silhouette recipe: blur_radius = ln(1 / 1e-4 - 1) * sigma."""
    return math.log(1.0 / 1e-4 - 1.0) * sigma


def pixel_centres(H, W, dtype=torch.float64):
    """(x [W], y [H]) of the pixel centres: x = (W - 2j - 1) / s, y = (H - 2i - 1) / s, s = min(H, W), computed in float32
    as the rasteriser does (they are inputs of the arithmetic, like the float32 vertices), returned as `dtype`."""
    s = min(H, W)
    x = (W - 2 * torch.arange(W, dtype=torch.float32) - 1) / s
    y = (H - 2 * torch.arange(H, dtype=torch.float32) - 1) / s
    return x.to(dtype), y.to(dtype)


def edge_fn(px, py, ax, ay, bx, by):
    return (px - ax) * (by - ay) - (py - ay) * (bx - ax)


def barycentric(px, py, v):
    """v [..., 3, 2] -> screen barycentrics [..., 3] (area + 1e-8 in the denominator, as BarycentricCoordsForward)."""
    x0, y0, x1, y1, x2, y2 = v[..., 0, 0], v[..., 0, 1], v[..., 1, 0], v[..., 1, 1], v[..., 2, 0], v[..., 2, 1]
    area = edge_fn(x2, y2, x0, y0, x1, y1) + EPS
    return torch.stack([edge_fn(px, py, x1, y1, x2, y2) / area, edge_fn(px, py, x2, y2, x0, y0) / area,
                        edge_fn(px, py, x0, y0, x1, y1) / area], -1)


def perspective_correct(b, z):
    t = torch.stack([b[..., 0] * z[..., 1] * z[..., 2], z[..., 0] * b[..., 1] * z[..., 2], z[..., 0] * z[..., 1] * b[..., 2]], -1)
    return t / t.sum(-1, keepdim=True).clamp_min(EPS)


def clip_barycentric(b):
    c = b.clamp_min(0.0)
    return c / c.sum(-1, keepdim=True).clamp_min(EPS)


def seg_sqdist(px, py, a, b):
    """Squared distance from p to segment a-b (a, b [..., 2]); a segment of squared length <= 1e-8 counts as its end b."""
    ba = b - a
    pa = torch.stack([px - a[..., 0], py - a[..., 1]], -1)
    l2 = (ba * ba).sum(-1)
    t = ((ba * pa).sum(-1) / torch.where(l2 <= EPS, torch.ones_like(l2), l2)).clamp(0.0, 1.0)
    d = pa - t[..., None] * ba
    pb = torch.stack([px - b[..., 0], py - b[..., 1]], -1)
    return torch.where(l2 <= EPS, (pb * pb).sum(-1), (d * d).sum(-1))


def tri_sqdist(px, py, v):
    """Squared distance to the nearest of the edges (v0, v1), (v0, v2), (v1, v2) -> (dist, edge: the first of equals)."""
    d = torch.stack([seg_sqdist(px, py, v[..., 0, :], v[..., 1, :]), seg_sqdist(px, py, v[..., 0, :], v[..., 2, :]),
                     seg_sqdist(px, py, v[..., 1, :], v[..., 2, :])], -1)
    e = torch.argmin(d.detach(), -1)   # argmin returns the first minimal index
    return d.gather(-1, e[..., None])[..., 0], e


def candidates(verts_ndc, faces, H, W, blur_radius, perspective_correct_=True, clip_barycentric_coords=None, cull_backfaces=False):
    """Every (pixel, face) candidate of frame-batched meshes, float64.  verts_ndc [B,V,3], faces [F,3].
    Returns dict of [B, H*W, F] tensors: ok (candidate), pz, dist, inside, and csum = sum |c| of the barycentrics pz
    interpolates with (> 1 where an unclipped pz extrapolates the face's plane)."""
    if clip_barycentric_coords is None:
        clip_barycentric_coords = blur_radius > 0
    v = verts_ndc.double()
    fv = v[:, faces.long()]                                       # [B,F,3,3]
    xy, z = fv[..., :2], fv[..., 2]
    xs, ys = pixel_centres(H, W)
    py = ys[:, None].expand(H, W).reshape(1, -1, 1)
    px = xs[None, :].expand(H, W).reshape(1, -1, 1)
    xy_, z_ = xy[:, None], z[:, None]                              # [B,1,F,3,(2)]
    area = edge_fn(xy[..., 0, 0], xy[..., 0, 1], xy[..., 1, 0], xy[..., 1, 1], xy[..., 2, 0], xy[..., 2, 1])
    skip_face = (z.amax(-1) < 0) | (area.abs() <= EPS) | (cull_backfaces & (area < 0))      # [B,F]
    r = math.sqrt(blur_radius)
    xmin, xmax = xy[..., 0].amin(-1) - r, xy[..., 0].amax(-1) + r
    ymin, ymax = xy[..., 1].amin(-1) - r, xy[..., 1].amax(-1) + r
    outside = (px > xmax[:, None]) | (px < xmin[:, None]) | (py > ymax[:, None]) | (py < ymin[:, None])
    b = barycentric(px, py, xy_)
    if perspective_correct_:
        b = perspective_correct(b, z_)
    c = clip_barycentric(b) if clip_barycentric_coords else b
    pz = (c * z_).sum(-1)
    dist, _ = tri_sqdist(px, py, xy_)
    inside = (b > 0).all(-1)
    ok = ~skip_face[:, None] & ~outside & (pz >= 0) & (inside | (dist < blur_radius))
    return {"ok": ok, "pz": pz, "dist": dist, "inside": inside, "csum": c.abs().sum(-1)}


def select(cand, K):
    """pytorch3d's per-pixel queue, faces in index order: keep the K candidates of smallest (pz, face).
    Returns face [B, P, K] int64 sorted by (pz, face), -1 in empty slots."""
    ok, pz = cand["ok"], cand["pz"]
    B, P, F = ok.shape
    qz = torch.full((B, P, K), math.inf, dtype=torch.float64)
    qf = torch.full((B, P, K), -1, dtype=torch.int64)
    for f in range(F):
        # the slot to replace: the largest key (pz, face); empty slots hold +inf.  A later face has the larger index, so it
        # replaces only a strictly larger pz.
        mz = qz.amax(-1, keepdim=True)
        slot = torch.where(qz == mz, qf, torch.full_like(qf, -2)).argmax(-1, keepdim=True)
        take = ok[:, :, f] & (pz[:, :, f] < mz[..., 0])
        qz.scatter_(-1, slot, torch.where(take[..., None], pz[:, :, f:f + 1], qz.gather(-1, slot)))
        qf.scatter_(-1, slot, torch.where(take[..., None], torch.full_like(slot, f), qf.gather(-1, slot)))
    o = torch.argsort(qf, dim=-1, stable=True)                    # secondary key: the face
    qz, qf = qz.gather(-1, o), qf.gather(-1, o)
    o = torch.argsort(qz, dim=-1, stable=True)                    # primary key: pz (empty slots hold +inf: last)
    return qf.gather(-1, o)


def silhouette_from_selection(verts_ndc, faces, H, W, sel, sigma, perspective_correct_=True):
    """silhouette [B,H,W] = 1 - prod_k sigmoid(signed_dist_k / sigma) over the selected faces sel [B, H*W, K] (-1 = empty),
    differentiable with respect to verts_ndc (through the nearest edge's squared distance; inside/outside is held fixed)."""
    B = verts_ndc.shape[0]
    K = sel.shape[-1]
    fidx = sel.clamp_min(0)
    fv = verts_ndc[:, faces.long()]                                # [B,F,3,3]
    g = torch.gather(fv, 1, fidx.reshape(B, -1)[..., None, None].expand(-1, -1, 3, 3)).reshape(B, H * W, K, 3, 3)
    xs, ys = pixel_centres(H, W, verts_ndc.dtype)
    py = ys[:, None].expand(H, W).reshape(1, -1, 1)
    px = xs[None, :].expand(H, W).reshape(1, -1, 1)
    with torch.no_grad():
        b = barycentric(px, py, g[..., :2])
        if perspective_correct_:
            b = perspective_correct(b, g[..., 2])
        inside = (b > 0).all(-1)
    dist, _ = tri_sqdist(px, py, g[..., :2])
    sd = torch.where(inside, -dist, dist)
    q = torch.where(sel >= 0, torch.sigmoid(sd / sigma), torch.ones_like(sd))     # 1 - p, exact when p is near 1
    return (1.0 - q.prod(-1)).reshape(B, H, W)


def fragments(verts_ndc, faces, H, W, sel, cand):
    """pytorch3d's fragments for the selection: pix_to_face (packed b*F + f), zbuf, dists [B,H,W,K], -1 in empty slots."""
    B, P, K = sel.shape
    F = faces.shape[0]
    idx = sel.clamp_min(0)
    empty = sel < 0
    pz = cand["pz"].gather(-1, idx).masked_fill(empty, -1.0)
    sd = torch.where(cand["inside"], -cand["dist"], cand["dist"]).gather(-1, idx).masked_fill(empty, -1.0)
    p2f = (sel + torch.arange(B)[:, None, None] * F).masked_fill(empty, -1)
    return p2f.reshape(B, H, W, K), pz.reshape(B, H, W, K), sd.reshape(B, H, W, K)


def soft_silhouette(verts_ndc, faces, H, W, K, sigma=1e-4, blur_radius=None, perspective_correct_=True,
                    clip_barycentric_coords=None, cull_backfaces=False):
    """The whole contract: (silhouette [B,H,W], selection [B,H*W,K], candidates)."""
    if blur_radius is None:
        blur_radius = default_blur_radius(sigma)
    if clip_barycentric_coords is None:
        clip_barycentric_coords = blur_radius > 0
    cand = candidates(verts_ndc.detach(), faces, H, W, blur_radius, perspective_correct_, clip_barycentric_coords, cull_backfaces)
    sel = select(cand, K)
    sil = silhouette_from_selection(verts_ndc.double(), faces, H, W, sel, sigma, perspective_correct_)
    return sil, sel, cand
