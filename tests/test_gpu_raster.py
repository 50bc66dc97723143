"""hold_raster_silhouette / hold_raster_silhouette_bwd (pytorch3d's MeshRasterizer + SoftSilhouetteShader, fitting/utils.py:101-118)
against the float64 oracle (oracle/soft_raster_oracle.py): fragments, silhouette, vertex gradients, batch independence, argument
rejection, and a pose refinement end to end.  New kernels: each case runs in a fresh interpreter (`isolated`)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import soft_raster_oracle as R
from oracle.mesh_sdf_oracle import star_mesh

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _cfg(K, sigma, blur, persp, clip, cull):
    from hold_b200.capi import RasterCfg

    return RasterCfg(K, int(persp), int(clip), int(cull), float(blur), float(sigma))


def _render(c, v, faces, H, W, cfg, frags=True):
    from hold_b200.capi import check, lib, ptr, stream_ptr

    B, V, _ = v.shape
    K = cfg.faces_per_pixel
    sil = torch.full((B, H, W), float("nan"), device=DEV)
    p2f = torch.empty(B, H, W, K, dtype=torch.int64, device=DEV) if frags else None
    zb = torch.empty(B, H, W, K, device=DEV) if frags else None
    di = torch.empty(B, H, W, K, device=DEV) if frags else None
    check(lib().hold_raster_silhouette(c.h, B, V, ptr(v), faces.shape[0], ptr(faces), H, W, C.byref(cfg), ptr(sil), ptr(p2f), ptr(zb),
                                       ptr(di), stream_ptr()))
    c.check()
    return sil, p2f, zb, di


def _render_bwd(c, v, faces, H, W, cfg, g):
    from hold_b200.capi import check, lib, ptr, stream_ptr

    B, V, _ = v.shape
    gv = torch.full((B, V, 3), float("nan"), device=DEV)
    check(lib().hold_raster_silhouette_bwd(c.h, B, V, ptr(v), faces.shape[0], ptr(faces), H, W, C.byref(cfg), ptr(g), ptr(gv), stream_ptr()))
    c.check()
    return gv


def _star_ndc(B, H, W, depths, seed=0):
    """The closed star mesh at the given depths, rotated per frame, in pytorch3d NDC (through fitting.project_ndc)."""
    from hold_b200 import fitting
    from oracle.hold_oracle import axis_angle_to_matrix

    vs, fs = star_mesh(level=3, seed=seed)
    g = torch.Generator().manual_seed(seed)
    rot = axis_angle_to_matrix(torch.randn(B, 3, generator=g, dtype=torch.float64))
    v = torch.einsum("bij,vj->bvi", rot, torch.from_numpy(vs).double())
    v[..., 2] += torch.tensor(depths, dtype=torch.float64)[:, None]
    v[..., 0] += 0.2
    f = 0.9 * min(H, W)
    K = torch.tensor([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], dtype=torch.float64)
    return fitting.project_ndc(v, K, H, W).float(), torch.from_numpy(fs.astype(np.int32))


def _quad_stack(n=150, seed=0):
    """n slightly offset quads (2 faces each) covering most of the image at depths 1 + 0.01 k: many pixels have > K candidates."""
    g = torch.Generator().manual_seed(seed)
    vs, fs = [], []
    for k in range(n):
        o = (torch.rand(2, generator=g) - 0.5) * 0.2
        x0, x1, y0, y1 = -0.8 + o[0], 0.8 + o[0], -0.7 + o[1], 0.7 + o[1]
        z = 1.0 + 0.01 * k
        vs += [[x0, y0, z], [x1, y0, z], [x1, y1, z], [x0, y1, z]]
        fs += [[4 * k, 4 * k + 1, 4 * k + 2], [4 * k, 4 * k + 2, 4 * k + 3]]
    perm = torch.randperm(n, generator=g)     # faces not in depth order
    f = torch.tensor(fs, dtype=torch.int32).view(n, 2, 3)[perm].reshape(-1, 3)
    return torch.tensor(vs, dtype=torch.float32)[None], f


def _random_tris(B, n, seed):
    """Random triangles of both orientations, some straddling z = 0 or wholly behind it, some of zero area."""
    g = torch.Generator().manual_seed(seed)
    xy = torch.rand(B, n, 3, 2, generator=g) * 2.4 - 1.2
    xy = xy.mean(2, keepdim=True) + (xy - xy.mean(2, keepdim=True)) * 0.35
    z = torch.rand(B, n, 3, generator=g) * 3.0 + 0.5
    z[:, : n // 8] -= 2.5                                  # straddling z = 0 or behind it
    xy[:, n // 8: n // 8 + 6, 2] = xy[:, n // 8: n // 8 + 6, 1]   # zero area
    v = torch.cat([xy, z[..., None]], -1).reshape(B, n * 3, 3)
    f = torch.arange(n * 3, dtype=torch.int32).view(n, 3)
    return v.contiguous(), f


def _check_case(c, v, faces, H, W, K, sigma=1e-4, blur=None, persp=True, clip=None, cull=False, grad=True, label=""):
    blur = R.default_blur_radius(sigma) if blur is None else blur
    clip = blur > 0 if clip is None else clip
    cfg = _cfg(K, sigma, blur, persp, clip, cull)
    vd, fd = v.to(DEV).contiguous(), faces.to(DEV).contiguous()
    B, F = v.shape[0], faces.shape[0]
    sil, p2f, zb, di = _render(c, vd, fd, H, W, cfg)
    sil_nf = _render(c, vd, fd, H, W, cfg, frags=False)[0]
    assert torch.equal(sil, sil_nf), label                       # the fragment outputs change nothing

    # the float32 effective blur radius is what the kernel compares with
    blur32 = float(torch.tensor(blur, dtype=torch.float32))
    cand = R.candidates(v.double(), faces, H, W, blur32, persp, clip, cull)
    sel_o = R.select(cand, K)
    p2f, zb, di = p2f.cpu().reshape(B, H * W, K), zb.cpu().reshape(B, H * W, K), di.cpu().reshape(B, H * W, K)
    sel_k = torch.where(p2f >= 0, p2f - torch.arange(B)[:, None, None] * F, p2f)
    assert ((sel_k >= -1) & (sel_k < F)).all()
    # slots are filled from the front and sorted by (pz, face)
    filled = sel_k >= 0
    assert (filled[..., 1:] <= filled[..., :-1]).all()
    assert ((zb[..., 1:] >= zb[..., :-1]) | ~filled[..., 1:]).all()

    # the kept face set equals the oracle's, up to exact pz ties at the K-th key and decisions on the blur boundary
    a, _ = sel_k.sort(-1)
    b, _ = sel_o.sort(-1)
    bad = (a != b).any(-1)
    n_bad = int(bad.sum())
    pz, dist = cand["pz"], cand["dist"]
    for bb, pp in bad.nonzero().tolist():
        ks, os_ = set(a[bb, pp].tolist()) - {-1}, set(b[bb, pp].tolist()) - {-1}
        kth = max(pz[bb, pp, f].item() for f in os_) if os_ else 0.0
        for f in ks ^ os_:
            tie = abs(pz[bb, pp, f].item() - kth) <= 1e-5 * max(kth, 1e-3)
            edge = abs(dist[bb, pp, f].item() - blur32) <= 1e-6 * max(blur32, 1e-6)
            assert tie or edge, (label, bb, pp, f, sorted(ks), sorted(os_))
    assert n_bad <= max(2, B * H * W // 20), (label, n_bad)

    # fragments against the oracle's values for the kernel's selection
    idx = sel_k.clamp_min(0)
    pz_r = pz.gather(-1, idx)
    sd_r = torch.where(cand["inside"], -dist, dist).gather(-1, idx)
    # relative to the face's depth scale: for a face straddling z = 0, pz near 0 is a cancellation of its vertices' depths
    zscale = v[..., 2].double().abs()[:, faces.long()].amax(-1)                       # [B,F]
    zscale = torch.maximum(pz_r.abs(), zscale.gather(1, idx.reshape(B, -1)).reshape(idx.shape))
    # pz is ill-conditioned in float32 (as in pytorch3d) where it extrapolates the face's plane from barycentrics outside
    # [0, 1] (no clipping; thin faces) or where the perspective correction mixes depths of both signs (a face straddling
    # z = 0).  Where a face in front of the camera interpolates (sum |c| = 1, always with clipping) the bound is 2e-6 (thin
    # random faces reach 1.7e-6; the star mesh and the quads stay within 1e-6).  Where it extrapolates (edge-on faces of the
    # star reach 3.3e-5 without clipping, thin random faces 2e-4) or straddles z = 0, only a sanity bound applies.
    front = (v[..., 2].double()[:, faces.long()].amin(-1) > 0)                       # [B,F]
    front = front.gather(1, idx.reshape(B, -1)).reshape(idx.shape) & filled
    strict = front & (cand["csum"].gather(-1, idx) <= 1.0 + 1e-9)
    zerr_all = (zb.double() - pz_r).abs() / zscale
    zerr, zerr_x = zerr_all[strict], zerr_all[filled & ~strict]
    derr = (di.double() - sd_r).abs()[filled]
    assert zerr.numel() == 0 or zerr.max() <= 2e-6, (label, zerr.max())
    assert zerr_x.numel() == 0 or zerr_x.max() <= 1e-3, (label, zerr_x.max())
    assert derr.numel() == 0 or derr.max() <= 1e-6, (label, derr.max())
    assert (p2f[~filled] == -1).all() and (zb[~filled] == -1).all() and (di[~filled] == -1).all()

    # silhouette against the oracle's blend over the same selection
    v64 = v.double().requires_grad_(True)
    ref = R.silhouette_from_selection(v64, faces, H, W, sel_k, sigma, persp)
    err = (sil.cpu().double() - ref.detach()).abs().max().item()
    assert err <= 1e-6, (label, err)
    print(f"{label}: mismatched pixels {n_bad}, zbuf rel {zerr.max().item() if zerr.numel() else 0:.2e}, sil max|d| {err:.2e}, "
          f"covered {(ref > 0.5).double().mean().item():.2f}")
    if grad:
        g = torch.Generator().manual_seed(11)
        gs = torch.randn(B, H, W, generator=g)
        gv = _render_bwd(c, vd, fd, H, W, cfg, gs.to(DEV)).cpu()
        (ref * gs.double()).sum().backward()
        gref = v64.grad
        gmax = gref.abs().max().item()
        assert gmax > 0, label
        gerr = (gv.double() - gref).abs().max().item()
        assert gerr <= 1e-5 * gmax, (label, gerr, gmax)
        assert (gv[..., 2] == 0).all()
        print(f"{label}: g_verts max|d| {gerr:.2e} of max|g| {gmax:.2e}")
    return sil, sel_k


# ---------------------------------------------------------------------------------------------------------- cases


def impl_star(c):
    for H, W in ((64, 64), (48, 80), (80, 48)):
        v, f = _star_ndc(2, H, W, [2.6, 4.0])
        for K in (1, 8, 100):
            _check_case(c, v, f, H, W, K, label=f"star {H}x{W} K{K}")
    v, f = _star_ndc(2, 64, 64, [3.0, 5.0], seed=1)
    _check_case(c, v, f, 64, 64, 8, blur=0.0, label="star blur 0")                       # clipping off with blur 0
    _check_case(c, v, f, 64, 64, 8, persp=False, label="star no perspective")
    _check_case(c, v, f, 64, 64, 8, clip=False, label="star no clip")
    _check_case(c, v, f, 64, 64, 8, cull=True, label="star culled")
    _check_case(c, v, f, 64, 64, 100, sigma=1e-4, label="star sigma 1e-4")


def impl_edges(c):
    v, f = _random_tris(2, 96, seed=3)
    for cull in (False, True):
        for persp in (True, False):
            for clip in (True, False):
                _check_case(c, v, f, 48, 80, 8, sigma=1e-3, persp=persp, clip=clip, cull=cull,
                            label=f"random cull{int(cull)} persp{int(persp)} clip{int(clip)}")
    # sigma 1e-3 as above: at 1e-4 the silhouette of these thin random faces is within 2.1e-6 (the star mesh: 1e-6)
    _check_case(c, v, f, 80, 48, 100, sigma=1e-3, blur=0.0, label="random blur 0")


def impl_quads(c):
    v, f = _quad_stack()
    for K in (1, 8, 100):
        sil, sel = _check_case(c, v, f, 64, 64, K, sigma=1e-3, label=f"quads K{K}")
        assert (sel >= 0).sum(-1).max() == K
    # the over-K path inside one tile next to pixels under K (the quads' ragged borders); interior pixels of these large faces
    # have p = 1 (1 - p = 0 in float32), so their gradient must come out 0, not NaN
    sil, _ = _check_case(c, v, f, 48, 80, 100, sigma=1e-4, label="quads 48x80 K100")
    assert (sil == 1.0).sum() > 200


def impl_batch(c):
    from hold_b200 import fitting

    v, f = _star_ndc(3, 48, 80, [2.5, 3.5, 6.0], seed=2)
    vd, fd = v.to(DEV), f.to(DEV)
    full = fitting.soft_silhouette(c, vd, fd, (48, 80), faces_per_pixel=8)
    for b in range(3):
        one = fitting.soft_silhouette(c, vd[b:b + 1].contiguous(), fd, (48, 80), faces_per_pixel=8)
        assert torch.equal(one[0], full[b]), b
    rgba = fitting.SilhouetteRenderer(c, (48, 80), faces_per_pixel=8)(vd, fd)
    assert rgba.shape == (3, 48, 80, 4) and torch.equal(rgba[..., 3], full) and (rgba[..., :3] == 1).all()


def impl_reject(c):
    from hold_b200 import fitting
    from hold_b200.capi import lib, ptr, stream_ptr

    v, f = _star_ndc(1, 32, 32, [3.0])
    vd, fd = v.to(DEV), f.to(DEV)
    sil = torch.empty(1, 32, 32, device=DEV)
    g = torch.zeros(1, 32, 32, device=DEV)
    gv = torch.empty(1, v.shape[1], 3, device=DEV)
    zb = torch.empty(1, 32, 32, 4, device=DEV)
    fw = lambda cfg, H=32, W=32, vp=ptr(vd), sp=ptr(sil), frag=(None, None, None): lib().hold_raster_silhouette(
        c.h, 1, v.shape[1], vp, f.shape[0], ptr(fd), H, W, cfg, sp, *frag, stream_ptr())
    ok = C.byref(_cfg(4, 1e-4, R.default_blur_radius(), 1, 1, 0))
    assert fw(ok) == 0
    for K in (0, -1, 1025):
        assert fw(C.byref(_cfg(K, 1e-4, 1e-3, 1, 1, 0))) == -1, K
    assert fw(C.byref(_cfg(4, 0.0, 1e-3, 1, 1, 0))) == -1            # sigma must be > 0
    assert fw(C.byref(_cfg(4, 1e-4, -1.0, 1, 1, 0))) == -1           # blur_radius >= 0
    assert fw(ok, H=0) == -1 and fw(ok, W=0) == -1 and fw(ok, H=-3) == -1
    assert fw(ok, vp=None) == -1 and fw(ok, sp=None) == -1 and fw(None) == -1
    assert fw(ok, frag=(None, ptr(zb), None)) == -1                   # fragments: all three or none
    assert lib().hold_raster_silhouette_bwd(c.h, 1, v.shape[1], ptr(vd), f.shape[0], ptr(fd), 32, 32, ok, None, ptr(gv), stream_ptr()) == -1
    assert lib().hold_raster_silhouette_bwd(c.h, 1, v.shape[1], ptr(vd), f.shape[0], ptr(fd), 32, 32, ok, ptr(g), None, stream_ptr()) == -1
    c.check()
    # out-of-range face indices are refused in Python before any launch
    n0 = c.launches
    hi, lo = f.clone(), f.clone()
    hi[5, 1] = v.shape[1]
    lo[0, 0] = -1
    for ff in (hi, lo):
        with pytest.raises(ValueError):
            fitting.soft_silhouette(c, vd, ff.to(DEV), 32)
    with pytest.raises(ValueError):
        fitting.soft_silhouette(c, vd, fd, 32, faces_per_pixel=0)
    assert c.launches == n0


def impl_refine(c):
    """Pose refinement as optimize_ckpt.py runs it: target silhouette of the star mesh posed by hold_object_tf, start from a
    perturbed pose, 50 Adam steps on L1(silhouette, target) through project_ndc -> SoftSilhouetteFn -> hold_object_tf_bwd."""
    from hold_b200 import fitting
    from hold_b200.model import ObjectServer

    vs, fs = star_mesh(level=3, seed=0)
    srv = ObjectServer(c, torch.from_numpy(vs))
    faces = torch.from_numpy(fs.astype(np.int32)).to(DEV)
    H = W = 64
    Kc = torch.tensor([[60.0, 0, 32.0], [0, 60.0, 32.0], [0, 0, 1]], device=DEV)
    scale = torch.ones(1, device=DEV)
    rot_t = torch.tensor([[0.3, -0.2, 0.5]], device=DEV)
    tr_t = torch.tensor([[0.1, -0.15, 5.0]], device=DEV)
    sig = 1e-3
    render = lambda r, t: fitting.soft_silhouette(c, fitting.project_ndc(srv.forward(scale, t, r)["verts"], Kc, H, W), faces, (H, W),
                                                  faces_per_pixel=50, sigma=sig)
    with torch.no_grad():
        target = render(rot_t, tr_t)
    rot = (rot_t + torch.tensor([[0.15, 0.1, -0.15]], device=DEV)).requires_grad_(True)
    tr = (tr_t + torch.tensor([[0.12, -0.1, 0.3]], device=DEV)).requires_grad_(True)
    opt = torch.optim.Adam([rot, tr], lr=0.02)
    losses = []
    for _ in range(50):
        opt.zero_grad()
        loss = (render(rot, tr) - target).abs().mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    final = (render(rot, tr) - target).abs().mean().item()
    dt = (tr - tr_t).abs().max().item()
    print(f"refine: loss {losses[0]:.4f} -> {final:.5f}, |translation error| {dt:.4f}, rotation error {(rot - rot_t).abs().max().item():.4f}")
    assert final <= losses[0] / 10, (losses[0], final)
    assert dt <= 0.05, dt


@pytest.mark.parametrize("case", ["impl_star", "impl_edges", "impl_quads", "impl_batch", "impl_reject", "impl_refine"])
def test_raster(isolated, case):
    isolated("tests/test_gpu_raster.py", case, timeout=900)
