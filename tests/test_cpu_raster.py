"""CPU-only: the soft-silhouette rasteriser's per-pixel steps as the CUDA kernels run them (hold_b200/csrc/raster_phases.h
compiled for the host) against the float64 oracle (oracle/soft_raster_oracle.py); the oracle's gradient against finite
differences; fitting.project_ndc and fitting.knn_points."""
import ctypes as C
import math
import os
import subprocess

import pytest
import torch

from hold_b200 import fitting
from oracle import soft_raster_oracle as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    out = os.path.join(ROOT, "tests", "_build", "libraster_host.so")
    src = os.path.join(ROOT, "tests", "host", "raster_host.cpp")
    hdr = os.path.join(ROOT, "hold_b200", "csrc", "raster_phases.h")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    return C.CDLL(out)


_p = lambda t: C.c_void_p(t.data_ptr())


def _tris(n, g, zlo=0.5, zhi=3.0):
    """n random triangles [n,9] (x0 y0 x1 y1 x2 y2 z0 z1 z2) and a point near each [n,2], float32."""
    xy = torch.rand(n, 3, 2, generator=g) * 2 - 1
    z = torch.rand(n, 3, generator=g) * (zhi - zlo) + zlo
    v = torch.cat([xy.reshape(n, 6), z], 1).contiguous()
    p = (xy.mean(1) + torch.randn(n, 2, generator=g) * 0.4).contiguous()
    return v, p


@pytest.mark.parametrize("H,W", [(64, 64), (48, 80), (80, 48), (1, 7)])
def test_pixel_centres(H, W):
    lib = _lib()
    x, y = torch.empty(W), torch.empty(H)
    lib.pix_ndc_host(H, W, _p(x), _p(y))
    xr, yr = R.pixel_centres(H, W)
    assert torch.equal(x, xr.float()) and torch.equal(y, yr.float())
    s = min(H, W)
    assert x[0].item() == pytest.approx((W - 1) / s) and x[-1].item() == pytest.approx(-(W - 1) / s)   # col 0 is left: +x
    assert y[0].item() == pytest.approx((H - 1) / s)                                                  # row 0 is the top: +y


def test_barycentrics_perspective_and_clip():
    lib = _lib()
    g = torch.Generator().manual_seed(0)
    n = 4000
    v, p = _tris(n, g)
    b, bp, c = (torch.empty(n, 3) for _ in range(3))
    lib.bary_host(n, _p(p), _p(v), _p(b), _p(bp), _p(c))
    v64, p64 = v.double(), p.double()
    xy = torch.stack([v64[:, 0:2], v64[:, 2:4], v64[:, 4:6]], 1)
    z = torch.stack([v64[:, 6], v64[:, 7], v64[:, 8]], 1)
    area = R.edge_fn(xy[:, 0, 0], xy[:, 0, 1], xy[:, 1, 0], xy[:, 1, 1], xy[:, 2, 0], xy[:, 2, 1]).abs()
    good = area > 5e-2                                              # well-conditioned triangles: float32 vs float64
    rb = R.barycentric(p64[:, 0], p64[:, 1], xy)
    rbp = R.perspective_correct(rb, z)
    rc = R.clip_barycentric(rbp)
    for a, r in ((b, rb), (bp, rbp), (c, rc)):
        err = ((a.double() - r).abs() / r.abs().clamp_min(1.0))[good].max().item()
        assert err < 1e-4, err
    assert (bp.sum(1) - 1).abs()[(b > 0).all(1) & good].max() < 1e-5  # inside the face perspective correction renormalises
    assert (c >= 0).all() and ((c.sum(1) - 1).abs() < 1e-5).all()    # clipping: non-negative, sums to 1
    inner = (bp > 0).all(1) & good
    assert ((c - bp)[inner].abs() < 1e-6).all()                      # inside the face clipping changes nothing


def test_segment_distance_and_reverse_mode():
    lib = _lib()
    g = torch.Generator().manual_seed(1)
    n = 4000
    p, a, b = (torch.rand(n, 2, generator=g) * 2 - 1 for _ in range(3))
    b[:50] = a[:50] + 1e-5                                           # degenerate segments: the distance to b
    p[50:100] = a[50:100] + 0.3 * (b[50:100] - a[50:100])            # on the segment
    gg = torch.randn(n, generator=g)
    d, ga, gb = torch.empty(n), torch.empty(n, 2), torch.empty(n, 2)
    lib.seg_host(n, _p(p), _p(a), _p(b), _p(gg), _p(d), _p(ga), _p(gb))
    a64, b64 = a.double().requires_grad_(True), b.double().requires_grad_(True)
    p64 = p.double()
    r = R.seg_sqdist(p64[:, 0], p64[:, 1], a64, b64)
    (r * gg.double()).sum().backward()
    assert (d.double() - r.detach()).abs().max() < 1e-6
    for x, ref in ((ga, a64.grad), (gb, b64.grad)):
        assert ((x.double() - ref).abs() / ref.abs().max()).max() < 1e-5


@pytest.mark.parametrize("persp,clip,cull", [(1, 1, 0), (0, 0, 0), (1, 0, 1), (0, 1, 1)])
def test_pixel_face_candidates(persp, clip, cull):
    """The whole per-(pixel, face) test: candidate or not, pz, squared distance, inside."""
    lib = _lib()
    g = torch.Generator().manual_seed(2 + persp + 2 * clip + 4 * cull)
    n = 6000
    v, p = _tris(n, g, zlo=-0.5)                                      # some faces straddle z = 0 or lie behind it
    v[:100, 2:4] = v[:100, 0:2]                                       # zero-area faces
    blur = 0.02
    ok, inside = torch.empty(n, dtype=torch.int32), torch.empty(n, dtype=torch.int32)
    pz, dist = torch.empty(n), torch.empty(n)
    lib.pixel_face_host(n, _p(p), _p(v), C.c_float(blur), C.c_float(1e-4), persp, clip, cull, _p(ok), _p(pz), _p(dist), _p(inside))
    p64 = p.double()
    xy = torch.stack([v[:, 0:2], v[:, 2:4], v[:, 4:6]], 1).double()
    z = v[:, 6:9].double()
    vv = torch.cat([xy, z[..., None]], -1)                           # [n,3,3] -> one face per frame
    ok_r, pz_r, d_r, in_r = [], [], [], []
    for k in range(0, n, 500):
        sl = slice(k, k + 500)
        # frame = one triangle, image = none: evaluate the oracle's candidate rule at the given point
        c = _oracle_point(p64[sl], vv[sl], blur, persp, clip, cull)
        ok_r.append(c[0]), pz_r.append(c[1]), d_r.append(c[2]), in_r.append(c[3])
    ok_r, pz_r, d_r, in_r = (torch.cat(t) for t in (ok_r, pz_r, d_r, in_r))
    assert ok_r[:100].sum() == 0 and ok[:100].sum() == 0
    # away from the decision boundaries the two agree exactly on the decisions
    clear = (d_r - blur).abs() > 1e-5
    assert torch.equal(ok.bool()[clear], ok_r[clear]), (ok.bool() != ok_r)[clear].sum()
    both = ok.bool() & ok_r
    assert both.sum() > n // 10
    assert ((pz.double() - pz_r).abs() / pz_r.abs().clamp_min(1e-3))[both].max() < 1e-4
    assert (dist.double() - d_r)[both].abs().max() < 1e-6
    edge = d_r < 1e-9
    assert torch.equal(inside.bool()[both & ~edge], in_r[both & ~edge])


def _oracle_point(p, vv, blur, persp, clip, cull):
    """The oracle's candidate rule at one point per triangle (the oracle's `candidates` over a 1-pixel image is the same
    arithmetic; this calls its pieces directly)."""
    xy, z = vv[..., :2], vv[..., 2]
    area = R.edge_fn(xy[:, 0, 0], xy[:, 0, 1], xy[:, 1, 0], xy[:, 1, 1], xy[:, 2, 0], xy[:, 2, 1])
    skip = (z.amax(-1) < 0) | (area.abs() <= R.EPS) | (bool(cull) & (area < 0))
    r = math.sqrt(blur)
    px, py = p[:, 0], p[:, 1]
    out = (px > xy[..., 0].amax(-1) + r) | (px < xy[..., 0].amin(-1) - r) | (py > xy[..., 1].amax(-1) + r) | (py < xy[..., 1].amin(-1) - r)
    b = R.barycentric(px, py, xy)
    if persp:
        b = R.perspective_correct(b, z)
    c = R.clip_barycentric(b) if clip else b
    pz = (c * z).sum(-1)
    d, _ = R.tri_sqdist(px, py, xy)
    inside = (b > 0).all(-1)
    return ~skip & ~out & (pz >= 0) & (inside | (d < blur)), pz, d, inside


def test_blend_with_exact_zero_factors():
    """silhouette and d sil / d signed_dist, with factors 1 - p that are exactly 0 in float32 (p = 1) and factors near 1."""
    lib = _lib()
    sigma = 1e-4
    cases = [
        [-0.05, 2e-4, 5e-4],             # one face deep inside: 1 - p = 0 in float32
        [-0.05, -0.02, 1e-4],            # two zero factors
        [1e-5, -1e-5, 3e-4, 8e-4],       # near the edges, no zero factor
        [-2e-3, 0.0],                    # 1 - p ~ 2e-9: tiny but non-zero
        [],                              # no kept face
    ]
    for sd in cases:
        m = len(sd)
        s32 = torch.tensor(sd, dtype=torch.float32)
        sil, dsd = torch.empty(1), torch.empty(max(m, 1))
        lib.blend_host(m, _p(s32) if m else None, C.c_float(sigma), _p(sil), _p(dsd))
        s64 = s32.double().requires_grad_(True)
        ref = 1.0 - torch.sigmoid(s64 / sigma).prod()
        if m:
            ref.backward()
            gmax = s64.grad.abs().max().item()
            assert (dsd[:m].double() - s64.grad).abs().max().item() <= 1e-6 * max(gmax, 1.0), (sd, dsd, s64.grad)
        assert abs(sil.item() - ref.item()) < 1e-6, (sd, sil, ref)
    # with a zero factor the silhouette is exactly 1
    sil, dsd, s32 = torch.empty(1), torch.empty(3), torch.tensor(cases[0], dtype=torch.float32)
    lib.blend_host(3, _p(s32), C.c_float(sigma), _p(sil), _p(dsd))
    assert sil.item() == 1.0 and (dsd[:3] == 0).all()


def test_oracle_gradient_matches_finite_differences():
    """The oracle's silhouette, for a fixed selection, is differentiable: its autograd gradient equals central differences."""
    g = torch.Generator().manual_seed(3)
    v = torch.tensor([[[0.5, 0.4, 2.0], [-0.3, 0.5, 2.2], [0.1, -0.5, 1.8], [-0.6, -0.2, 2.5]]], dtype=torch.float64)
    faces = torch.tensor([[0, 1, 2], [1, 3, 2]])
    H, W, sigma = 12, 10, 0.02
    blur = R.default_blur_radius(sigma)
    cand = R.candidates(v, faces, H, W, blur)
    sel = R.select(cand, 2)
    w = torch.randn(1, H, W, generator=g, dtype=torch.float64)
    vv = v.clone().requires_grad_(True)
    (R.silhouette_from_selection(vv, faces, H, W, sel, sigma) * w).sum().backward()
    h = 1e-6
    fd = torch.zeros_like(v)
    for k in range(v.numel()):
        vp, vm = v.clone().view(-1), v.clone().view(-1)
        vp[k] += h
        vm[k] -= h
        fp = (R.silhouette_from_selection(vp.view_as(v), faces, H, W, sel, sigma) * w).sum()
        fm = (R.silhouette_from_selection(vm.view_as(v), faces, H, W, sel, sigma) * w).sum()
        fd.view(-1)[k] = (fp - fm) / (2 * h)
    assert vv.grad.abs().max() > 1.0
    assert (vv.grad - fd).abs().max() <= 1e-5 * vv.grad.abs().max()
    assert (vv.grad[..., 2] == 0).all()                               # z carries no gradient


def test_oracle_selection_keeps_the_nearest():
    """select() keeps the K smallest (pz, face); equal pz: the lower face index."""
    cand = {"ok": torch.tensor([[[True, True, True, False, True]]]),
            "pz": torch.tensor([[[3.0, 1.0, 2.0, 0.5, 1.0]]], dtype=torch.float64)}
    assert R.select(cand, 2).tolist() == [[[1, 4]]]
    assert R.select(cand, 3).tolist() == [[[1, 4, 2]]]
    assert R.select(cand, 6).tolist() == [[[1, 4, 2, 0, -1, -1]]]


def test_project_ndc():
    g = torch.Generator().manual_seed(4)
    B, V, H, W = 2, 50, 48, 80
    X = torch.randn(B, V, 3, generator=g, dtype=torch.float64)
    X[..., 2] = X[..., 2].abs() + 2.0
    K = torch.zeros(B, 3, 3, dtype=torch.float64)
    K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = 90.0, 95.0, 41.0, 23.0, 1.0
    out = fitting.project_ndc(X, K, H, W)
    s = min(H, W)
    u = 90.0 * X[..., 0] / X[..., 2] + 41.0
    v = 95.0 * X[..., 1] / X[..., 2] + 23.0
    assert torch.allclose(out[..., 0], (W / 2 - u) * 2 / s)
    assert torch.allclose(out[..., 1], (H / 2 - v) * 2 / s)
    assert torch.equal(out[..., 2], X[..., 2])
    # hand-computed pinhole: f = 100, principal point at the image centre, W = 80, H = 48 (s = 48).  The point (0.24, -0.12, 2)
    # projects to u = 100 * 0.12 + 40 = 52, v = 100 * -0.06 + 24 = 18: 12 px right of centre -> x = -12 * 2/48 = -0.5;
    # 6 px above -> y = +0.25.
    K1 = torch.tensor([[100.0, 0, 40.0], [0, 100.0, 24.0], [0, 0, 1]], dtype=torch.float64)
    p = fitting.project_ndc(torch.tensor([[[0.24, -0.12, 2.0]]], dtype=torch.float64), K1, 48, 80)
    assert torch.allclose(p, torch.tensor([[[-0.5, 0.25, 2.0]]], dtype=torch.float64))
    # a pixel centre maps back to itself: pixel (row i, col j) at u = j + 0.5, v = i + 0.5
    i, j = 7, 61
    q = fitting.project_ndc(torch.tensor([[[(j + 0.5 - 40.0) / 100.0, (i + 0.5 - 24.0) / 100.0, 1.0]]], dtype=torch.float64), K1, 48, 80)
    xs, ys = R.pixel_centres(48, 80)
    assert torch.allclose(q[0, 0, :2], torch.stack([xs[j], ys[i]]))


def test_knn_points():
    g = torch.Generator().manual_seed(5)
    p1 = torch.randn(2, 10, 3, generator=g, dtype=torch.float64, requires_grad=True)
    p2 = torch.randn(2, 300, 3, generator=g, dtype=torch.float64, requires_grad=True)
    K = 4
    out = fitting.knn_points(p1, p2, K)
    assert out.dists.shape == (2, 10, K) and out.idx.shape == (2, 10, K) and out.knn.shape == (2, 10, K, 3)
    assert out.idx.dtype == torch.int64
    for n in range(2):
        for i in range(10):
            d = [((p1[n, i] - p2[n, j]) ** 2).sum().item() for j in range(300)]
            order = sorted(range(300), key=lambda j: d[j])[:K]
            assert out.idx[n, i].tolist() == order
            assert torch.allclose(out.dists[n, i], torch.tensor([d[j] for j in order], dtype=torch.float64))
    assert torch.equal(out.knn, torch.stack([p2[n][out.idx[n]] for n in range(2)]))
    w = torch.randn(2, 10, K, generator=g, dtype=torch.float64)
    (out.dists * w).sum().backward()
    ga, gb = p1.grad.clone(), p2.grad.clone()
    q1, q2 = p1.detach().clone().requires_grad_(True), p2.detach().clone().requires_grad_(True)
    ref = ((q1[:, :, None] - torch.stack([q2[n][out.idx[n]] for n in range(2)])) ** 2).sum(-1)
    (ref * w).sum().backward()
    assert torch.allclose(ga, q1.grad) and torch.allclose(gb, q2.grad)
