"""Time the soft-silhouette rasteriser (hold_raster_silhouette / _bwd) on the pose refinement's workload.

Workloads (pytorch3d's soft-silhouette settings: K = 100, sigma = 1e-4, blur_radius = ln(1/1e-4 - 1) sigma, 512 x 512):
  scene  B frames of a hand-sized closed mesh (1 536 faces) next to an object mesh (2 976 faces), drawn together as one mesh,
         as fitting/utils.py draws the hand and the object;
  quads  150 stacked quads over most of the image, so that most pixels have more than K candidates (the exact-selection path).
Prints one JSON line per workload: ms per forward and per forward + backward (CUDA events, after warm-up), the card's name and
power limit read in the same run, the peak device memory of a forward + backward, and the nominal pixel-face pairs
(B H W F, counted from shapes) per second of the forward.

    python tools/bench_silhouette.py [--frames 8] [--iters 20]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def sphere(n_lat, n_lon, r, centre):
    """Closed latitude-longitude sphere (n_lat - 2 rings between the poles): 2 n_lon (n_lat - 2) faces."""
    th = torch.linspace(0, math.pi, n_lat)[1:-1]
    ph = torch.arange(n_lon) * (2 * math.pi / n_lon)
    ring = torch.stack([torch.sin(th)[:, None] * torch.cos(ph), torch.sin(th)[:, None] * torch.sin(ph),
                        torch.cos(th)[:, None].expand(-1, n_lon)], -1).reshape(-1, 3)
    v = torch.cat([torch.tensor([[0.0, 0.0, 1.0]]), ring, torch.tensor([[0.0, 0.0, -1.0]])]) * r + torch.tensor(centre)
    f = []
    last = 1 + (n_lat - 2) * n_lon
    for j in range(n_lon):
        f.append([0, 1 + j, 1 + (j + 1) % n_lon])
        f.append([last, 1 + (n_lat - 3) * n_lon + (j + 1) % n_lon, 1 + (n_lat - 3) * n_lon + j])
    for i in range(n_lat - 3):
        for j in range(n_lon):
            a, b = 1 + i * n_lon + j, 1 + i * n_lon + (j + 1) % n_lon
            f += [[a, a + n_lon, b], [b, a + n_lon, b + n_lon]]
    return v, torch.tensor(f, dtype=torch.int32)


def scene(B):
    from hold_b200 import fitting

    vh, fh = sphere(26, 32, 0.09, (-0.06, 0.0, 0.6))       # hand-sized: 1 536 faces, ~18 cm across at 60 cm
    vo, fo = sphere(33, 48, 0.12, (0.1, 0.02, 0.7))        # object: 2 976 faces
    v = torch.cat([vh, vo])
    f = torch.cat([fh, fo + vh.shape[0]])
    g = torch.Generator().manual_seed(0)
    vb = v[None] + torch.randn(B, 1, 3, generator=g) * torch.tensor([0.02, 0.02, 0.03])   # frames differ a little
    Kc = torch.tensor([[600.0, 0, 256.0], [0, 600.0, 256.0], [0, 0, 1]])
    return fitting.project_ndc(vb, Kc, 512, 512).contiguous(), f


def quads(B, n=150):
    g = torch.Generator().manual_seed(0)
    vs, fs = [], []
    for k in range(n):
        o = (torch.rand(2, generator=g) - 0.5) * 0.2
        x0, x1, y0, y1 = -0.8 + o[0], 0.8 + o[0], -0.7 + o[1], 0.7 + o[1]
        z = 1.0 + 0.01 * k
        vs += [[x0, y0, z], [x1, y0, z], [x1, y1, z], [x0, y1, z]]
        fs += [[4 * k, 4 * k + 1, 4 * k + 2], [4 * k, 4 * k + 2, 4 * k + 3]]
    return torch.tensor(vs)[None].expand(B, -1, -1).contiguous(), torch.tensor(fs, dtype=torch.int32)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def run(ctx, name, v, f, iters, H=512, W=512, K=100, sigma=1e-4):
    from hold_b200 import fitting

    dev = torch.device("cuda", 0)
    v, f = v.to(dev), f.to(dev)
    B, F = v.shape[0], f.shape[0]
    fc = fitting.check_faces(f, v.shape[1], dev)          # once: the host sync of the face check stays out of the timing
    cfg = fitting._cfg(K, None, sigma, True, None, False)
    vg = v.clone().requires_grad_(True)
    g = torch.randn(B, H, W, device=dev)
    fwd = lambda: fitting.SoftSilhouetteFn.apply(v, fc, ctx, H, W, cfg)
    fb = lambda: fitting.SoftSilhouetteFn.apply(vg, fc, ctx, H, W, cfg).backward(g)
    for _ in range(3):
        fwd(), fb()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(dev)[0]
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    fb()
    torch.cuda.synchronize()
    peak_torch = torch.cuda.max_memory_allocated(dev) - base
    ws = B * F * 64                                       # the library's face records (grow-only workspace, already allocated)
    ms_f = timed(fwd, iters)
    ms_fb = timed(fb, iters)
    ctx.check()
    sil = fwd()
    return {"workload": name, "card": card(), "B": B, "H": H, "W": W, "F": F, "K": K, "sigma": sigma,
            "ms_forward": round(ms_f, 4), "ms_forward_backward": round(ms_fb, 4),
            "peak_bytes_torch": int(peak_torch), "workspace_bytes": ws, "pytorch3d_fragment_bytes": B * H * W * K * 28,
            "pixel_face_pairs_per_s_forward": B * H * W * F / (ms_f * 1e-3),
            "coverage": round((sil > 0.5).float().mean().item(), 4), "free_bytes_before": int(free0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import __graft_entry__ as g

    g.build()
    from hold_b200 import capi

    torch.cuda.set_device(0)
    ctx = capi.Context(0)
    for name, (v, f) in (("scene", scene(a.frames)), ("quads", quads(a.frames))):
        print(json.dumps(run(ctx, name, v, f, a.iters)), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
