"""Time the canonical-mesh signed distance of the training loss targets: the brute force (hold_mesh_sdf) against the BVH query
(hold_mesh_sdf_bvh), alternating the two in one run.

Points: 125 440, the canonical points of the object node in one forward_train on bench.py's training scene (10 frames x 128
rays x 98 samples), moved affinely into each mesh's box; and as many uniform points in the mesh's box.
Meshes:
  hand     a closed marching-cubes mesh of about 7 k faces (the size of the reference's subdivided MANO mesh);
  object   the synthetic object node's generate_mesh(backend="gpu") mesh at the reference's resolution (491 148 faces, open);
  object3k that mesh after meshing.decimate(..., 3000).
Prints one JSON line per (mesh, point set): median call times from CUDA events over --iters calls (BVH build and query split by a
torch.profiler pass of its own), the fraction of points in the winding-number trust band, whether both give the same bits, and
the card's name and power limit read in the same run.  Then one line with the time of an eager training step (forward_train + Loss +
backward + Adam, as bench.py --config train runs it) on that scene with no mesh, with the object mesh attached, and with none again.

    python tools/bench_mesh_sdf.py [--iters 10]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

WS_MESH_BVH = 24   # hold_b200/csrc/common.cuh WsSlot; its first two ints: bad-face flag, band count of the last call
BUILD = ("k_bvh_bounds", "k_bvh_codes", "k_bvh_link", "k_bvh_refit", "k_im_hist", "k_im_scan", "k_im_scatter", "Memset")
QUERY = ("k_bvh_query", "k_bvh_band")


def train_scene(ctx):
    """bench.py's training scene and batch (run_train): the whole model, 10 frames x 128 pixels"""
    import bench
    from hold_b200 import capi, scene_io, synth
    from hold_b200.model import HOLDNet

    dev = torch.device("cuda", 0)
    sc = synth.make_scene(H=bench.H, W=bench.W, S=bench.S, nodes=bench.NODES, B=10, seed=0)
    for nid in sc.node_ids:
        sc.beta[nid] = torch.tensor(bench.BETA)
    fg = scene_io.build_net(sc, ctx, capi.MLP_TC)
    bg, _, _ = scene_io.build_background(sc, ctx, mlp_mode=capi.MLP_TC)
    net = HOLDNet(ctx, dict(fg.nodes), background=bg)
    gen = torch.Generator().manual_seed(100)
    ids = torch.stack([torch.randperm(bench.H * bench.W, generator=gen)[:128] for _ in range(10)])
    inp = scene_io.scene_input(sc, dev)
    inp["uv"] = torch.gather(inp["uv"], 1, ids.to(dev)[:, :, None].expand(-1, -1, 2)).contiguous()
    inp.update({"current_epoch": 30, "global_step": 12000})
    return sc, net, inp


def object_canonical_points(net, inp):
    from hold_b200 import train

    got, orig = {}, train.prepare_loss_targets

    def spy(out, node, B, P, canonical_pts, generator=None):
        got[node.node_id] = canonical_pts.detach().reshape(-1, 3).clone()
        return orig(out, node, B, P, canonical_pts, generator)

    train.prepare_loss_targets = spy
    try:
        with torch.no_grad():
            train.forward_train(net, inp, generator=torch.Generator(device="cuda").manual_seed(0))
    finally:
        train.prepare_loss_targets = orig
    return got["object"]


def hand_mesh(ctx, n=48):
    from hold_b200 import meshing

    a = torch.linspace(-1.0, 1.0, n, device="cuda")
    x, y, z = torch.meshgrid(a, a, a, indexing="ij")
    vol = (x * x + y * y + z * z).sqrt() - 0.7 - 0.05 * torch.sin(5 * x) * torch.sin(4 * y) * torch.sin(3 * z)
    v, f = meshing.marching_cubes(ctx, vol, 0.0)
    return meshing.largest_component(v.cpu().numpy() * (2.0 / (n - 1)) - 1.0, f.cpu().numpy())


def call(ctx, fn, pts, v, f, sdf, fi):
    from hold_b200.capi import check, lib, stream_ptr

    g = getattr(lib(), fn)
    p = lambda t: C.c_void_p(t.data_ptr())
    check(g(ctx.h, 1, pts.shape[0], p(pts), v.shape[0], p(v), 0, f.shape[0], p(f), p(sdf), p(fi), stream_ptr()))


def timed(fn, iters):
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def kernel_split(fn):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    build = query = 0.0
    for e in prof.key_averages():
        us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if any(k in e.key for k in QUERY):
            query += us
        elif any(k in e.key for k in BUILD):
            build += us
    return build / 1e3, query / 1e3


def step_ms(ctx, net, inp, iters):
    """one eager TrainStep as bench.py --config train runs it: forward_train, Loss, backward, Adam"""
    from hold_b200 import train

    dev = torch.device("cuda", 0)
    R = 10 * 128
    gt_rgb = torch.rand(R, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(7))
    gt_mask = torch.zeros(R, 4, device=dev)
    gt_mask[:, 0] = 1.0
    ts = train.TrainStep(net, group=None, capturable=False)
    ts.step(inp, gt_rgb, gt_mask)
    ctx.check()
    torch.cuda.reset_peak_memory_stats()
    ms = timed(lambda: ts.step(inp, gt_rgb, gt_mask), iters)
    return ms, torch.cuda.max_memory_allocated() / 2**30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--step-iters", type=int, default=3)
    args = ap.parse_args()
    from bench_decimate import card, object_mesh
    from hold_b200 import capi, meshing

    ctx = capi.Context(0)
    name, power = card()
    sc, net, inp = train_scene(ctx)
    xc = object_canonical_points(net, inp)
    ov, of = object_mesh(ctx)
    ov, of = np.ascontiguousarray(ov, np.float32), np.ascontiguousarray(of, np.int32)
    dv, df = meshing.decimate(ctx, ov, of, 3000)
    meshes = {"hand": hand_mesh(ctx), "object": (ov, of), "object3k": (dv.cpu().numpy(), df.cpu().numpy())}
    lo0, hi0 = torch.from_numpy(ov.min(0)).cuda(), torch.from_numpy(ov.max(0)).cuda()
    g = torch.Generator(device="cuda").manual_seed(3)
    for label, (v, f) in meshes.items():
        v = torch.as_tensor(np.ascontiguousarray(v, np.float32)).cuda()
        f = torch.as_tensor(np.ascontiguousarray(f, np.int32)).cuda()
        lo, hi = v.min(0).values, v.max(0).values
        sets = {"canonical": ((xc - lo0) / (hi0 - lo0) * (hi - lo) + lo).contiguous(),
                "uniform": (lo + torch.rand(xc.shape[0], 3, device="cuda", generator=g) * (hi - lo)).contiguous()}
        for sname, pts in sets.items():
            out = {}
            for fn in ("hold_mesh_sdf", "hold_mesh_sdf_bvh"):
                sdf = torch.empty(pts.shape[0], device="cuda")
                fi = torch.empty(pts.shape[0], dtype=torch.int32, device="cuda")
                call(ctx, fn, pts, v, f, sdf, fi)
                out[fn] = (sdf, fi)
            ctx.check()
            state = torch.zeros(2, dtype=torch.int32, device="cuda")
            ws_copy = capi.lib().hold_debug_ws_copy
            ws_copy.restype, ws_copy.argtypes = C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]
            capi.check(ws_copy(ctx.h, WS_MESH_BVH, state.data_ptr(), 8))
            band = state.cpu().numpy()
            same = bool(torch.equal(out["hold_mesh_sdf"][0].view(torch.int32), out["hold_mesh_sdf_bvh"][0].view(torch.int32))
                        and torch.equal(out["hold_mesh_sdf"][1], out["hold_mesh_sdf_bvh"][1]))
            ms = {fn: [] for fn in out}
            for _ in range(3):                                              # alternate the two
                for fn, (sdf, fi) in out.items():
                    ms[fn].append(timed(lambda: call(ctx, fn, pts, v, f, sdf, fi), max(1, args.iters // 3)))
            build, query = kernel_split(lambda: call(ctx, "hold_mesh_sdf_bvh", pts, v, f, *out["hold_mesh_sdf_bvh"]))
            print(json.dumps({"mesh": label, "points": sname, "P": int(pts.shape[0]), "F": int(f.shape[0]),
                              "brute_ms": round(statistics.median(ms["hold_mesh_sdf"]), 3),
                              "bvh_ms": round(statistics.median(ms["hold_mesh_sdf_bvh"]), 3),
                              "bvh_build_ms": round(build, 3), "bvh_query_ms": round(query, 3),
                              "band_fraction": round(int(band[1]) / pts.shape[0], 5), "same_bits": same,
                              "gpu": name, "power_limit": power}), flush=True)
    obj = net.nodes["object"]
    torch.cuda.empty_cache()
    for label in ("none", "object", "none"):
        obj.mesh_vo_cano, obj.mesh_fo_cano = (torch.from_numpy(ov).cuda(), torch.from_numpy(of).cuda()) if label == "object" else (None, None)
        ms, gib = step_ms(ctx, net, inp, args.step_iters)
        print(json.dumps({"step": "TrainStep (forward_train + Loss + backward + Adam), eager", "mesh": label,
                          "faces": int(of.shape[0]) if label == "object" else 0, "ms_median": round(ms, 2), "peak_gib": round(gib, 2),
                          "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
