"""Time the canonical-mesh refresh (HOLD.meshing_cano) on the synthetic object node at the reference's resolution (res_init 32,
3 upsampling steps): the host composition generate_mesh(backend="gpu") ran before the selection moved to the device, against
meshing.extract_mesh, alternating the two in one run.

  host    MISE + SDF queries on the device; the dense grid to the host as float64 and back; marching cubes on the device; the
          mesh to the host; the grid-to-world transform in numpy; largest_component (scipy); the result back to the device, where
          a training caller needs it;
  device  MISE + SDF queries; marching cubes; the transform in torch; hold_largest_component; everything stays on the device.

Every stage is timed with a host clock between device synchronisations (each pipeline also reads sizes on the host on its own).
Prints one JSON line per pipeline with the median of each stage over --iters runs and whether the two results are equal bit for
bit, then one line with the CUDA time of each hold_largest_component kernel (torch.profiler, in a run of its own, averaged over
its calls), and the card's name and power limit read in the same run.

    python tools/bench_meshing.py [--iters 5]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ["?, ?"])[0].split(", ")
    return name, power


class Stages:
    def __init__(self):
        self.ms = {}
        torch.cuda.synchronize()
        self.t = time.perf_counter()

    def mark(self, name):
        torch.cuda.synchronize()
        t = time.perf_counter()
        self.ms[name] = self.ms.get(name, 0.0) + (t - self.t) * 1e3
        self.t = t


def host_pipeline(ctx, func, box, res_init, res_up):
    from hold_b200 import meshing

    st = Stages()
    grid, res, gt_scale, gt_center = meshing._dense_grid(ctx, func, box, 0.0, res_init, res_up, 1.1)
    st.mark("mise_queries")
    grid = grid.cpu().numpy().astype(np.float64)
    dev = torch.device("cuda", ctx.device)
    gd = torch.as_tensor(grid, device=dev)
    st.mark("copies")
    v, f = meshing.marching_cubes(ctx, gd, 0.0)
    st.mark("marching_cubes")
    v, f = v.cpu().numpy(), f.cpu().numpy()
    st.mark("copies")
    verts_mc = ((v / res - 0.5) * 1.1) * gt_scale + gt_center
    faces = f.astype(np.int64)
    st.mark("transform")
    v, f = meshing.largest_component(verts_mc, faces)
    st.mark("component_selection")
    v, f = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
    st.mark("copies")
    return (v, f), st.ms


def device_pipeline(ctx, func, box, res_init, res_up):
    from hold_b200 import meshing

    st = Stages()
    grid, res, gt_scale, gt_center = meshing._dense_grid(ctx, func, box, 0.0, res_init, res_up, 1.1)
    st.mark("mise_queries")
    v, f = meshing.marching_cubes(ctx, grid, 0.0)
    st.mark("marching_cubes")
    v = meshing.grid_to_world(v, res, gt_scale, gt_center)
    st.mark("transform")
    out = meshing.largest_component_device(ctx, v, f)
    st.mark("component_selection")
    return out, st.ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--res-init", type=int, default=32)
    ap.add_argument("--res-up", type=int, default=3)
    args = ap.parse_args()
    from hold_b200 import capi, meshing, scene_io, synth

    ctx = capi.Context(0)
    name, power = card()
    sc = synth.make_scene(H=8, W=8, S=32, nodes=("right", "object"), seed=4)
    net = scene_io.build_net(sc, ctx, capi.MLP_TC)
    func = meshing.node_sdf_func(ctx, net.nodes["object"])
    box = sc.obj_pts_cano.numpy()
    pipes = {"host": host_pipeline, "device": device_pipeline}
    res = {k: p(ctx, func, box, args.res_init, args.res_up)[0] for k, p in pipes.items()}    # warm-up
    runs = {k: [] for k in pipes}
    for _ in range(args.iters):
        for k, p in pipes.items():                                        # alternated in one loop
            res[k], ms = p(ctx, func, box, args.res_init, args.res_up)
            runs[k].append(ms)
    (hv, hf), (dv, df) = res["host"], res["device"]
    same = hv.shape == dv.shape and torch.equal(hv.view(torch.int32), dv.view(torch.int32)) and torch.equal(hf, df.long())
    for k in pipes:
        stages = {s: round(statistics.median(r[s] for r in runs[k]), 3) for s in runs[k][0]}
        total = round(statistics.median(sum(r.values()) for r in runs[k]), 3)
        print(json.dumps({"pipeline": k, "res_init": args.res_init, "res_up": args.res_up, "faces_out": int(hf.shape[0]),
                          "verts_out": int(hv.shape[0]), "ms_median": stages, "ms_total_median": total, "bitwise_equal": bool(same),
                          "card": name, "power_limit": power}))
    # per-kernel CUDA time of hold_largest_component on the object's marching-cubes mesh
    grid, r, gs, gc = meshing._dense_grid(ctx, func, box, 0.0, args.res_init, args.res_up, 1.1)
    v, f = meshing.marching_cubes(ctx, grid, 0.0)
    v = meshing.grid_to_world(v, r, gs, gc)
    meshing.largest_component_device(ctx, v, f)
    n = 10
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            meshing.largest_component_device(ctx, v, f)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if "k_cc_" in e.key or "k_im_" in e.key:
            short = e.key.split("(")[0].replace("hold::", "")
            kern[short] = round(kern.get(short, 0.0) + e.device_time_total / 1e3 / n, 4)
    print(json.dumps({"hold_largest_component_kernels_ms_per_call": kern, "faces_in": int(f.shape[0]), "verts_in": int(v.shape[0]),
                      "card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
