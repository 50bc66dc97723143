"""Time the quadric edge-collapse decimation (hold_decimate, hold_b200.meshing.decimate) on the pose refinement's workload.

Workloads, both down to 3 000 faces (the object size tools/bench_silhouette.py draws):
  object  the canonical object mesh generate_mesh(backend="gpu") extracts from a synthetic object node at the reference's
          resolution (res_init 32, 3 upsampling steps), as load_data would receive it;
  bumpy   a 5 * 10^4-face closed mesh, the GPU marching cubes of a bumpy sphere.
Prints one JSON line per workload: the median wall time of a call over --iters calls after a warm-up (the call synchronises its
stream every round, so a host clock around it measures the device work and the per-round reads), the round count and whether the
device output equals the host restatement bit for bit (both from tests/host/decimate_host.cpp), and the card's name and power
limit read in the same run.

    python tools/bench_decimate.py [--iters 10]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ["?, ?"])[0].split(", ")
    return name, power


def object_mesh(ctx):
    from hold_b200 import capi, meshing, scene_io, synth

    sc = synth.make_scene(H=8, W=8, S=32, nodes=("right", "object"), seed=4)
    net = scene_io.build_net(sc, ctx, capi.MLP_TC)
    return meshing.generate_mesh(ctx, meshing.node_sdf_func(ctx, net.nodes["object"]), sc.obj_pts_cano.numpy(), backend="gpu")


def bumpy_mesh(ctx, n=107):
    from hold_b200 import meshing

    a = torch.linspace(-1.0, 1.0, n, device="cuda")
    x, y, z = torch.meshgrid(a, a, a, indexing="ij")
    vol = (x * x + y * y + z * z).sqrt() - 0.7 - 0.04 * torch.sin(6 * x) * torch.sin(6 * y) * torch.sin(6 * z)
    v, f = meshing.marching_cubes(ctx, vol, 0.0)
    return meshing.largest_component(v.cpu().numpy() * (2.0 / (n - 1)) - 1.0, f.cpu().numpy())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--target", type=int, default=3000)
    args = ap.parse_args()
    from hold_b200 import capi, meshing
    from test_cpu_decimate import euler, host_decimate

    ctx = capi.Context(0)
    name, power = card()
    for label, (v, f) in (("object", object_mesh(ctx)), ("bumpy", bumpy_mesh(ctx))):
        v, f = np.ascontiguousarray(v, np.float32), np.ascontiguousarray(f, np.int32)
        vd, fd = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
        out = meshing.decimate(ctx, vd, fd, args.target)                  # warm-up
        times = []
        for _ in range(args.iters):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = meshing.decimate(ctx, vd, fd, args.target)
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
        hv, hf, rounds = host_decimate(v, f, args.target)
        same = np.array_equal(out[0].cpu().numpy().view(np.int32), hv.view(np.int32)) and np.array_equal(out[1].cpu().numpy(), hf)
        print(json.dumps({"workload": label, "faces_in": int(f.shape[0]), "verts_in": int(v.shape[0]), "faces_out": int(out[1].shape[0]), "euler": int(euler(v, f)),
                          "rounds": rounds, "ms_median": round(statistics.median(times), 3), "ms_min": round(min(times), 3),
                          "device_equals_host": bool(same), "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
