"""Timings of the SURVEY §8f rank-4 rows against their CPU counterparts on the same box (VERDICT r1 item 10):
 (a) canonical mesh value grid at the reference's resolution (res_init 32, 3 upsampling steps -> 257^3 lattice, utils/meshing.py:10-47):
     GPU MISE + fused tensor-core SDF queries (meshing.generate_grid) vs the reference's OWN compiled Cython MISE (oracle/_ref) driven
     by the oracle's SDF net on the host cores (what hold.py:139-167 runs on the CPU);
 (b) the pose-refinement server path of optimize_ckpt.py (fitting/model.py:113-117): MANO lbs forward + backward for B frames,
     hold_mano_lbs(+_bwd) vs torch autograd through the oracle's lbs() on the host cores.
Prints one JSON line per row."""
import glob
import json
import os
import sys
import time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from hold_b200 import capi, meshing, scene_io, synth
from oracle import hold_oracle as O

ctx = capi.Context(0); dev = torch.device("cuda", 0)
sc = synth.make_scene(H=8, W=8, S=32, nodes=("right", "object"), seed=4)
net = scene_io.build_net(sc, ctx, capi.MLP_TC)
threads = min(16, len(os.sched_getaffinity(0)))
torch.set_num_threads(threads)

# ---------------------------------------------------------------- (a) value grid
node = net.nodes["object"]
func = meshing.node_sdf_func(ctx, node)
verts = sc.obj_pts_cano.numpy()
meshing.generate_grid(ctx, func, verts, 0.0, res_init=32, res_up=3); torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(3):
    grid, res, gt_scale, gt_center = meshing.generate_grid(ctx, func, verts, 0.0, res_init=32, res_up=3)
torch.cuda.synchronize()
t_gpu = (time.perf_counter() - t0) / 3
so = next(iter(glob.glob(os.path.join(ROOT, "oracle", "_ref", "mise*.so"))), None)
t_cpu, n_q, same = None, 0, None
if so is not None:
    sys.path.insert(0, os.path.dirname(so))
    import mise
    sd = sc.sdf_state["object"]
    t0 = time.perf_counter()
    ex = mise.MISE(32, 3, 0.0)
    pts = ex.query()
    with torch.no_grad():
        while pts.shape[0] != 0:
            p = pts.astype(np.float32)
            p = (p / ex.resolution - 0.5) * 1.1
            p = p * gt_scale + gt_center
            vals = O.sdf_mlp(torch.tensor(p).float(), sd)[:, 0].numpy().astype(np.float64)
            n_q += pts.shape[0]
            ex.update(pts, vals)
            pts = ex.query()
    ref = ex.to_dense()
    t_cpu = time.perf_counter() - t0
    same = float((np.sign(ref) == np.sign(grid)).mean())
print(json.dumps({"row": "8f-4a generate_grid (MISE 32 -> 256, canonical object SDF)", "gpu_s": t_gpu, "cpu_reference_s": t_cpu, "speedup": (t_cpu / t_gpu) if t_cpu else None,
                  "sdf_queries": n_q, "cpu_threads": threads, "inside_outside_agreement": same,
                  "note": "CPU: the reference's own compiled libmise + oracle SDF net (torch fp32); GPU: hold_mise_* + hold_sdf_eval (tensor cores)"}))

# ---------------------------------------------------------------- (b) pose-refinement server path
from hold_b200.model import MANOServer
B = 64
m = sc.mano["right"]
srv = net.nodes["right"].server
g = torch.Generator().manual_seed(0)
pose = (torch.randn(B, 48, generator=g) * 0.3)
transl = torch.randn(B, 3, generator=g) * 0.1
betas = sc.betas["right"][None].repeat(B, 1)
scale = torch.full((B,), float(sc.scene_scale))
gv = torch.randn(B, 778, 3, generator=g)
def gpu_step():
    p, t, b = pose.to(dev).requires_grad_(True), transl.to(dev).requires_grad_(True), betas.to(dev).requires_grad_(True)
    out = srv(scale.to(dev), t, p, b)
    (out["verts"] * gv.to(dev)).sum().backward()
    return p.grad
gpu_step(); torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(20):
    gp = gpu_step()
torch.cuda.synchronize()
t_gpu = (time.perf_counter() - t0) / 20
verts_c, tfs_c_inv = O.mano_canonical(m, sc.betas["right"])
def cpu_step():
    p, t, b = pose.clone().requires_grad_(True), transl.clone().requires_grad_(True), betas.clone().requires_grad_(True)
    out = O.mano_server(m, scale, t, p, b, tfs_c_inv)
    (out["verts"] * gv).sum().backward()
    return p.grad
cpu_step()
t0 = time.perf_counter()
for _ in range(5):
    cp = cpu_step()
t_cpu = (time.perf_counter() - t0) / 5
err = ((gp.cpu() - cp).abs().max() / cp.abs().max()).item()
print(json.dumps({"row": "8f-4b MANO server forward + backward (optimize_ckpt.py server path)", "frames": B, "gpu_s": t_gpu, "cpu_reference_s": t_cpu,
                  "speedup": t_cpu / t_gpu, "cpu_threads": threads, "grad_rel_err": err,
                  "note": "CPU: torch autograd through the oracle's lbs() restatement (pinned to the vendored lbs()); GPU: hold_mano_lbs + hold_mano_lbs_bwd"}))
