"""Kernel times of the background leg of a training step (train.background_forward_train forward + backward, bench.py's
training workload: 10 frames x 128 rays), fixed shells and stratified depths: CUDA-event time per leg and a torch.profiler
kernel table.  Writes the table under $PROF_OUT (default prof_out/)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
from hold_b200 import capi, ops, scene_io, synth, train

ctx = capi.Context(0)
dev = torch.device("cuda", 0)
Bf, px = 10, 128
sc = synth.make_scene(H=bench.H, W=bench.W, S=bench.S, nodes=bench.NODES, B=Bf, seed=0)
scene_io.build_net(sc, ctx, capi.MLP_TC)
bg, _, _ = scene_io.build_background(sc, ctx, mlp_mode=capi.MLP_TC)
gen = torch.Generator().manual_seed(100)
ids = torch.stack([torch.randperm(bench.H * bench.W, generator=gen)[:px] for _ in range(Bf)])
inp = scene_io.scene_input(sc, dev)
uv = torch.gather(inp["uv"], 1, ids.to(dev)[:, :, None].expand(-1, -1, 2)).contiguous()
dirs, cam = ops.camera_rays(ctx, uv, inp["extrinsics"], inp["intrinsics"])
R = Bf * px
bgw = torch.rand(R, device=dev).requires_grad_(True)
seed = torch.randn(R, 3, device=dev)


def leg(jitter):
    out = train.background_forward_train(bg, bgw, dirs, cam, inp["idx"], Bf, sc.bounding_sphere, jitter=jitter)
    (out["bg_rgb"] * seed).sum().backward()


for name, jit in (("fixed shells", None), ("stratified", torch.rand(R, 32, device=dev))):
    for _ in range(3):
        leg(jit)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 50
    e0.record()
    for _ in range(n):
        leg(jit)
    e1.record()
    torch.cuda.synchronize()
    print(f"background leg, {name}: {e0.elapsed_time(e1) / n:.3f} ms per forward + backward ({R} rays x 32 samples)")

from torch.profiler import ProfilerActivity, profile

with profile(activities=[ProfilerActivity.CUDA]) as p:
    for _ in range(10):
        leg(torch.rand(R, 32, device=dev))
    torch.cuda.synchronize()
table = p.key_averages().table(sort_by="cuda_time_total", row_limit=30, max_name_column_width=70)
print(table)
out_dir = os.environ.get("PROF_OUT", "prof_out")
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "bg_train_kernels.txt"), "w") as f:
    f.write(table)
print(torch.cuda.get_device_name(0))
