"""Fixed launch order for ncu captures: [0] k_mlp_tc<0> sdf-only (2^22 points), [1] k_mlp_tc<3> sdf + gradient + feature
(2^20 points), then one colour-net launch through hold_shade on a small frame.
  ncu --set full --clock-control none --import-source on -k regex:k_mlp_tc -s 1 -c 1 -o prof_out/x python tools/prof_kernels.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from hold_b200 import capi, scene_io, synth

ctx = capi.Context(0); dev = torch.device("cuda", 0)
sc = synth.make_scene(H=8, W=8, S=128, nodes=("right", "object"))
node = scene_io.build_net(sc, ctx, capi.MLP_TC).nodes["right"]
P0, P1 = 1 << 22, 1 << 20
g = torch.Generator().manual_seed(0)
xc = ((torch.rand(P0, 3, generator=g) - 0.5) * 1.6).to(dev)
sdf = torch.empty(P0, device=dev); grad = torch.empty(P1, 3, device=dev); feat = torch.empty(P1, 256, device=dev)
L = capi.lib()
capi.check(L.hold_sdf_eval(ctx.h, node.slot, P0, capi.ptr(xc), None, capi.ptr(sdf), None, None, capi.stream_ptr()))
torch.cuda.synchronize()
capi.check(L.hold_sdf_eval(ctx.h, node.slot, P1, capi.ptr(xc), None, capi.ptr(sdf), capi.ptr(grad), capi.ptr(feat), capi.stream_ptr()))
torch.cuda.synchronize()
ctx.check()
print("prof_kernels done")
