"""GPU experiments in one process (section 3 drove KNN kernel variants that have since been removed from the library):
 1. tensor-core SDF chains vs float64: signed / max error of sdf (sampler-round kernel and reverse-mode kernel) and of the gradient,
    for accumulator compensation factors 1 + c 2^-24 (is the residual a truncation bias of the tensor core's accumulator?)
 2. kernel times: sampler-round SDF launch, reverse-mode launch
 3. hand KNN / inverse-LBS kernel variants inside hold_sample (A/B/A/B order)
 4. background nets: exact fp32 vs tensor cores"""
import ctypes as C
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from hold_b200 import capi, scene_io, synth
from oracle import hold_oracle as O

ctx = capi.Context(0); dev = torch.device("cuda", 0)
L = capi.lib()
L.hold_debug_set.restype = C.c_int
L.hold_debug_set.argtypes = [C.c_void_p, C.c_int, C.c_int]

def timed(fn, n=3):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n

# ---------------------------------------------------------------- 1. error vs float64
print("== 1. tensor-core SDF chains vs float64 (c = accumulator compensation, scale 1 + c 2^-24)")
for perturb in (0.0, 0.02, 0.05):
    sc = synth.make_scene(H=8, W=8, S=32, nodes=("right", "object"), seed=4, perturb=perturb)
    net = scene_io.build_net(sc, ctx, capi.MLP_TC)
    g = torch.Generator().manual_seed(9)
    x = ((torch.rand(20000, 3, generator=g) - 0.5) * 1.6)
    for nid in sc.node_ids:
        sd = {k: v.double() for k, v in sc.sdf_state[nid].items()}
        xg = x.double().requires_grad_(True)
        ref = O.sdf_mlp(xg, sd, torch.zeros(x.shape[0], 45, dtype=torch.float64) if nid != "object" else None)
        gref = torch.autograd.grad(ref[:, 0].sum(), xg)[0].detach()
        ref = ref.detach()
        near = ref[:, 0].abs() < 0.05
        if not near.any():
            near = ref[:, 0].abs() <= ref[:, 0].abs().kthvalue(200).values
        node = net.nodes[nid]
        xd = x.to(dev).contiguous()
        for c in (0, 8, 10, 11, 12, 14):
            assert L.hold_debug_set(ctx.h, 2, c) == 0
            s0 = torch.empty(x.shape[0], device=dev)
            capi.check(L.hold_sdf_eval(ctx.h, node.slot, x.shape[0], capi.ptr(xd), None, capi.ptr(s0), None, None, capi.stream_ptr()))
            s1, g1, f1 = torch.empty(x.shape[0], device=dev), torch.empty(x.shape[0], 3, device=dev), torch.empty(x.shape[0], 256, device=dev)
            capi.check(L.hold_sdf_eval(ctx.h, node.slot, x.shape[0], capi.ptr(xd), None, capi.ptr(s1), capi.ptr(g1), capi.ptr(f1), capi.stream_ptr()))
            ctx.check()
            e0 = (s0.cpu().double() - ref[:, 0]); e1 = (s1.cpu().double() - ref[:, 0])
            eg = (g1.cpu().double() - gref).abs().max().item() / gref.abs().max().item()
            ef = (f1.cpu().double() - ref[:, 1:]).abs().max().item() / ref[:, 1:].abs().max().item()
            print(f"perturb {perturb} {nid:6s} c={c:2d}: sdf-only mean {e0.mean().item():+.2e} max {e0.abs().max().item():.2e} near-surface max {e0[near].abs().max().item():.2e} | "
                  f"rev sdf mean {e1.mean().item():+.2e} max {e1.abs().max().item():.2e} | grad rel {eg:.2e} feat rel {ef:.2e}", flush=True)
        L.hold_debug_set(ctx.h, 2, -1)

# ---------------------------------------------------------------- 2. kernel times
print("== 2. kernel times")
sc = synth.make_scene(H=8, W=8, S=128, nodes=("right", "object"))
node = scene_io.build_net(sc, ctx, capi.MLP_TC).nodes["right"]
P0, P1 = 1 << 23, 1 << 20
xc = ((torch.rand(P0, 3, generator=torch.Generator().manual_seed(0)) - 0.5) * 1.6).to(dev)
sdf = torch.empty(P0, device=dev); grad = torch.empty(P1, 3, device=dev); feat = torch.empty(P1, 256, device=dev)
t0 = timed(lambda: capi.check(L.hold_sdf_eval(ctx.h, node.slot, P0, capi.ptr(xc), None, capi.ptr(sdf), None, None, capi.stream_ptr())))
t1 = timed(lambda: capi.check(L.hold_sdf_eval(ctx.h, node.slot, P1, capi.ptr(xc), None, capi.ptr(sdf), capi.ptr(grad), capi.ptr(feat), capi.stream_ptr())), n=5)
ctx.check()
print(f"sampler-round SDF launch: {t0:.2f} ms per 2^23 points ({2 * 459008 * P0 / t0 / 1e9:.1f} TFLOP/s algorithmic); reverse mode: {t1:.2f} ms per Mi points "
      f"({2 * (524544 + 459008) * P1 / t1 / 1e9:.1f} TFLOP/s algorithmic)", flush=True)
del xc, sdf, grad, feat

# ---------------------------------------------------------------- 3. KNN variants inside hold_sample
print("== 3. hand KNN variants (hold_sample of the hand node, 256x256 frame, beta 0.03)")
sc2 = synth.make_scene(H=256, W=256, S=128, nodes=("right", "object"), B=1, seed=0)
for nid in sc2.node_ids:
    sc2.beta[nid] = torch.tensor(0.03)
net2 = scene_io.build_net(sc2, ctx, capi.MLP_TC)
inp2 = scene_io.scene_input(sc2, dev)
from hold_b200 import ops
from hold_b200.model import ErrorBoundSampler
hn = net2.nodes["right"]
dirs, cam = ops.camera_rays(ctx, inp2["uv"], inp2["extrinsics"], inp2["intrinsics"])
pose, keep, _, _ = hn.articulate(inp2)
smp = ErrorBoundSampler(hn)
zs = {}
for rep in range(2):
    for v, name in ((0, "default"), (1, "filtered scan"), (2, "6 blocks/SM")):
        L.hold_debug_set(ctx.h, 1, v)
        out = {}
        def run():
            out["z"], out["it"] = smp.get_z_vals(dirs, cam, pose, 1)
        t = timed(run, n=2)
        ctx.check()
        zs[v] = out["z"].clone()
        print(f"  pass {rep} {name:14s}: hold_sample {t:8.2f} ms  rounds {int(out['it'].item())}  z identical to default: {bool(torch.equal(zs[v], zs[0]))}", flush=True)
L.hold_debug_set(ctx.h, 1, 0)
# whole step for reference
t = timed(lambda: net2.forward_fg(inp2, return_factors=False, want_weights=False), n=2)
print(f"  whole foreground step 256x256: {t:.1f} ms ({256 * 256 / t:.1f} k rays/s)")

# ---------------------------------------------------------------- 4. background
print("== 4. background nets, 256x256 rays")
for mm, name in ((capi.MLP_FP32, "fp32 CUDA cores"), (capi.MLP_TC, "tensor cores")):
    bg, _, _ = scene_io.build_background(sc2, ctx, mlp_mode=mm)
    w = torch.rand(dirs.shape[0], device=dev)
    res = {}
    def runbg():
        res["o"] = bg(w, dirs, cam, sc2.frame_idx.to(dev), 1)
    t = timed(runbg, n=2)
    ctx.check()
    if mm == capi.MLP_FP32:
        base = res["o"]["bg_rgb"].clone()
    print(f"  {name:16s}: {t:8.2f} ms  max|d bg_rgb| vs fp32 {(res['o']['bg_rgb'] - base).abs().max().item():.2e}", flush=True)
print("exp_r2b done")
