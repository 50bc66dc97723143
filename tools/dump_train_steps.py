"""Run N training steps of the benchmark's training scene and dump the state after every step, for bit-for-bit comparison of
two builds or two runs (the training counterpart of `bench.py --dump-outputs`).

  python tools/dump_train_steps.py DIR [--steps N] [--graph | --stratified] [--frames F] [--pixels P] [--size HW] [--seed S]
  python tools/compare_dumps.py DIR_A DIR_B

The scene is the one `bench.py --config train` builds from its seeds: bench.py's resolution, samples per ray, beta and nodes,
the NeRF++ background, `--frames` frames x `--pixels` pixels chosen by the bench's generator, the per-frame poses as leaves.
`--size` renders a smaller image for quick runs.  After every step DIR holds, as float32 / float64 .npy files named
`stepNNN.<what>.<parameter>`: the loss and its terms, every parameter, its .grad and Adam's moments (exp_avg, exp_avg_sq).
--graph captures the step as one CUDA graph (TrainStep.capture, whose warm-up takes three eager steps) and dumps the replays;
--stratified draws the training-mode samples from a generator seeded with --seed; the eikonal samples come from the default
generator, seeded with --seed as well."""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def build(args, ctx, dev):
    """bench.run_train's scene, batch and targets (its seeds), at --frames x --pixels of an --size image."""
    import bench
    from hold_b200 import capi, scene_io, synth
    from hold_b200.model import HOLDNet

    hw = args.size or bench.H
    sc = synth.make_scene(H=hw, W=hw, S=bench.S, nodes=bench.NODES, B=args.frames, seed=0)
    for nid in sc.node_ids:
        sc.beta[nid] = torch.tensor(bench.BETA)
    fg = scene_io.build_net(sc, ctx, capi.MLP_TC)
    bg, _, _ = scene_io.build_background(sc, ctx, mlp_mode=capi.MLP_TC)
    net = HOLDNet(ctx, dict(fg.nodes), background=bg)
    gen = torch.Generator().manual_seed(100)
    ids = torch.stack([torch.randperm(hw * hw, generator=gen)[:args.pixels] for _ in range(args.frames)])
    inp = scene_io.scene_input(sc, dev)
    inp["uv"] = torch.gather(inp["uv"], 1, ids.to(dev)[:, :, None].expand(-1, -1, 2)).contiguous()
    leaves = {}
    for k in list(inp):
        if torch.is_tensor(inp[k]) and inp[k].is_floating_point() and any(k.endswith(s) for s in (".full_pose", ".transl", ".global_orient")):
            inp[k] = inp[k].clone().requires_grad_(True)
            leaves[f"input.{k}"] = inp[k]
    R = args.frames * args.pixels
    gt_rgb = torch.rand(R, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(7))
    gt_mask = torch.zeros(R, 4, device=dev)
    gt_mask[:, 0] = 1.0
    return net, inp, leaves, gt_rgb, gt_mask


def dump(d, step, ts, names, loss, parts):
    pre = os.path.join(d, f"step{step:03d}")

    def save(what, t, dtype=torch.float32):
        if t.numel():      # as bench.py's dump: empty tensors (the object's unused pose layer) are left out
            np.save(f"{pre}.{what}.npy", t.detach().to(dtype).cpu().numpy())

    save("loss", loss, torch.float64)
    for k, v in parts.items():
        save(f"loss_{k}", v, torch.float64)
    for p in ts.params:
        n = names[id(p)]
        save(f"param.{n}", p)
        if p.grad is not None:
            save(f"grad.{n}", p.grad)
        st = ts.opt.state.get(p, {})
        for k in ("exp_avg", "exp_avg_sq"):
            if k in st:
                save(f"adam_{k}.{n}", st[k])


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("dir")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--graph", action="store_true", help="capture the step as one CUDA graph and dump its replays")
    ap.add_argument("--stratified", action="store_true", help="training-mode (stratified) sampling")
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--pixels", type=int, default=128)
    ap.add_argument("--size", type=int, default=0, help="image height = width (default: the bench's)")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if args.graph and args.stratified:
        ap.error("a stratified training step cannot be captured as a CUDA graph (TrainStep)")
    import __graft_entry__ as g

    g.build()
    from hold_b200 import capi, train

    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    ctx = capi.Context(0)
    torch.manual_seed(args.seed)
    net, inp, leaves, gt_rgb, gt_mask = build(args, ctx, dev)
    ts = train.TrainStep(net, capturable=args.graph, stratified=args.stratified)
    ts.params = ts.params + list(leaves.values())
    names = {id(p): n for n, p in net.named_parameters()}
    names.update({id(p): n for n, p in leaves.items()})
    os.makedirs(args.dir, exist_ok=True)
    gen = torch.Generator(device=dev).manual_seed(args.seed) if args.stratified else None
    if args.graph:
        ts.capture(inp, gt_rgb, gt_mask, warmup=3)
    for i in range(args.steps):
        loss, parts = ts.replay() if args.graph else ts.step(inp, gt_rgb, gt_mask, generator=gen)
        torch.cuda.synchronize()
        dump(args.dir, i, ts, names, loss, parts)
    ctx.check()
    print(f"dump_train_steps: {args.steps} steps ({'graph replays' if args.graph else 'eager'}"
          f"{', stratified' if args.stratified else ''}) -> {args.dir}")


if __name__ == "__main__":
    main()
