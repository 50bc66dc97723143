"""Run N Adam steps of the pose-refinement scene of tests/test_gpu_fit_repro.py and dump the state after every step, for
bit-for-bit comparison of two builds or two runs (the refinement counterpart of tools/dump_train_steps.py).

  python tools/dump_fit_steps.py DIR [--steps N] [--graph]
  python tools/compare_dumps.py DIR_A DIR_B

The scene: the synthetic MANO rig (hold_mano_lbs / _bwd) with convex-hull faces and an object (hold_object_tf / _bwd, obj_scale
frozen), drawn together by the soft-silhouette rasteriser, with an L1 silhouette loss and a fingertip-to-object contact term on
pointcloud.knn_points.  After every step DIR holds, as float32 .npy files named `stepNNN.<what>.<leaf>`: the loss, every pose
leaf, its .grad and Adam's state (adam_exp_avg, adam_exp_avg_sq, adam_step).  --graph captures one step as a CUDA graph
(after three eager warm-up steps) and dumps its replays."""
import argparse
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("dir")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--graph", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dump_fit_steps.py needs a GPU")
    spec = importlib.util.spec_from_file_location("fit_repro", os.path.join(ROOT, "tests", "test_gpu_fit_repro.py"))
    scene = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(scene)
    from hold_b200 import capi

    torch.cuda.set_device(0)
    ctx = capi.Context(0)
    snaps = scene.refine_run(ctx, args.steps, graph=args.graph)
    os.makedirs(args.dir, exist_ok=True)
    for i, snap in enumerate(snaps):
        for k, v in snap.items():
            np.save(os.path.join(args.dir, f"step{i:03d}.{k}.npy"), v.detach().float().cpu().numpy())
    print(f"{len(snaps)} steps, loss {snaps[0]['loss'].item():.6f} -> {snaps[-1]['loss'].item():.6f}, written to {args.dir}")
    ctx.close()


if __name__ == "__main__":
    main()
