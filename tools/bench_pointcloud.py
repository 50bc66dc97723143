"""Time the point-cloud evaluation kernels (hold_knn_points, hold_icp) at the sizes an evaluation meets.

Workloads:
  hands   K = 1 KNN and chamfer_distance over 256 frames of 778 vs 778 points (MANO vertices);
  object  K = 1 KNN and chamfer_distance of 1 x 2^17 points against 2^15;
  icp     point-to-point ICP, 30 iterations enqueued (convergence disabled), on 1 and on 16 pairs of 2^15 points;
and, where its [N,P1,P2] chunk fits in 2 GB, the torch brute force (fitting.knn_points' expression, in chunks of queries) for
comparison.  Prints one JSON line per workload: ms per call (CUDA events after warm-up), the card's name and power limit read
in the same run, and the point pairs evaluated per second (counted from shapes).

    python tools/bench_pointcloud.py [--iters 20]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def torch_knn1(p1, p2, chunk):
    """K = 1 brute force in torch, `chunk` queries at a time ([N,chunk,P2] distances per step)."""
    out = []
    for a in range(0, p1.shape[1], chunk):
        d = ((p1[:, a:a + chunk, None, :] - p2[:, None, :, :]) ** 2).sum(-1)
        out.append(d.min(-1).values)
    return torch.cat(out, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import __graft_entry__ as g

    g.build()
    from hold_b200 import capi
    from hold_b200 import pointcloud as PC

    assert torch.cuda.is_available(), "bench_pointcloud needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    ctx = capi.Context(0)
    info = card()
    gen = torch.Generator(device=dev).manual_seed(0)

    def emit(name, ms, pairs, **kw):
        print(json.dumps(dict(workload=name, ms=round(ms, 4), pair_evals_per_s=float(f"{pairs / (ms * 1e-3):.4g}"), card=info, **kw)),
              flush=True)

    for name, N, P1, P2 in (("hands", 256, 778, 778), ("object", 1, 2**17, 2**15)):
        x = torch.rand(N, P1, 3, device=dev, generator=gen)
        y = torch.rand(N, P2, 3, device=dev, generator=gen)
        emit(f"{name}_knn_k1", timed(lambda: PC.knn_points(ctx, x, y, K=1), args.iters), N * P1 * P2, N=N, P1=P1, P2=P2)
        emit(f"{name}_chamfer", timed(lambda: PC.chamfer_distance(ctx, x, y), args.iters), 2 * N * P1 * P2, N=N, P1=P1, P2=P2)
        chunk = max(1, min(P1, (2 << 30) // (N * P2 * 3 * 4)))
        ref = torch_knn1(x, y, chunk)
        got = PC.knn_points(ctx, x, y, K=1).dists[..., 0]
        ctx.check()
        emit(f"{name}_torch_knn_k1", timed(lambda: torch_knn1(x, y, chunk), max(2, args.iters // 4), warmup=1), N * P1 * P2, N=N, P1=P1,
             P2=P2, chunk=chunk, max_abs_diff_vs_kernel=float((ref - got).abs().max()))
    for N in (1, 16):
        P = 2**15
        src = torch.rand(N, P, 3, device=dev, generator=gen)
        tgt = (src + 0.01 * torch.randn(N, P, 3, device=dev, generator=gen)).contiguous()
        # relative thresholds < 0: the test never holds, so all 30 iterations run for every pair
        fn = lambda: PC.icp(ctx, src, tgt, 0.05, relative_fitness=-1.0, relative_rmse=-1.0, max_iteration=30)
        r = fn()
        ctx.check()
        assert int(r.iterations.min()) == 30
        emit(f"icp_{N}x{P}", timed(fn, max(2, args.iters // 4), warmup=1), N * P * P * 31, N=N, Ps=P, Pt=P, iterations=30,
             fitness=float(r.fitness.mean()))
    print(json.dumps(dict(done=True, card=info, launches=ctx.launches)))


if __name__ == "__main__":
    main()
