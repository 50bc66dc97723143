"""Where a layer of the tensor-core MLP kernel (hold_b200/csrc/mlp_tc.cuh) spends its clocks.

Builds the library a second time with -DHOLD_TC_PHASE_TIMING into the output directory (the default build and its output stay as
they are), and runs, once against each library in a process of its own:
  sdf_only : the bench-size sampler-round launch, 262 144 x 128 points, sdf head only, on both nodes' nets (k_mlp_tc<0>)
  sdf_rev  : sdf + gradient + feature on 2^20 points (k_mlp_tc<3>)
  colour   : the colour net on 2^20 points (k_mlp_tc<2>)
Prints ONE JSON line: per launch kind the mean SM clocks per phase (per consumer warp and layer-tile, by layer and over the whole
chain), each phase's share of a layer, the drift between the two warpgroups, the kernel's ms in the timed and in the untimed
library (the probe's own cost), and the card's name, power limit and SM clock as nvidia-smi reports them in the same call (sm_mhz_during: read while the sdf_only launches run).

  python tools/prof_mlp_phases.py [--out prof_out] [--reps 3]
Needs an H100; exits non-zero without a GPU."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SLOTS = ("wait_full", "stage_agree", "head", "mma", "epilogue", "fence_barrier", "prologue", "drift", "drift_abs", "count")
MAX_STEPS = 17
LAYER_PHASES = ("head", "mma", "epilogue", "fence_barrier")   # these four add up to a layer


def smi():
    try:
        o = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=10).stdout.strip().split(",")
        return {"name": o[0].strip(), "power_limit_w": float(o[1]), "sm_mhz": int(o[2]), "sm_max_mhz": int(o[3])}
    except Exception as e:   # noqa: BLE001 - the query is a label beside the numbers, not a measurement
        return {"unavailable": str(e)}


def summarise(raw, n_layers):
    """raw[l][wg][slot] sums -> mean clocks per consumer warp and layer-tile."""
    layers, tot = [], {k: 0.0 for k in SLOTS[:7]}
    for l in range(n_layers):
        n = raw[l][0][9] + raw[l][1][9]
        if n == 0:
            continue
        row = {k: (raw[l][0][i] + raw[l][1][i]) / n for i, k in enumerate(SLOTS[:7])}
        nd = raw[l][0][9] / 4.0                      # drift: warp 0 of warpgroup 0 records it, once per tile
        row["drift_wg0_minus_wg1"] = (raw[l][0][7] - (1 << 64) if raw[l][0][7] >= (1 << 63) else raw[l][0][7]) / nd
        row["drift_abs"] = raw[l][0][8] / nd
        row["layer"] = sum(row[k] for k in LAYER_PHASES)
        layers.append({"l": l, **{k: round(v, 1) for k, v in row.items()}})
        for k in tot:
            tot[k] += row[k]
    chain = sum(tot[k] for k in LAYER_PHASES) + tot["prologue"]
    share = {k: round(tot[k] / chain, 4) for k in tot}
    return {"clocks_per_tile": {k: round(v, 1) for k, v in tot.items()}, "tile": round(chain, 1), "share_of_tile": share, "layers": layers}


def worker(lib_path, reps):
    import torch

    from hold_b200 import capi

    capi.LIB_PATH = lib_path
    from hold_b200 import scene_io, synth

    L = capi.lib()
    timed = hasattr(L, "hold_tc_phase_read")
    if timed:
        L.hold_tc_phase_read.restype, L.hold_tc_phase_read.argtypes = C.c_int, [C.c_void_p, C.c_void_p]
    ctx, dev = capi.Context(0), torch.device("cuda", 0)
    sc = synth.make_scene(H=8, W=8, S=128, nodes=("right", "object"))
    nodes = scene_io.build_net(sc, ctx, capi.MLP_TC).nodes
    P0, P1 = 512 * 512 * 128, 1 << 20
    g = torch.Generator().manual_seed(0)
    xc = ((torch.rand(P0, 3, generator=g) - 0.5) * 1.6).to(dev)
    sdf = torch.empty(P0, device=dev)
    grad, feat, rgb = torch.empty(P1, 3, device=dev), torch.empty(P1, 256, device=dev), torch.empty(P1, 3, device=dev)
    nrm = torch.nn.functional.normalize(torch.randn(P1, 3, generator=g), dim=1).to(dev)
    tcode = torch.randn(1, 32, generator=g).to(dev)
    s = capi.stream_ptr()

    def sdf_only():
        for nid in ("right", "object"):
            capi.check(L.hold_sdf_eval(ctx.h, nodes[nid].slot, P0, capi.ptr(xc), None, capi.ptr(sdf), None, None, s))

    def sdf_rev():
        capi.check(L.hold_sdf_eval(ctx.h, nodes["right"].slot, P1, capi.ptr(xc), None, capi.ptr(sdf), capi.ptr(grad), capi.ptr(feat), s))

    def colour():
        capi.check(L.hold_rgb_eval(ctx.h, nodes["object"].slot, 1, P1, capi.ptr(xc), capi.ptr(nrm), None, capi.ptr(feat), capi.ptr(tcode), capi.ptr(rgb), s))

    raw = (C.c_ulonglong * (MAX_STEPS * 2 * len(SLOTS)))()
    out = {}
    for name, fn, launches, n_layers in (("sdf_only", sdf_only, 2, 8), ("sdf_rev", sdf_rev, 1, 17), ("colour", colour, 1, MAX_STEPS)):
        fn()
        torch.cuda.synchronize()
        if timed:
            capi.check(L.hold_tc_phase_read(ctx.h, raw))   # drop the warm-up's clocks
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        during = smi() if name == "sdf_only" else None   # the launches are still running: the SM clock under this load
        torch.cuda.synchronize()
        ctx.check()
        out[name] = {"ms_per_launch": e0.elapsed_time(e1) / (reps * launches)}
        if during is not None:
            out[name]["sm_mhz_during"] = during.get("sm_mhz")
        if timed:
            capi.check(L.hold_tc_phase_read(ctx.h, raw))
            r = [[[int(raw[(l * 2 + w) * len(SLOTS) + k]) for k in range(len(SLOTS))] for w in range(2)] for l in range(MAX_STEPS)]
            out[name].update(summarise(r, n_layers))
    print("PHASES " + json.dumps(out))


def run_worker(lib_path, reps):
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", lib_path, "--reps", str(reps)], capture_output=True, text=True)
    for line in p.stdout.splitlines():
        if line.startswith("PHASES "):
            return json.loads(line[7:])
    sys.stderr.write(p.stdout + p.stderr)
    raise SystemExit(f"worker on {lib_path} failed (exit {p.returncode})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "prof_out"))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--untimed-lib", default=None, help="library for the untimed ms (default: the tree's build)")
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("prof_mlp_phases: needs a GPU (no CPU fallback)")
    if args.worker:
        return worker(args.worker, args.reps)
    import __graft_entry__ as g

    g.build()
    os.makedirs(args.out, exist_ok=True)
    timing_lib = os.path.join(args.out, "libhold_b200_phase_timing.so")
    srcs = [os.path.join(g.CSRC, f) for f in os.listdir(g.CSRC)] + [os.path.join(ROOT, "include", "hold_b200.h")]
    if not os.path.exists(timing_lib) or any(os.path.getmtime(f) > os.path.getmtime(timing_lib) for f in srcs):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.run([nvcc] + g.NVCC_FLAGS + ["-DHOLD_TC_PHASE_TIMING", "-o", timing_lib, os.path.join(g.CSRC, "api.cu")], check=True, cwd=g.CSRC)
    gpu = smi()
    timed = run_worker(timing_lib, args.reps)
    untimed = run_worker(args.untimed_lib or g.LIB, args.reps)
    for k in timed:
        timed[k]["ms_per_launch_untimed"] = untimed[k]["ms_per_launch"]
    print(json.dumps({"tool": "prof_mlp_phases", "unit": "SM clocks per consumer warp and 128-row tile (mean)", "gpu": gpu, "kinds": timed}))


if __name__ == "__main__":
    main()
