"""Compare two output dumps of `python bench.py --steps K --dump-outputs DIR` (same seed, two builds of the library).

  python tools/compare_dumps.py DIR_A DIR_B

Prints, per array present in both: max and mean absolute difference, and for per-ray arrays the share of rays whose every
component agrees within 1e-4 (times max(1, max|A|), the bar of tests/test_gpu_e2e.py); then one JSON line with the same numbers.
Exits 1 if an array exists on one side only or the shapes differ."""
import json
import os
import sys

import numpy as np


def compare(a, b):
    d = np.abs(a.astype(np.float64) - b.astype(np.float64))
    row = {"max_abs": float(d.max()) if d.size else 0.0, "mean_abs": float(d.mean()) if d.size else 0.0, "identical": bool(np.array_equal(a, b))}
    if a.ndim >= 1 and a.shape[0] > 1:
        tol = 1e-4 * max(1.0, float(np.abs(a).max()))
        row["rays_within_1e-4"] = float((d.reshape(a.shape[0], -1).max(axis=1) <= tol).mean())
    return row


def main(dir_a, dir_b):
    names = lambda d: {f[:-4] for f in os.listdir(d) if f.endswith(".npy")}
    na, nb = names(dir_a), names(dir_b)
    bad = sorted(na ^ nb)
    out = {}
    for k in sorted(na & nb):
        a, b = np.load(os.path.join(dir_a, k + ".npy")), np.load(os.path.join(dir_b, k + ".npy"))
        if a.shape != b.shape:
            bad.append(k)
            continue
        out[k] = r = compare(a, b)
        share = f"  rays within 1e-4: {r['rays_within_1e-4']:.6f}" if "rays_within_1e-4" in r else ""
        print(f"{k:24s} {str(a.shape):18s} max|d| {r['max_abs']:.3e}  mean|d| {r['mean_abs']:.3e}{'  identical' if r['identical'] else ''}{share}")
    print(json.dumps({"tool": "compare_dumps", "a": dir_a, "b": dir_b, "arrays": out, "mismatched": bad}))
    return 1 if bad else 0


if __name__ == "__main__":
    if len(sys.argv) != 3:
        raise SystemExit(__doc__)
    sys.exit(main(sys.argv[1], sys.argv[2]))
