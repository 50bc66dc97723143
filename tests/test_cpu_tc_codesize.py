"""CPU-only: properties of the shipped tensor-core MLP kernels that the phase timing (tools/prof_mlp_phases.py, DESIGN.md §3.1)
showed to matter, read from the library's SASS, and the dump comparison tool on synthetic arrays.

* The epilogues are straight-line code and run at pace only while a layer's body fits the instruction cache.  The sampler-round
  kernel k_mlp_tc<0> once carried an inlined Fourier embedding in all 64 column-pair instances of its skip layer (14 216
  instructions, 227 KB; that layer's epilogue took 6x a plain layer's clocks); it is held below 7 000 instructions here.
* The phase-timing probes are compiled out of the shipped library."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sass_instruction_counts(lib_path):
    out = subprocess.run(["cuobjdump", "-sass", lib_path], capture_output=True, text=True).stdout
    if not out:
        pytest.skip("cuobjdump unavailable")
    counts, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = 0
        elif cur is not None and re.match(r"\s+/\*[0-9a-f]{4,6}\*/\s+\S", line):
            counts[cur] += 1
    return counts


def test_sampler_round_kernel_fits_the_instruction_cache_budget(built):
    from hold_b200 import capi

    counts = _sass_instruction_counts(capi.LIB_PATH)
    name = [k for k in counts if "k_mlp_tcILi0E" in k]
    assert len(name) == 1, name
    n = counts[name[0]]
    print(f"k_mlp_tc<0>: {n} SASS instructions ({16 * n / 1024:.0f} KB)")
    assert 3000 < n < 7000, n


def test_phase_timing_is_compiled_out_of_the_shipped_library(built):
    from hold_b200 import capi

    assert not hasattr(capi.lib(), "hold_tc_phase_read")
    syms = subprocess.run(["nm", "-D", capi.LIB_PATH], capture_output=True, text=True).stdout
    assert "g_tc_phase" not in syms and "hold_tc_phase_read" not in syms


def test_compare_dumps(tmp_path):
    rng = np.random.default_rng(0)
    a, b = tmp_path / "a", tmp_path / "b"
    a.mkdir(), b.mkdir()
    x = rng.random((1000, 3)).astype(np.float32)
    y = x.copy()
    y[:10, 1] += 1e-3                      # 1 % of the rays move beyond 1e-4
    y[10:, 0] += 1e-6
    for d, v in ((a, x), (b, y)):
        np.save(d / "fg_rgb.npy", v)
        np.save(d / "sampler_iters.npy", np.array([5.0, 5.0]))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "compare_dumps.py"), str(a), str(b)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    import json

    res = json.loads(r.stdout.strip().splitlines()[-1])["arrays"]
    assert res["sampler_iters"]["identical"] and res["sampler_iters"]["max_abs"] == 0.0
    assert abs(res["fg_rgb"]["rays_within_1e-4"] - 0.99) < 1e-9 and 9e-4 < res["fg_rgb"]["max_abs"] < 1.1e-3
    np.save(b / "extra.npy", x)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "compare_dumps.py"), str(a), str(b)], capture_output=True, text=True)
    assert r.returncode == 1
