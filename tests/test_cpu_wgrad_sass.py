"""CPU-only: the weight-gradient reduction (hold_wgrad) reduces in a fixed order.  Its kernels, k_wgrad_tc and k_wgrad_sum, must
not add floating-point values into global memory with atomics (RED / ATOM): the order of such adds is the order in which CTAs
finish, and the result's last bits would change from run to run (wgrad_tc.cuh)."""
import re
import subprocess

import pytest


def _sass_by_function(lib_path):
    out = subprocess.run(["cuobjdump", "-sass", lib_path], capture_output=True, text=True).stdout
    if not out:
        pytest.skip("cuobjdump unavailable")
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9._]*)", line)
        if cur is not None and m:
            funcs[cur].append(m.group(1))
    return funcs


# global reductions / atomics whose operation is a floating-point add, e.g. REDG.E.ADD.F32.FTZ.RN.STRONG.GPU
FLOAT_GLOBAL_ADD = re.compile(r"^(RED|REDG|ATOM|ATOMG)\..*\bADD\.(F16|BF16|F16x2|BF16x2|F32|F64)\b")


def test_float_global_add_pattern():
    assert FLOAT_GLOBAL_ADD.match("REDG.E.ADD.F32.FTZ.RN.STRONG.GPU")
    assert FLOAT_GLOBAL_ADD.match("ATOMG.E.ADD.F32.FTZ.RN.STRONG.GPU")
    assert not FLOAT_GLOBAL_ADD.match("ATOMG.E.ADD.STRONG.GPU")      # integer add
    assert not FLOAT_GLOBAL_ADD.match("ATOMS.ADD.F32")                # shared memory
    assert not FLOAT_GLOBAL_ADD.match("RED.AND.DEFER_BLOCKING")


def test_wgrad_kernels_have_no_float_atomics_to_global_memory(built):
    from hold_b200 import capi

    funcs = _sass_by_function(capi.LIB_PATH)
    names = [k for k in funcs if "k_wgrad_" in k]
    assert any("k_wgrad_tc" in k for k in names), names
    for k in names:
        bad = [op for op in funcs[k] if FLOAT_GLOBAL_ADD.match(op)]
        print(f"{k}: {len(funcs[k])} SASS instructions, {len(bad)} floating-point global atomics")
        assert not bad, (k, sorted(set(bad)))
