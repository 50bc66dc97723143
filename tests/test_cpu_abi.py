"""CPU-only: the C-ABI library builds, loads and exports every symbol include/hold_b200.h declares, and the
product path fails loudly without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "hold_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(hold_[a-z_0-9]+)\s*\(", src)))


def test_header_symbols_exported(built):
    from hold_b200 import capi

    lib = capi.lib()
    names = declared_symbols()
    assert len(names) >= 17
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/hold_b200.h but not exported"
    assert set(names) == set(capi.EXPORTS), "ctypes table and header disagree"
    assert lib.hold_version() == 200


def test_struct_layouts_match_header(built):
    from hold_b200 import capi

    # field counts/sizes of the POD structs as the header lays them out (LP64)
    assert C.sizeof(capi.NodeCfg) == 8 * 4 + 5 * 4
    assert C.sizeof(capi.MlpWeights) == 4 + 9 * 4 + 9 * 4 + 4 + 3 * 9 * 8  # n_layers, in, out, pad, 3 pointer arrays
    assert C.sizeof(capi.NodePose) == 6 * 8 and C.sizeof(capi.Factors) == 6 * 8 and C.sizeof(capi.RenderOut) == 7 * 8
    assert C.sizeof(capi.SamplerRand) == 3 * 8 and C.sizeof(capi.ManoModel) == 8 * 8


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_no_cpu_fallback(built):
    from hold_b200 import capi

    h = C.c_void_p()
    rc = capi.lib().hold_ctx_create(C.byref(h), 0)
    assert rc == -2 and b"no CPU fallback" in capi.lib().hold_last_error()
    with pytest.raises(capi.HoldError):
        capi.Context(0)


def test_bad_arguments_are_errors_not_crashes(built):
    from hold_b200 import capi

    lib = capi.lib()
    assert lib.hold_ctx_create(None, 0) == -1
    assert lib.hold_ctx_destroy(None) == 0
    assert lib.hold_ctx_launch_count(None) == -1
    assert lib.hold_node_configure(None, 0, None) == -1


def test_sass_is_hopper_native(built):
    """The shipped .so carries wgmma / bulk-async / mbarrier / setmaxnreg SASS for sm_90a."""
    import subprocess

    from hold_b200 import capi

    out = subprocess.run(["cuobjdump", "-sass", capi.LIB_PATH], capture_output=True, text=True).stdout
    if not out:
        pytest.skip("cuobjdump unavailable")
    assert "sm_90a" in out
    for mnem in ("HGMMA", "UBLKCP", "SYNCS", "USETMAXREG"):
        assert mnem in out, f"{mnem} missing from SASS"
