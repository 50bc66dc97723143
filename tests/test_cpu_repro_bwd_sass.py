"""CPU-only: the soft-silhouette backward (hold_raster_silhouette_bwd) and the K-NN backward (hold_knn_points_bwd) add in a fixed
order.  None of their kernels may add floating-point values into global memory with atomics (RED / ATOM), nor use a
shared-memory atomic (ATOMS: an fp32 atomicAdd to shared memory compiles to an ATOMS.CAST.SPIN loop): the order of such adds is
the order in which threads get there, and the result's last bits would change from run to run (raster.cuh, pointcloud.cuh,
inverse_map.cuh)."""
import pytest

from test_cpu_wgrad_sass import FLOAT_GLOBAL_ADD, _sass_by_function

RASTER_BWD = ("k_rasterILb1E", "k_raster_bwd_faces", "k_raster_bwd_verts", "k_raster_vert_keys")
KNN_BWD = ("k_knn_bwd_rows", "k_knn_bwd_targets")
INVERSE_MAP = ("k_im_hist", "k_im_scan", "k_im_scatter", "k_im_first")   # shared by both


def _unordered_adds(ops):
    return sorted({op for op in ops if FLOAT_GLOBAL_ADD.match(op) or op.startswith("ATOMS")})


@pytest.mark.parametrize("path", ["raster", "knn"])
def test_backward_kernels_have_no_float_atomics(built, path):
    from hold_b200 import capi

    funcs = _sass_by_function(capi.LIB_PATH)
    want = (RASTER_BWD if path == "raster" else KNN_BWD) + INVERSE_MAP
    for w in want:
        names = [k for k in funcs if w in k]
        assert names, f"no kernel named {w}"
        for k in names:
            bad = _unordered_adds(funcs[k])
            print(f"{k}: {len(funcs[k])} SASS instructions, unordered adds {bad}")
            assert not bad, (k, bad)


def test_shared_float_add_is_caught():
    assert _unordered_adds(["ATOMS.CAST.SPIN", "REDG.E.ADD.F32.FTZ.RN.STRONG.GPU", "ATOMS.ADD", "FADD"]) == [
        "ATOMS.ADD", "ATOMS.CAST.SPIN", "REDG.E.ADD.F32.FTZ.RN.STRONG.GPU"]
