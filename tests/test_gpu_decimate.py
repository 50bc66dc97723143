"""Quadric edge-collapse decimation on the GPU (hold_decimate, hold_b200.meshing.decimate) against its host restatement
(tests/host/decimate_host.cpp over the same decimate_phases.h): counts, vertices and faces bit for bit on every mesh of
test_cpu_decimate.py and on the canonical object mesh that generate_mesh(backend="gpu") extracts from a synthetic object node at
the reference's resolution, decimated to 3 000 faces; repeated calls bit-identical; bad arguments and out-of-range indices
caught; the decimated object's soft silhouette at 512 x 512 close to the full mesh's (IoU)."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_cpu_decimate import check_closed_oriented, euler, host_decimate, latlong_sphere, meshes

pytestmark = pytest.mark.gpu


def _same(dev, host):
    (v0, f0), (v1, f1) = dev, host
    v0, f0 = v0.cpu().numpy(), f0.cpu().numpy()
    return v0.shape == v1.shape and f0.shape == f1.shape and np.array_equal(v0.view(np.int32), v1.view(np.int32)) and np.array_equal(f0, f1)


@pytest.fixture(scope="module")
def cpu_meshes():
    m = meshes()
    v, f = latlong_sphere(20, 24)
    keep = (v[f][:, :, 2] > -1e-6).all(1)
    m["hemisphere"] = (v, f[keep])                  # open: a boundary loop, and unused vertices below the equator
    m["octahedron"] = (np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32),
                       np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]], np.int32))
    return m


@pytest.fixture(scope="module")
def object_mesh(ctx):
    """generate_mesh(backend="gpu") of a synthetic object node at the reference's resolution (res_init 32, 3 upsampling steps)"""
    from hold_b200 import capi, meshing, scene_io, synth

    sc = synth.make_scene(H=8, W=8, S=32, nodes=("right", "object"), seed=4)
    net = scene_io.build_net(sc, ctx, capi.MLP_TC)
    v, f = meshing.generate_mesh(ctx, meshing.node_sdf_func(ctx, net.nodes["object"]), sc.obj_pts_cano.numpy(), backend="gpu")
    ctx.check()
    return np.ascontiguousarray(v, np.float32), np.ascontiguousarray(f, np.int32)


def test_device_equals_host_restatement(ctx, cpu_meshes):
    from hold_b200 import meshing

    for name, (v, f) in cpu_meshes.items():
        for frac in (0.5, 0.1, 0.02, 0.0):
            t = int(f.shape[0] * frac)
            dv, df = meshing.decimate(ctx, v, f, t)
            hv, hf, _ = host_decimate(v, f, t)
            assert _same((dv, df), (hv, hf)), f"{name} at {frac}: device and host differ"


def test_object_mesh_to_3000_faces(ctx, object_mesh):
    from hold_b200 import meshing

    v, f = object_mesh
    hv, hf, rounds = host_decimate(v, f, 3000)
    dev = meshing.decimate(ctx, v, f, 3000)
    print(f"object mesh: {v.shape[0]} vertices, {f.shape[0]} faces, chi {euler(v, f)} -> {hf.shape[0]} faces in {rounds} rounds")
    assert _same(dev, (hv, hf))
    for _ in range(3):                                                    # repeated calls: the same bits
        assert _same(meshing.decimate(ctx, torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), 3000), (hv, hf))
    assert euler(hv, hf) == euler(v, f)
    # the target, or a stop below the round cap where no edge passes the rules: this object's surface leaves the grid (chi -1, an
    # open mesh) and its boundary vertices never move; it stopped at 6 038 faces when this test was written
    assert hf.shape[0] in (3000, 2999) or (rounds < 1000 and 3000 < hf.shape[0] < f.shape[0] // 50)


def test_target_at_least_f_and_bad_arguments(ctx, cpu_meshes):
    from hold_b200 import capi, meshing

    v, f = cpu_meshes["latlong"]
    dv, df = meshing.decimate(ctx, v, f, f.shape[0])
    assert np.array_equal(dv.cpu().numpy(), v) and np.array_equal(df.cpu().numpy(), f)
    with pytest.raises(capi.HoldError):
        meshing.decimate(ctx, v, f, -1)
    bad = f.copy()
    bad[7, 2] = v.shape[0]
    with pytest.raises(capi.HoldError, match="outside"):
        meshing.decimate(ctx, v, bad, 100)
    bad[7, 2] = -1
    with pytest.raises(capi.HoldError, match="outside"):
        meshing.decimate(ctx, v, bad, 100)
    ctx.check()                                                           # the error word was cleared
    lib, nv, nf = capi.lib(), C.c_int(0), C.c_int(0)
    s = capi.stream_ptr()
    assert lib.hold_decimate(None, 3, None, 1, None, 0, C.c_float(0.3), None, None, C.byref(nv), C.byref(nf), s) == -1
    assert lib.hold_decimate(ctx.h, 3, None, 1, None, 0, C.c_float(0.3), None, None, C.byref(nv), C.byref(nf), s) == -1
    assert lib.hold_decimate(ctx.h, 3, None, 1 << 30, None, 0, C.c_float(0.3), None, None, C.byref(nv), C.byref(nf), s) == -1
    assert "2^31" in lib.hold_last_error().decode()
    assert lib.hold_decimate(ctx.h, 3, None, 1, None, 0, C.c_float(float("nan")), None, None, C.byref(nv), C.byref(nf), s) == -1
    dv, df = meshing.decimate(ctx, v, f, 300)                             # still works after the errors
    assert _same((dv, df), host_decimate(v, f, 300)[:2])


# IoU of the decimated object's silhouette against the full mesh's at 512 x 512.  The first run, on an NVIDIA H100 80GB HBM3,
# gave 0.919 (491 148 -> 6 038 faces, 142 878 silhouette pixels of the full mesh)
IOU_MIN = 0.90


def test_silhouette_of_the_decimated_object(ctx, object_mesh):
    from hold_b200 import fitting, meshing

    v, f = object_mesh
    dv, df = meshing.decimate(ctx, v, f, 3000)
    vt = torch.from_numpy(v).cuda()
    c, ext = (vt.max(0).values + vt.min(0).values) / 2, (vt.max(0).values - vt.min(0).values).max()
    K = torch.tensor([[1024.0, 0, 256.0], [0, 1024.0, 256.0], [0, 0, 1]], device="cuda")
    R = fitting.SilhouetteRenderer(ctx, 512)

    def sil(verts, faces):
        cam = (verts - c) / ext + torch.tensor([0.0, 0.0, 2.5], device="cuda")     # the object ~400 px across
        return R(fitting.project_ndc(cam[None], K, 512, 512).contiguous(), faces.int().contiguous())[0, ..., 3] > 0.5

    a, b = sil(vt, torch.from_numpy(f).cuda()), sil(dv, df)
    ctx.check()
    iou = ((a & b).sum() / (a | b).sum()).item()
    print(f"silhouette IoU at 512 x 512, {f.shape[0]} -> {df.shape[0]} faces: {iou:.5f} ({a.sum().item()} px)")
    assert a.sum() > 10000 and iou >= IOU_MIN
