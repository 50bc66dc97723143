"""SURVEY §8f rank 4 on the GPU: (1) the device MISE (hold_mise_*) driven with the analytic fields of tests/test_cpu_mise.py,
round by round against the stored outputs of the reference's own MISE (tests/golden/mise/mise_cases.json); (2) generate_grid,
the GPU MISE fed by the fused-MLP SDF queries, against the host restatement (tests/host/mise_host.cpp, which test_cpu_mise.py
holds to the same goldens) fed with the SAME SDF values round by round -> identical dense grids."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def impl_generate_grid_matches_host_mise(ctx):
    from hold_b200 import capi, meshing, scene_io, synth

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_cpu_mise import _host

    lib = _host()
    dev = torch.device("cuda", 0)
    sc = synth.make_scene(H=8, W=8, S=32, nodes=("right", "object"), seed=4)
    net = scene_io.build_net(sc, ctx, capi.MLP_FP32)
    node = net.nodes["object"]
    func = meshing.node_sdf_func(ctx, node)
    verts = sc.obj_pts_cano.numpy()
    grid, res, gt_scale, gt_center = meshing.generate_grid(ctx, func, verts, 0.0, res_init=8, res_up=2)
    ctx.check()
    # the reference loop (utils/meshing.py:19-47) with the same SDF function
    G = (8 << 2) + 1
    h = lib.mise_host_create(8, 2, C.c_float(0.0))
    buf = np.zeros((G**3, 3), np.int32)
    rounds = 0
    while True:
        n = lib.mise_host_query(h, buf.ctypes.data_as(C.c_void_p), C.c_int(G**3))
        if n == 0:
            break
        p = buf[:n].astype(np.float32)
        p = (p / (G - 1) - 0.5) * 1.1
        p = p * gt_scale + gt_center
        vals = np.ascontiguousarray(func(torch.tensor(p).float().to(dev).contiguous()).cpu().numpy().astype(np.float32))
        lib.mise_host_update(h, vals.ctypes.data_as(C.c_void_p))
        rounds += 1
    ref = np.empty(G**3, np.float32)
    lib.mise_host_to_dense(h, ref.ctypes.data_as(C.c_void_p))
    lib.mise_host_destroy(h)
    ref = ref.reshape(G, G, G).astype(np.float64)
    assert rounds >= 2 and grid.shape == ref.shape == (33, 33, 33)
    assert np.array_equal(grid, ref)
    assert (grid < 0).any() and (grid > 0).any()


def impl_device_mise_matches_reference_mise_goldens(ctx):
    from hold_b200 import meshing

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_cpu_mise as T

    for res0, depth, seed in T.CASES:
        ex = meshing.MISE(ctx, res0, depth, 0.0)
        query = lambda: ex.query().cpu().numpy()
        update = lambda pts, vals: ex.update(None, torch.from_numpy(vals).to(ex._dev))
        dense = lambda: ex.to_dense().cpu().numpy()
        d = T.digest(*T.run_mise(query, update, dense, res0, depth, seed))
        ctx.check()
        ex.close()
        T.assert_matches_golden(d, res0, depth, seed, f"device MISE {res0},{depth},{seed} vs reference MISE goldens")


def test_device_mise_matches_reference_mise_goldens(isolated):
    isolated("tests/test_gpu_mise.py", "impl_device_mise_matches_reference_mise_goldens")


def test_generate_grid_matches_host_mise(isolated):
    isolated("tests/test_gpu_mise.py", "impl_generate_grid_matches_host_mise")
