"""Largest-component selection and canonical meshing on the GPU (hold_largest_component, meshing.largest_component_device,
meshing.extract_mesh, Node.meshing_cano, train.meshing_cano) against the host: the device selection equals
meshing.largest_component bit for bit on every mesh of test_cpu_mesh_cc.py and on the synthetic object node's marching-cubes mesh
at the reference's resolution; repeated calls bit-identical; an out-of-range index raises HoldError; generate_mesh(backend="gpu")
equals the host composition it replaced (kept inline below) bit for bit, on an analytic field and on the object node; an empty
level set raises ValueError; training after train.meshing_cano equals training with the host-built mesh attached by hand; the
mesh follows the current BARF mask; a captured TrainStep refuses to replay after a refresh and replays after a new capture."""
import math

import numpy as np
import pytest
import torch

from test_cpu_mesh_cc import cases
from test_gpu_train_repro import _assert_equal_runs, _batch, _make, _snapshot

pytestmark = pytest.mark.gpu


def host_generate_mesh(ctx, func, verts, level_set=0.0, res_init=32, res_up=3):
    """generate_mesh(backend="gpu") as it was before the selection moved to the device: the float64 grid on the host, back to
    the device for marching cubes, the grid-to-world transform in numpy and largest_component with scipy.  Also returns the
    marching-cubes mesh."""
    from hold_b200 import meshing

    grid, res, gt_scale, gt_center = meshing.generate_grid(ctx, func, verts, level_set, res_init, res_up)
    dev = torch.device("cuda", ctx.device)
    v, f = meshing.marching_cubes(ctx, torch.as_tensor(grid, device=dev), level_set)
    verts_mc = ((v.cpu().numpy() / res - 0.5) * 1.1) * gt_scale + gt_center
    faces = f.cpu().numpy().astype(np.int64)
    return meshing.largest_component(verts_mc, faces), (verts_mc, faces)


def same(a, b):
    (v0, f0), (v1, f1) = a, b
    v0, f0, v1, f1 = (t.cpu().numpy() if torch.is_tensor(t) else np.asarray(t) for t in (v0, f0, v1, f1))
    return (v0.dtype == v1.dtype == np.float32 and v0.shape == v1.shape and f0.shape == f1.shape
            and np.array_equal(v0.view(np.int32), v1.view(np.int32)) and np.array_equal(f0, f1))


def two_spheres(pts):
    d0 = (pts - torch.tensor([0.3, 0.0, 0.0], device=pts.device)).norm(dim=1) - 0.25
    d1 = (pts - torch.tensor([-0.3, 0.1, 0.0], device=pts.device)).norm(dim=1) - 0.15
    return torch.minimum(d0, d1)


@pytest.fixture(scope="module")
def object_node(ctx):
    from hold_b200 import capi, meshing, scene_io, synth

    sc = synth.make_scene(H=8, W=8, S=32, nodes=("right", "object"), seed=4)
    net = scene_io.build_net(sc, ctx, capi.MLP_TC)
    obj = net.nodes["object"]
    return sc, obj, meshing.node_sdf_func(ctx, obj)


def test_device_equals_host_on_every_case(ctx):
    from hold_b200 import meshing

    for name, (v, f) in cases().items():
        ref = meshing.largest_component(v, f.astype(np.int64))
        dev = meshing.largest_component_device(ctx, v, f)
        assert dev[1].dtype == torch.int32 and same(dev, ref), name
        for _ in range(2):
            assert same(meshing.largest_component_device(ctx, torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()), ref), name
    ctx.check()


def test_bad_index_and_no_face(ctx):
    from hold_b200 import capi, meshing

    v, f = cases()["soup0"]
    for bad_value in (v.shape[0], -1):
        bad = f.copy()
        bad[11, 1] = bad_value
        with pytest.raises(capi.HoldError, match="outside"):
            meshing.largest_component_device(ctx, v, bad)
    ctx.check()                                                           # the error word was cleared
    with pytest.raises(ValueError):
        meshing.largest_component_device(ctx, v, f[:0])
    assert same(meshing.largest_component_device(ctx, v, f), meshing.largest_component(v, f.astype(np.int64)))


def test_generate_mesh_on_an_analytic_field(ctx):
    from hold_b200 import meshing

    box = np.array([[-0.6, -0.6, -0.6], [0.6, 0.6, 0.6]], np.float32)
    for res_init, res_up in ((16, 2), (20, 2), (32, 3)):
        ref, (mv, mf) = host_generate_mesh(ctx, two_spheres, box, 0.0, res_init, res_up)
        got = meshing.generate_mesh(ctx, two_spheres, box, res_init=res_init, res_up=res_up, backend="gpu")
        assert got[1].dtype == np.int64 and same(got, ref), (res_init, res_up)
        assert same(meshing.extract_mesh(ctx, two_spheres, box, 0.0, res_init, res_up), ref)
        print(f"two spheres at {res_init} / {res_up}: {mf.shape[0]} marching-cubes faces -> {ref[1].shape[0]}")
    # the grid-to-world transform alone at power-of-two and other resolutions, against numpy's
    rng = np.random.default_rng(0)
    idx = (rng.random((100000, 3)) * 160).astype(np.float32)
    for res in (160, 256, 96):
        gt_scale, gt_center = np.float32(1.37), np.array([0.1, -0.2, 0.3], np.float32)
        ref_w = ((idx / res - 0.5) * 1.1) * gt_scale + gt_center
        got_w = meshing.grid_to_world(torch.from_numpy(idx).cuda(), res, gt_scale, gt_center).cpu().numpy()
        assert np.array_equal(got_w.view(np.int32), ref_w.view(np.int32)), res


def test_empty_level_set_raises(ctx):
    from hold_b200 import meshing

    box = np.array([[-0.6, -0.6, -0.6], [0.6, 0.6, 0.6]], np.float32)
    outside = lambda p: torch.ones(p.shape[0], device=p.device)
    with pytest.raises(ValueError):
        host_generate_mesh(ctx, outside, box, 0.0, 16, 1)
    with pytest.raises(ValueError):
        meshing.generate_mesh(ctx, outside, box, res_init=16, res_up=1, backend="gpu")
    with pytest.raises(ValueError):
        meshing.extract_mesh(ctx, outside, box, 0.0, 16, 1)


def test_object_node_mesh(ctx, object_node):
    from hold_b200 import meshing

    sc, obj, func = object_node
    ref, (mv, mf) = host_generate_mesh(ctx, func, sc.obj_pts_cano.numpy())
    got = meshing.generate_mesh(ctx, func, sc.obj_pts_cano.numpy(), backend="gpu")
    print(f"object node: {mf.shape[0]} marching-cubes faces, largest component {ref[1].shape[0]} faces, {ref[0].shape[0]} vertices")
    assert mf.shape[0] > 400000
    assert same(got, ref)
    vd, fd = torch.from_numpy(mv).cuda(), torch.from_numpy(mf).cuda()
    for _ in range(3):                                                    # repeated calls: the same bits
        assert same(meshing.largest_component_device(ctx, vd, fd), ref)
    ctx.check()


def test_node_meshing_cano(ctx, object_node):
    from hold_b200 import meshing

    sc, obj, func = object_node
    v, f = obj.meshing_cano(16, 2)
    assert v.is_cuda and f.dtype == torch.int32 and obj.mesh_vo_cano is v and obj.mesh_fo_cano is f
    ref, _ = host_generate_mesh(ctx, func, obj.server.verts_c[0], 0.0, 16, 2)
    assert same((v, f), ref)


def test_meshing_follows_the_barf_mask(ctx):
    from hold_b200 import capi, meshing, scene_io, synth

    sc = synth.make_scene(H=8, W=8, S=32, nodes=("right", "object"), seed=4)
    net = scene_io.build_net(sc, ctx, capi.MLP_TC)
    obj = net.nodes["object"]
    with torch.no_grad():                                                 # the geometric init gives the frequencies no weight
        g = torch.Generator(device="cuda").manual_seed(2)
        w0 = obj.implicit_network.state_dict()["lin0.weight_v"]
        w0[:, 3:] += 0.05 * torch.randn(w0[:, 3:].shape, device=w0.device, generator=g)
    obj.start_barf(0, 12)
    for _ in range(5):
        obj.step_embedding()
    w = obj.barf_weights.clone()
    assert 0 < float(w.min()) < 1 or (w == 0).any()                       # a partial mask: some frequencies are off
    v, f = obj.meshing_cano(16, 2)
    box = obj.server.verts_c[0]
    masked = meshing.extract_mesh(ctx, meshing.node_sdf_func(ctx, obj, embed_w=w), box, 0.0, 16, 2)
    plain = meshing.extract_mesh(ctx, meshing.node_sdf_func(ctx, obj), box, 0.0, 16, 2)
    assert same((v, f), masked)
    assert not same((v, f), plain)


def _steps_with_mesh(ctx, refresh):
    from hold_b200 import meshing, train

    sc, net = _make(ctx)
    obj = net.nodes["object"]
    if refresh:
        meshes = train.meshing_cano(net, 16, 2)
        assert set(meshes) == {"right", "object"} and obj.mesh_vo_cano is meshes["object"][0]
        assert getattr(net.nodes["right"], "mesh_v_cano_div", None) is None
    else:
        (v, f), _ = host_generate_mesh(ctx, meshing.node_sdf_func(ctx, obj), obj.server.verts_c[0], 0.0, 16, 2)
        obj.mesh_vo_cano, obj.mesh_fo_cano = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    mesh = (obj.mesh_vo_cano.cpu().numpy(), obj.mesh_fo_cano.cpu().numpy())
    inp, _, _ = _batch(sc)
    dev = torch.device("cuda", 0)
    B, P = inp["uv"].shape[:2]
    gt = torch.Generator(device=dev).manual_seed(1)
    batch = {"idx": inp["idx"], "gt.rgb": torch.rand(B, P, 3, device=dev, generator=gt),
             "gt.mask": torch.tensor([0, 50, 150], device=dev)[torch.randint(0, 3, (B, P), device=dev, generator=gt)]}
    g = torch.Generator(device=dev).manual_seed(4)
    opt = torch.optim.Adam([p for p in net.parameters() if p.requires_grad], lr=1e-4)
    snaps = []
    for it in range(2):
        opt.zero_grad(set_to_none=False)
        out = train.forward_train(net, {**inp, "current_epoch": 30, "global_step": 12000 + it}, generator=g)
        assert "object.index_off_surface" in out
        ld = train.Loss()(batch, out)
        ld["loss"].backward()
        opt.step()
        snaps.append(_snapshot(net, opt, {k: torch.as_tensor(v) for k, v in ld.items()}))
    ctx.check()
    return mesh, snaps


def test_training_after_meshing_cano_equals_the_host_mesh(ctx):
    mesh_a, a = _steps_with_mesh(ctx, refresh=True)
    mesh_b, b = _steps_with_mesh(ctx, refresh=False)
    assert mesh_a[0].shape == mesh_b[0].shape and np.array_equal(mesh_a[0].view(np.int32), mesh_b[0].view(np.int32))
    assert np.array_equal(mesh_a[1], mesh_b[1])
    print(f"object mesh at 16 / 2: {mesh_a[1].shape[0]} faces; losses", [s["loss.loss"].item() for s in a])
    _assert_equal_runs(a, b)


def test_replay_after_a_refresh_raises_and_a_new_capture_replays(ctx):
    from hold_b200 import train

    sc, net = _make(ctx)
    inp, gt_rgb, gt_mask = _batch(sc)
    train.meshing_cano(net, 16, 1)
    torch.manual_seed(3)
    ts = train.TrainStep(net, lr=1e-4, n_eik=64, capturable=True)
    ts.capture(inp, gt_rgb, gt_mask, warmup=2)
    l0 = ts.replay()[0].item()
    n_small = net.nodes["object"].mesh_fo_cano.shape[0]
    train.meshing_cano(net, 16, 2)                                       # a larger mesh: new tensors, a larger BVH workspace
    assert net.nodes["object"].mesh_fo_cano.shape[0] > n_small
    with pytest.raises(RuntimeError, match="capture"):
        ts.replay()
    ts.capture(inp, gt_rgb, gt_mask, warmup=2)
    l1, l2 = ts.replay()[0].item(), ts.replay()[0].item()
    torch.cuda.synchronize()
    ctx.check()
    print("replay losses", l0, l1, l2)
    assert all(math.isfinite(x) for x in (l0, l1, l2)) and l2 < l0
