"""Bitwise-reproducible training on one GPU: two nets built from the same seeds and trained on the same batches stay identical bit
for bit -- every loss, parameter, gradient and Adam moment -- eager (default and stratified sampling), through forward_train +
train.Loss with the canonical meshes attached, and as replays of a captured TrainStep graph.  The weight gradients reduce in a
fixed order (hold_wgrad), and no torch op of the step has a nondeterministic CUDA kernel (checked under torch's deterministic-
algorithms mode in a child process).  tools/dump_train_steps.py twice gives identical dumps."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS = 5


def _make(ctx, background=True, meshes=False):
    """The scene and model of test_gpu_train.py::test_train_step_cuda_graph_replay, optionally with the canonical meshes of
    test_forward_train_outputs_and_loss attached."""
    from hold_b200 import capi, scene_io, synth
    from hold_b200.model import HOLDNet

    sc = synth.make_scene(H=8, W=8, S=32, nodes=("right", "object"), B=2, seed=5)
    sc.intrinsics[:, 0, 2] += 0.37
    net = scene_io.build_net(sc, ctx, capi.MLP_TC)
    bg = scene_io.build_background(sc, ctx, mlp_mode=capi.MLP_TC)[0] if background else None
    full = HOLDNet(ctx, dict(net.nodes), background=bg)
    if meshes:
        from scipy.spatial import ConvexHull

        hull = lambda p: torch.as_tensor(ConvexHull(p.detach().cpu().double().numpy()).simplices.astype("int32")).cuda()
        right, obj = full.nodes["right"], full.nodes["object"]
        right.mesh_v_cano_div = right.server.verts_c[0].detach().clone()
        right.mesh_f_cano_div = hull(right.mesh_v_cano_div)
        obj.mesh_vo_cano = sc.obj_pts_cano.cuda()
        obj.mesh_fo_cano = hull(sc.obj_pts_cano)
    return sc, full


def _batch(sc):
    from hold_b200 import scene_io

    dev = torch.device("cuda", 0)
    inp = scene_io.scene_input(sc, dev)
    R = sc.B * sc.uv.shape[1]
    g = torch.Generator(device=dev).manual_seed(0)
    gt_rgb, gt_mask = torch.rand(R, 3, device=dev, generator=g), torch.zeros(R, 4, device=dev)
    gt_mask[:, 0] = 1.0
    return inp, gt_rgb, gt_mask


def _snapshot(net, opt, losses):
    snap = {f"loss.{k}": v.detach().clone() for k, v in losses.items()}
    for n, p in net.named_parameters():
        snap[f"param.{n}"] = p.detach().clone()
        if p.grad is not None:
            snap[f"grad.{n}"] = p.grad.clone()
        for k, v in opt.state.get(p, {}).items():
            snap[f"adam.{k}.{n}"] = v.clone()
    return snap


def _assert_equal_runs(a, b):
    assert len(a) == len(b)
    for i, (sa, sb) in enumerate(zip(a, b)):
        assert sa.keys() == sb.keys(), (i, sorted(sa.keys() ^ sb.keys()))
        diff = [k for k in sa if not torch.equal(sa[k], sb[k])]
        assert not diff, f"step {i}: {len(diff)} of {len(sa)} tensors differ, e.g. {diff[:6]}"
    assert any(k.startswith("grad.") for k in a[0]) and any(k.startswith("adam.") for k in a[-1])


def _train_steps(ctx, stratified, background=True):
    from hold_b200 import train

    sc, net = _make(ctx, background)
    inp, gt_rgb, gt_mask = _batch(sc)
    torch.manual_seed(3)
    gen = torch.Generator(device="cuda").manual_seed(9) if stratified else None
    ts = train.TrainStep(net, lr=1e-4, n_eik=64, stratified=stratified)
    snaps = []
    for _ in range(STEPS):
        loss, parts = ts.step(inp, gt_rgb, gt_mask, generator=gen)
        snaps.append(_snapshot(net, ts.opt, dict(loss=loss, **parts)))
    ctx.check()
    return snaps


@pytest.mark.parametrize("background", [True, False])
@pytest.mark.parametrize("stratified", [False, True])
def test_eager_train_steps_bitwise(ctx, stratified, background):
    a = _train_steps(ctx, stratified, background)
    b = _train_steps(ctx, stratified, background)      # built after a is done: both use the context's node slots in turn
    print("losses", [s["loss.loss"].item() for s in a])
    _assert_equal_runs(a, b)


def _loss_steps(ctx, stratified):
    from hold_b200 import train

    sc, net = _make(ctx, meshes=True)
    inp, _, _ = _batch(sc)
    dev = torch.device("cuda", 0)
    B, P = inp["uv"].shape[:2]
    gt = torch.Generator(device=dev).manual_seed(1)
    batch = {"idx": inp["idx"], "gt.rgb": torch.rand(B, P, 3, device=dev, generator=gt),
             "gt.mask": torch.tensor([0, 50, 150], device=dev)[torch.randint(0, 3, (B, P), device=dev, generator=gt)]}
    g = torch.Generator(device=dev).manual_seed(4)
    opt = torch.optim.Adam([p for p in net.parameters() if p.requires_grad], lr=1e-4)
    snaps = []
    for it in range(STEPS):
        opt.zero_grad(set_to_none=False)
        out = train.forward_train(net, {**inp, "current_epoch": 30, "global_step": 12000 + it}, generator=g, stratified=stratified)
        ld = train.Loss()(batch, out)
        ld["loss"].backward()
        opt.step()
        snaps.append(_snapshot(net, opt, {k: torch.as_tensor(v) for k, v in ld.items()}))
    ctx.check()
    return snaps


@pytest.mark.parametrize("stratified", [False, True])
def test_forward_train_loss_backward_bitwise(ctx, stratified):
    a = _loss_steps(ctx, stratified)
    b = _loss_steps(ctx, stratified)
    assert "loss.loss/mano_cano" in a[0] and "loss.loss/opacity_sparse" in a[0]
    _assert_equal_runs(a, b)


def _graph_replays(ctx):
    from hold_b200 import train

    sc, net = _make(ctx)
    inp, gt_rgb, gt_mask = _batch(sc)
    torch.manual_seed(3)
    ts = train.TrainStep(net, lr=1e-4, n_eik=64, capturable=True)
    ts.capture(inp, gt_rgb, gt_mask, warmup=3)
    snaps = []
    for _ in range(STEPS):
        loss, parts = ts.replay()
        snaps.append(_snapshot(net, ts.opt, dict(loss=loss, **parts)))
    torch.cuda.synchronize()
    ctx.check()
    del ts
    return snaps


def test_graph_replays_bitwise(ctx):
    a = _graph_replays(ctx)
    b = _graph_replays(ctx)
    print("replay losses", [s["loss.loss"].item() for s in a])
    _assert_equal_runs(a, b)


def audit_deterministic_ops(ctx):
    """Child process: every op of the training step under torch.use_deterministic_algorithms(True, warn_only=True), which warns
    for each op whose CUDA kernel has no deterministic implementation.  The library itself never switches that mode on."""
    import warnings

    from hold_b200 import train

    torch.use_deterministic_algorithms(True, warn_only=True)
    found = []
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        for stratified in (False, True):
            for background in (True, False):
                _train_steps(ctx, stratified, background)
            _loss_steps(ctx, stratified)
        sc, net = _make(ctx)
        inp, gt_rgb, gt_mask = _batch(sc)
        ts = train.TrainStep(net, lr=1e-4, n_eik=64, capturable=True)
        ts.capture(inp, gt_rgb, gt_mask, warmup=1)
        ts.replay()
        torch.cuda.synchronize()
        found = sorted({str(w.message).splitlines()[0] for w in rec if "determinis" in str(w.message)})
    for f in found:
        print("nondeterministic:", f)
    assert not found, found
    with warnings.catch_warnings(record=True) as rec:      # the check itself works: histc's CUDA kernel is flagged
        warnings.simplefilter("always")
        torch.histc(torch.rand(64, device="cuda"), bins=4)
    assert any("determinis" in str(w.message) for w in rec), [str(w.message) for w in rec]


def test_train_step_has_no_nondeterministic_torch_op(isolated):
    isolated("tests/test_gpu_train_repro.py", "audit_deterministic_ops", timeout=900, env={"CUBLAS_WORKSPACE_CONFIG": ":4096:8"})


def test_dump_train_steps_twice_identical(ctx, tmp_path):
    tool = os.path.join(ROOT, "tools", "dump_train_steps.py")
    small = ["--steps", "3", "--frames", "2", "--pixels", "32", "--size", "32"]
    for mode in (["--stratified"], ["--graph"]):
        dirs = []
        for run in ("a", "b"):
            d = str(tmp_path / ("_".join(m.strip("-") for m in mode) or "eager") / run)
            r = subprocess.run([sys.executable, tool, d] + small + mode, cwd=ROOT, capture_output=True, text=True, timeout=600)
            assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
            dirs.append(d)
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "compare_dumps.py"), *dirs], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        rep = json.loads(r.stdout.strip().splitlines()[-1])
        assert not rep["mismatched"] and len(rep["arrays"]) > 3 * 50
        names = sorted(rep["arrays"])
        assert any(".grad." in k for k in names) and any(".adam_exp_avg_sq." in k for k in names) and "step002.loss" in names
        diff = [k for k, v in rep["arrays"].items() if not v["identical"]]
        assert not diff, (mode, diff[:8])
