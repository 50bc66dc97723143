"""hold_linear against every matrix id documented in include/hold_b200.h, for a hand node, an object node and the background:
C = A . M^T (+ bias) is compared with a float64 product of the folded reference weights in the documented operand order.
Also the background's two rejections: hold_linear(node -1) after the background was re-packed in fp32 mode, and background
weights that carry weight_g (the reference's background nets are plain nn.Linear)."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
E_BADARG, E_STATE = -1, -6


@pytest.fixture(scope="module")
def env(built):
    from hold_b200 import capi, scene_io, synth

    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    torch.cuda.set_device(0)
    c = capi.Context(0)   # its own context: this module re-packs the background in both modes
    sc = synth.make_scene(H=8, W=8, S=32, nodes=("right", "object"), B=1, seed=4, perturb=0.02)
    net = scene_io.build_net(sc, c, capi.MLP_TC)
    _, bg_sdf, bg_rgb = scene_io.build_background(sc, c, mlp_mode=capi.MLP_TC)
    yield dict(ctx=c, sc=sc, net=net, bg_sdf=bg_sdf, bg_rgb=bg_rgb)
    c.close()


def _fold(sd, l):
    if f"lin{l}.weight_v" in sd:
        v, g = sd[f"lin{l}.weight_v"].double(), sd[f"lin{l}.weight_g"].double()
        return v * (g / v.norm(dim=1, keepdim=True)), sd[f"lin{l}.bias"].double()
    return sd[f"lin{l}.weight"].double(), sd[f"lin{l}.bias"].double()


def _matrices(sdf_sd, rgb_sd, k_in, lead, n_hidden):
    """{mat: (M [nvalid, kvalid] float64, bias or None)} in the header's operand order."""
    out = {}
    for l in range(9):
        W, b = _fold(sdf_sd, l)
        if l == 0:
            W = W[:, :k_in]                                            # hand: the 45 pose columns are dropped
        if l == 4:
            W = W * (1.0 / math.sqrt(2.0))                             # the skip's 1/sqrt 2
        if l == 8:
            W, b = W[1:], b[1:]                                        # the 256 feature rows
        out[l], out[16 + l] = (W, b), (W.T, None)
    Ws = [_fold(rgb_sd, l) for l in range(n_hidden)]          # the colour GEMM layers (the 3-row head is not a matrix id)
    W0, b0 = Ws[0]
    feat, other = W0[:, lead:lead + 256], torch.cat([W0[:, :lead], W0[:, lead + 256:]], 1)
    out[32] = (torch.cat([feat, other], 1), b0)                        # A = [feature | the other inputs]
    out[48], out[49] = (feat.T, None), (other.T, None)
    for l in range(1, n_hidden):
        out[32 + l], out[49 + l] = Ws[l], (Ws[l][0].T, None)
    return out


def _check(ctx, slot, mats, label):
    from hold_b200 import capi

    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(7)
    P = 1000
    for mat, (M, b) in sorted(mats.items()):
        n, k = M.shape
        A = torch.randn(P, (k + 3) // 4 * 4, generator=g)
        Cm = torch.full((P, (n + 3) // 4 * 4), float("nan"), device=dev)
        Ad = A.to(dev)
        capi.check(capi.lib().hold_linear(ctx.h, slot, mat, P, capi.ptr(Ad), Ad.stride(0), k, 0 if b is None else 1, None,
                                          capi.ptr(Cm), Cm.stride(0), n, capi.stream_ptr()))
        ctx.check()
        ref = A[:, :k].double() @ M.T + (0.0 if b is None else b)
        err = ((Cm[:, :n].cpu().double() - ref).abs().max() / ref.abs().max()).item()
        print(f"{label} mat {mat}: [{n} x {k}] rel err {err:.2e}")
        assert err <= 1e-5, f"{label} mat {mat}: {err:.2e}"


@pytest.mark.parametrize("nid", ["right", "object"])
def test_node_matrices(env, nid):
    sc, node = env["sc"], env["net"].nodes[nid]
    mats = _matrices(sc.sdf_state[nid], sc.rgb_state[nid], 39, 14, 4)
    assert sorted(mats) == list(range(9)) + list(range(16, 25)) + list(range(32, 36)) + list(range(48, 53))
    _check(env["ctx"], node.slot, mats, nid)


def test_background_matrices(env):
    mats = _matrices(env["bg_sdf"], env["bg_rgb"], 116, 59, 1)
    assert sorted(mats) == list(range(9)) + list(range(16, 25)) + [32, 48, 49]
    _check(env["ctx"], -1, mats, "background")


def _bg_set(ctx, sdf_sd, rgb_sd, mode):
    from hold_b200 import capi

    dev = torch.device("cuda", 0)
    wi, k1 = capi.mlp_weights({k: v.to(dev) for k, v in sdf_sd.items()}, 9)
    wr, k2 = capi.mlp_weights({k: v.to(dev) for k, v in rgb_sd.items()}, 2)
    rc = capi.lib().hold_bg_set_weights(ctx.h, C.byref(wi), C.byref(wr), mode, capi.stream_ptr())
    torch.cuda.synchronize()
    return rc


def _linear_rc(ctx, slot):
    from hold_b200 import capi

    A = torch.zeros(128, 256, device="cuda")
    out = torch.empty(128, 256, device="cuda")
    return capi.lib().hold_linear(ctx.h, slot, 1, 128, capi.ptr(A), 256, 256, 0, None, capi.ptr(out), 256, 256, capi.stream_ptr())


def test_background_fp32_repack_retires_tc_images(env):
    """After the background is re-packed in fp32 mode, its tensor-core images are stale: hold_linear(node -1) refuses them."""
    from hold_b200 import capi

    ctx = env["ctx"]
    try:
        assert _bg_set(ctx, env["bg_sdf"], env["bg_rgb"], capi.MLP_FP32) == 0, capi.lib().hold_last_error()
        assert _linear_rc(ctx, -1) == E_STATE
        assert _bg_set(ctx, env["bg_sdf"], env["bg_rgb"], capi.MLP_TC) == 0, capi.lib().hold_last_error()
        assert _linear_rc(ctx, -1) == 0, capi.lib().hold_last_error()
    finally:
        _bg_set(ctx, env["bg_sdf"], env["bg_rgb"], capi.MLP_TC)


def test_background_rejects_weight_g(env):
    """The background nets have no weight-norm: weights that carry weight_g are malformed input in either mode."""
    from hold_b200 import capi

    ctx = env["ctx"]
    W = env["bg_sdf"]["lin2.weight"]
    sdf_wn = {k: v for k, v in env["bg_sdf"].items() if k != "lin2.weight"}
    sdf_wn["lin2.weight_v"], sdf_wn["lin2.weight_g"] = W, W.norm(dim=1, keepdim=True)
    try:
        for mode in (capi.MLP_FP32, capi.MLP_TC):
            assert _bg_set(ctx, sdf_wn, env["bg_rgb"], mode) == E_BADARG, mode
            assert b"weight_g" in capi.lib().hold_last_error()
    finally:
        _bg_set(ctx, env["bg_sdf"], env["bg_rgb"], capi.MLP_TC)
