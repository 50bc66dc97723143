"""The first link of every training gradient on the device: hold_composite / hold_composite_bwd (merge_factors + density2weight +
the integrals of volumetric_render, hold/hold_utils.py:76-121,243-271) and hold_bg_integrate / hold_bg_integrate_bwd
(bg_volume_rendering, background.py:137-165) against float64 torch.autograd, at the training batch and at the opacities a trained
scene reaches.  Inputs, references and error measures are tests/test_cpu_composite.py's and tests/test_cpu_bg_integrate.py's."""
import ctypes as C

import pytest
import torch

import test_cpu_composite as T
from test_cpu_bg_integrate import _reference as bg_reference

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _calls(ctx):
    from hold_b200 import capi

    lib = capi.lib()

    def fwd(n, R, S, f, c, comp, per):
        capi.check(lib.hold_composite(ctx.h, n, R, S, f, c, comp, per, capi.stream_ptr()))
        torch.cuda.synchronize()
        ctx.check()

    def bwd(n, R, S, f, c, gc, gp, d):
        capi.check(lib.hold_composite_bwd(ctx.h, n, R, S, f, c, gc, gp, d, capi.stream_ptr()))
        torch.cuda.synchronize()
        ctx.check()

    return fwd, bwd


@pytest.mark.parametrize("n", [1, 2, 3, 4])
@pytest.mark.parametrize("beta", T.BETAS)
def test_composite_opacity_sweep(ctx, beta, n):
    """Forward at 1e-5; all six outputs seeded; every gradient tensor at 1e-4 of float64 and the worst ray within 4x of float32
    autograd's worst ray on the same inputs."""
    fwd, bwd = _calls(ctx)
    T.check_sweep(fwd, bwd, T.make_case(n, beta), DEV, f"device beta={beta} n={n}")


def _check_grads(d, ref, label):
    for k in range(len(d)):
        for name in T.GRADS:
            e = T.rel(d[k][name], ref[k][name])
            assert e <= T.BWD_TOL, f"{label} node {k} d_{name}: {e:.2e}"


@pytest.mark.parametrize("n", [1, 3, 4])
def test_per_node_branch(ctx, n):
    """hold_composite_bwd's per-node renders (z_max = the node's own last z): g_per_node alone overwrites each node's
    d_factors[k]; with g_comp the per-node passes accumulate onto the composite's gradients; g_comp alone overwrites."""
    fwd, bwd = _calls(ctx)
    case = T.make_case(n, 0.01, seed=7)
    R = case["R"]
    comp, per = T.run_forward(fwd, case, DEV)
    gc, gp = T.gate(comp["fg_weights"]), [T.gate(p["fg_weights"]) for p in per]
    g_comp = T.seeds(R, case["gen"])
    g_per = [T.seeds(R, case["gen"]) for _ in range(n)]
    print(f"per-node n={n}: optical depth {T.optical_depth(case)}")
    for label, a, b in (("per-node only", None, g_per), ("comp + per-node", g_comp, g_per), ("comp only", g_comp, None)):
        _, ref = T.reference(case, a, b, gc, gp)
        _check_grads(T.run_backward(bwd, case, DEV, a, b), ref, f"n={n} {label}")


@pytest.mark.parametrize("seeded", T.KEYS + ("none",))
def test_null_upstream_gradients(ctx, seeded):
    """One of the six composite outputs seeded, every other upstream gradient NULL (bg_weights alone = every one NULL except
    bg_weights); "none": all six NULL, the gradients are exactly 0."""
    fwd, bwd = _calls(ctx)
    case = T.make_case(3, 0.01, seed=11)
    comp, _ = T.run_forward(fwd, case, DEV)
    gc = T.gate(comp["fg_weights"])
    g = T.seeds(case["R"], case["gen"], keys=() if seeded == "none" else (seeded,))
    _, ref = T.reference(case, g, None, gc, None)
    d = T.run_backward(bwd, case, DEV, g, None)
    if seeded == "none":
        assert all((d[k][name] == 0).all() for k in range(3) for name in T.GRADS)
    else:
        _check_grads(d, ref, f"{seeded} alone")


def test_composite_boundaries(ctx):
    """R = 1 against float64; R = 0 writes nothing; n = 0, n = 5, S < 2 and no upstream gradient at all are rejected."""
    from hold_b200 import capi

    fwd, bwd = _calls(ctx)
    case = T.make_case(2, 0.01, R=1, seed=3)
    comp, per = T.run_forward(fwd, case, DEV)
    gc, gp = T.gate(comp["fg_weights"]), [T.gate(p["fg_weights"]) for p in per]
    g_comp, g_per = T.seeds(1, case["gen"]), [T.seeds(1, case["gen"]) for _ in range(2)]
    out, ref = T.reference(case, g_comp, g_per, gc, gp)
    T.check_forward(comp, per, out["comp"], [out[k] for k in range(2)], "R=1")
    _check_grads(T.run_backward(bwd, case, DEV, g_comp, g_per), ref, "R=1")

    lib = capi.lib()
    case = T.make_case(4, 0.01, R=4, seed=5)
    fac = [{k: v.to(DEV) for k, v in f.items()} for f in case["fac"]]
    d = [{name: torch.full(fac[k][name].shape, 7.0, device=DEV) for name in T.GRADS} for k in range(4)]
    g = {k: v.to(DEV) for k, v in T.seeds(4, case["gen"]).items()}
    facs, dfs, cls, gro = T.factors(fac), T.factors(d), (C.c_int32 * 5)(*case["cls"], 0), T.render_out(g)
    capi.check(lib.hold_composite_bwd(ctx.h, 4, 0, T.S_TRAIN, facs, cls, C.byref(gro), None, dfs, capi.stream_ptr()))
    torch.cuda.synchronize()
    assert all((d[k][name] == 7.0).all() for k in range(4) for name in T.GRADS)
    for n, S, gc_ in ((0, T.S_TRAIN, gro), (5, T.S_TRAIN, gro), (4, 1, gro), (4, T.S_TRAIN, None)):
        with pytest.raises(capi.HoldError):
            capi.check(lib.hold_composite_bwd(ctx.h, n, 4, S, facs, cls, None if gc_ is None else C.byref(gc_), None, dfs,
                                              capi.stream_ptr()))
    ctx.check()


# ------------------------------------------------------------------------------------------------ background integral
BG_N = 32


def _bg_case(jittered, seed):
    """R = 4k + 1 rays (four rays per 128-thread block of the reverse kernel: the last block is partial)."""
    from oracle import hold_oracle as O

    g = torch.Generator().manual_seed(seed)
    R, R_s = 4 * 300 + 1, 3.0
    z = O.uniform_z(0.0, torch.ones(R, 1), BG_N, torch.rand(R, BG_N, generator=g) if jittered else None) * (1.0 / R_s)
    sdf = torch.randn(R, BG_N, generator=g) * 3.0
    sdf[0::5] = (sdf[0::5] * 300.0).clamp(-1e3, 1e3)                     # opaque first shells: |sdf| up to 1e3
    sdf[1::5] = torch.randn(sdf[1::5].shape, generator=g) * 1e-6         # near zero: the 1e10 last interval carries the weight
    sdf.view(-1)[::7] = 0.0                                                # |sdf|'s kink: torch's subgradient 0
    sdf[-1] = -sdf[-1].abs()
    rgb = torch.rand(R * BG_N, 3, generator=g)
    wfg = torch.rand(R, generator=g)
    wfg[::6], wfg[3::6] = 0.0, 1.0
    return z.contiguous(), sdf.reshape(-1).contiguous(), rgb, wfg, g


def _bg_terms(z, sdf, rgb, wfg, g_rgb, g_only, g_sem):
    """Per ray, in float64, the size of the terms that d_sdf and d_fg_bg_weights are differences of (bg_phases.h):
    d sdf_k = (dw_k e_k T_k - sum_{i>k} dw_i w_i) dist_k sign(sdf_k) -> max_k (|dw_k| e_k T_k + sum_{i>k} |dw_i| w_i) dist_k over
    sdf_k != 0;  d w_fg = <only, g_rgb> + g_sem[0] -> sum_c |only_c g_rgb_c| + |g_sem[0]|."""
    R = z.shape[0]
    zf = torch.flip(z.double(), dims=[-1])
    dist = torch.cat([zf[:, :-1] - zf[:, 1:], torch.full((R, 1), 1e10, dtype=torch.float64)], -1)
    s = sdf.double().reshape(R, BG_N)
    fe = dist * s.abs()
    T_ = torch.exp(-torch.cumsum(torch.cat([torch.zeros(R, 1, dtype=torch.float64), fe[:, :-1]], -1), -1))
    e = torch.exp(-fe)
    w = (1 - e) * T_
    zero3 = torch.zeros(R, 3, dtype=torch.float64)
    gr = g_rgb.double() if g_rgb is not None else zero3
    g = (g_only.double() if g_only is not None else zero3) + wfg.double()[:, None] * gr
    c = rgb.double().reshape(R, BG_N, 3)
    dw = (c * g[:, None, :]).sum(-1).abs()
    after = torch.flip(torch.cumsum(torch.flip(dw * w, dims=[-1]), -1), dims=[-1]) - dw * w
    t_sdf = ((dw * e * T_ + after) * dist * (s != 0)).amax(1)
    only = (w[:, :, None] * c).sum(1)
    t_w = (only * gr).abs().sum(1) + (g_sem.double()[:, 0].abs() if g_sem is not None else 0.0)
    return t_sdf, t_w


@pytest.mark.parametrize("jittered", [False, True])
@pytest.mark.parametrize("null", ["none", "g_rgb", "g_only", "g_sem"])
def test_bg_integrate(ctx, jittered, null):
    """Forward at 1e-5; every gradient tensor at 1e-4 of float64 and the worst ray within 4x of float32 autograd's worst ray on
    the same inputs.  d_sdf and d_fg_bg_weights are differences of larger terms (an opaque shell's d_sdf is e^{-fe} times the
    difference of two samples' dw), so their rays are measured against the size of those terms."""
    from hold_b200 import capi

    lib = capi.lib()
    z, sdf, rgb, wfg, g = _bg_case(jittered, 20 + jittered)
    R = z.shape[0]
    gs = dict(g_rgb=torch.randn(R, 3, generator=g), g_only=torch.randn(R, 3, generator=g), g_sem=torch.randn(R, 4, generator=g))
    if null != "none":
        gs[null] = None

    def grads(dtype):
        leaves = [t.to(dtype).requires_grad_(True) for t in (sdf, rgb, wfg)]
        ref = bg_reference(z.to(dtype), *leaves)
        loss = sum((o * s.to(dtype)).sum() for o, s in zip(ref, gs.values()) if s is not None)
        return ref, torch.autograd.grad(loss, leaves)

    ref, r64 = grads(torch.float64)
    _, r32 = grads(torch.float32)
    dz, ds, dr, dw = (t.to(DEV).contiguous() for t in (z, sdf, rgb, wfg))
    out = [torch.full((R, k), float("nan"), device=DEV) for k in (3, 3, 4)]
    capi.check(lib.hold_bg_integrate(ctx.h, R, capi.ptr(dz), capi.ptr(ds), capi.ptr(dr), capi.ptr(dw), *(capi.ptr(t) for t in out),
                                     capi.stream_ptr()))
    dg = [None if t is None else t.to(DEV).contiguous() for t in gs.values()]
    d = [torch.full_like(t, float("nan")) for t in (ds, dr, dw)]
    capi.check(lib.hold_bg_integrate_bwd(ctx.h, R, capi.ptr(dz), capi.ptr(ds), capi.ptr(dr), capi.ptr(dw), *(capi.ptr(t) for t in dg),
                                         *(capi.ptr(t) for t in d), capi.stream_ptr()))
    torch.cuda.synchronize()
    ctx.check()
    for name, a, r in zip(("bg_rgb", "bg_rgb_only", "bg_semantics"), out, ref):
        e = T.rel(a, r)
        assert e <= T.FWD_TOL, (name, e)
    t_sdf, t_w = _bg_terms(z, sdf, rgb, wfg, *gs.values())
    print(f"bg jittered={jittered} null={null}: R={R}, |sdf| max {sdf.abs().max().item():.3g}, exact zeros {(sdf == 0).sum().item()}")
    for name, a, r, x, terms in zip(("d_sdf", "d_rgb", "d_fg_bg_weights"), d, r64, r32, (t_sdf, None, t_w)):
        e = T.rel(a, r)
        wk = T.worst_ray([a.reshape(R, -1)], [r.reshape(R, -1)], terms)
        w32 = T.worst_ray([x.reshape(R, -1)], [r.reshape(R, -1)], terms)
        print(f"  {name:16s} rel {e:.2e}  worst ray {wk:.2e}  float32 autograd worst ray {w32:.2e}")
        assert e <= T.BWD_TOL, (name, e)
        assert wk <= T.F32_FACTOR * max(w32, T.F32_FLOOR), f"{name}: worst ray {wk:.2e} > {T.F32_FACTOR} x float32 autograd's {w32:.2e}"
    assert (d[0].cpu()[sdf == 0] == 0).all()
