"""CPU-only: the composite and per-node renders with their reverse mode, as the CUDA kernels run them
(hold_b200/csrc/composite_phases.h compiled for the host), against float64 torch.autograd through merge_factors + density2weight +
the integrals of volumetric_render (hold/hold_utils.py:76-121,243-271), at training sizes and at the opacities a trained scene
reaches (Laplace densities down to beta = 0.001, optical depths into the thousands).

The helpers here (inputs, references, error measures) are shared with tests/test_gpu_composite_bwd.py, which holds the device
kernels to the same bars."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from hold_b200 import train
from hold_b200.capi import Factors, RenderOut

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R_TRAIN = 10 * 128 + 37          # the training batch (10 frames x 128 pixels) plus a partial 128-thread block
S_TRAIN = 98                     # N_samples 64 + N_samples_extra 32 + 2 per node
BETAS = (0.1, 0.03, 0.01, 0.003, 0.001)
CLS = (2, 1, 3, 0)
KEYS = ("fg_rgb", "mask_prob", "normal", "depth", "fg_semantics", "bg_weights")
WIDTH = dict(fg_rgb=3, mask_prob=0, normal=3, depth=0, fg_semantics=4, bg_weights=0)
GRADS = ("color", "normal", "density")
# the worst ray may be F32_FACTOR x float32 autograd's worst ray (run where the kernel runs, so with the same expf), and never
# needs to beat F32_FLOOR (8 float32 ulps): below that the two differ only in the order of their float32 sums
FWD_TOL, BWD_TOL, F32_FACTOR, F32_FLOOR = 1e-5, 1e-4, 4.0, 2.0 ** -20


def _lib():
    out = os.path.join(ROOT, "tests", "_build", "libcomposite_host.so")
    src = os.path.join(ROOT, "tests", "host", "composite_host.cpp")
    hdr = os.path.join(ROOT, "hold_b200", "csrc", "composite_phases.h")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    return C.CDLL(out)


# ------------------------------------------------------------------------------------------------ inputs
def laplace_density(sdf, beta):
    """LaplaceDensity (volsdf_utils.py): (1 / beta) (0.5 + 0.5 sign(s) expm1(-|s| / beta))."""
    return (0.5 + 0.5 * sdf.sign() * torch.expm1(-sdf.abs() / beta)) / beta


def make_case(n, beta, R=R_TRAIN, S=S_TRAIN, seed=0):
    """n nodes of R rays x S samples (float32, CPU).  Per ray one density profile, each node with its own parameters:
    ray % 4 == 0 solid from a surface crossing to the far end, 1 a slab 0.05-0.5 thick, 2 empty (density 0), 3 one opaque spike
    (fe up to ~1e4: exp underflows behind it).  Six z values per ray are shared by all nodes (exact ties in the merge) and every
    fifth ray of node 0 repeats a z (a zero-length interval inside the node)."""
    g = torch.Generator().manual_seed(1000 * n + seed + int(round(-1000 * torch.log10(torch.tensor(beta)).item())))
    zshared = torch.rand(R, 6, generator=g, dtype=torch.float64) * 3.5 + 0.5
    kind = torch.arange(R) % 4
    fac = []
    for k in range(n):
        z = torch.sort(torch.cat([zshared, torch.rand(R, S - 6, generator=g, dtype=torch.float64) * 3.5 + 0.5], 1), 1).values
        if k == 0:
            z[::5, S // 2] = z[::5, S // 2 - 1]
        z = z.float().double()
        zs = 1.0 + torch.rand(R, 1, generator=g, dtype=torch.float64)                    # surface crossing in [1, 2)
        zc = 1.0 + 2.0 * torch.rand(R, 1, generator=g, dtype=torch.float64)              # slab centre in [1, 3)
        th = 0.05 + 0.45 * torch.rand(R, 1, generator=g, dtype=torch.float64)            # slab thickness
        sdf = torch.where((kind == 0)[:, None], zs - z, (z - zc).abs() - 0.5 * th)
        dens = laplace_density(sdf, beta)
        dens[kind == 2] = 0.0
        spike = torch.zeros(R, S, dtype=torch.float64)
        j = torch.randint(0, S - 1, (R,), generator=g)
        spike[torch.arange(R), j] = 10.0 ** (1.0 + 4.5 * torch.rand(R, generator=g, dtype=torch.float64))
        dens = torch.where((kind == 3)[:, None], spike, dens)
        fac.append(dict(color=torch.rand(R, S, 3, generator=g), normal=torch.randn(R, S, 3, generator=g), density=dens.float(),
                        z_vals=z.float()))
    return dict(fac=fac, cls=list(CLS[:n]), n=n, R=R, S=S, gen=g)


def seeds(R, gen, keys=KEYS):
    return {k: (torch.randn(R, WIDTH[k], generator=gen) if WIDTH[k] else torch.randn(R, generator=gen)) if k in keys else None
            for k in KEYS}


def optical_depth(case):
    """min / max over rays of the composite's total optical depth sum(fe), in float64."""
    m = train.merge_factors([{k: f[k].double() for k in ("color", "normal", "density", "z_vals")} | dict(semantics=f["color"].double())
                             for f in case["fac"]])
    z = torch.cat([m["z_vals"], m["z_max"][:, None]], 1)
    tot = ((z[:, 1:] - z[:, :-1]) * m["density"]).sum(1)
    return tot.min().item(), tot.max().item()


# ------------------------------------------------------------------------------------------------ calls (host library or device)
def factors(fac):
    fs = (Factors * len(fac))()
    for k, f in enumerate(fac):
        for name, t in f.items():
            assert t.is_contiguous()
            setattr(fs[k], name, t.data_ptr())
    return fs


def render_out(d):
    ro = RenderOut()
    for name, t in d.items():
        if t is not None:
            assert t.is_contiguous()
            setattr(ro, name, t.data_ptr())
    return ro


def outputs(R, M, dev, fill=float("nan")):
    d = {k: torch.full((R, WIDTH[k]) if WIDTH[k] else (R,), fill, device=dev) for k in KEYS}
    d["fg_weights"] = torch.full((R, M), fill, device=dev)
    return d


def run_forward(fwd, case, dev):
    """fwd(n, R, S, factors, cls, comp, per_node) with hold_composite's arguments -> (comp, [per-node]) dicts incl. fg_weights."""
    n, R, S = case["n"], case["R"], case["S"]
    fac = [{k: v.to(dev).contiguous() for k, v in f.items()} for f in case["fac"]]
    comp, per = outputs(R, n * S - 2 * n + 1, dev), [outputs(R, S, dev) for _ in range(n)]
    per_ro = (RenderOut * n)(*[render_out(p) for p in per])
    fwd(n, R, S, factors(fac), (C.c_int32 * n)(*case["cls"]), C.byref(render_out(comp)), per_ro)
    return comp, per


def run_backward(bwd, case, dev, g_comp, g_per, fill=float("nan"), prefill=None):
    """bwd(n, R, S, factors, cls, g_comp, g_per_node, d_factors) with hold_composite_bwd's arguments.  g_comp: dict of seeds (None
    entries = NULL) or None; g_per: list of n such dicts or None.  prefill: per-node dict of initial d_* values (else `fill`)."""
    n, R, S = case["n"], case["R"], case["S"]
    fac = [{k: v.to(dev).contiguous() for k, v in f.items()} for f in case["fac"]]
    keep = []

    def ro(d):
        t = {k: (None if v is None else v.to(dev).contiguous()) for k, v in d.items()}
        keep.append(t)
        return render_out(t)

    d = [{name: (prefill[k][name].to(dev).clone() if prefill else torch.full(fac[k][name].shape, fill, device=dev)) for name in GRADS}
         for k in range(n)]
    gc = C.byref(ro(g_comp)) if g_comp is not None else None
    gp = (RenderOut * n)(*[ro(g_per[k]) for k in range(n)]) if g_per is not None else None
    bwd(n, R, S, factors(fac), (C.c_int32 * n)(*case["cls"]), gc, gp, factors(d))
    return d


# ------------------------------------------------------------------------------------------------ references
def _sem(R, S, c, dtype, device):
    s = torch.zeros(R, S, 4, dtype=dtype, device=device)
    s[:, :, c] = 1.0
    return s


def render_comp(leaves, cls):
    R, S = leaves[0]["z_vals"].shape
    return train.volumetric_render(train.merge_factors([dict(f, semantics=_sem(R, S, cls[k], f["z_vals"].dtype, f["z_vals"].device)) for k, f in enumerate(leaves)]))


def render_node(f, c):
    R, S = f["z_vals"].shape
    return train.volumetric_render(dict(f, semantics=_sem(R, S, c, f["z_vals"].dtype, f["z_vals"].device), z_max=f["z_vals"][:, -1]))


def gate(fg_weights):
    """mask_prob's clamp(0, 1) passes the gradient where 0 <= sum(w) <= 1.  The decision is taken from the float32 sum of the
    kernel's own weights in merge order (the sum a float32 training sees), not from the float64 sum: an opaque ray's float64
    sum 1 - bg can sit on the other side of 1.  (Either side gives the same gradient up to bg * delta, which vanishes there.)"""
    w = fg_weights.detach().float().cpu()
    acc = torch.zeros(w.shape[0])
    for i in range(w.shape[1]):
        acc = acc + w[:, i]
    return ((acc >= 0) & (acc <= 1)).double()


def reference(case, g_comp, g_per, gate_comp, gate_per, dtype=torch.float64, dev=torch.device("cpu")):
    """Forward outputs and d_color / d_normal / d_density of sum over the seeded renders of <render, seed>, by torch.autograd in
    `dtype` on `dev` over the same float32 inputs.  mask_prob's clamp gate per render comes from gate()."""
    leaves = [{k: f[k].to(dev, dtype).clone().requires_grad_(k in GRADS) for k in ("color", "normal", "density", "z_vals")}
              for f in case["fac"]]
    loss, outs = 0.0, {}
    renders = []
    if g_comp is not None:
        renders.append(("comp", render_comp(leaves, case["cls"]), g_comp, gate_comp))
    if g_per is not None:
        renders += [(k, render_node(leaves[k], case["cls"][k]), g_per[k], gate_per[k]) for k in range(case["n"])]
    for name, out, sd, gt in renders:
        outs[name] = out
        for key, s in sd.items():
            if s is None:
                continue
            o = out["fg_weights"].sum(1) * gt.to(dev, dtype) if key == "mask_prob" else out[key]
            loss = loss + (o.reshape(s.shape) * s.to(dev, dtype)).sum()
    params = [f[name] for f in leaves for name in GRADS]
    if not torch.is_tensor(loss):
        return outs, [{name: torch.zeros_like(f[name]) for name in GRADS} for f in leaves]
    gr = torch.autograd.grad(loss, params, allow_unused=True)
    gr = [torch.zeros_like(p) if x is None else x for p, x in zip(params, gr)]
    return outs, [{name: x.cpu() for name, x in zip(GRADS, gr[3 * k: 3 * k + 3])} for k in range(case["n"])]


def rel(a, r):
    a, r = a.detach().double().cpu(), r.detach().double().cpu()
    return ((a - r).abs().max() / r.abs().max().clamp_min(1e-30)).item()


def worst_ray(a, r, terms=None):
    """a, r: lists of one gradient tensor per node.  max over rays of (max |a - r| over the ray's entries in all nodes) / (max |r|
    over the same entries).  Each ray's scale is floored at 2^-24 of the tensor's largest entry: float32 resolves a weight
    1 - exp(-fe) to 2^-24 only, so a ray that is nearly empty (a slab between two samples at small beta) or lies wholly behind
    an opaque spike has no float32 digits of its own in any float32 arithmetic.  terms [R] (optional): per ray, the size of the
    terms the gradient sums, used as the scale where it is larger than max |r| (a gradient that is a difference of larger terms
    is known to float32 only relative to them)."""
    a = torch.cat([t.detach().double().cpu().reshape(t.shape[0], -1) for t in a], 1)
    r = torch.cat([t.detach().double().cpu().reshape(t.shape[0], -1) for t in r], 1)
    scale = r.abs().amax(1)
    if terms is not None:
        scale = torch.maximum(scale, terms.double())
    scale = scale.clamp_min(r.abs().max().item() * 2.0 ** -24).clamp_min(1e-30)
    return ((a - r).abs().amax(1) / scale).max().item()


def check_forward(comp, per, ref_comp, ref_per, label):
    for key in KEYS + ("fg_weights",):
        e = rel(comp[key], ref_comp[key].reshape(comp[key].shape))
        assert e <= FWD_TOL, f"{label} comp.{key}: {e:.2e}"
        for k, p in enumerate(per):
            e = rel(p[key], ref_per[k][key].reshape(p[key].shape))
            assert e <= FWD_TOL, f"{label} node {k}.{key}: {e:.2e}"


def check_sweep(fwd, bwd, case, dev, label):
    """The opacity sweep: forward at 1e-5, all six outputs of the composite seeded, every gradient tensor at 1e-4 of float64 and
    the worst ray at most F32_FACTOR x float32 autograd's worst ray on the same inputs and device."""
    n, R = case["n"], case["R"]
    comp, per = run_forward(fwd, case, dev)
    gc = gate(comp["fg_weights"])
    g_comp = seeds(R, case["gen"])
    ref_out, ref = reference(case, g_comp, None, gc, None)
    per_ref = [render_node({k: f[k].double() for k in ("color", "normal", "density", "z_vals")}, case["cls"][k]) for k, f in enumerate(case["fac"])]
    check_forward(comp, per, ref_out["comp"], per_ref, label)
    _, r32 = reference(case, g_comp, None, gc, None, dtype=torch.float32, dev=dev)
    d = run_backward(bwd, case, dev, g_comp, None)
    lo, hi = optical_depth(case)
    print(f"{label}: optical depth {lo:.3g} .. {hi:.3g}, clamp gate closed on {int((gc == 0).sum())} of {R} rays")
    for name in GRADS:
        e = max(rel(d[k][name], ref[k][name]) for k in range(n))
        wk = worst_ray([x[name] for x in d], [x[name] for x in ref])
        w32 = worst_ray([x[name] for x in r32], [x[name] for x in ref])
        print(f"  d_{name:7s} rel {e:.2e}  worst ray {wk:.2e}  float32 autograd worst ray {w32:.2e}")
        assert e <= BWD_TOL, f"{label} d_{name}: rel {e:.2e}"
        assert wk <= F32_FACTOR * max(w32, F32_FLOOR), f"{label} d_{name}: worst ray {wk:.2e} > {F32_FACTOR} x float32 autograd's {w32:.2e}"


@pytest.mark.parametrize("n", [1, 2, 3, 4])
@pytest.mark.parametrize("beta", BETAS)
def test_composite_opacity_sweep(beta, n):
    lib = _lib()
    case = make_case(n, beta)
    check_sweep(lib.composite_host, lib.composite_bwd_host, case, torch.device("cpu"), f"host beta={beta} n={n}")
