"""CPU-only: the background's sample depths and its 32-sample integral with the reverse mode, as the CUDA kernels run them
(hold_b200/csrc/bg_phases.h compiled for the host), against the oracle's float32 depths bit for bit and float64 torch.autograd
over bg_volume_rendering (model/renderables/background.py:137-165)."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from oracle import hold_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 32


def _lib():
    out = os.path.join(ROOT, "tests", "_build", "libbg_host.so")
    src = os.path.join(ROOT, "tests", "host", "bg_host.cpp")
    hdr = os.path.join(ROOT, "hold_b200", "csrc", "bg_phases.h")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    return C.CDLL(out)


_p = lambda t: None if t is None else C.c_void_p(t.data_ptr())


def _depths(lib, R, R_s, jitter):
    z = torch.full((R, N), float("nan"))
    lib.bg_depths_host(C.c_int(R), C.c_float(R_s), _p(jitter), _p(z))
    return z


@pytest.mark.parametrize("R_s", [6.0, 3.0, 2.5])
def test_background_depths_match_inverse_sample(R_s):
    """Fixed shells = inverse_sample's linspace(0, 1, 32) / R_s (what hold_background computes); with jitter = the oracle's float32
    uniform_z(0, 1, 32, jitter) / R_s, every depth inside its stratum."""
    lib = _lib()
    R = 200
    g = torch.Generator().manual_seed(0)
    fixed = O.uniform_z(0.0, torch.ones(R, 1), N) * (1.0 / R_s)
    assert torch.equal(_depths(lib, R, R_s, None), fixed)
    assert torch.equal(fixed[0], torch.linspace(0.0, 1.0, N) * (1.0 / R_s))
    jitter = torch.rand(R, N, generator=g)
    jitter[0], jitter[1] = 0.0, 1.0 - 2 ** -24                          # stratum edges
    z = _depths(lib, R, R_s, jitter)
    assert torch.equal(z, O.uniform_z(0.0, torch.ones(R, 1), N, jitter) * (1.0 / R_s))
    lo, hi = (_depths(lib, 1, R_s, torch.full((1, N), v)) for v in (0.0, 1.0))     # the strata's edges
    assert (z >= lo).all() and (z <= hi).all() and (lo[:, 1:] == hi[:, :-1]).all()


def test_foreground_stratified_z_matches_uniform_sampler():
    """The same helper serves the foreground sampler (k_sampler_init): UniformSampler.get_z_vals with and without jitter."""
    lib = _lib()
    g = torch.Generator().manual_seed(1)
    R, n, near = 300, 64, 0.05
    far = (torch.rand(R, generator=g) * 3.0 + 0.5).contiguous()
    u = torch.rand(R, n, generator=g)
    for jit in (None, u):
        z = torch.full((R, n), float("nan"))
        lib.stratified_z_host(C.c_int(R), C.c_int(n), C.c_float(near), _p(far), _p(jit), _p(z))
        assert torch.equal(z, O.uniform_z(near, far[:, None], n, jit))


def _reference(z, sdf, rgb, wfg):
    """bg_volume_rendering over the flipped depths (the oracle's `background` after its nets), float64."""
    R = z.shape[0]
    zf = torch.flip(z, dims=[-1])
    d = torch.cat([zf[:, :-1] - zf[:, 1:], torch.full((R, 1), 1e10, dtype=z.dtype)], -1)
    fe = d * sdf.reshape(R, N).abs()
    alpha = 1 - torch.exp(-fe)
    T = torch.exp(-torch.cumsum(torch.cat([torch.zeros(R, 1, dtype=z.dtype), fe[:, :-1]], -1), -1))
    w = alpha * T
    only = (w.unsqueeze(-1) * rgb.reshape(R, N, 3)).sum(1)
    sem = torch.zeros(R, 4, dtype=z.dtype)
    sem[:, 0] = 1.0
    return wfg[:, None] * only, only, wfg[:, None] * sem


def _rel(a, r):
    return ((a.double() - r).abs().max() / r.abs().max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("jittered", [False, True])
@pytest.mark.parametrize("seeds", ["all", "no_only", "rgb_only"])
def test_integral_forward_and_backward(jittered, seeds):
    lib = _lib()
    g = torch.Generator().manual_seed(7 + jittered)
    R, R_s = 256, 6.0
    z = _depths(lib, R, R_s, torch.rand(R, N, generator=g) if jittered else None)
    sdf = torch.randn(R * N, generator=g) * 3.0
    sdf[: 40 * N] *= 60.0                                                # opaque rays: the transmittance reaches ~0
    sdf[::7] = 0.0                                                       # |sdf|'s kink: torch's subgradient 0
    sdf[R * N - N:] = -sdf[R * N - N:].abs()                             # a ray of negative sdf only
    rgb = torch.rand(R * N, 3, generator=g)
    wfg = torch.rand(R, generator=g)
    wfg[::5] = 0.0                                                       # the foreground takes the whole ray
    g_rgb, g_only, g_sem = torch.randn(R, 3, generator=g), torch.randn(R, 3, generator=g), torch.randn(R, 4, generator=g)
    if seeds == "no_only":
        g_only = None
    elif seeds == "rgb_only":
        g_only, g_sem = None, None

    s64, c64, w64 = (t.double().requires_grad_(True) for t in (sdf, rgb, wfg))
    ref = _reference(z.double(), s64, c64, w64)
    loss = sum((o * s.double()).sum() for o, s in zip(ref, (g_rgb, g_only, g_sem)) if s is not None)
    loss.backward()

    out = [torch.full((R, n), float("nan")) for n in (3, 3, 4)]
    lib.bg_integrate_host(C.c_int(R), _p(z), _p(sdf), _p(rgb), _p(wfg), *(_p(t) for t in out))
    for name, a, r in zip(("bg_rgb", "bg_rgb_only", "bg_semantics"), out, ref):
        assert _rel(a, r.detach()) <= 1e-6, (name, _rel(a, r.detach()))
    d_sdf, d_rgb, d_w = torch.full_like(sdf, float("nan")), torch.full_like(rgb, float("nan")), torch.full_like(wfg, float("nan"))
    lib.bg_integrate_bwd_host(C.c_int(R), _p(z), _p(sdf), _p(rgb), _p(wfg), _p(g_rgb), _p(g_only), _p(g_sem), _p(d_sdf), _p(d_rgb), _p(d_w))
    for name, a, r in (("d_sdf", d_sdf, s64.grad), ("d_rgb", d_rgb, c64.grad), ("d_fg_bg_weights", d_w, w64.grad)):
        e = _rel(a, r)
        print(f"jittered={jittered} seeds={seeds} {name}: {e:.2e}")
        assert e <= 1e-6, (name, e)
    assert (d_sdf[::7] == 0).all()
