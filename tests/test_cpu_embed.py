"""CPU-only: the Fourier embedding the tensor-core chains inline (hold_b200/csrc/embed_phases.h, compiled here with g++) against the
oracle's embedder (engine/embedders.py:48-51 restated, pinned to the reference): values and derivatives for the 39-element
canonical-point embedding (with and without BARF weights), the 84-element inverted-sphere embedding of the background and the
27-element view embedding, at every group offset the kernels use (layer-0 operand: e0 = 0, 8, ...; skip columns: e0 = n0 - 217,
including the negative offset of the mixed hand-off), and the sin/cos kernel against float64."""
import ctypes as C
import os
import subprocess

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    out = os.path.join(ROOT, "tests", "_build", "libembed_host.so")
    src = os.path.join(ROOT, "tests", "host", "embed_host.cpp")
    hdr = os.path.join(ROOT, "hold_b200", "csrc", "embed_phases.h")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    return C.CDLL(out)


def _groups(lib, D, deriv, n_embed, x, ew, e0):
    P, G = x.shape[0], len(e0)
    x = np.ascontiguousarray(x, np.float32)
    e0 = np.ascontiguousarray(e0, np.int32)
    out = np.zeros((P, G, 8), np.float32)
    ok = np.zeros(G, np.uint32)
    ewp = None if ew is None else np.ascontiguousarray(ew, np.float32).ctypes.data_as(C.c_void_p)
    lib.embed_groups(D, int(deriv), n_embed, P, x.ctypes.data_as(C.c_void_p), ewp, G, e0.ctypes.data_as(C.c_void_p),
                     out.ctypes.data_as(C.c_void_p), ok.ctypes.data_as(C.c_void_p))
    return out, ok


def _assemble(out, ok, e0, n_embed):
    """scatter the groups back into [P, n_embed]; every element must be produced by exactly the groups that cover it"""
    P = out.shape[0]
    full = np.full((P, n_embed), np.nan, np.float32)
    for g, s in enumerate(e0):
        for i in range(8):
            e = s + i
            exists = 0 <= e < n_embed
            assert bool((ok[g] >> i) & 1) == exists, (s, i)
            if exists:
                full[:, e] = out[:, g, i]
    assert not np.isnan(full).any()
    return full


def test_sincos_kernel_accuracy():
    lib = _lib()
    rng = np.random.default_rng(0)
    x = np.concatenate([(rng.random(200000) - 0.5) * 4 * f for f in (1, 2, 4, 8, 16, 32, 64, 128, 256, 512)]).astype(np.float32)
    s, c = np.zeros_like(x), np.zeros_like(x)
    lib.sincos_host(x.size, x.ctypes.data_as(C.c_void_p), s.ctypes.data_as(C.c_void_p), c.ctypes.data_as(C.c_void_p))
    es, ec = np.abs(s - np.sin(x.astype(np.float64))).max(), np.abs(c - np.cos(x.astype(np.float64))).max()
    print(f"sincos_cw max abs error: sin {es:.2e} cos {ec:.2e}")
    assert es <= 1.0e-7 and ec <= 1.0e-7


def test_embedding_groups_match_the_oracle():
    from oracle import hold_oracle as O

    lib = _lib()
    g = torch.Generator().manual_seed(0)
    x3 = (torch.rand(500, 3, generator=g) - 0.5) * 2.4
    ref = O.embed_n(x3, 6).numpy()                                  # [P, 39]
    for e0 in ([0, 8, 16, 24, 32], [-1, 7, 15, 23, 31], [-1 + 0, 3 + 4, 11 + 4, 19 + 4, 27 + 4, 35 + 4]):
        out, ok = _groups(lib, 3, False, 39, x3.numpy(), None, e0)
        full = _assemble(out, ok, e0, 39)
        err = np.abs(full - ref).max()
        assert err <= 2e-7, (e0, err)
    ew = np.linspace(0.1, 1.0, 39).astype(np.float32)               # BarfEmbedder weights
    out, ok = _groups(lib, 3, False, 39, x3.numpy(), ew, [0, 8, 16, 24, 32])
    assert np.abs(_assemble(out, ok, [0, 8, 16, 24, 32], 39) - ref * ew).max() <= 2e-7
    # derivative w.r.t. the element's own coordinate: autograd over the oracle's embedder
    xg = x3.double().clone().requires_grad_(True)
    eg = O.embed_n(xg, 6)
    dref = np.zeros((500, 39))
    for e in range(39):
        (gr,) = torch.autograd.grad(eg[:, e].sum(), xg, retain_graph=True)
        dref[:, e] = gr[:, e % 3].numpy()
    out, ok = _groups(lib, 3, True, 39, x3.numpy(), None, [0, 8, 16, 24, 32])
    dfull = _assemble(out, ok, [0, 8, 16, 24, 32], 39)
    assert np.abs(dfull - dref).max() <= 4e-6                        # |d/dx| up to 32
    # background: 4-d inverted-sphere point, 10 frequencies (84); view direction, 4 frequencies (27)
    x4 = torch.rand(300, 4, generator=g) * 2 - 1
    e0 = list(range(0, 88, 8))
    out, ok = _groups(lib, 4, False, 84, x4.numpy(), None, e0)
    assert np.abs(_assemble(out, ok, e0, 84) - O.embed_n(x4, 10).numpy()).max() <= 2e-7
    v = torch.nn.functional.normalize(torch.randn(300, 3, generator=g), dim=1)
    e0 = [0, 8, 16, 24]
    out, ok = _groups(lib, 3, False, 27, v.numpy(), None, e0)
    assert np.abs(_assemble(out, ok, e0, 27) - O.embed_n(v, 4).numpy()).max() <= 2e-7
