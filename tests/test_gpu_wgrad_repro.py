"""hold_wgrad reduces in a fixed order: every call with the same inputs gives the same bits, eager or replayed from a CUDA graph,
at the training step's sizes (1 280 rays x 98 or 128 samples; the (N, K) blocks of the SDF, colour and background nets) and at
edge sizes (a partial slab, one row, one row past an n-block, strided operands, with and without power-of-two operand scales).
The sums stay within 1e-5 of max |OUT| of the float64 product."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

TRAIN = [(P, N, K, 0, True) for P in (1280 * 98, 1280 * 128)
         for (N, K) in ((256, 256), (256, 39), (217, 256), (1, 256), (3, 256), (256, 84))]
EDGE = [(P, N, K, 5, scaled) for P in (1, 31, 33, 4097) for (N, K) in ((1, 256), (129, 39)) for scaled in (False, True)]


def _case(P, N, K, pad, scaled):
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(P * 1000 + N * 10 + K)
    mag = 1e-5 if scaled else 1.0        # gradients this small need the operand scales to keep their fp16 split
    D = torch.randn(P, N + pad, device=dev, generator=g) * mag
    A = torch.randn(P, K + 2 * pad, device=dev, generator=g)
    return D, A


def _wgrad(ctx, D, A, N, K, sd, sa, out):
    from hold_b200 import capi

    capi.check(capi.lib().hold_wgrad(ctx.h, D.shape[0], capi.ptr(D), D.stride(0), N, capi.ptr(A), A.stride(0), K, capi.ptr(sd),
                                     capi.ptr(sa), capi.ptr(out), out.stride(0), capi.stream_ptr()))


def _scale(ctx, t, ncols):
    from hold_b200 import capi

    s = torch.empty(1, device=t.device)
    capi.check(capi.lib().hold_pow2_scale(ctx.h, t.shape[0], ncols, capi.ptr(t), t.stride(0), capi.ptr(s), capi.stream_ptr()))
    return s


@pytest.mark.parametrize("P,N,K,pad,scaled", TRAIN + EDGE)
def test_wgrad_bitwise_reproducible(ctx, P, N, K, pad, scaled):
    D, A = _case(P, N, K, pad, scaled)
    sd, sa = (_scale(ctx, D, N), _scale(ctx, A, K)) if scaled else (None, None)
    sentinel = 7.0
    outs = []
    for _ in range(10):
        o = torch.full((N, K + 3 * pad), sentinel, device=D.device)
        _wgrad(ctx, D, A, N, K, sd, sa, o)
        outs.append(o)
    ctx.check()
    first = outs[0]
    assert all(torch.equal(o, first) for o in outs[1:]), "repeated calls differ"
    assert (first[:, K:] == sentinel).all(), "hold_wgrad wrote beyond column K of OUT"
    # the same call captured in a CUDA graph: each replay equals the eager result bit for bit
    og = torch.full_like(first, sentinel)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        _wgrad(ctx, D, A, N, K, sd, sa, og)
    for _ in range(3):
        og[:, :K].fill_(-1.0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(og, first), "graph replay differs from the eager call"
    ctx.check()
    ref = D[:, :N].double().T @ A[:, :K].double()
    err = ((first[:, :K].double() - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item()
    print(f"P={P} N={N} K={K} pad={pad} scaled={scaled}: rel err {err:.2e}")
    assert err < 1e-5, err


def test_wgrad_p0_zeroes_out(ctx):
    D = torch.randn(4, 8, device="cuda")
    A = torch.randn(4, 8, device="cuda")
    o = torch.full((8, 10), 3.0, device="cuda")
    from hold_b200 import capi

    capi.check(capi.lib().hold_wgrad(ctx.h, 0, capi.ptr(D), 8, 8, capi.ptr(A), 8, 8, None, None, capi.ptr(o), 10, capi.stream_ptr()))
    torch.cuda.synchronize()
    assert (o[:, :8] == 0).all() and (o[:, 8:] == 3.0).all()
