"""Reverse mode of the SDF net with its input gradient as an OUTPUT, and of the colour net — the algebra of SURVEY §8f rank 2
(train.py's step: hold/hold.py:110-137; the second-order path engine/volsdf_utils.py:123-131 `create_graph=is_training`).

The reference gets these gradients from torch.autograd, including a double backward through d sdf / d x_c (the normal fed to
the colour net).  Here the normal's gradient g = d sdf / d x_c is an output of ONE function (sdf, feat, g) = F(x_c; W), and the
backward of F for seeds (d_sdf, d_feat, d_g) is written out: it is a forward-mode sweep along E'(x) d_g (which is what the
reverse-over-reverse pass reduces to) followed by one ordinary reverse sweep with the second-order terms
softplus''(z_l) * h_l * q_l added to the pre-activation gradients.  Notation (rows = points):

  forward     A_0 = e = E(x);  z_l = A_l W_l^T + b_l;  a_l = softplus(z_l), s_l = softplus'(z_l);  A_{l+1} = a_l,
              A_4 = [a_3 | e] / sqrt 2;  out = A_8 W_8^T + b_8  (sdf = out[:,0], feat = out[:,1:])
  gradient    gbar_7 = w * s_7 (w = W_8[0]);  q_{l-1} = gbar_l W_l;  gbar_{l-1} = q_{l-1} * s_{l-1};  g_e = gbar_0 W_0 + skip;  g = E'(x)^T g_e
  backward I  d_ge = E'(x) d_g;  h_0 = d_ge W_0^T;  u_{l-1} = h_{l-1} * s_{l-1};  h_l = u'_{l-1} W_l^T  (u' = [u_3 | d_ge] / sqrt 2 at l = 4)
              dW_l += gbar_l^T u'_{l-1};  second-order seeds  dz2_l = softplus''(z_l) * h_l * q_l  (q_7 := w)
  backward II dA_8 = d_out W_8;  dz_l = dA_{l+1} * s_l + dz2_l;  dW_l += dz_l^T A_l;  dA_l = dz_l W_l;  d_x = E'(x)^T d_e + E''-term

Every product with a weight matrix goes through `ops.lin` / `ops.lin_t` (the tensor-core split-precision GEMM against the packed
weight images on the GPU: hold_linear), every weight-gradient reduction over the points through `ops.wgrad` (a plain GEMM), the
pointwise steps through `ops.*` elementwise kernels.  `TorchOps` (below) runs the same algorithm with torch on the CPU in any
dtype; tests/test_cpu_train_bwd.py checks it against torch.autograd over the oracle in float64."""
from __future__ import annotations

import math

import torch

N_FREQ = 6
D_EMBED = 3 + 3 * 2 * N_FREQ   # 39
SKIP = 4
N_SKIP_A = 256 - D_EMBED       # 217 activation columns feeding layer 4


# ------------------------------------------------------------------------------------------------ embedding (engine/embedders.py:48-51)
def embed_terms(x, embed_w=None, order=0):
    """E(x) [P,39] (order 0), dE_e/dx_{c(e)} (order 1) or d2E_e/dx_{c(e)}^2 (order 2): every component depends on ONE
    coordinate c(e) = e % 3.  Layout [x, sin(x), cos(x), sin(2x), cos(2x), ...]."""
    outs = []
    if order == 0:
        outs.append(x)
    elif order == 1:
        outs.append(torch.ones_like(x))
    else:
        outs.append(torch.zeros_like(x))
    for k in range(N_FREQ):
        f = float(2.0 ** k)
        s, c = torch.sin(x * f), torch.cos(x * f)
        if order == 0:
            outs += [s, c]
        elif order == 1:
            outs += [f * c, -f * s]
        else:
            outs += [-f * f * s, -f * f * c]
    e = torch.cat(outs, -1)
    return e if embed_w is None else e * embed_w[None, :]


def embed_vjp(d1, ge):
    """E'(x)^T ge: [P,39] -> [P,3] given d1 = dE_e/dx_{c(e)}."""
    return (d1 * ge).reshape(ge.shape[0], -1, 3).sum(1)


def embed_jvp(d1, v):
    """E'(x) v: [P,3] -> [P,39]."""
    return d1 * v.repeat(1, d1.shape[1] // 3)


class TorchOps:
    """Reference backend: the matrices are plain tensors W[l] ([N,K], the folded weight-norm weights), any dtype."""

    def __init__(self, W, b):
        self.W, self.b = W, b

    def lin(self, A, l, bias=True):          # A W_l^T (+ b_l)
        y = A @ self.W[l].T
        return y + self.b[l] if bias else y

    def lin_t(self, A, l):                   # A W_l
        return A @ self.W[l]

    def wgrad(self, D, A):                   # D^T A : [N,K]
        return D.T @ A

    def w_row(self):                         # W_8[0]: the sdf head
        return self.W[8][0]

    def act(self, z, e=None):
        """a = softplus(z), s = softplus'(z); with e (layer 3): the next operand [a | e] (the 1/sqrt 2 of the skip lives in W_4)."""
        a, s = torch.nn.functional.softplus(z, beta=100), torch.sigmoid(100 * z)
        return (a if e is None else torch.cat([a, e], 1)), s

    def colsum(self, D):
        return D.sum(0)

    # pointwise steps (fused CUDA kernels in the GPU backend)
    def mul(self, x, y):
        return x * y

    def mulrow(self, row, y):
        return row[None, :] * y

    def u_dz2(self, h, s, q):                # u = h s;  dz2 = h q softplus''(z) with softplus'' = 100 s (1 - s)
        return h * s, h * q * (100.0 * s * (1.0 - s))

    def dz(self, dA, s, dz2):
        return dA * s if dz2 is None else dA * s + dz2

    def embed(self, x, embed_w, order):
        return embed_terms(x, embed_w, order)

    def embed_vjp(self, d1, ge):
        return embed_vjp(d1, ge)

    def embed_jvp(self, d1, v):
        return embed_jvp(d1, v)

    def relu(self, z):
        return torch.relu(z)

    def relu_bwd(self, dA, a):
        return dA * (a > 0)


SQ2 = 1.0 / math.sqrt(2.0)


def sdf_forward(ops, x, embed_w=None):
    """-> sdf [P], feat [P,256], g [P,3], stash.  The skip's 1/sqrt 2 is carried by W_4 itself (`ops` holds W_4 / sqrt 2, as
    the packed weight images do), so A_4 = [a_3 | e]."""
    e = ops.embed(x, embed_w, 0)
    d1 = ops.embed(x, embed_w, 1)
    A, S = [e], []
    for l in range(8):
        z = ops.lin(A[l], l)
        a, s = ops.act(z, e if l + 1 == SKIP else None)
        S.append(s)
        A.append(a)
    out = ops.lin(A[8], 8)
    sdf, feat = out[:, 0], out[:, 1:]
    w = ops.w_row()
    gbar, q = [None] * 8, [None] * 8
    gbar[7] = ops.mulrow(w, S[7])
    q[7] = w[None, :].expand_as(S[7])
    ge_skip = None
    for l in range(7, 0, -1):
        ql = ops.lin_t(gbar[l], l)
        if l == SKIP:
            ge_skip, ql = ql[:, N_SKIP_A:], ql[:, :N_SKIP_A]
        q[l - 1] = ql
        gbar[l - 1] = ops.mul(ql, S[l - 1])
    ge = ops.lin_t(gbar[0], 0) + ge_skip
    g = ops.embed_vjp(d1, ge)
    return sdf, feat, g, dict(x=x, e=e, d1=d1, A=A, S=S, gbar=gbar, q=q, ge=ge, w=w, embed_w=embed_w)


def sdf_backward(ops, st, d_sdf, d_feat, d_g):
    """-> d_x [P,3], dW[0..8], db[0..8] for upstream gradients of (sdf, feat, g); any of them may be None.
    dW[4] is the gradient w.r.t. the matrix `ops` holds (W_4 / sqrt 2): the caller multiplies by 1/sqrt 2 for W_4 itself."""
    x, e, d1, A, S, gbar, q, ge, w = st["x"], st["e"], st["d1"], st["A"], st["S"], st["gbar"], st["q"], st["ge"], st["w"]
    P = x.shape[0]
    zero = lambda *shape: torch.zeros(*shape, dtype=x.dtype, device=x.device)
    dW = [None] * 9
    db = [None] * 9
    d_x = zero(P, 3)
    dz2 = [None] * 8
    if d_g is not None:
        # ---- I: through g = E'(x)^T ge.  d_ge = E'(x) d_g; the E'' term goes straight to d_x
        d_ge = ops.embed_jvp(d1, d_g)
        d2 = ops.embed(x, st["embed_w"], 2)
        d_x = d_x + ops.embed_vjp(ops.embed_jvp(d2, d_g), ge)
        h = ops.lin(d_ge, 0, bias=False)                    # dL/d gbar_0
        dW[0] = ops.wgrad(gbar[0], d_ge)
        for l in range(1, 8):
            u, dz2[l - 1] = ops.u_dz2(h, S[l - 1], q[l - 1])  # dL/d q_{l-1};  dL/d s_{l-1} x softplus''
            uf = torch.cat([u, d_ge], 1) if l == SKIP else u
            dW[l] = ops.wgrad(gbar[l], uf)
            h = ops.lin(uf, l, bias=False)                  # dL/d gbar_l
        hs, dz2[7] = ops.u_dz2(h, S[7], q[7])
        d_w = ops.colsum(hs)                                # gbar_7 = w * s_7
    else:
        d_w = zero(256)
    # ---- II: ordinary reverse sweep
    d_out = torch.cat([(d_sdf if d_sdf is not None else zero(P))[:, None], d_feat if d_feat is not None else zero(P, 256)], 1)
    dW[8] = ops.wgrad(d_out, A[8])
    dW[8][0] = dW[8][0] + d_w
    db[8] = ops.colsum(d_out)
    dA = ops.lin_t(d_out, 8)
    d_e = zero(P, D_EMBED)
    for l in range(7, -1, -1):
        dzl = ops.dz(dA, S[l], dz2[l])
        g_w = ops.wgrad(dzl, A[l])
        dW[l] = g_w if dW[l] is None else dW[l] + g_w
        db[l] = ops.colsum(dzl)
        dA = ops.lin_t(dzl, l)
        if l == SKIP:
            d_e = d_e + dA[:, N_SKIP_A:]
            dA = dA[:, :N_SKIP_A]
    d_e = d_e + dA
    d_x = d_x + ops.embed_vjp(d1, d_e)
    return d_x, dW, db


# ------------------------------------------------------------------------------------------------ colour net (networks/texture_net.py:69-101)
def rgb_forward(ops, inp):
    """inp [P, K0] = [x_c, n, pose_embed, feat(+time)] -> rgb [P,3], stash.  4 ReLU layers + sigmoid head."""
    A = [inp]
    for l in range(4):
        A.append(ops.relu(ops.lin(A[l], l)))
    rgb = torch.sigmoid(ops.lin(A[4], 4))
    return rgb, dict(A=A, rgb=rgb)


def rgb_backward(ops, st, d_rgb):
    A, rgb = st["A"], st["rgb"]
    dW, db = [None] * 5, [None] * 5
    dz = d_rgb * rgb * (1.0 - rgb)
    dW[4], db[4] = ops.wgrad(dz, A[4]), ops.colsum(dz)
    dA = ops.lin_t(dz, 4)
    for l in range(3, -1, -1):
        dz = ops.relu_bwd(dA, A[l + 1])
        dW[l], db[l] = ops.wgrad(dz, A[l]), ops.colsum(dz)
        dA = ops.lin_t(dz, l)
    return dA, dW, db


# ------------------------------------------------------------------------------------------------ background nets (renderables/background.py)
def skipnet_forward(ops, inp, skip=4, d_skip=None):
    """A Softplus(100) chain with one skip connection and no input gradient output (the NeRF++ background's implicit net,
    confs/general.yaml:34-54; shape_net.py:116-126): A_0 = inp [P, d_in] = [e | cond];  z_l = A_l W_l^T + b_l;  A_{l+1} = softplus(z_l),
    A_skip = [a | e] with e = the first d_skip columns of inp (the embedding; the 1/sqrt 2 lives in W_skip);  out = A_8 W_8^T + b_8."""
    d_skip = inp.shape[1] if d_skip is None else d_skip
    e = inp[:, :d_skip]
    A, S = [inp], []
    for l in range(8):
        a, s = ops.act(ops.lin(A[l], l), e if l + 1 == skip else None)
        S.append(s)
        A.append(a)
    return ops.lin(A[8], 8), dict(A=A, S=S, skip=skip, d_skip=d_skip)


def skipnet_backward(ops, st, d_out):
    """-> d_inp [P, d_in], dW[0..8], db[0..8] (dW[skip] w.r.t. the matrix `ops` holds, W_skip / sqrt 2)."""
    A, S, skip, d_skip = st["A"], st["S"], st["skip"], st["d_skip"]
    dW, db = [None] * 9, [None] * 9
    dW[8], db[8] = ops.wgrad(d_out, A[8]), ops.colsum(d_out)
    dA = ops.lin_t(d_out, 8)
    d_e = None
    for l in range(7, -1, -1):
        dz = ops.dz(dA, S[l], None)
        dW[l], db[l] = ops.wgrad(dz, A[l]), ops.colsum(dz)
        dA = ops.lin_t(dz, l)
        if l == skip:
            n_a = dA.shape[1] - d_skip
            d_e, dA = dA[:, n_a:], dA[:, :n_a]
    d_inp = dA.clone() if d_e is None else torch.cat([dA[:, :d_skip] + d_e, dA[:, d_skip:]], 1)
    return d_inp, dW, db


def head_forward(ops, inp):
    """ReLU layer + 3-row sigmoid head (the background's colour net, 315 -> 128 -> 3)."""
    a1 = ops.relu(ops.lin(inp, 0))
    rgb = torch.sigmoid(ops.lin(a1, 1))
    return rgb, dict(inp=inp, a1=a1, rgb=rgb)


def head_backward(ops, st, d_rgb):
    inp, a1, rgb = st["inp"], st["a1"], st["rgb"]
    dz1 = d_rgb * rgb * (1.0 - rgb)
    dW1, db1 = ops.wgrad(dz1, a1), ops.colsum(dz1)
    dz0 = ops.relu_bwd(ops.lin_t(dz1, 1), a1)
    return ops.lin_t(dz0, 0), [ops.wgrad(dz0, inp), dW1], [ops.colsum(dz0), db1]

