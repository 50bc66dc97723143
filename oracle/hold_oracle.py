"""CPU ORACLE — TEST INFRASTRUCTURE ONLY.

A plain torch-CPU (fp32) restatement of HOLD's volumetric-rendering hot path, written from the
reference's behaviour (file:line cited per function, all relative to the reference's code/src unless
noted).  It exists only to *check* the CUDA path: only `tests/`, `__graft_entry__.smoke()` and
`bench.py`'s cpu_baseline / `--impl reference` legs may import it.  Nothing under `hold_b200/` does.

Parity status: **pinned against the reference's own modules**
(`oracle/ref_harness.py` imports `$HOLD_REFERENCE/code/src/{engine,networks,model,...}` behind
harness-side shims and compares every function below; the committed fixtures in `tests/golden/` were
produced by that script).  The reference has no golden vectors / KATs / tests of its own (SURVEY §4),
and `pytorch3d.ops.knn_points` (pytorch3d 35badc08) is not in the tree, so KNN is restated from its
documented contract (squared L2, K smallest, ascending) and is unpinned at that boundary.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


class RayMissesSphere(RuntimeError):
    """ray_sampler.py:16-18 calls exit(); the oracle raises instead."""


# ----------------------------------------------------------------------------- a1: rays


def camera_rays(uv, pose, intrinsics):
    """datasets/utils.py:230-282 `lift` + `get_camera_params` (pose-matrix branch).
    uv [B,R,2], pose [B,4,4] c2w, intrinsics [B,4,4] -> ray_dirs [B,R,3], cam_loc [B,3]."""
    fx, fy = intrinsics[:, 0, 0:1], intrinsics[:, 1, 1:2]
    cx, cy = intrinsics[:, 0, 2:3], intrinsics[:, 1, 2:3]
    sk = intrinsics[:, 0, 1:2]
    x, y = uv[:, :, 0], uv[:, :, 1]
    z = torch.ones_like(x)
    xl = (x - cx + cy * sk / fy - sk * y / fy) / fx * z
    yl = (y - cy) / fy * z
    pc = torch.stack([xl, yl, z, torch.ones_like(z)], -1)           # [B,R,4]
    world = torch.bmm(pose, pc.permute(0, 2, 1)).permute(0, 2, 1)[:, :, :3]
    cam = pose[:, :3, 3]
    d = F.normalize(world - cam[:, None, :], dim=2)
    return d, cam


# ----------------------------------------------------------------------------- a2/a3: sphere + uniform


def sphere_far(cam, dirs, r):
    """engine/ray_sampler.py:6-25, far root only (near is clamped to 0 and unused)."""
    b = torch.bmm(dirs.view(-1, 1, 3), cam.view(-1, 3, 1)).squeeze(-1)
    under = b**2 - (cam.norm(2, 1, keepdim=True) ** 2 - r**2)
    if (under <= 0).any():
        raise RayMissesSphere("BOUNDING SPHERE PROBLEM")
    return (torch.sqrt(under) - b).clamp_min(0.0)


def uniform_z(near, far, n, jitter=None):
    """UniformSampler.get_z_vals, ray_sampler.py:54-80. far [R,1]. jitter: [R,n] uniforms (training)."""
    t = torch.linspace(0.0, 1.0, steps=n)
    z = near * (1.0 - t) + far * t
    if jitter is not None:
        mids = 0.5 * (z[..., 1:] + z[..., :-1])
        upper = torch.cat([mids, z[..., -1:]], -1)
        lower = torch.cat([z[..., :1], mids], -1)
        z = lower + (upper - lower) * jitter
    return z


# ----------------------------------------------------------------------------- a12: density


def laplace_density(sdf, beta):
    """engine/density.py:21-26."""
    return (1.0 / beta) * (0.5 + 0.5 * sdf.sign() * torch.expm1(-sdf.abs() / beta))


def density_beta(beta_param, beta_min=1e-4):
    """engine/density.py:28-30."""
    return beta_param.abs() + beta_min


# ----------------------------------------------------------------------------- a4: error-bound sampler


def _error_bound(beta, sdf, dists, d_star):
    """ErrorBoundSampler.get_error_bound, ray_sampler.py:354-366.  sdf [R,n], dists/d_star [R,n-1]."""
    sigma = laplace_density(sdf, beta)
    fe = torch.cat([torch.zeros(dists.shape[0], 1, dtype=dists.dtype), dists * sigma[:, :-1]], -1)
    integral = torch.cumsum(fe, -1)
    eps_sec = torch.exp(-d_star / beta) * dists**2.0 / (4 * beta**2)
    eint = torch.cumsum(eps_sec, -1)
    bound = (torch.clamp(torch.exp(eint), max=1.0e6) - 1.0) * torch.exp(-integral[:, :-1])
    return bound.max(-1)[0]


def _inverse_cdf(cdf, bins, u):
    """ray_sampler.py:295-307."""
    inds = torch.searchsorted(cdf, u, right=True)
    below = (inds - 1).clamp_min(0)
    above = inds.clamp_max(cdf.shape[-1] - 1)
    c0, c1 = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    b0, b1 = torch.gather(bins, 1, below), torch.gather(bins, 1, above)
    den = c1 - c0
    den = torch.where(den < 1e-5, torch.ones_like(den), den)
    return b0 + (u - c0) / den * (b1 - b0), inds


def sampler_round(z, sdf, beta, beta0, cfg, it, rand=None, final_extras=None):
    """One iteration of the while loop of ErrorBoundSampler.get_z_vals (ray_sampler.py:160-311) as a pure function of the
    merged, sorted (z, sdf) [R,n], the per-ray beta [R] entering the round and the round index `it` (0-based).  Works in the
    dtype of its inputs (float64 inputs give the exact-arithmetic answer the fp32 results are measured against in
    tests/test_gpu_sampler_rounds.py).  Returns dict(beta, d_star, samples, inds, upsample, not_conv)."""
    Ne, N = cfg["N_samples_eval"], cfg["N_samples"]
    eps, add_tiny = cfg["eps"], cfg["add_tiny"]
    R, dt = z.shape[0], z.dtype
    beta = beta.clone()
    dists = z[:, 1:] - z[:, :-1]
    a, b, c = dists, sdf[:, :-1].abs(), sdf[:, 1:].abs()
    first = a.pow(2) + b.pow(2) <= c.pow(2)
    second = a.pow(2) + c.pow(2) <= b.pow(2)
    d_star = torch.zeros(R, z.shape[1] - 1, dtype=dt)
    d_star[first] = b[first]
    d_star[second] = c[second]
    s = (a + b + c) / 2.0
    area = s * (s - a) * (s - b) * (s - c)
    m = ~first & ~second & (b + c - a > 0)
    d_star[m] = (2.0 * torch.sqrt(area[m])) / a[m]
    d_star = (sdf[:, 1:].sign() * sdf[:, :-1].sign() == 1) * d_star
    err = _error_bound(beta0, sdf, dists, d_star)
    beta[err <= eps] = beta0
    bmin, bmax = beta0.reshape(1).repeat(R), beta
    for _ in range(cfg["beta_iters"]):
        mid = (bmin + bmax) / 2.0
        err = _error_bound(mid.unsqueeze(-1), sdf, dists, d_star)
        bmax[err <= eps] = mid[err <= eps]
        bmin[err > eps] = mid[err > eps]
    beta = bmax
    sigma = laplace_density(sdf, beta.unsqueeze(-1))
    dists1 = torch.cat([dists, torch.full((R, 1), 1e10, dtype=dt)], -1)
    fe = dists1 * sigma
    sfe = torch.cat([torch.zeros(R, 1, dtype=dt), fe[:, :-1]], -1)
    alpha = 1 - torch.exp(-fe)
    T = torch.exp(-torch.cumsum(sfe, -1))
    w = alpha * T
    not_conv = bool(beta.max() > beta0)
    upsample = not_conv and (it + 1) < cfg["max_total_iters"]
    if upsample:
        n_new = Ne
        eps_sec = torch.exp(-d_star / beta.unsqueeze(-1)) * dists**2.0 / (4 * beta.unsqueeze(-1) ** 2)
        eint = torch.cumsum(eps_sec, -1)
        pdf = (torch.clamp(torch.exp(eint), max=1.0e6) - 1.0) * T[:, :-1] + add_tiny
    else:
        n_new = N
        pdf = w[:, :-1] + 1e-5
    pdf = pdf / pdf.sum(-1, keepdim=True)
    cdf = torch.cat([torch.zeros(R, 1, dtype=dt), torch.cumsum(pdf, -1)], -1)
    if upsample or rand is None:
        u = torch.linspace(0.0, 1.0, steps=n_new, dtype=dt).unsqueeze(0).repeat(R, 1)
    else:
        u = rand["u"]
    samples, inds = _inverse_cdf(cdf, z, u.contiguous())
    return dict(beta=beta, d_star=d_star, samples=samples, inds=inds, upsample=upsample, not_conv=not_conv)


def final_z_vals(samples, z, far, cfg, rand=None):
    """ray_sampler.py:313-336: the N weight-CDF samples + near + far + N_extra strided (eval) entries of z, sorted."""
    Nx, R = cfg["N_samples_extra"], samples.shape[0]
    near = torch.full((R, 1), float(cfg["near"]), dtype=samples.dtype)
    if Nx > 0:
        if rand is None:
            eidx = torch.linspace(0, z.shape[1] - 1, Nx).long()
        else:
            eidx = rand["extra_idx"]
            if eidx.dim() == 2:   # one draw per possible round count (include/hold_b200.h, hold_sampler_rand): row rounds-1
                eidx = eidx[z.shape[1] // cfg["N_samples_eval"] - 1]
        extra = torch.cat([near, far, z[:, eidx]], -1)
    else:
        extra = torch.cat([near, far], -1)
    zf, _ = torch.sort(torch.cat([samples, extra], -1), -1)
    return zf


def error_bound_sample(sdf_query, dirs, cam, beta0, cfg, bounding_sphere, rand=None, trace=None):
    """ErrorBoundSampler.get_z_vals with inverse_sphere_bg=True, ray_sampler.py:128-352
    (VolSDF Algorithm 1).  sdf_query(points[P,3]) -> sdf[P] is `sdf_func_with_deformer(...)[0]`.
    rand: None for eval (deterministic linspace u / extras) or dict(jitter[R,Ne], u[R,N], extra_idx[Nx]).
    Returns z_vals [R, N + N_extra + 2] and the number of rounds run (batch-global, :244)."""
    Ne = cfg["N_samples_eval"]
    eps = cfg["eps"]
    R = dirs.shape[0]
    far = sphere_far(cam, dirs, bounding_sphere)
    z = uniform_z(cfg["near"], far, Ne, None if rand is None else rand["jitter"])
    samples, idx = z, None
    d0 = z[:, 1:] - z[:, :-1]
    beta = torch.sqrt((1.0 / (4.0 * math.log(eps + 1.0))) * (d0**2.0).sum(-1))
    it, not_conv, sdf = 0, True, None
    while not_conv and it < cfg["max_total_iters"]:
        pts = cam.unsqueeze(1) + samples.unsqueeze(2) * dirs.unsqueeze(1)
        s_new = sdf_query(pts.reshape(-1, 3)).reshape(R, -1)
        z_in, s_in, beta_in = samples.clone(), s_new.clone(), beta.clone()   # trace only: this round's inputs
        if idx is not None:
            sdf = torch.gather(torch.cat([sdf, s_new], -1), 1, idx)
        else:
            sdf = s_new
        rd = sampler_round(z, sdf, beta, beta0, cfg, it, rand)
        beta, samples, not_conv, upsample = rd["beta"], rd["samples"], rd["not_conv"], rd["upsample"]
        it += 1
        if trace is not None:
            trace.append(dict(it=it, z=z.clone(), sdf=sdf.clone(), beta=beta.clone(), d_star=rd["d_star"].clone(),
                              samples=samples.clone(), inds=rd["inds"].clone(), upsample=upsample,
                              z_in=z_in, s_in=s_in, beta_in=beta_in, far=far.clone()))
        if upsample:
            z, idx = torch.sort(torch.cat([z, samples], -1), -1)
    return final_z_vals(samples, z, far, cfg, rand), it


# ----------------------------------------------------------------------------- a8/a9/a11: embedder + MLPs


def embed(x, n_freq=6, weights=None):
    """engine/embedders.py:48-51 (+ BARF weights :118-122). Layout [x, sin(x), cos(x), sin(2x), ...]."""
    out = [x]
    for k in range(n_freq):
        f = float(2.0**k)
        out += [torch.sin(x * f), torch.cos(x * f)]
    e = torch.cat(out, -1)
    return e if weights is None else e * weights[None, :]


def barf_weights(alpha, L=6, input_dim=3):
    """engine/embedders.py:92-107."""
    k = torch.arange(L, dtype=torch.float32)
    ak = alpha - k
    w = torch.clamp(ak, 0, 1)
    m = torch.logical_and(0 <= ak, ak < 1)
    w[m] = ((1 - torch.cos(ak * math.pi)) / 2)[m]
    w = w[:, None].repeat(1, input_dim * 2).view(-1)
    return torch.cat([torch.ones(input_dim), w], 0)


def wn(sd, name):
    """weight-norm fold w = v * (g/||v||_row)  (nn.utils.weight_norm dim=0; shape_net.py:80)."""
    v, g = sd[name + ".weight_v"], sd[name + ".weight_g"]
    return v * (g / v.norm(dim=1, keepdim=True))


def sdf_mlp(x, sd, cond=None, embed_w=None):
    """ImplicitNet.forward, networks/shape_net.py:84-130. x [P,3] canonical points.
    cond: [P,45] (hand; multiplied by 0 at :104-106) or None.  Returns [P,257] (sdf, feat)."""
    e = embed(x, 6, embed_w)
    h = e
    for l in range(9):
        if l == 0 and cond is not None:
            h = torch.cat([h, cond * 0.0], -1)
        if l == 4:
            h = torch.cat([h, e], 1) / math.sqrt(2)
        h = F.linear(h, wn(sd, f"lin{l}"), sd[f"lin{l}.bias"])
        if l < 8:
            h = F.softplus(h, beta=100)
    return h


def rgb_mlp(x_c, normals, pose_cond, feat, sd):
    """RenderingNet.forward mode 'pose', networks/texture_net.py:69-101.
    pose_cond: [P,45] or None (object -> zeros(8)).  feat already includes the time code for objects."""
    if pose_cond is not None and pose_cond.shape[1] > 0:
        pe = F.linear(pose_cond, sd["lin_pose.weight"], sd["lin_pose.bias"])
    else:
        pe = torch.zeros(x_c.shape[0], 8)
    h = torch.cat([x_c, normals, pe, feat], -1)
    for l in range(5):
        h = F.linear(h, wn(sd, f"lin{l}"), sd[f"lin{l}.bias"])
        if l < 4:
            h = torch.relu(h)
    return torch.sigmoid(h)


# ----------------------------------------------------------------------------- a6/a7: deformers


def knn_points(p, v, K):
    """Contract of pytorch3d.ops.knn_points (35badc08; call site model/mano/deformer.py:85):
    squared L2, K smallest ascending. p [P,3], v [V,3] -> d2 [P,K], idx [P,K] (int64)."""
    d2 = ((p[:, None, :] - v[None, :, :]) ** 2).sum(-1)
    d, i = torch.topk(d2, K, dim=1, largest=False, sorted=True)
    return d, i


def skin_weights_query(p, verts, W, K=15):
    """KNNDeformer.query_skinning_weights_multi, model/mano/deformer.py:84-105. W [V,16]."""
    d2, idx = knn_points(p, verts, K)
    d2 = torch.clamp(d2, max=4)
    conf = torch.exp(-d2)
    conf = conf / conf.sum(-1, keepdim=True)
    w = (W[idx] * conf.unsqueeze(-1)).sum(1)
    outlier = torch.sqrt(d2).min(1).values > 0.1
    return w, outlier, idx


def hand_inverse_warp(x, posed_verts, W, tfs, K=15):
    """KNNDeformer.forward(inverse=True) + skinning(), model/mano/deformer.py:34-68,145-170.
    x [P,3] posed-space points of ONE frame, tfs [16,4,4] -> x_c [P,3], outlier mask, idx."""
    w, outlier, idx = skin_weights_query(x, posed_verts, W, K)
    T = torch.einsum("pn,nij->pij", w, tfs)
    xh = F.pad(x, (0, 1), value=1.0)
    xc = torch.einsum("pij,pj->pi", T.inverse(), xh)[:, :3]
    return xc, outlier, idx


def hand_forward_jacobian(x_c, cano_verts, W, tfs, K=15):
    """The 3x3 Jacobian of KNNDeformer.forward_skinning that volsdf_utils.py:66-81 builds with three
    autograd calls: weights are detached (deformer.py:101) so J = (sum_j w_j tfs_j)[:3,:3] exactly."""
    w, _, idx = skin_weights_query(x_c, cano_verts, W, K)
    T = torch.einsum("pn,nij->pij", w, tfs)
    return T[:, :3, :3], idx


def rigid_inverse_warp(x, tf):
    """ObjectDeformer.forward(inverse=True), model/obj/deformer.py:10-31. tf [4,4]."""
    xh = F.pad(x, (0, 1), value=1.0)
    return (torch.inverse(tf) @ xh.T).T[:, :3]


# ----------------------------------------------------------------------------- a16/a17: servers


def rodrigues(rv):
    """utils/external/lbs.py:298-329 batch_rodrigues. rv [N,3] -> [N,3,3]."""
    ang = torch.norm(rv + 1e-8, dim=1, keepdim=True)
    d = rv / ang
    c, s = torch.cos(ang)[:, None], torch.sin(ang)[:, None]
    rx, ry, rz = d[:, 0:1], d[:, 1:2], d[:, 2:3]
    z = torch.zeros_like(rx)
    Km = torch.cat([z, -rz, ry, rz, z, -rx, -ry, rx, z], 1).view(-1, 3, 3)
    return torch.eye(3, dtype=rv.dtype)[None] + s * Km + (1 - c) * torch.bmm(Km, Km)


def mano_lbs(m, betas, full_pose):
    """`lbs()` utils/external/lbs.py:139-251 as driven by MANO.forward (body_models.py:601-685,
    flat_hand_mean=False so pose += [0,0,0,hands_mean]).  Returns verts, joints(16), A, v_posed."""
    B = full_pose.shape[0]
    pose = full_pose + torch.cat([torch.zeros(3, dtype=full_pose.dtype), m["hands_mean"]])[None]
    v_shaped = m["v_template"][None] + torch.einsum("bl,mkl->bmk", betas, m["shapedirs"])
    J = torch.einsum("bik,ji->bjk", v_shaped, m["J_regressor"])
    Rm = rodrigues(pose.reshape(-1, 3)).view(B, 16, 3, 3)
    pf = (Rm[:, 1:] - torch.eye(3, dtype=Rm.dtype)).reshape(B, -1)
    v_posed = v_shaped + torch.matmul(pf, m["posedirs"]).view(B, -1, 3)
    par = m["parents"]
    rel = J.clone()
    rel[:, 1:] = rel[:, 1:] - J[:, par[1:]]
    Tm = torch.zeros(B, 16, 4, 4, dtype=full_pose.dtype)
    Tm[:, :, :3, :3] = Rm
    Tm[:, :, :3, 3] = rel
    Tm[:, :, 3, 3] = 1.0
    chain = [Tm[:, 0]]
    for i in range(1, 16):
        chain.append(torch.matmul(chain[int(par[i])], Tm[:, i]))
    G = torch.stack(chain, 1)
    Jh = F.pad(J, (0, 1))[..., None]                                  # [B,16,4,1] (w = 0)
    A = G - F.pad(torch.matmul(G, Jh), (3, 0))
    T = torch.matmul(m["lbs_weights"][None].expand(B, -1, -1), A.view(B, 16, 16)).view(B, -1, 4, 4)
    vh = F.pad(v_posed, (0, 1), value=1.0)[..., None]
    verts = torch.matmul(T, vh)[:, :, :3, 0]
    return verts, G[:, :, :3, 3], A, v_posed


def mano_server(m, scene_scale, transl, full_pose, betas, tfs_c_inv=None):
    """GenericServer.forward, model/mano/server.py:62-99. scene_scale [B], transl [B,3].
    tfs_c_inv None <=> absolute=True."""
    verts, joints, A, v_posed = mano_lbs(m, betas, full_pose)
    joints = torch.cat([joints, verts[:, m["tip_ids"]]], 1)          # vertex_joint_selector: +5 tips
    s = scene_scale.view(-1, 1, 1)
    t = transl.view(-1, 1, 3)
    out = {"verts": verts * s + t * s, "jnts": joints * s + t * s}
    top = A[:, :, :3, :] * s.view(-1, 1, 1, 1)                        # server.py:90-93, written without in-place
    tf = torch.cat([torch.cat([top[..., :3], (top[..., 3] + t * s)[..., None]], -1), A[:, :, 3:4, :]], 2)   # ops: differentiable
    if tfs_c_inv is not None:
        tf = torch.einsum("bnij,njk->bnik", tf, tfs_c_inv)
    out["tfs"] = tf
    out["skin_weights"] = m["lbs_weights"][None].expand(verts.shape[0], -1, -1)
    out["v_posed"] = v_posed
    return out


def mano_canonical(m, betas):
    """GenericServer.__init__ canonical pose (server.py:11-17,41-60): scale 1, transl 0,
    pose = -hands_mean (flat hand).  Returns verts_c [778,3], tfs_c_inv [16,4,4]."""
    fp = torch.cat([torch.zeros(3), -m["hands_mean"]])[None]
    out = mano_server(m, torch.ones(1), torch.zeros(1, 3), fp, betas.view(1, 10))
    return out["verts"][0], out["tfs"][0].inverse()


def axis_angle_to_matrix(aa):
    """common/rot.py:105-138,777-805 of the reference (quaternion route)."""
    ang = torch.norm(aa, p=2, dim=-1, keepdim=True)
    half = ang * 0.5
    small = ang.abs() < 1e-6
    k = torch.where(small, 0.5 - ang * ang / 48, torch.sin(half) / torch.where(small, torch.ones_like(ang), ang))
    q = torch.cat([torch.cos(half), aa * k], -1)
    r, i, j, kk = torch.unbind(q, -1)
    two_s = 2.0 / (q * q).sum(-1)
    o = torch.stack([1 - two_s * (j * j + kk * kk), two_s * (i * j - kk * r), two_s * (i * kk + j * r),
                     two_s * (i * j + kk * r), 1 - two_s * (i * i + kk * kk), two_s * (j * kk - i * r),
                     two_s * (i * kk - j * r), two_s * (j * kk + i * r), 1 - two_s * (i * i + j * j)], -1)
    return o.reshape(aa.shape[:-1] + (3, 3))


def object_server(rot, trans, scene_scale, obj_scale, denorm_mat, pts_cano):
    """ObjectModel.forward, model/obj/object_model.py:29-70 -> (obj_tfs [B,4,4], verts [B,Nv,3])."""
    B = rot.shape[0]
    eye = torch.eye(4, dtype=rot.dtype)
    tf = eye.repeat(B, 1, 1)
    tf[:, :3, :3] = axis_angle_to_matrix(rot)
    tf[:, :3, 3] = trans
    sm = eye.repeat(B, 1, 1) * scene_scale[:, None, None]
    sm[:, 3, 3] = 1
    om = eye.repeat(B, 1, 1) * obj_scale
    om[:, 3, 3] = 1
    tf = torch.matmul(torch.matmul(torch.matmul(sm, tf), om), denorm_mat[None].repeat(B, 1, 1))
    vh = F.pad(pts_cano, (0, 1), value=1.0)[None].repeat(B, 1, 1)
    v = torch.bmm(tf, vh.permute(0, 2, 1)).permute(0, 2, 1)
    return tf, v[:, :, :3] / v[:, :, 3:4]


# ----------------------------------------------------------------------------- a13/a14: merge + integrate


def density2weight(density, z, z_max):
    """engine/volsdf_utils.py:220-251. density [R,S], z [R,S], z_max [R]."""
    d = torch.cat([z[:, 1:] - z[:, :-1], z_max.unsqueeze(-1) - z[:, -1:]], -1)
    fe = d * density
    alpha = 1 - torch.exp(-fe)
    T = torch.exp(-torch.cumsum(torch.cat([torch.zeros(d.shape[0], 1), fe], -1), -1))
    return alpha * T[:, :-1], T[:, -1]


def volumetric_render(f, is_training=False):
    """hold/hold_utils.py:243-271 + engine/rendering.py:18-22."""
    w, bgw = density2weight(f["density"].reshape(f["z_vals"].shape), f["z_vals"], f["z_max"])
    integ = lambda c: (c * w[:, :, None]).sum(1)
    out = {
        "fg_rgb": integ(f["color"]),
        "fg_weights": w,
        "mask_prob": torch.clamp(integ(torch.ones_like(f["color"][:, :, :1])), 0, 1),
        "normal": integ(f["normal"]),
        "depth": integ(f["z_vals"][:, :, None]),
        "fg_semantics": integ(f["semantics"]),
        "bg_weights": bgw,
    }
    if not is_training:
        out["fg_rgb.vis"] = out["fg_rgb"] + bgw[:, None]
    return out


def merge_factors(fl, stable=False):
    """hold/hold_utils.py:76-121: concat on the sample axis, sort by z, drop (n-1) head / n tail.
    The reference calls torch.sort without stable=True, so the order of EXACT z ties between nodes (common: all
    nodes share the ray's uniform grid, near and far) is implementation-defined (CPU introsort != CUDA segmented
    sort).  `stable=True` fixes the canonical order hold_b200 implements (lower node first)."""
    n = len(fl)
    keys = ["color", "normal", "density", "semantics", "z_vals"]
    cat = {k: torch.cat([f[k] for f in fl], 1) for k in keys}
    zs, ind = torch.sort(cat["z_vals"], dim=1, stable=stable)
    out = {}
    for k in keys:
        if k == "z_vals":
            out[k] = zs[:, (n - 1): -n]
        else:
            out[k] = torch.gather(cat[k], 1, ind[:, :, None].expand(-1, -1, cat[k].shape[-1]))[:, (n - 1): -n]
    out["z_max"] = zs[:, -n]
    out["indices"] = ind
    return out


# ----------------------------------------------------------------------------- a5/a10/a15/a18: node + scene


def node_forward(kind, class_id, dirs, cam, frame_of_ray, sdf_sd, rgb_sd, beta_param, cfg, R_s,
                 tfs, posed_verts=None, cano_verts=None, skin_W=None, pose_cond=None, time_code=None,
                 embed_w=None, rand=None, trace=None):
    """Node.forward (model/renderables/node.py:49-87) with sample_points of mano_node.py:71-124 /
    object_node.py:57-110, eval mode.  dirs/cam [R,3]; frame_of_ray [R] (rays grouped by frame,
    contiguous, as the reference's view(num_images,-1,3) assumes).
    kind 'hand': tfs [B,16,4,4]; 'object': tfs [B,4,4].  Returns factors dict + extras."""
    R = dirs.shape[0]
    beta = density_beta(beta_param)

    def warp(x, fr):
        xc = torch.empty_like(x)
        for b in fr.unique().tolist():
            m = fr == b
            if kind == "hand":
                xc[m] = hand_inverse_warp(x[m], posed_verts[b], skin_W, tfs[b])[0]
            else:
                xc[m] = rigid_inverse_warp(x[m], tfs[b])
        return xc

    def cond_of(fr):
        return None if kind != "hand" else torch.zeros(fr.shape[0], 45)

    def sdf_query(pts):
        fr = frame_of_ray.repeat_interleave(pts.shape[0] // R)
        return sdf_mlp(warp(pts, fr), sdf_sd, cond_of(fr), embed_w)[:, 0]

    with torch.no_grad():
        z, iters = error_bound_sample(sdf_query, dirs, cam, beta, cfg, R_s, rand, trace)
    S = z.shape[1]
    pts = (cam.unsqueeze(1) + z.unsqueeze(2) * dirs.unsqueeze(1)).reshape(-1, 3)
    fr = frame_of_ray.repeat_interleave(S)
    with torch.no_grad():
        x_c = warp(pts, fr)
    # extract_features, volsdf_utils.py:51-105: SDF again with grad wrt x_c; J of forward skinning
    xg = x_c.clone().requires_grad_(True)
    out = sdf_mlp(xg, sdf_sd, cond_of(fr), embed_w)
    sdf, feat = out[:, :1], out[:, 1:]
    g = torch.autograd.grad(sdf, xg, torch.ones_like(sdf))[0]
    J = torch.empty(x_c.shape[0], 3, 3)
    for b in fr.unique().tolist():
        m = fr == b
        if kind == "hand":
            J[m] = hand_forward_jacobian(x_c[m], cano_verts, skin_W, tfs[b])[0]
        else:
            J[m] = tfs[b][:3, :3]
    normals = F.normalize(torch.einsum("bi,bij->bj", g, J.inverse()), dim=1, eps=1e-6)
    feat = feat.detach()
    if time_code is not None:
        feat = torch.cat([feat, time_code[fr]], -1)
    pc = None if pose_cond is None else pose_cond[fr]
    with torch.no_grad():
        rgb = rgb_mlp(x_c, normals.detach(), pc, feat, rgb_sd)
        dens = laplace_density(sdf.detach(), beta)
    sem = torch.zeros(R, S, 4)
    sem[:, :, class_id] = 1.0
    return {
        "color": rgb.reshape(R, S, 3), "normal": normals.detach().reshape(R, S, 3),
        "density": dens.reshape(R, S, 1), "semantics": sem, "z_vals": z,
        "sdf": sdf.detach().reshape(R, S), "canonical_pts": x_c.reshape(R, S, 3),
        "grad": g.reshape(R, S, 3), "iters": iters, "feat": feat,
    }


def node_forward_train(kind, x, frame_of_point, sdf_sd, rgb_sd, beta_param, tfs, posed_verts=None, cano_verts=None, skin_W=None,
                       pose_cond=None, time_code=None, embed_w=None):
    """Node.forward after sampling in TRAINING mode (node.py:57-87; extract_features with create_graph=True,
    volsdf_utils.py:51-147): deformed points x [P,3] (frames given by frame_of_point) -> dict(sdf, x_c, feat, grad, normal, color,
    density) with the autograd graph attached to every tensor among (state dicts, beta_param, tfs, pose_cond, time_code) that
    requires grad.  Skinning weights are detached (mano/deformer.py:101)."""
    xc = torch.empty_like(x)
    Jl = torch.empty(x.shape[0], 3, 3, dtype=x.dtype)
    parts = []
    order = []
    for b in frame_of_point.unique().tolist():
        m = (frame_of_point == b).nonzero()[:, 0]
        if kind == "hand":
            w, _, _ = skin_weights_query(x[m].detach(), posed_verts[b].detach(), skin_W)
            Tm = torch.einsum("pn,nij->pij", w.detach(), tfs[b])
            xh = F.pad(x[m], (0, 1), value=1.0)
            parts.append(torch.einsum("pij,pj->pi", Tm.inverse(), xh)[:, :3])
        else:
            xh = F.pad(x[m], (0, 1), value=1.0)
            parts.append((xh @ tfs[b].inverse().T)[:, :3])
        order.append(m)
    perm = torch.cat(order)
    x_c = torch.empty_like(x).index_copy(0, perm, torch.cat(parts))
    cond = torch.zeros(x.shape[0], 45, dtype=x.dtype) if kind == "hand" else None
    xg = x_c if x_c.requires_grad else x_c.clone().requires_grad_(True)
    out = sdf_mlp(xg, sdf_sd, cond, embed_w)
    sdf, feat = out[:, 0], out[:, 1:]
    g = torch.autograd.grad(sdf.sum(), xg, create_graph=True)[0]
    Js = []
    for b in frame_of_point.unique().tolist():
        m = (frame_of_point == b).nonzero()[:, 0]
        if kind == "hand":
            w, _, _ = skin_weights_query(x_c[m].detach(), cano_verts, skin_W)
            Js.append(torch.einsum("pn,nij->pij", w.detach(), tfs[b])[:, :3, :3])
        else:
            Js.append(tfs[b][:3, :3][None].expand(m.shape[0], 3, 3))
    J = torch.empty(x.shape[0], 3, 3, dtype=x.dtype).index_copy(0, perm, torch.cat(Js))
    normal = F.normalize(torch.einsum("bi,bij->bj", g, J.inverse()), dim=1, eps=1e-6)
    f2 = feat if time_code is None else torch.cat([feat, time_code[frame_of_point]], -1)
    pc = None if pose_cond is None else pose_cond[frame_of_point]
    color = rgb_mlp(x_c, normal, pc, f2, rgb_sd)
    density = laplace_density(sdf, density_beta(beta_param))
    return dict(sdf=sdf, x_c=x_c, feat=feat, grad=g, normal=normal, color=color, density=density)


def composite(factors_list, stable=False):
    """HOLDNet.forward_fg, hold/hold_net.py:76-88: composite render + per-node renders."""
    comp = merge_factors(factors_list, stable)
    out = {"comp": volumetric_render(comp)}
    out["comp"]["z_vals"] = comp["z_vals"]
    out["comp"]["indices"] = comp["indices"]
    for k, f in enumerate(factors_list):
        ff = dict(f)
        ff["z_max"] = f["z_vals"][:, -1]
        out[k] = volumetric_render(ff)
    return out


# ----------------------------------------------------------------------------- scene driver (tests/bench)


def scene_articulation(sc):
    """Per-node server outputs for a hold_b200.synth.SynthScene (a16/a17)."""
    art = {}
    B = sc.B
    scale = torch.full((B,), float(sc.scene_scale))
    for nid in sc.node_ids:
        p = sc.params[nid]
        if nid in ("right", "left"):
            m = sc.mano[nid]
            verts_c, tfs_c_inv = mano_canonical(m, sc.betas[nid])
            full_pose = torch.cat([p["global_orient"], p["pose"]], 1)
            out = mano_server(m, scale, p["transl"], full_pose, sc.betas[nid][None].repeat(B, 1), tfs_c_inv)
            art[nid] = dict(kind="hand", tfs=out["tfs"], verts=out["verts"], jnts=out["jnts"],
                            cano_verts=verts_c, skin_W=m["lbs_weights"], pose_cond=full_pose[:, 3:] / math.pi,
                            v_posed=out["v_posed"], tfs_c_inv=tfs_c_inv)
        else:
            tf, v = object_server(p["global_orient"], p["transl"], scale, 1.0, torch.eye(4), sc.obj_pts_cano)
            art[nid] = dict(kind="object", tfs=tf, verts=v)
    return art


CLASS_ID = {"object": 1, "right": 2, "left": 3}


def render_scene(sc, ray_ids=None, chunk=None, trace=None, stable_ties=False):
    """Whole foreground path a1 -> a14 for the rays `ray_ids` (flat index into [B*H*W]) of a
    SynthScene, processed in calls of `chunk` rays (the reference renders 512-pixel chunks,
    datasets/eval_datasets.py:13; the sampler's convergence flag is per call, ray_sampler.py:244)."""
    art = scene_articulation(sc)
    dirs, cam = camera_rays(sc.uv, sc.extrinsics, sc.intrinsics)
    P = dirs.shape[1]
    dirs = dirs.reshape(-1, 3)
    cam = cam.unsqueeze(1).repeat(1, P, 1).reshape(-1, 3)
    frame = torch.arange(sc.B).repeat_interleave(P)
    if ray_ids is None:
        ray_ids = torch.arange(dirs.shape[0])
    chunk = chunk or ray_ids.numel()
    outs = []
    for s in range(0, ray_ids.numel(), chunk):
        ids = ray_ids[s:s + chunk]
        fl = []
        for nid in sc.node_ids:
            a = art[nid]
            f = node_forward(a["kind"], CLASS_ID[nid], dirs[ids], cam[ids], frame[ids], sc.sdf_state[nid],
                             sc.rgb_state[nid], sc.beta[nid], sc.sampler, sc.bounding_sphere, a["tfs"],
                             posed_verts=a.get("verts") if a["kind"] == "hand" else None,
                             cano_verts=a.get("cano_verts"), skin_W=a.get("skin_W"),
                             pose_cond=a.get("pose_cond"),
                             time_code=sc.time_code if a["kind"] == "object" else None,
                             trace=None if trace is None else trace.setdefault(nid, []))
            fl.append(f)
        comp = composite(fl, stable_ties)
        outs.append(dict(nodes=fl, render=comp))
    return outs, art


# ----------------------------------------------------------------------------- §8f rank 1: NeRF++ background


def embed_n(x, n_freq):
    """engine/embedders.py:48-51 for any input width (background: 4-d points x 10 freqs, view dirs x 4 freqs)."""
    out = [x]
    for k in range(n_freq):
        f = float(2.0**k)
        out += [torch.sin(x * f), torch.cos(x * f)]
    return torch.cat(out, -1)


def bg_sdf_mlp(p4, frame_code, sd):
    """Background ImplicitNet (confs/general.yaml:34-54): d_in 4, multires 10 (84), cond 'frame' (32) at layer 0,
    8x256, skip_in [4], no weight-norm, Softplus(100).  p4 [P,4], frame_code [P,32] -> [P,257]."""
    e = embed_n(p4, 10)
    h = e
    for l in range(9):
        if l == 0:
            h = torch.cat([h, frame_code], -1)
        if l == 4:
            h = torch.cat([h, e], 1) / math.sqrt(2)
        h = F.linear(h, sd[f"lin{l}.weight"], sd[f"lin{l}.bias"])
        if l < 8:
            h = F.softplus(h, beta=100)
    return h


def bg_rgb_mlp(view_dirs, frame_code, feat, sd):
    """Background RenderingNet, mode 'nerf_frame_encoding' (texture_net.py:55-68,93-101; general.yaml:55-64)."""
    h = torch.cat([embed_n(view_dirs, 4), frame_code, feat], -1)
    h = torch.relu(F.linear(h, sd["lin0.weight"], sd["lin0.bias"]))
    return torch.sigmoid(F.linear(h, sd["lin1.weight"], sd["lin1.bias"]))


def depth2pts_outside(ray_o, ray_d, depth, R_s):
    """Background.depth2pts_outside, model/renderables/background.py:102-135 (NeRF++ inverted sphere)."""
    o_dot_d = torch.sum(ray_d * ray_o, dim=-1)
    under = o_dot_d**2 - ((ray_o**2).sum(-1) - R_s**2)
    d_sphere = torch.sqrt(under) - o_dot_d
    p_sphere = ray_o + d_sphere.unsqueeze(-1) * ray_d
    p_mid = ray_o - o_dot_d.unsqueeze(-1) * ray_d
    p_mid_norm = torch.norm(p_mid, dim=-1)
    axis = torch.cross(ray_o, p_sphere, dim=-1)
    axis = axis / torch.norm(axis, dim=-1, keepdim=True)
    phi = torch.asin(p_mid_norm / R_s)
    theta = torch.asin(p_mid_norm * depth)
    ang = (phi - theta).unsqueeze(-1)
    pn = (p_sphere * torch.cos(ang) + torch.cross(axis, p_sphere, dim=-1) * torch.sin(ang)
          + axis * torch.sum(axis * p_sphere, dim=-1, keepdim=True) * (1.0 - torch.cos(ang)))
    pn = pn / torch.norm(pn, dim=-1, keepdim=True)
    return torch.cat((pn, depth.unsqueeze(-1)), dim=-1)


def background(bg_weights, ray_dirs, cam_loc, frame_code, frame_of_ray, bg_sdf_sd, bg_rgb_sd, R_s, n_bg=32):
    """HOLDNet.forward's background leg (hold_net.py:91-118) = inverse_sample (ray_sampler.py:82-85) +
    Background.forward (background.py:35-100) + bg_volume_rendering (:137-165).  Eval mode.
    Returns bg_rgb [R,3], bg_rgb_only [R,3], bg_semantics [R,4], z_bg [R,n_bg]."""
    R = ray_dirs.shape[0]
    z_bg = uniform_z(0.0, torch.ones(R, 1), n_bg) * (1.0 / R_s)
    zf = torch.flip(z_bg, dims=[-1])
    dirs = ray_dirs.unsqueeze(1).repeat(1, n_bg, 1)
    locs = cam_loc.unsqueeze(1).repeat(1, n_bg, 1)
    p4 = depth2pts_outside(locs, dirs, zf, R_s).reshape(-1, 4)
    fc = frame_code[frame_of_ray].repeat_interleave(n_bg, 0)
    o = bg_sdf_mlp(p4, fc, bg_sdf_sd)
    sdf, feat = o[:, :1], o[:, 1:]
    rgb = bg_rgb_mlp(dirs.reshape(-1, 3), fc, feat, bg_rgb_sd).reshape(R, n_bg, 3)
    dens = sdf.abs().reshape(R, n_bg)                                  # AbsDensity, engine/density.py:33-35
    d = torch.cat([zf[:, :-1] - zf[:, 1:], torch.full((R, 1), 1e10)], -1)
    fe = d * dens
    alpha = 1 - torch.exp(-fe)
    T = torch.exp(-torch.cumsum(torch.cat([torch.zeros(R, 1), fe[:, :-1]], -1), -1))
    w = alpha * T
    only = (w.unsqueeze(-1) * rgb).sum(1)
    sem = torch.zeros(R, 4)
    sem[:, 0] = 1.0
    return bg_weights.unsqueeze(-1) * only, only, bg_weights.unsqueeze(-1) * sem, z_bg
