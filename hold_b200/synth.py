"""Seeded synthetic scenes for parity tests and benchmarks (SURVEY.md §8d).

Nothing here touches the reference: no dataset, MANO pickle or checkpoint is
available offline, so the rig is a MANO-*shaped* struct (778 verts, 16 joints,
same kinematic tree as MANO: parents of `utils/external/lbs.py:378-383`'s loop)
and the networks use the reference constructors' init recipe
(`networks/shape_net.py:51-73`, geometric init).

Everything is generated with numpy's MT19937 / torch's CPU generator so that every machine, with or without a GPU,
produces bit-identical inputs.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
import torch

MANO_PARENTS = np.array([-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 0, 10, 11, 0, 13, 14], dtype=np.int64)
# thumb, index, middle, ring, pinky tip vertices (utils/external/vertex_ids.py:69-75)
MANO_TIP_IDS = np.array([744, 320, 443, 554, 671], dtype=np.int64)
N_VERTS = 778
RIG_SCALE = 4.0
N_JOINTS = 16


def make_mano_struct(seed: int = 0, is_rhand: bool = True) -> dict:
    """A MANO-shaped model struct: same tensor shapes/semantics as MANO_{RIGHT,LEFT}.pkl."""
    rs = np.random.RandomState(1000 + seed)
    # --- rest joints: wrist + 5 fingers x 3 joints (metres, hand ~0.19 long)
    J = np.zeros((N_JOINTS, 3), np.float64)
    finger_dirs = []
    for f in range(5):
        ang = (-0.55 + 0.28 * f) if f > 0 else -1.05
        d = np.array([math.sin(ang), math.cos(ang), 0.0])
        finger_dirs.append(d)
        base = 0.085 * d + np.array([0.0, 0.0, 0.004 * (f - 2)])
        seg = [0.036, 0.026, 0.020] if f > 0 else [0.034, 0.028, 0.022]
        p = base.copy()
        for s in range(3):
            J[1 + 3 * f + s] = p
            p = p + seg[s] * d
    # tips (not joints, used to place verts)
    tips = [J[3 + 3 * f] + 0.02 * finger_dirs[f] for f in range(5)]
    # --- vertices: capsules around bones + palm slab
    verts = np.zeros((N_VERTS, 3), np.float64)
    owner = np.zeros(N_VERTS, np.int64)
    n_palm = 250
    for i in range(N_VERTS):
        if i < n_palm:
            u, v = rs.rand(), rs.rand()
            p = np.array([(-0.045 + 0.09 * u), 0.095 * v, 0.0])
            p[2] = (0.011 + 0.003 * rs.rand()) * (1 if rs.rand() > 0.5 else -1)
            verts[i] = p
            owner[i] = 0
        else:
            f = (i - n_palm) % 5
            s = rs.randint(0, 3)
            j0 = 1 + 3 * f + s
            a = J[j0]
            b = J[j0 + 1] if s < 2 else tips[f]
            t = rs.rand()
            c = a + t * (b - a)
            d = finger_dirs[f]
            e1 = np.cross(d, np.array([0.0, 0.0, 1.0]))
            e1 /= np.linalg.norm(e1)
            e2 = np.cross(d, e1)
            th = 2 * math.pi * rs.rand()
            r = 0.0085 - 0.0008 * s + 0.0008 * rs.rand()
            verts[i] = c + r * (math.cos(th) * e1 + math.sin(th) * e2)
            owner[i] = j0
    # make the 5 MANO tip ids actual finger tips
    for f in range(5):
        verts[MANO_TIP_IDS[f]] = tips[f]
        owner[MANO_TIP_IDS[f]] = 3 + 3 * f
    # --- skinning weights: soft assignment to the 4 nearest joints, rows sum to 1
    d2 = ((verts[:, None, :] - J[None, :, :]) ** 2).sum(-1)
    w = np.exp(-d2 / (2 * 0.018**2))
    w[np.arange(N_VERTS), owner] += 0.5
    order = np.argsort(-w, axis=1)
    mask = np.zeros_like(w)
    np.put_along_axis(mask, order[:, :4], 1.0, axis=1)
    w = w * mask
    w = w / w.sum(1, keepdims=True)
    # --- joint regressor: sparse convex combination of nearby verts
    Jr = np.exp(-d2.T / (2 * 0.012**2)) + 1e-12
    Jr = Jr / Jr.sum(1, keepdims=True)
    # shift the template so that regressed joints coincide with J as well as possible (cosmetic)
    shapedirs = 0.0025 * rs.randn(N_VERTS, 3, 10)
    posedirs = 0.0006 * rs.randn(135, N_VERTS * 3)
    hands_mean = 0.12 * rs.randn(45)
    if not is_rhand:
        verts[:, 0] *= -1
        shapedirs[:, 0, :] *= -1
        hands_mean = hands_mean.reshape(15, 3) * np.array([1.0, -1.0, -1.0])
        hands_mean = hands_mean.reshape(45)
    f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    # canonical units: x RIG_SCALE so the rig is O(1) like the SDF net's geometric init (radius ~0.5)
    verts, shapedirs, posedirs = verts * RIG_SCALE, shapedirs * RIG_SCALE, posedirs * RIG_SCALE
    return {
        "v_template": f32(verts),
        "shapedirs": f32(shapedirs),
        "posedirs": f32(posedirs),
        "J_regressor": f32(Jr),
        "lbs_weights": f32(w / w.sum(1, keepdims=True)),
        "parents": torch.from_numpy(MANO_PARENTS.copy()),
        "hands_mean": f32(hands_mean),
        "tip_ids": torch.from_numpy(MANO_TIP_IDS.copy()),
        "is_rhand": is_rhand,
    }


# ----------------------------------------------------------------------------- network weights


def _geometric_linear(l, n_lin, in_dim, out_dim, d_embed, bias_radius, gen):
    """Geometric init of one ImplicitNet layer (shape_net.py:51-73), own generator."""
    w = torch.empty(out_dim, in_dim)
    b = torch.zeros(out_dim)
    std = math.sqrt(2.0) / math.sqrt(out_dim)
    if l == n_lin - 1:
        w.normal_(math.sqrt(math.pi) / math.sqrt(in_dim), 1e-4, generator=gen)
        b.fill_(-bias_radius)
    elif l == 0:
        w.zero_()
        w[:, :3].normal_(0.0, std, generator=gen)
    elif l == 4:  # skip_in
        w.normal_(0.0, std, generator=gen)
        w[:, -(d_embed - 3):] = 0.0
    else:
        w.normal_(0.0, std, generator=gen)
    return w, b


def make_sdf_state(kind: str, seed: int, radius: float, perturb: float = 0.0) -> dict:
    """state_dict of one ImplicitNet in the reference's key format
    (`lin<k>.{weight_g,weight_v,bias}`; SURVEY §5 checkpoint row).

    kind: "hand" (cond=pose 45 zeroed columns, lin0 in=84) or "object" (lin0 in=39).
    """
    gen = torch.Generator().manual_seed(2000 + seed)
    d_embed = 39
    cond = 45 if kind == "hand" else 0
    dims = [d_embed] + [256] * 8 + [257]
    sd = {}
    n_lin = len(dims) - 1
    for l in range(n_lin):
        out_dim = dims[l + 1] - d_embed if (l + 1) == 4 else dims[l + 1]
        in_dim = dims[l] + (cond if l == 0 else 0)
        w, b = _geometric_linear(l, n_lin, in_dim, out_dim, d_embed, radius, gen)
        if perturb > 0:
            w = w + perturb * torch.randn(w.shape, generator=gen)
        sd[f"lin{l}.weight_v"] = w.contiguous()
        sd[f"lin{l}.weight_g"] = w.norm(dim=1, keepdim=True).contiguous()
        sd[f"lin{l}.bias"] = b
    return sd


def make_rgb_state(kind: str, seed: int) -> dict:
    """state_dict of one RenderingNet (mode 'pose', texture_net.py:22-42): default nn.Linear init
    + weight-norm; hand d_in = 3+3+8+256 = 270, object + 32 time code = 302."""
    gen = torch.Generator().manual_seed(3000 + seed)
    d0 = 270 if kind == "hand" else 302
    dims = [d0, 256, 256, 256, 256, 3]
    sd = {}

    def lin(i, o):
        k = 1.0 / math.sqrt(i)
        w = (torch.rand(o, i, generator=gen) * 2 - 1) * k
        b = (torch.rand(o, generator=gen) * 2 - 1) * k
        return w, b

    for l in range(5):
        w, b = lin(dims[l], dims[l + 1])
        sd[f"lin{l}.weight_v"] = w
        sd[f"lin{l}.weight_g"] = w.norm(dim=1, keepdim=True)
        sd[f"lin{l}.bias"] = b
    pose_dim = 45 if kind == "hand" else 0
    w, b = lin(max(pose_dim, 1), 8)
    if pose_dim == 0:
        w = torch.zeros(8, 0)
    sd["lin_pose.weight"] = w
    sd["lin_pose.bias"] = b
    return sd


def make_bg_state(seed: int) -> tuple[dict, dict]:
    """Background nets (confs/general.yaml:34-64): ImplicitNet d_in 4 / multires 10 / cond frame(32), init 'none',
    no weight-norm -> plain `lin<k>.{weight,bias}`; RenderingNet 315 -> 128 -> 3.  Default nn.Linear init."""
    gen = torch.Generator().manual_seed(4000 + seed)

    def lin(i, o):
        k = 1.0 / math.sqrt(i)
        return (torch.rand(o, i, generator=gen) * 2 - 1) * k, (torch.rand(o, generator=gen) * 2 - 1) * k

    dims = [84] + [256] * 8 + [257]
    sdf, rgb = {}, {}
    for l in range(9):
        out_dim = dims[l + 1] - 84 if (l + 1) == 4 else dims[l + 1]
        in_dim = dims[l] + (32 if l == 0 else 0)
        sdf[f"lin{l}.weight"], sdf[f"lin{l}.bias"] = lin(in_dim, out_dim)
    rgb["lin0.weight"], rgb["lin0.bias"] = lin(315, 128)
    rgb["lin1.weight"], rgb["lin1.bias"] = lin(128, 3)
    return sdf, rgb


# ----------------------------------------------------------------------------- scenes


@dataclass
class SynthScene:
    """One synthetic HOLD scene: B frames, n nodes, H x W pixels per frame."""

    H: int
    W: int
    B: int
    node_ids: list
    uv: torch.Tensor          # [B, H*W, 2] (x=col, y=row), image_dataset.py:66-67
    intrinsics: torch.Tensor  # [B, 4, 4]
    extrinsics: torch.Tensor  # [B, 4, 4] camera-to-world (get_camera_params uses pose[:, :3, 3] as centre)
    scene_scale: float
    bounding_sphere: float
    sampler: dict
    mano: dict = field(default_factory=dict)       # node_id -> mano struct
    betas: dict = field(default_factory=dict)      # node_id -> [10]
    params: dict = field(default_factory=dict)     # node_id -> dict(global_orient, pose, transl [, betas])
    sdf_state: dict = field(default_factory=dict)  # node_id -> ImplicitNet state_dict
    rgb_state: dict = field(default_factory=dict)  # node_id -> RenderingNet state_dict
    beta: dict = field(default_factory=dict)       # node_id -> density.beta parameter (scalar tensor)
    time_code: torch.Tensor | None = None          # [B, 32] object frame latent
    obj_pts_cano: torch.Tensor | None = None       # [Nv, 3]
    frame_idx: torch.Tensor | None = None          # [B]


def sampler_cfg(S: int = 128) -> dict:
    """'S samples/ray' == the reference ratios of confs/general.yaml:69-78 (SURVEY D2)."""
    return dict(near=0.0, N_samples=S // 2, N_samples_eval=S, N_samples_extra=S // 4,
                eps=0.1, beta_iters=10, max_total_iters=5, add_tiny=1.0e-6)


def _look_at(cam, target=np.zeros(3)):
    z = target - cam
    z = z / np.linalg.norm(z)
    up = np.array([0.0, -1.0, 0.0])
    x = np.cross(z, up)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = x, y, z, cam
    return c2w


def make_scene(H=64, W=64, S=128, nodes=("right", "object"), B=1, seed=0, perturb=0.0,
               hand_radius=0.45, obj_radius=0.5) -> SynthScene:
    rs = np.random.RandomState(seed)
    scene_scale = 1.3
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    uv1 = np.stack([xs.reshape(-1), ys.reshape(-1)], -1).astype(np.float32)
    uv = torch.from_numpy(np.broadcast_to(uv1[None], (B, H * W, 2)).copy())
    K = np.eye(4, dtype=np.float32)
    K[0, 0] = K[1, 1] = 1.2 * W
    K[0, 2], K[1, 2] = W / 2.0, H / 2.0
    intr = torch.from_numpy(np.broadcast_to(K[None], (B, 4, 4)).copy())
    ext = []
    for b in range(B):
        ang = 0.15 * b
        cam = 2.0 * np.array([math.sin(ang) * 0.3, 0.1 * math.sin(0.7 * b), -math.cos(ang * 0.3)])
        cam = 2.0 * cam / np.linalg.norm(cam)
        ext.append(_look_at(cam))
    ext = torch.from_numpy(np.stack(ext).astype(np.float32))
    sc = SynthScene(H=H, W=W, B=B, node_ids=list(nodes), uv=uv, intrinsics=intr, extrinsics=ext,
                    scene_scale=scene_scale, bounding_sphere=6.0, sampler=sampler_cfg(S))
    sc.frame_idx = torch.arange(B)
    walk = lambda dim, s: np.cumsum(s * rs.randn(B, dim), 0).astype(np.float32)
    for k, nid in enumerate(nodes):
        if nid in ("right", "left"):
            sc.mano[nid] = make_mano_struct(seed, is_rhand=(nid == "right"))
            sc.betas[nid] = torch.from_numpy((0.5 * rs.randn(10)).astype(np.float32))
            off = 0.45 if len([n for n in nodes if n in ("right", "left")]) == 2 else 0.0
            sx = off if nid == "right" else -off
            go = 0.3 * rs.randn(1, 3).astype(np.float32) + walk(3, 0.03)
            pose = 0.3 * rs.randn(1, 45).astype(np.float32) + walk(45, 0.02)
            tr = np.array([[sx - 0.08, -0.36, 0.0]], np.float32) + 0.02 * rs.randn(1, 3).astype(np.float32) + walk(3, 0.002)
            sc.params[nid] = dict(global_orient=torch.from_numpy(go), pose=torch.from_numpy(pose),
                                  transl=torch.from_numpy(tr.astype(np.float32)))
            sc.sdf_state[nid] = make_sdf_state("hand", seed + 10 * k, hand_radius, perturb)
            sc.rgb_state[nid] = make_rgb_state("hand", seed + 10 * k)
        else:
            go = 0.3 * rs.randn(1, 3).astype(np.float32) + walk(3, 0.03)
            tr = 0.02 * rs.randn(1, 3).astype(np.float32) + np.array([[0.22, 0.1, 0.1]], np.float32) + walk(3, 0.002)
            sc.params[nid] = dict(global_orient=torch.from_numpy(go), transl=torch.from_numpy(tr.astype(np.float32)))
            sc.sdf_state[nid] = make_sdf_state("object", seed + 10 * k, obj_radius, perturb)
            sc.rgb_state[nid] = make_rgb_state("object", seed + 10 * k)
            pts = rs.randn(512, 3)
            pts = obj_radius * pts / np.linalg.norm(pts, axis=1, keepdims=True)
            sc.obj_pts_cano = torch.from_numpy(pts.astype(np.float32))
            sc.time_code = torch.from_numpy((0.1 * rs.randn(B, 32)).astype(np.float32))
        sc.beta[nid] = torch.tensor(0.1)
    return sc
