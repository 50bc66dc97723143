"""CPU-only: the references, case generators and error measures of tests/test_gpu_skin_warps.py, run at tiny sizes against the
oracle (knn_points / skin_weights_query / hand_inverse_warp / rigid_inverse_warp and torch.autograd over them), and the generated
ray cases through knn_phases.h on the host, so that the first GPU run is not the first run of the reference code.

What the device tests compare:
  - the ray-walk KNN of k_inverse_warp_hand_rays against the full scan of k_inverse_warp, bit for bit;
  - hold_inverse_warp / hold_forward_warp against a float32 brute-force KNN in lexicographic (distance, index) order and a float64
    blend-and-solve on the same neighbours;
  - hold_inverse_warp_bwd against float64 autograd with the skinning weights detached (deformer.py:101)."""
import math

import numpy as np
import torch

from hold_b200 import synth
from oracle import hold_oracle as O

K, NV, NJ = 15, 778, 16
REL_TOL = 1e-4                    # the project's relative bar on forward values
BWD_TOL = 1e-5                    # g_tfs entries, relative to the sum of the magnitudes of the terms they add up
F32_FACTOR, F32_FLOOR = 4.0, 2.0 ** -20
# exact duplicate posed vertices (distance ties resolved by index): a triple and a pair
DUPS = ((7, 100), (7, 650), (201, 412))
TIE_JC = (1, 5, 13, 30)           # sample index of the constructed tie on each tie ray (previous sample = index - 1)
N_SPECIAL = len(TIE_JC) + 6 + 6 + 4   # the special rays of frame_rays: tie, through duplicates, inside the hand, on vertices


# ------------------------------------------------------------------------------------------------ poses and posed vertices
def mano(nid):
    return synth.make_mano_struct(0, is_rhand=(nid == "right"))


def tie_vertices(W):
    """u < w with different dominant bones, and 14 fillers: the vertices moved into the tie construction of `posed_hand`."""
    reserved = {v for p in DUPS for v in p}
    bone = W.argmax(1)
    free = [v for v in range(NV) if v not in reserved]
    u = free[0]
    w = next(v for v in reversed(free) if bone[v] != bone[u])
    fill = [v for v in free[1:] if v != w][::37][:14]
    assert len(fill) == 14
    return u, w, fill


def posed_hand(nid, B, seed):
    """A strongly articulated hand per frame (different poses per frame), tfs with the constant last row (0, 0, 0, 1), exact
    duplicate vertices, and 16 vertices moved (per frame) into the tie construction of `tie_rays`.  Returns (verts [B,778,3],
    tfs [B,16,4,4], ties: per frame (cam_x0, y0, z0, m)) on the CPU."""
    m = mano(nid)
    g = torch.Generator().manual_seed(seed)
    pose = torch.randn(B, 48, generator=g) * 0.5
    transl = torch.tensor([[-0.08, -0.36, 0.0]]) + 0.05 * torch.randn(B, 3, generator=g)
    out = O.mano_server(m, torch.full((B,), 1.3), transl, pose, 0.5 * torch.randn(B, 10, generator=g))
    verts, tfs = out["verts"].float().contiguous(), out["tfs"].float().clone()
    tfs[:, :, 3, :] = torch.tensor([0.0, 0.0, 0.0, 1.0])
    u, w, fill = tie_vertices(m["lbs_weights"])
    ties = []
    for b in range(B):
        v = verts[b]
        hi, c = v.max(0).values, v.mean(0)
        x0, y0, z0 = float(math.ceil(hi[0].item()) + 2), round(c[1].item() * 64) / 64, round(c[2].item() * 64) / 64
        mid = x0 + 0.5
        v[u] = torch.tensor([mid + 0.125, y0 + 0.125, z0])
        v[w] = torch.tensor([mid - 0.125, y0 + 0.125, z0])
        for k, f in enumerate(fill):
            v[f] = torch.tensor([mid + k / 512, y0 + 1 / 1024, z0])
        for a, d in DUPS:
            v[d] = v[a]
        ties.append((mid, y0, z0))
    return verts.contiguous(), tfs.contiguous(), ties


def object_tfs(B, seed):
    """Per frame T = [[c R, t], [0, s]] . D with D a denorm-like matrix ([[sigma Q, t'], [0, 1]]); c cycles through 0.01, 100 and
    moderate values, s through 1 and values != 1 (the / s of the inverse, the / w of the forward)."""
    g = torch.Generator().manual_seed(seed)
    cs, ss = (0.01, 100.0, 1.3, 0.7, 2.5), (1.0, 1.0, 1.7, 0.6, 1.25)
    out = torch.zeros(B, 4, 4, dtype=torch.float64)
    for b in range(B):
        M = torch.eye(4, dtype=torch.float64)
        M[:3, :3] = cs[b % 5] * O.axis_angle_to_matrix(torch.randn(1, 3, generator=g))[0].double()
        M[:3, 3] = torch.randn(3, generator=g).double() * 0.3 * cs[b % 5]
        M[3, 3] = ss[b % 5]
        D = torch.eye(4, dtype=torch.float64)
        D[:3, :3] = 1.7 * torch.linalg.qr(torch.randn(3, 3, generator=g).double())[0]
        D[:3, 3] = torch.tensor([0.11, -0.07, 0.23], dtype=torch.float64)
        out[b] = M @ D
    return out.float().contiguous()


# ------------------------------------------------------------------------------------------------ rays (hot path cases)
def expected_seg_len(B, rays, S, sm_count):
    """launch_inverse_warp's walk length (api.cu): 32, halved while B * rays * ceil(S / len) < sm_count * 4 * 128 * 2."""
    seg = 32
    while seg > 4 and B * rays * (-(-S // seg)) < sm_count * 4 * 128 * 2:
        seg //= 2
    return seg


def rays_for_seg_len(L, B, S, sm_count, odd=True):
    """Rays per frame whose launch walks L samples per thread; odd: not a multiple of 128."""
    T = sm_count * 4 * 128 * 2
    lo = -(-T // (-(-S // L)))                      # smallest total ray count at which length L stays
    rpf = -(-lo // B) + 37
    if odd and rpf % 128 == 0:
        rpf += 1
    return rpf


def pixel_dirs(seed=0):
    """Ray directions of one synthetic 512 x 512 camera looking at the hand (synth.make_scene's camera set-up)."""
    sc = synth.make_scene(H=512, W=512, S=8, nodes=(), B=1, seed=seed)
    d, c = O.camera_rays(sc.uv, sc.extrinsics, sc.intrinsics)
    return d[0].contiguous(), c[0].contiguous()


def nearest_on_ray(cam, dirs, verts, chunk=16384):
    """Depth along each ray of its closest approach to the nearest vertex (for depths near the surface)."""
    t_out = torch.empty(cam.shape[0], device=cam.device)
    for a in range(0, cam.shape[0], chunk):
        c, d = cam[a:a + chunk], dirs[a:a + chunk]
        rel = verts[None] - c[:, None]                              # [n, 778, 3]
        t = (rel * d[:, None]).sum(-1).clamp_min(0.0)
        d2 = ((rel - t[..., None] * d[:, None]) ** 2).sum(-1)
        t_out[a:a + chunk] = t.gather(1, d2.argmin(1, keepdim=True))[:, 0]
    return t_out


def frame_rays(verts, tie, n, S, seed, pix=None, dev=torch.device("cpu")):
    """n rays of one frame, S samples each: (cam [n,3], dirs [n,3], z [n,S]) float32 on `dev`, and the number of special rays.
    Special rays first: the tie rays of `posed_hand`, rays through duplicated vertices (dense samples: the duplicates straddle
    the 15th / 16th cut on some), cameras inside the hand's bounding box and cameras exactly at vertices; the rest are 512 x 512
    pixel rays (every (262144 / n)-th pixel) with most samples within a few mm of the hand, a quarter spread from 0 to beyond the
    hand (large jumps along the ray: the seeds fail and the walk falls back to its full scan).  Odd z on a subset of the rays:
    repeated z, z = 0, and non-monotone z inside a walk."""
    g = torch.Generator().manual_seed(seed)
    vc = verts.cpu()
    cams, dirs, zs = [], [], []
    mid, y0, z0 = tie
    for jc in TIE_JC:
        if jc >= S or len(zs) >= n:
            continue
        zc = jc / 16 + 0.25
        cams.append(torch.tensor([mid - zc, y0, z0]))
        dirs.append(torch.tensor([1.0, 0.0, 0.0]))
        zs.append(torch.arange(S, dtype=torch.float32) / 16 + 0.25)     # sample jc at x = mid, jc - 1 at mid - 1/16
    hand = (vc[:, 0] < mid - 1.0)                                        # the vertices not moved into the tie construction
    lo, hi = vc[hand].min(0).values, vc[hand].max(0).values
    for a, _ in DUPS[1:]:                                                # through the triple (7, 100, 650) and the pair (201, 412)
        for _ in range(3):
            d = torch.nn.functional.normalize(torch.randn(3, generator=g), dim=0)
            cams.append(vc[a] - 0.06 * d)
            dirs.append(d)
            zs.append(torch.linspace(0.0, 0.12, S))
    for _ in range(6):                                                   # inside the bounding box
        cams.append(lo + (hi - lo) * torch.rand(3, generator=g))
        dirs.append(torch.nn.functional.normalize(torch.randn(3, generator=g), dim=0))
        zs.append(torch.sort(torch.cat([torch.rand(S - S // 4, generator=g) * 0.3, 1.0 + 2.0 * torch.rand(S // 4, generator=g)]))[0])
    for v in (7, 650, 33, 500):                                          # exactly at a vertex
        cams.append(vc[v].clone())
        dirs.append(torch.nn.functional.normalize(torch.randn(3, generator=g), dim=0))
        z = torch.sort(torch.rand(S, generator=g) * 0.1)[0]
        z[0] = 0.0
        zs.append(z)
    ns = min(len(zs), n)
    cam = torch.stack(cams[:ns]).to(dev)
    dr = torch.stack(dirs[:ns]).to(dev)
    z = torch.stack(zs[:ns]).to(dev)
    npix = n - ns
    if npix > 0:
        pd, pc = pix if pix is not None else pixel_dirs()
        ids = (torch.arange(npix, dtype=torch.float64) * (pd.shape[0] / npix)).long()
        pdir = pd[ids].to(dev)
        pcam = pc.to(dev)[None].expand(npix, 3).contiguous()
        th = nearest_on_ray(pcam, pdir, verts.to(dev)[hand.to(dev)])
        nn_ = S - S // 4
        zn = th[:, None] + 0.004 * torch.randn(npix, nn_, generator=g).to(dev)
        zf = torch.rand(npix, S // 4, generator=g).to(dev) * (th[:, None] + 1.0)
        zp = torch.sort(torch.cat([zn, zf], 1).clamp_min(0.0), 1)[0]
        r = torch.arange(npix, device=dev)
        zp[r % 5 == 0, 0] = 0.0                                          # z = 0
        rep = r % 7 == 1
        if S >= 12:
            zp[rep, 3:11:2] = zp[rep, 2:10:2]                            # exact repeats (the sampler's merge makes these)
        swp = r % 11 == 2
        if S >= 48:
            zp[swp, 40:48] = zp[swp, 40:48].flip(1)                      # non-monotone inside a walk
        a = zp[swp, 3].clone()
        zp[swp, 3] = zp[swp, 4]
        zp[swp, 4] = a
        cam = torch.cat([cam, pcam])
        dr = torch.cat([dr, pdir])
        z = torch.cat([z, zp])
    return cam.float().contiguous(), dr.float().contiguous(), z.float().contiguous(), ns


def ray_points(cam, dirs, z):
    """x = cam + z * dir as two float32 ops (no contraction), as the kernels form them: [n, S, 3]."""
    x = z[..., None] * dirs[:, None, :]
    return cam[:, None, :] + x


# ------------------------------------------------------------------------------------------------ references
def sq_dist(x, v):
    """float32 (dx^2 + dy^2) + dz^2 with every op its own kernel (no contraction): x [P,3], v [V,3] -> [P,V]."""
    s = []
    for c in range(3):
        d = x[:, c:c + 1] - v[None, :, c]
        s.append(d * d)
    return (s[0] + s[1]) + s[2]


def brute_knn(x, v, chunk=65536):
    """float32 brute force in lexicographic (distance, index) order: (d2 [P,15], idx [P,15] int64)."""
    ds, ids = [], []
    for a in range(0, x.shape[0], chunk):
        d, i = torch.sort(sq_dist(x[a:a + chunk], v), dim=1, stable=True)
        ds.append(d[:, :K])
        ids.append(i[:, :K])
    return torch.cat(ds), torch.cat(ids)


def straddles(x, v, chunk=65536):
    """Points whose 15th and 16th neighbours are at exactly the same distance (a tie across the cut)."""
    n = 0
    for a in range(0, x.shape[0], chunk):
        d = torch.sort(sq_dist(x[a:a + chunk], v), dim=1)[0]
        n += int((d[:, K - 1] == d[:, K]).sum())
    return n


def skin_weights(x, idx, v, W, dtype):
    """query_skinning_weights_multi on given neighbours: weights [P,16] and d2 [P,15] in `dtype` from float32 inputs."""
    nb = v[idx].to(dtype)                                     # [P,15,3]
    d2 = ((x.to(dtype)[:, None, :] - nb) ** 2).sum(-1)
    conf = torch.exp(-d2.clamp(max=4.0))
    conf = conf / conf.sum(-1, keepdim=True)
    return (W.to(dtype)[idx] * conf[..., None]).sum(1), d2


def hand_warp_ref(x, idx, v, W, tfs, dtype, forward=False):
    """x [P,3] float32, idx [P,15], v [778,3], tfs [16,4,4] -> x_c (inverse: (T^-1 [x;1])[:3]) or x_d (forward: (T [x;1])[:3] / s)
    with T = sum_j w_j tfs_j, in `dtype`.  float32 is the oracle's einsum + T.inverse()."""
    w, _ = skin_weights(x, idx, v, W, dtype)
    T = torch.einsum("pn,nij->pij", w, tfs.to(dtype))
    xh = torch.nn.functional.pad(x.to(dtype), (0, 1), value=1.0)
    if forward:
        y = torch.einsum("pij,pj->pi", T, xh)
        return y[:, :3] / y[:, 3:]
    return torch.einsum("pij,pj->pi", T.inverse(), xh)[:, :3]


def rigid_ref(x, tf, dtype, forward=False):
    xh = torch.nn.functional.pad(x.to(dtype), (0, 1), value=1.0)
    if forward:
        y = xh @ tf.to(dtype).T
        return y[:, :3] / y[:, 3:]
    return (xh @ torch.linalg.inv(tf.to(dtype)).T)[:, :3]


def worst(a, r):
    """max |a - r| over all entries, relative to the tensor's scale max(1, max |r|)."""
    a, r = a.double(), r.double()
    return ((a - r).abs().max() / r.abs().max().clamp_min(1.0)).item()


def point_grads(T, x, g):
    """Per point, the gradient of g . x_c w.r.t. the rows 0..2 of T and T[3][3] (warp_bwd_phases.h's formulas, float64):
    x_c = M^-1 (x - t / s), q = M^-T g -> G [P,13] (row-major 3x4, then d/ds) and q = dL/dx [P,3]."""
    M, t, s = T[:, :3, :3], T[:, :3, 3], T[:, 3, 3]
    Mi = torch.linalg.inv(M)
    xc = torch.einsum("pij,pj->pi", Mi, x - t / s[:, None])
    q = torch.einsum("pji,pj->pi", Mi, g)
    G = torch.cat([(-q[:, :, None] * xc[:, None, :]), (-q / s[:, None])[..., None]], 2).reshape(-1, 12)
    G = torch.cat([G, ((q * t).sum(1) / (s * s))[:, None]], 1)
    return G, q


def bwd_ref(x, g, tfs, w, dtype):
    """Autograd of sum g . x_c with x_c = (sum_j w_j tfs_j)^-1 [x;1] (weights detached; hand: w [P,16] and tfs [16,4,4], object:
    w None and tfs [4,4]) in `dtype`: (g_tfs, g_x)."""
    tr = tfs.to(dtype).clone().requires_grad_()
    xr = x.to(dtype).clone().requires_grad_()
    T = torch.einsum("pn,nij->pij", w.to(dtype), tr) if w is not None else tr[None].expand(x.shape[0], 4, 4)
    xh = torch.nn.functional.pad(xr, (0, 1), value=1.0)
    xc = torch.einsum("pij,pj->pi", T.inverse(), xh)[:, :3]
    return torch.autograd.grad((xc * g.to(dtype)).sum(), (tr, xr))


def bwd_terms(x, g, tfs, w, magnitude=False):
    """float64 sum over points of |term| of each g_tfs entry (rows 0..2 and [3][3]): hand [16,4,4], object [4,4]; other entries 0.
    magnitude: each term's factors formed from absolute values (|M^-1|, |x| + |t / s|, |g|), the size of what float32 rounds
    inside one term (a single point's term is itself a difference: x - t / s and M^-1 u cancel on and near the vertices)."""
    x, g = x.double(), g.double()
    if w is not None:
        T = torch.einsum("pn,nij->pij", w.double(), tfs.double())
    else:
        T = tfs.double()[None].expand(x.shape[0], 4, 4)
    if magnitude:
        Mi, t, s = torch.linalg.inv(T[:, :3, :3]).abs(), T[:, :3, 3].abs(), T[:, 3, 3].abs()
        qa = torch.einsum("pji,pj->pi", Mi, g.abs())
        xa = torch.einsum("pij,pj->pi", Mi, x.abs() + t / s[:, None])
        Ga = torch.cat([(qa[:, :, None] * xa[:, None, :]), (qa / s[:, None])[..., None]], 2).reshape(-1, 12)
        Ga = torch.cat([Ga, ((qa * t).sum(1) / (s * s))[:, None]], 1)
    else:
        Ga = point_grads(T, x, g)[0].abs()
    out = torch.zeros(*(tfs.shape[:-2]), 16, dtype=torch.float64, device=x.device)
    if w is not None:
        s = torch.einsum("pj,pe->je", w.double().abs(), Ga)            # [16, 13]
        out[:, :12] = s[:, :12]
        out[:, 15] = s[:, 12]
    else:
        s = Ga.sum(0)
        out[:12] = s[:12]
        out[15] = s[12]
    return out.reshape(*(tfs.shape[:-2]), 4, 4)


def worst_entry(a, r, terms):
    """max over the entries of rows 0..2 and [3][3] of |a - r| / sum |terms| (0 where both the error and the terms are 0)."""
    mask = torch.ones(4, 4, dtype=torch.bool)
    mask[3, :3] = False
    e = (a.double() - r.double()).abs()[..., mask]
    t = terms[..., mask]
    return (e / t.clamp_min(1e-300)).max().item()


# ------------------------------------------------------------------------------------------------ CPU tests
def _host_knn():
    import test_cpu_knn

    return test_cpu_knn._lib()


def test_brute_knn_matches_the_oracle_and_lexicographic_order():
    verts, tfs, ties = posed_hand("right", 1, 0)
    v = verts[0]
    g = torch.Generator().manual_seed(0)
    x = v[torch.randint(0, NV, (500,), generator=g)] + 0.03 * torch.randn(500, 3, generator=g)
    d, i = brute_knn(x, v, chunk=128)
    do, io = O.knn_points(x, v, K)
    assert torch.equal(d, do)
    # topk breaks ties arbitrarily: the sets agree where no tie straddles the cut, and the brute force is in (distance, index) order
    d16 = torch.sort(sq_dist(x, v), 1)[0][:, K]
    clean = d16 != d[:, K - 1]
    assert (~clean).any() and clean.float().mean().item() > 0.9
    assert torch.equal(i.sort(1)[0][clean], io.sort(1)[0][clean])
    full = sq_dist(x, v).numpy()
    order = np.lexsort((np.broadcast_to(np.arange(NV), full.shape), full), axis=-1)[:, :K]
    assert np.array_equal(i.numpy(), order)
    # a point on the triple (7, 100, 650): indices in that order at distance 0
    d, i = brute_knn(v[7][None], v)
    assert i[0, :3].tolist() == [7, 100, 650] and (d[0, :3] == 0).all()


def test_warp_references_match_the_oracle():
    W = mano("right")["lbs_weights"]
    verts, tfs, _ = posed_hand("right", 1, 1)
    v, tf = verts[0], tfs[0]
    g = torch.Generator().manual_seed(1)
    x = v[torch.randint(0, NV, (400,), generator=g)] + 0.02 * torch.randn(400, 3, generator=g)
    x[:10] += 4.0                                                        # far: every confidence clamps at d2 = 4
    _, idx = brute_knn(x, v)
    xo, out_o, idx_o = O.hand_inverse_warp(x, v, W, tf)
    wo, _, _ = O.skin_weights_query(x, v, W)
    same = (idx_o == idx).all(1)
    assert same.float().mean().item() > 0.9                              # topk breaks the duplicates' ties its own way
    w32, d2 = skin_weights(x, idx, v, W, torch.float32)
    assert (w32 - wo)[same].abs().max().item() < 1e-6
    x32 = hand_warp_ref(x, idx, v, W, tf, torch.float32)
    x64 = hand_warp_ref(x, idx, v, W, tf, torch.float64)
    assert torch.equal(x32[same], xo[same])                              # the float32 reference is the oracle's arithmetic
    assert worst(x32, x64) < REL_TOL
    assert ((torch.sqrt(d2[:, 0].float().clamp(max=4.0)) > 0.1) == out_o)[same].all() and out_o[:10].all()
    # forward (KNN against the canonical vertices): forward_skinning's (T [x_c;1])[:3], T = sum_j w_j tfs_j
    cano = O.mano_lbs(mano("right"), torch.zeros(1, 10), torch.cat([torch.zeros(1, 3), -mano("right")["hands_mean"][None]], 1))[0][0]
    xc = cano[torch.randint(0, NV, (400,), generator=g)] + 0.02 * torch.randn(400, 3, generator=g)
    _, idx = brute_knn(xc, cano)
    wo, _, idx_o = O.skin_weights_query(xc, cano, W)
    same = (idx_o == idx).all(1)
    assert same.float().mean().item() > 0.9
    xd_o = torch.einsum("pij,pj->pi", torch.einsum("pn,nij->pij", wo, tf), torch.nn.functional.pad(xc, (0, 1), value=1.0))[:, :3]
    xd = hand_warp_ref(xc, idx, cano, W, tf, torch.float64, forward=True)
    assert worst(hand_warp_ref(xc, idx, cano, W, tf, torch.float32, forward=True)[same], xd_o[same]) < 1e-6
    assert worst(xd_o[same], xd[same]) < 1e-5
    # object: both directions
    T = object_tfs(5, 2)
    for b in range(5):
        p = torch.randn(300, 3, generator=g) * 0.5
        r64 = rigid_ref(p, T[b], torch.float64)
        assert worst(O.rigid_inverse_warp(p, T[b]), r64) < REL_TOL
        # the forward's homogeneous divide undoes the full inverse: x = fwd(y[:3] / y[3]), y = T^-1 [x;1]
        y = torch.nn.functional.pad(p.double(), (0, 1), value=1.0) @ torch.linalg.inv(T[b].double()).T
        assert worst(rigid_ref(y[:, :3] / y[:, 3:], T[b], torch.float64, forward=True), p) < 1e-10


def test_backward_references_match_autograd():
    W = mano("left")["lbs_weights"]
    verts, tfs, _ = posed_hand("left", 1, 2)
    v, tf = verts[0], tfs[0]
    g = torch.Generator().manual_seed(2)
    P = 300
    x = v[torch.randint(0, NV, (P,), generator=g)] + 0.05 * torch.randn(P, 3, generator=g)
    _, idx = brute_knn(x, v)
    x, idx = x[(O.knn_points(x, v, K)[1] == idx).all(1)], idx[(O.knn_points(x, v, K)[1] == idx).all(1)]   # same neighbours
    P = x.shape[0]
    assert P > 250
    gx = torch.randn(P, 3, generator=g)
    # the oracle's autograd (test_cpu_warp_bwd.py's construction) on float32
    xr, tr = x.clone().requires_grad_(), tf.clone().requires_grad_()
    w, _, _ = O.skin_weights_query(x, v, W)
    T = torch.einsum("pn,nij->pij", w.detach(), tr)
    xc = torch.einsum("pij,pj->pi", T.inverse(), torch.nn.functional.pad(xr, (0, 1), value=1.0))[:, :3]
    ref_t, ref_x = torch.autograd.grad((xc * gx).sum(), (tr, xr))
    w64, _ = skin_weights(x, idx, v, W, torch.float64)
    g_t, g_x = bwd_ref(x, gx, tf, w64, torch.float64)
    terms = bwd_terms(x, gx, tf, w64)
    assert worst_entry(ref_t, g_t, terms) < 1e-5
    assert worst(ref_x, g_x) < 1e-5
    # the closed form (warp_bwd_phases.h) is the autograd gradient, and sum |term| bounds it
    T64 = torch.einsum("pn,nij->pij", w64, tf.double())
    G, q = point_grads(T64, x.double(), gx.double())
    cf = torch.einsum("pj,pe->je", w64, G)
    mask = torch.ones(4, 4, dtype=torch.bool)
    mask[3, :3] = False
    assert torch.allclose(torch.cat([cf[:, :12], cf[:, 12:]], 1), g_t.reshape(16, 16)[:, mask.flatten()], rtol=1e-10, atol=1e-12)
    assert torch.allclose(q, g_x, rtol=1e-10, atol=1e-12)
    assert (g_t.abs()[:, mask] <= terms[:, mask] * (1 + 1e-12)).all()
    assert (terms[:, mask] <= bwd_terms(x, gx, tf, w64, magnitude=True)[:, mask] * (1 + 1e-12)).all()
    # object, s != 1: d/ds carries the / s^2
    tfo = object_tfs(3, 3)[2]
    assert tfo[3, 3].item() != 1.0
    p = torch.randn(P, 3, generator=g)
    pr, tr = p.clone().requires_grad_(), tfo.clone().requires_grad_()
    ot, ox = torch.autograd.grad((O.rigid_inverse_warp(pr, tr) * gx).sum(), (tr, pr))
    g_t, g_x = bwd_ref(p, gx, tfo, None, torch.float64)
    assert worst_entry(ot, g_t, bwd_terms(p, gx, tfo, None)) < 1e-5 and worst(ox, g_x) < 1e-5
    G, q = point_grads(tfo.double()[None].expand(P, 4, 4), p.double(), gx.double())
    assert abs(G[:, 12].sum().item() - g_t[3, 3].item()) < 1e-9 * max(1.0, abs(g_t[3, 3].item()))


def test_ray_cases_reach_the_walks_branches_on_the_host():
    """The generated rays through knn_phases.h on the host (one walk per ray): exact against the brute force, with full-scan
    fallbacks, straddling duplicate ties, and the constructed tie where the lower-index vertex enters at the 15th place only
    through the tie clause (the previous sample's 15th is the higher-index one)."""
    import ctypes as C

    lib = _host_knn()
    m = mano("right")
    S, n = 40, 64
    verts, tfs, ties = posed_hand("right", 1, 3)
    cano = np.ascontiguousarray(m["v_template"].numpy())
    skin = np.ascontiguousarray(m["lbs_weights"].numpy())
    cam, dirs, z, ns = frame_rays(verts[0], ties[0], n, S, seed=3, pix=pixel_dirs())
    vn = np.ascontiguousarray(verts[0].numpy())
    idx = np.zeros((n, S, K), np.int32)
    dist = np.zeros((n, S, K), np.float32)
    fb, vis = C.c_int(0), C.c_double(0.0)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    cn, dn, zn = (np.ascontiguousarray(t.numpy()) for t in (cam, dirs, z))
    assert lib.knn_cluster_host(C.c_int(n), C.c_int(S), vp(vn), vp(cano), vp(skin), vp(cn), vp(dn), vp(zn), vp(idx), vp(dist),
                                C.byref(fb), C.byref(vis)) == 0
    x = ray_points(cam, dirs, z).reshape(-1, 3)
    d, i = brute_knn(x, verts[0])
    assert np.array_equal(idx.reshape(-1, K), i.numpy())
    assert fb.value > 0, "the cases must force the full-scan fallback"
    assert straddles(ray_points(cam[:ns], dirs[:ns], z[:ns]).reshape(-1, 3), verts[0]) > 0
    u, w, _ = tie_vertices(m["lbs_weights"])
    ii = i.reshape(n, S, K)
    for r, jc in enumerate(TIE_JC[:4]):
        assert w in ii[r, jc - 1].tolist() and u not in ii[r, jc - 1].tolist()
        assert ii[r, jc, K - 1].item() == u and w not in ii[r, jc].tolist()
        assert d.reshape(n, S, K)[r, jc, K - 1].item() == sq_dist(x.reshape(n, S, 3)[r, jc][None], verts[0])[0, w].item()


def test_seg_len_rule():
    assert expected_seg_len(1, 512 * 512, 128, 132) == 32
    assert expected_seg_len(10, 128, 98, 132) == 4
    for L in (32, 16, 8, 4):
        for S in (128, 98, 33):
            for B in (1, 3, 10):
                if L == 4:
                    continue
                assert expected_seg_len(B, rays_for_seg_len(L, B, S, 132), S, 132) == L
