"""TEST INFRASTRUCTURE (oracle/): signed distance of points to a closed triangle mesh, restating what the reference gets
from kaolin v0.10.0 (not in the reference's tree; parity UNPINNED at that boundary, anchored on the call sites
engine/volsdf_utils.py:172-217): `point_to_mesh_distance` = squared distance to the nearest face, `check_sign` =
inside/outside by ray parity.  Deliberately a different formulation from the kernels' (plane projection + edge
segments instead of Voronoi regions; ray parity instead of the winding number), in float64."""
import numpy as np


def _seg_sqdist(p, a, b):
    ab = b - a
    t = np.clip(((p - a) * ab).sum(-1) / np.maximum((ab * ab).sum(-1), 1e-300), 0.0, 1.0)
    q = a + t[..., None] * ab
    return ((p - q) ** 2).sum(-1)


def point_to_mesh_sqdist(points, verts, faces):
    """points [P,3], verts [V,3], faces [F,3] -> (squared distance [P], nearest face [P]) in float64."""
    p = np.asarray(points, np.float64)[:, None, :]
    v = np.asarray(verts, np.float64)
    a, b, c = v[faces[:, 0]][None], v[faces[:, 1]][None], v[faces[:, 2]][None]
    n = np.cross(b - a, c - a)
    nn = np.maximum((n * n).sum(-1), 1e-300)
    dist_plane = ((p - a) * n).sum(-1)
    proj = p - (dist_plane / nn)[..., None] * n
    # inside test by barycentric signs
    def side(u, w):
        return (np.cross(w - u, proj - u) * n).sum(-1)
    inside = (side(a, b) >= 0) & (side(b, c) >= 0) & (side(c, a) >= 0)
    d_plane = dist_plane**2 / nn
    d_edge = np.minimum(np.minimum(_seg_sqdist(p, a, b), _seg_sqdist(p, b, c)), _seg_sqdist(p, c, a))
    d = np.where(inside, d_plane, d_edge)
    return d.min(1), d.argmin(1)


def check_sign(points, verts, faces, direction=(0.5377, 0.2941, 0.7902)):
    """inside [P] (bool) by ray parity along a generic direction (Moeller-Trumbore), float64."""
    p = np.asarray(points, np.float64)[:, None, :]
    v = np.asarray(verts, np.float64)
    d = np.asarray(direction, np.float64)
    d = d / np.linalg.norm(d)
    a, b, c = v[faces[:, 0]][None], v[faces[:, 1]][None], v[faces[:, 2]][None]
    e1, e2 = b - a, c - a
    h = np.cross(np.broadcast_to(d, e2.shape), e2)
    det = (e1 * h).sum(-1)
    ok = np.abs(det) > 1e-18
    inv = 1.0 / np.where(ok, det, 1.0)
    s = p - a
    u = (s * h).sum(-1) * inv
    q = np.cross(s, e1)
    w = (q * d).sum(-1) * inv
    t = (q * e2).sum(-1) * inv
    hit = ok & (u >= 0) & (w >= 0) & (u + w <= 1) & (t > 0)
    return (hit.sum(1) % 2) == 1


def signed_distance(points, verts, faces):
    """compute_mano_cano_sdf (engine/volsdf_utils.py:172-186): sqrt(kaolin distance) * (1 - 2 * inside)."""
    d, f = point_to_mesh_sqdist(points, verts, faces)
    return np.sqrt(d) * (1.0 - 2.0 * check_sign(points, verts, faces)), f


def star_mesh(level=3, seed=0, amp=0.25):
    """A closed, non-convex test mesh: subdivided octahedron pushed to radius 1 + amp * smooth(direction)."""
    v = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]
    f = [(0, 2, 4), (2, 1, 4), (1, 3, 4), (3, 0, 4), (2, 0, 5), (1, 2, 5), (3, 1, 5), (0, 3, 5)]
    v = [np.array(x, np.float64) for x in v]
    for _ in range(level):
        cache, nf = {}, []

        def mid(i, j):
            k = (min(i, j), max(i, j))
            if k not in cache:
                m = v[i] + v[j]
                v.append(m / np.linalg.norm(m))
                cache[k] = len(v) - 1
            return cache[k]

        for a, b, c in f:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [(a, ab, ca), (ab, b, bc), (ca, bc, c), (ab, bc, ca)]
        f = nf
    v = np.stack(v)
    rng = np.random.default_rng(seed)
    k = rng.normal(size=(4, 3))
    r = 1.0 + amp * np.sin(3.0 * v @ k.T).mean(1)
    return (v * r[:, None]).astype(np.float32), np.asarray(f, np.int32)
