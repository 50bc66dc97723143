"""Canonical mesh extraction (SURVEY §8f rank 4): the reference's `generate_mesh` (utils/meshing.py:9-72) with its two hot
parts on the GPU — the SDF queries (hold_sdf_eval, the fused MLP) and the MISE octree (hold_mise_*, a restatement of
code/src/libmise/mise.pyx that reproduces its dense value grid bit for bit).  Marching cubes: skimage on the host when it is
installed (the reference's own call, Lewiner's variant), otherwise / on request `marching_cubes` below on the GPU (hold_mc_*: a
classic case-table marching cubes with derived tables, watertight, pinned to oracle/marching_cubes.py — not to Lewiner's
triangulation, which this image cannot run)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .capi import check, lib, ptr, stream_ptr


class MISE:
    """`mise.MISE(resolution_0, depth, threshold)` (libmise/mise.pyx:36-88) on the device: query / update / to_dense."""

    def __init__(self, ctx, resolution_0: int, depth: int, threshold: float):
        self.ctx = ctx
        self.resolution_0, self.depth, self.threshold = resolution_0, depth, float(threshold)
        self.resolution = resolution_0 * (1 << depth)
        self._h = C.c_void_p()
        check(lib().hold_mise_create(ctx.h, resolution_0, depth, C.c_float(threshold), C.byref(self._h), stream_ptr()))
        self._dev = torch.device("cuda", ctx.device)

    def query(self) -> torch.Tensor:
        """Lattice coordinates [n,3] (int64, device) of the points to evaluate; n == 0 ends the loop (mise.pyx:113-136)."""
        n = C.c_int(0)
        check(lib().hold_mise_query(self._h, None, 0, C.byref(n), stream_ptr()))
        coords = torch.empty(n.value, 3, dtype=torch.int32, device=self._dev)
        if n.value:
            check(lib().hold_mise_query(self._h, ptr(coords), n.value, C.byref(n), stream_ptr()))
        return coords.long()

    def update(self, points, values: torch.Tensor):
        """Values of the points of the LAST query, in its order (mise.pyx:96-111)."""
        v = values.detach().reshape(-1).float().contiguous()
        check(lib().hold_mise_update(self._h, ptr(v), v.numel(), stream_ptr()))

    def to_dense(self) -> torch.Tensor:
        g = self.resolution + 1
        out = torch.empty(g, g, g, device=self._dev)
        check(lib().hold_mise_to_dense(self._h, ptr(out), stream_ptr()))
        return out

    def close(self):
        if self._h:
            lib().hold_mise_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _dense_grid(ctx, func, verts, level_set, res_init, res_up, scale):
    """The MISE rounds of `generate_grid` -> (value grid float32 [(R+1)^3 as R+1 cubed] on the device, resolution, gt_scale,
    gt_center)."""
    v = np.asarray(verts.detach().cpu() if torch.is_tensor(verts) else verts, dtype=np.float32)
    gt_bbox = np.stack([v.min(axis=0), v.max(axis=0)], axis=0)
    gt_center = (gt_bbox[0] + gt_bbox[1]) * 0.5
    gt_scale = (gt_bbox[1] - gt_bbox[0]).max()
    ex = MISE(ctx, res_init, res_up, level_set)
    dev = torch.device("cuda", ctx.device)
    center = torch.from_numpy(gt_center).to(dev)
    while True:
        coords = ex.query()
        if coords.shape[0] == 0:
            break
        pts = coords.float()                                   # same float32 operation order as meshing.py:24-32
        pts = (pts / ex.resolution - 0.5) * scale
        pts = pts * float(gt_scale) + center
        out = func(pts.contiguous())
        ex.update(coords, out["sdf"] if isinstance(out, dict) else out)
    grid = ex.to_dense()
    res = ex.resolution
    torch.cuda.current_stream().synchronize()              # to_dense reads the octree that close() frees
    ex.close()
    return grid, res, gt_scale, gt_center


def generate_grid(ctx, func, verts, level_set=0.0, res_init=32, res_up=3, scale=1.1):
    """The value grid `generate_mesh` hands to marching cubes (utils/meshing.py:10-47).  `func(points [n,3] cuda float32)`
    returns their SDF ([n] or {"sdf": ...}); `verts` = canonical mesh vertices (numpy / tensor [V,3]) for the bounding box.
    Returns (value_grid float64 numpy [(R+1)^3 as R+1 cubed], resolution, gt_scale, gt_center)."""
    grid, res, gt_scale, gt_center = _dense_grid(ctx, func, verts, level_set, res_init, res_up, scale)
    return grid.cpu().numpy().astype(np.float64), res, gt_scale, gt_center


def node_sdf_func(ctx, node, embed_w=None):
    """`lambda x: query_oc(implicit_network, x, cond)` of hold.py:139-167 for a hold_b200 Node: SDF of canonical points.
    embed_w: the BARF weights [39] of the object's embedder (Node.embed_w()); None = every frequency passes."""
    def f(pts):
        sdf = torch.empty(pts.shape[0], device=pts.device)
        check(lib().hold_sdf_eval(ctx.h, node.slot, pts.shape[0], ptr(pts), ptr(embed_w), ptr(sdf), None, None, stream_ptr()))
        return sdf
    return f


def largest_component(verts, faces):
    """The reference keeps the connected component of largest surface area (utils/meshing.py:58-70: trimesh.split(only_watertight=
    False) + argmax of `area`).  Same selection with scipy's connected components over the face-adjacency-by-shared-vertex graph
    (what trimesh.split uses for only_watertight=False); returns (verts, faces) re-indexed to the kept component."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components

    f = np.asarray(faces, dtype=np.int64)
    nv = int(verts.shape[0])
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]], 0)
    g = sp.coo_matrix((np.ones(e.shape[0], np.int8), (e[:, 0], e[:, 1])), shape=(nv, nv))
    _, label = connected_components(g, directed=False)
    fl = label[f[:, 0]]
    tri = verts[f]
    area = 0.5 * np.linalg.norm(np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), axis=1)
    per = np.bincount(fl, weights=area)
    keep_f = fl == int(np.argmax(per))
    used = np.unique(f[keep_f])
    remap = -np.ones(nv, np.int64)
    remap[used] = np.arange(used.shape[0])
    return verts[used], remap[f[keep_f]]


def largest_component_device(ctx, verts, faces):
    """`largest_component` on the device (hold_largest_component), bit for bit: verts [V,3], faces [F,3] (numpy or torch) ->
    (verts [V',3] float32, faces [F',3] int32) on the context's device.  No face raises ValueError, as np.argmax of no component
    does; a face index outside [0, V) raises HoldError."""
    dev = torch.device("cuda", ctx.device)
    v = torch.as_tensor(verts).to(device=dev, dtype=torch.float32).reshape(-1, 3).contiguous()
    f = torch.as_tensor(faces).to(device=dev, dtype=torch.int32).reshape(-1, 3).contiguous()
    if f.shape[0] == 0:
        raise ValueError("attempt to get argmax of an empty sequence: the mesh has no face")
    v_out, f_out = torch.empty_like(v), torch.empty_like(f)
    nv, nf = C.c_int(0), C.c_int(0)
    check(lib().hold_largest_component(ctx.h, v.shape[0], ptr(v), f.shape[0], ptr(f), ptr(v_out), ptr(f_out), C.byref(nv),
                                       C.byref(nf), stream_ptr()))
    ctx.check()
    return v_out[: nv.value], f_out[: nf.value]


def marching_cubes(ctx, volume: torch.Tensor, level: float = 0.0):
    """(verts [Nv,3] float32 in index coordinates, faces [Nt,3] int32) of the level set of a dense grid on the device (hold_mc_mark /
    hold_mc_emit + two torch.cumsum scans).  Inside = value < level; normals (right-hand rule) towards increasing values."""
    vol = volume.detach().float().contiguous()
    n0, n1, n2 = vol.shape
    dev = vol.device
    flags = torch.empty(n0 * n1 * n2 * 3, dtype=torch.int32, device=dev)
    ntri = torch.zeros((n0 - 1) * (n1 - 1) * (n2 - 1), dtype=torch.int32, device=dev)
    vp = lambda t: C.c_void_p(t.data_ptr())
    check(lib().hold_mc_mark(ctx.h, n0, n1, n2, ptr(vol), float(level), vp(flags), vp(ntri), stream_ptr()))
    vid = torch.cumsum(flags, 0, dtype=torch.int64)
    toff = torch.cumsum(ntri, 0, dtype=torch.int64)
    nv, nt = int(vid[-1]), int(toff[-1])                 # the one host sync: the outputs are sized by these
    vid -= flags
    toff -= ntri
    verts = torch.empty(nv, 3, device=dev)
    faces = torch.empty(nt, 3, dtype=torch.int32, device=dev)
    if nv:
        check(lib().hold_mc_emit(ctx.h, n0, n1, n2, ptr(vol), float(level), vp(flags), vp(vid), vp(toff), ptr(verts), vp(faces), stream_ptr()))
    return verts, faces


def grid_to_world(verts, res, gt_scale, gt_center):
    """Marching-cubes index coordinates [n,3] float32 (device) -> the bounding box of generate_grid (utils/meshing.py:52-53):
    ((v / res - 0.5) * 1.1) * gt_scale + gt_center, in float32 one operation at a time, as numpy rounds it.  res is divided as
    a device tensor: torch multiplies by the reciprocal of a host scalar divisor, which rounds differently."""
    res_t = torch.full((), float(res), device=verts.device)
    center = torch.from_numpy(np.asarray(gt_center, np.float32)).to(verts.device)
    return ((verts / res_t - 0.5) * 1.1) * float(gt_scale) + center


def extract_mesh(ctx, func, verts, level_set=0.0, res_init=32, res_up=3):
    """generate_mesh(backend="gpu") kept on the device: the MISE grid (float32, the values generate_grid's float64 grid holds),
    marching_cubes, grid_to_world and largest_component_device -> (verts [n,3] float32, faces [m,3] int32), device tensors.
    An empty level set raises ValueError, as generate_mesh's np.argmax does."""
    grid, res, gt_scale, gt_center = _dense_grid(ctx, func, verts, level_set, res_init, res_up, 1.1)
    v, f = marching_cubes(ctx, grid, level_set)
    return largest_component_device(ctx, grid_to_world(v, res, gt_scale, gt_center), f)


def generate_mesh(ctx, func, verts, level_set=0.0, res_init=32, res_up=3, keep_largest=True, backend="auto"):
    """utils/meshing.py:9-72 -> (verts [n,3], faces [m,3]) of the largest connected component (keep_largest=False: the raw
    marching-cubes tuple (verts, faces, normals, values)).  backend: "skimage" (the reference's call), "gpu" (hold_mc_*), "auto" =
    skimage when importable, else gpu.  The component selection (trimesh in the reference) is `largest_component` above, and on
    the gpu backend its device equal `largest_component_device`: the gpu result is `extract_mesh`'s, copied to the host."""
    if backend == "auto":
        try:
            import skimage.measure  # noqa: F401  (the reference's own dependency for this step)
            backend = "skimage"
        except ImportError:
            backend = "gpu"
    if backend == "gpu" and keep_largest:
        v, f = extract_mesh(ctx, func, verts, level_set, res_init, res_up)
        return v.cpu().numpy(), f.cpu().numpy().astype(np.int64)
    grid, res, gt_scale, gt_center = generate_grid(ctx, func, verts, level_set, res_init, res_up)
    if backend == "gpu":
        # hold_mc_*: outward normals (towards increasing SDF); normals / values of the skimage tuple are not produced
        dev = torch.device("cuda", ctx.device)
        v, f = marching_cubes(ctx, torch.as_tensor(grid, device=dev), level_set)
        verts_mc = ((v.cpu().numpy() / res - 0.5) * 1.1) * gt_scale + gt_center
        return verts_mc, f.cpu().numpy().astype(np.int64), None, None
    from skimage import measure

    mc = getattr(measure, "marching_cubes_lewiner", None) or measure.marching_cubes
    verts_mc, faces, normals, values = mc(volume=grid, gradient_direction="ascent", level=level_set)
    verts_mc = (verts_mc / res - 0.5) * 1.1
    verts_mc = verts_mc * gt_scale + gt_center
    faces = faces[:, [0, 2, 1]]
    if not keep_largest:
        return verts_mc, faces, normals, values
    return largest_component(verts_mc, faces)


def decimate(ctx, verts, faces, target_faces: int, quality_threshold: float = 0.3):
    """The object mesh brought down to `target_faces` faces by quadric edge collapse (hold_decimate), where the reference's
    load_data calls pymeshlab's meshing_decimation_quadric_edge_collapse.  verts [V,3], faces [F,3] as numpy (generate_mesh's
    output) or torch -> (verts [V',3] float32, faces [F',3] int32) on the context's device.  The result has target_faces or
    target_faces - 1 faces unless the collapse rules stop it earlier; target_faces >= F returns the input unchanged.  Not
    meshlab's result (DESIGN.md §6): the same rules in parallel rounds, bitwise reproducible.  A face index outside [0, V)
    raises HoldError."""
    dev = torch.device("cuda", ctx.device)
    v = torch.as_tensor(verts).to(device=dev, dtype=torch.float32).reshape(-1, 3).contiguous()
    f = torch.as_tensor(faces).to(device=dev, dtype=torch.int32).reshape(-1, 3).contiguous()
    if int(target_faces) >= f.shape[0]:
        return v, f
    v_out, f_out = torch.empty_like(v), torch.empty_like(f)
    nv, nf = C.c_int(0), C.c_int(0)
    check(lib().hold_decimate(ctx.h, v.shape[0], ptr(v), f.shape[0], ptr(f), int(target_faces), C.c_float(quality_threshold),
                              ptr(v_out), ptr(f_out), C.byref(nv), C.byref(nf), stream_ptr()))
    ctx.check()
    return v_out[: nv.value], f_out[: nf.value]
