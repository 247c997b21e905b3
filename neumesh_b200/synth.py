"""Synthetic inputs for the NeuMesh hot path (no dataset / checkpoint is reachable offline).

Everything here is deterministic given its seed and is shared by the tests, ``bench.py`` and
``__graft_entry__.smoke()`` so the CUDA path, the oracle and the reference see identical inputs.

* ``icosphere_mesh``  - displaced, subdivided icosahedron (SURVEY.md section 8d "scan63-like" mesh) with
  area-weighted vertex normals (what Open3D's ``compute_vertex_normals`` produces for the reference at
  ``models/mesh_grid.py:20``).
* ``make_state_dict`` - a NeuMesh ``state_dict`` with the reference's key set
  (``models/frameworks/neumesh/neumesh.py:43-102``) whose geometry MLP is *trained-like*:
  ``sdf ~= ds + small smooth residual`` (SURVEY.md section 4: random-init weights make the render chaotic and
  a 1e-4 / 1e-5 parity bar meaningless).
* ``spiral_poses`` / ``pinhole_rays`` - camera track and ray generation in the conventions of
  ``render.py:56-96`` and ``utils/rend_util.py:123-176``.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch


# ----------------------------------------------------------------------------------------------------------------
# mesh
# ----------------------------------------------------------------------------------------------------------------
@dataclass
class SynthMesh:
    """Minimal stand-in for the ``open3d.geometry.TriangleMesh`` the reference passes to ``MeshGrid``."""

    vertices: np.ndarray  # [V,3] float64 (Open3D stores doubles)
    triangles: np.ndarray  # [T,3] int32
    vertex_normals: np.ndarray  # [V,3] float64

    def compute_vertex_normals(self):
        self.vertex_normals = area_weighted_normals(self.vertices, self.triangles)
        return self


def area_weighted_normals(vertices: np.ndarray, triangles: np.ndarray) -> np.ndarray:
    """Sum of un-normalised face normals (cross products, i.e. weighted by twice the face area) per vertex,
    then normalised - the scheme Open3D uses."""
    v = vertices.astype(np.float64)
    a, b, c = v[triangles[:, 0]], v[triangles[:, 1]], v[triangles[:, 2]]
    fn = np.cross(b - a, c - a)
    vn = np.zeros_like(v)
    for k in range(3):
        np.add.at(vn, triangles[:, k], fn)
    nrm = np.linalg.norm(vn, axis=1, keepdims=True)
    nrm[nrm == 0] = 1.0
    return vn / nrm


def _icosahedron():
    t = (1.0 + math.sqrt(5.0)) / 2.0
    v = np.array(
        [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
         [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], dtype=np.float64)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    f = np.array(
        [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
         [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5],
         [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]], dtype=np.int64)
    return v, f


def _subdivide(v: np.ndarray, f: np.ndarray):
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]], axis=0)
    e_sorted = np.sort(e, axis=1)
    key = e_sorted[:, 0] * (v.shape[0] + 1) + e_sorted[:, 1]
    uniq, inv = np.unique(key, return_inverse=True)
    first = np.zeros(uniq.shape[0], dtype=np.int64)
    first[inv] = np.arange(e.shape[0])
    mid = v[e_sorted[first, 0]] + v[e_sorted[first, 1]]
    mid /= np.linalg.norm(mid, axis=1, keepdims=True)
    nv = v.shape[0]
    m = inv + nv
    T = f.shape[0]
    m01, m12, m20 = m[:T], m[T:2 * T], m[2 * T:]
    f_new = np.concatenate(
        [np.stack([f[:, 0], m01, m20], 1), np.stack([f[:, 1], m12, m01], 1),
         np.stack([f[:, 2], m20, m12], 1), np.stack([m01, m12, m20], 1)], axis=0)
    return np.concatenate([v, mid], axis=0), f_new


def icosphere_mesh(level: int = 5, radius: float = 0.5, bump: float = 0.05, seed: int = 0,
                   jitter: float = 0.15) -> SynthMesh:
    """V = 10*4**level + 2 vertices on a radially displaced sphere: r = radius + bump * smooth(dir).

    ``jitter`` (fraction of the mean edge length) moves vertices tangentially so that no two query-vertex
    distances tie exactly (tie order among equidistant vertices is implementation-defined, SURVEY.md section 4).
    """
    v, f = _icosahedron()
    for _ in range(level):
        v, f = _subdivide(v, f)
    rng = np.random.default_rng(seed)
    freqs = rng.normal(size=(6, 3)) * 2.5
    phase = rng.uniform(0, 2 * np.pi, size=(6,))
    amp = rng.uniform(0.4, 1.0, size=(6,))
    s = (np.sin(v @ freqs.T + phase) * amp).sum(1) / amp.sum()
    if jitter > 0:
        edge = math.sqrt(4 * math.pi / max(f.shape[0], 1) * 4 / math.sqrt(3)) * 0.5
        t = rng.normal(size=v.shape) * (jitter * edge)
        v = v + t
        v /= np.linalg.norm(v, axis=1, keepdims=True)
    p = v * (radius + bump * s)[:, None]
    # round through fp32 so that every consumer (which stores fp32) sees identical coordinates
    p = p.astype(np.float32).astype(np.float64)
    mesh = SynthMesh(vertices=p, triangles=f.astype(np.int32), vertex_normals=np.zeros_like(p))
    return mesh.compute_vertex_normals()


# Meshes unlike the icosphere, for the tests of everything whose correctness depends on the mesh's shape (the exact
# octree walks, the shell certificate, the bounded near / far scan).  Scans and edited meshes are open, non-convex,
# unevenly dense, and may carry duplicate or exactly coplanar vertices; each generator below stresses one of these.
def _finish(p: np.ndarray, f: np.ndarray) -> SynthMesh:
    p = np.ascontiguousarray(p).astype(np.float32).astype(np.float64)
    mesh = SynthMesh(vertices=p, triangles=np.ascontiguousarray(f).astype(np.int32), vertex_normals=np.zeros_like(p))
    return mesh.compute_vertex_normals()


def _rotation(rng) -> np.ndarray:
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))[None, :]
    if np.linalg.det(q) < 0:
        q[:, 0] = -q[:, 0]
    return q


def _drop_vertices(v: np.ndarray, f: np.ndarray, keep: np.ndarray):
    """Keep the faces whose three vertices are kept, then drop the vertices no face references."""
    f = f[keep[f].all(axis=1)]
    used = np.zeros(v.shape[0], dtype=bool)
    used[f.reshape(-1)] = True
    new_id = np.cumsum(used) - 1
    return v[used], new_id[f]


def _grid_faces(nu: int, nv: int, wrap_u: bool, wrap_v: bool) -> np.ndarray:
    """Two triangles per quad of an nu x nv vertex grid (vertex (i, j) at i * nv + j)."""
    iu = np.arange(nu if wrap_u else nu - 1)
    jv = np.arange(nv if wrap_v else nv - 1)
    i, j = np.meshgrid(iu, jv, indexing="ij")
    i, j = i.reshape(-1), j.reshape(-1)
    i1, j1 = (i + 1) % nu, (j + 1) % nv
    a, b, c, d = i * nv + j, i1 * nv + j, i1 * nv + j1, i * nv + j1
    return np.concatenate([np.stack([a, b, c], 1), np.stack([a, c, d], 1)], axis=0)


def open_bowl(level: int = 6, radius: float = 0.45, seed: int = 0, cap: float = 0.55,
              centre=(0.12, -0.08, 0.05)) -> SynthMesh:
    """A jittered icosphere with the cap dir_z < -cap cut off: an open boundary, off-centre, with its concave inside
    facing the spiral track's centre camera (which looks down +z from z = -2.5)."""
    m = icosphere_mesh(level, radius=1.0, bump=0.0, seed=seed)
    v = m.vertices / np.linalg.norm(m.vertices, axis=1, keepdims=True)
    v, f = _drop_vertices(v, m.triangles.astype(np.int64), v[:, 2] >= -cap)
    return _finish(v * radius + np.asarray(centre, dtype=np.float64), f)


def torus(R: float = 0.55, r: float = 0.15, nu: int = 256, nv: int = 64, seed: int = 0) -> SynthMesh:
    """A tilted, jittered torus: not star-shaped, rays pass through the hole, some rays cross it twice."""
    rng = np.random.default_rng(seed)
    u = (np.arange(nu)[:, None] + 0.3 * rng.uniform(-1, 1, size=(nu, nv))) * (2 * np.pi / nu)
    w = (np.arange(nv)[None, :] + 0.3 * rng.uniform(-1, 1, size=(nu, nv))) * (2 * np.pi / nv)
    p = np.stack([(R + r * np.cos(w)) * np.cos(u), (R + r * np.cos(w)) * np.sin(u), r * np.sin(w)], -1).reshape(-1, 3)
    return _finish(p @ _rotation(rng).T, _grid_faces(nu, nv, True, True))


def double_sheet(radius: float = 0.6, spacing: float = 0.01, gap: float = 0.03, seed: int = 0) -> SynthMesh:
    """Two jittered, tilted disks `gap` apart with opposite normals, each inside the other's 0.1 shell: a query between
    them has neighbours on both sheets, whose indicator vectors point in opposite directions."""
    rng = np.random.default_rng(seed)
    n = int(round(2 * radius / spacing)) + 1
    x = np.linspace(-radius, radius, n)
    gx, gy = np.meshgrid(x, x, indexing="ij")
    base = np.stack([gx.reshape(-1), gy.reshape(-1)], -1)
    f0 = _grid_faces(n, n, False, False)
    keep = (base ** 2).sum(1) <= radius * radius
    vs, fs = [], []
    for k, (z, flip) in enumerate(((0.5 * gap, False), (-0.5 * gap, True))):
        xy = base + rng.uniform(-0.3, 0.3, size=base.shape) * spacing
        p = np.concatenate([xy, np.full((xy.shape[0], 1), z)], 1)
        p, f = _drop_vertices(p, f0, keep)
        if flip:
            f = f[:, ::-1]
        fs.append(f + sum(q.shape[0] for q in vs))
        vs.append(p)
    return _finish(np.concatenate(vs) @ _rotation(rng).T, np.concatenate(fs))


def lattice_plane(n: int = 257, spacing: float = 1.0 / 256) -> SynthMesh:
    """An n x n grid at z = 0 with a power-of-two spacing: every coordinate is exact in fp32, so squared distances tie
    exactly everywhere (2-, 4- and 8-way ties at cell centres and edge midpoints) and every node has a zero-thickness
    disc."""
    x = (np.arange(n) - (n - 1) // 2) * spacing
    gx, gy = np.meshgrid(x, x, indexing="ij")
    p = np.stack([gx.reshape(-1), gy.reshape(-1), np.zeros(n * n)], -1)
    return _finish(p, _grid_faces(n, n, False, False))


def clustered(seed: int = 0, n_dup: int = 200) -> SynthMesh:
    """A coarse sphere (level 3, radius 0.5), a dense level-6 icosphere of radius 0.02 sitting on its surface, and
    `n_dup` exact copies of one of the dense vertices (unreferenced by any face).  The cluster packs ~100 vertices into
    each finest octree cell, so the deepest leaves hold far more than LEAF_MAX points."""
    coarse = icosphere_mesh(3, radius=0.5, bump=0.02, seed=seed)
    dense = icosphere_mesh(6, radius=0.02, bump=0.0, seed=seed + 1)
    c = coarse.vertices[7]
    v = np.concatenate([coarse.vertices, dense.vertices + c])
    f = np.concatenate([coarse.triangles, dense.triangles + coarse.vertices.shape[0]])
    dup = np.repeat(v[coarse.vertices.shape[0] + 5][None], n_dup, axis=0)
    return _finish(np.concatenate([v, dup]), f)


def fan_mesh(V: int, seed: int = 0) -> SynthMesh:
    """A tiny triangle fan: one apex and V - 1 rim vertices at seeded radii and heights."""
    rng = np.random.default_rng(seed)
    a = np.sort(rng.uniform(0, 2 * np.pi, size=V - 1))
    rr = rng.uniform(0.3, 0.8, size=V - 1)
    rim = np.stack([rr * np.cos(a), rr * np.sin(a), rng.uniform(-0.3, 0.3, size=V - 1)], -1)
    p = np.concatenate([np.array([[0.0, 0.0, 0.2]]), rim])
    i = np.arange(1, V)
    f = np.stack([np.zeros(V - 1, dtype=np.int64), i, np.where(i + 1 < V, i + 1, 1)], 1)
    return _finish(p, f)


FAR_BOWL_OFFSET = (100.0, -37.5, 12.25)
FAR_BOWL_SCALE = 1.0 / 64


def far_bowl(seed: int = 0) -> SynthMesh:
    """``open_bowl`` scaled by 1/64 and moved to about (100, -37.5, 12.25): the fp32 margins of the walk's bounds at
    coordinates whose ulp is ~1000 times coarser than at the unit scale, relative to the mesh."""
    m = open_bowl(seed=seed)
    return _finish(m.vertices * FAR_BOWL_SCALE + np.asarray(FAR_BOWL_OFFSET), m.triangles)


# ----------------------------------------------------------------------------------------------------------------
# model parameters
# ----------------------------------------------------------------------------------------------------------------
@dataclass
class ModelConfig:
    """Defaults = configs/neumesh_dtu_scan63.yaml:15-30 + models/frameworks/neumesh/__init__.py:19-45."""

    D_density: int = 3
    D_color: int = 4
    W: int = 256
    geometry_dim: int = 32
    color_dim: int = 32
    multires_view: int = 4
    multires_d: int = 8
    multires_fg: int = 2
    multires_ft: int = 2
    enable_nablas_input: bool = True
    ln_s: float = 0.55
    speed_factor: float = 10.0
    learn_indicator_weight: bool = False

    @property
    def ch_d(self):
        return 1 + 2 * self.multires_d

    @property
    def ch_view(self):
        return 3 * (1 + 2 * self.multires_view)

    @property
    def ch_fg(self):
        return self.geometry_dim * (1 + 2 * self.multires_fg)

    @property
    def ch_ft(self):
        return self.color_dim * (1 + 2 * self.multires_ft)

    @property
    def in_geo(self):
        return self.ch_d + self.ch_fg

    @property
    def in_color(self):
        return self.ch_d + self.ch_view + self.ch_ft + (3 if self.enable_nablas_input else 0)

    def model_kwargs(self):
        return dict(D_density=self.D_density, D_color=self.D_color, W=self.W, geometry_dim=self.geometry_dim,
                    color_dim=self.color_dim, multires_view=self.multires_view, multires_d=self.multires_d,
                    multires_fg=self.multires_fg, multires_ft=self.multires_ft,
                    enable_nablas_input=self.enable_nablas_input, ln_s=self.ln_s, speed_factor=self.speed_factor,
                    learn_indicator_weight=self.learn_indicator_weight)


def make_state_dict(mesh: SynthMesh, cfg: ModelConfig = ModelConfig(), seed: int = 1, residual: float = 0.02,
                    trained_like: bool = True) -> "dict[str, torch.Tensor]":
    """NeuMesh ``state_dict`` (reference key set, SURVEY.md section 5 'Checkpoint / resume').

    Geometry MLP (weight-norm ``g``/``v`` parametrisation, ``W_eff = g * v / ||v||_row``): hidden unit 0 carries
    ``ds + 1`` through every Softplus(beta=100) layer in its linear regime, the other units carry a smooth
    low-amplitude function of the embedding; the last layer returns ``unit0 - 1 + residual * mix(others)``.
    """
    g = torch.Generator().manual_seed(seed)
    V = mesh.vertices.shape[0]
    W = cfg.W

    def randn(*shape, scale=1.0):
        return torch.randn(*shape, generator=g, dtype=torch.float32) * scale

    sd: "dict[str, torch.Tensor]" = {}
    sd["ln_s"] = torch.tensor([cfg.ln_s], dtype=torch.float32)
    sd["geometry_features"] = randn(V, cfg.geometry_dim)
    sd["color_features"] = randn(V, cfg.color_dim)
    nrm = torch.from_numpy(mesh.vertex_normals).float()
    sd["indicator_vector"] = nrm + randn(V, 3, scale=0.05)
    if cfg.learn_indicator_weight:
        sd["indicator_weight_raw"] = torch.tensor([-2.0], dtype=torch.float32)

    def put_wn(prefix, weight, bias):
        nv = weight.norm(dim=1, keepdim=True)
        scale = 0.5 + torch.rand(weight.shape[0], 1, generator=g)  # v is NOT unit-norm: exercises g*v/||v||
        sd[prefix + ".weight_g"] = nv.clone()
        sd[prefix + ".weight_v"] = weight * scale
        sd[prefix + ".bias"] = bias

    # ---- geometry MLP -------------------------------------------------------------------------------------
    names = ["pts_linears.0"] + [f"pts_linears.{i}.0" for i in range(2, cfg.D_density + 1)]
    fan_in = cfg.in_geo
    for li, name in enumerate(names):
        if trained_like:
            w = randn(W, fan_in, scale=0.6 / math.sqrt(fan_in))
            b = 0.3 + 0.2 * torch.rand(W, generator=g)
            w[0].zero_()
            if li == 0:
                w[:, 0] *= 0.25  # keep the residual a gentle function of ds itself
                w[0, 0] = 1.0  # unit 0 <- ds (first channel of PE_8(ds))
            else:
                w[:, 0] = 0.0  # unit 0 does not leak into the residual units ...
                w[0, 0] = 1.0  # ... and is carried through unchanged
            b[0] = 1.0 if li == 0 else 0.0
        else:
            bound = 1.0 / math.sqrt(fan_in)
            w = (torch.rand(W, fan_in, generator=g) * 2 - 1) * bound
            b = (torch.rand(W, generator=g) * 2 - 1) * bound
        put_wn(name, w, b)
        fan_in = W
    if trained_like:
        w = randn(1, W, scale=residual / math.sqrt(W))
        w[0, 0] = 1.0
        b = torch.tensor([-1.0]) - residual * 0.0
        # remove the mean contribution of the residual units (each sits near softplus(~0.4) ~ 0.4)
        b = b - 0.4 * w[0, 1:].sum()
    else:
        bound = 1.0 / math.sqrt(W)
        w = (torch.rand(1, W, generator=g) * 2 - 1) * bound
        b = (torch.rand(1, generator=g) * 2 - 1) * bound
    put_wn("density_linear", w, b)

    # ---- colour MLP (plain Linear, default-init-like) -----------------------------------------------------
    names = ["views_linears.0"] + [f"views_linears.{i}.0" for i in range(2, cfg.D_color + 1)]
    fan_in = cfg.in_color
    for name in names:
        bound = 1.0 / math.sqrt(fan_in)
        sd[name + ".weight"] = (torch.rand(W, fan_in, generator=g) * 2 - 1) * bound
        sd[name + ".bias"] = (torch.rand(W, generator=g) * 2 - 1) * bound
        fan_in = W
    bound = 1.0 / math.sqrt(W)
    sd["color_linear.0.weight"] = (torch.rand(3, W, generator=g) * 2 - 1) * bound * 4.0
    sd["color_linear.0.bias"] = (torch.rand(3, generator=g) * 2 - 1) * bound
    return sd


# ----------------------------------------------------------------------------------------------------------------
# cameras / rays
# ----------------------------------------------------------------------------------------------------------------
def _normalize(v):
    return v / np.linalg.norm(v)


def look_at(cam_location, point, up=np.array([0.0, -1.0, 0.0])):
    """OpenCV-convention camera-to-world (camera looks down +z), as ``render.py:38-53``."""
    fwd = _normalize(point - cam_location)
    right = _normalize(np.cross(fwd, up))
    true_up = _normalize(np.cross(right, fwd))
    # columns: x = right, y = down (= -true_up ... the reference builds [-left, up, fwd]); keep a proper rotation
    x = np.cross(true_up, fwd)
    x = _normalize(x)
    y = np.cross(fwd, x)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = x, y, fwd, cam_location
    return c2w


def spiral_poses(n_views: int = 90, radius: float = 2.5, spiral_rad: float = 1.2, zrate: float = 0.5,
                 rots: int = 2, up=np.array([0.0, -1.0, 0.0])):
    """Spiral track around a centre pose that looks at the origin from distance ``radius``
    (``render.py:56-96``: positions ``c2w @ ([cos t, sin t, sin(t*zrate), 1] * rads)``, every pose looks at the
    focus point)."""
    centre = look_at(np.array([0.0, 0.0, -radius]), np.zeros(3), up)
    rads = np.array([spiral_rad, spiral_rad, spiral_rad * 0.1, 1.0])
    focus_world = centre[:3, :4] @ np.array([0.0, 0.0, radius, 1.0])
    poses = []
    for theta in np.linspace(0.0, 2.0 * np.pi * rots, n_views + 1)[:-1]:
        loc = centre[:3, :4] @ (np.array([math.cos(theta), math.sin(theta), math.sin(theta * zrate), 1.0]) * rads)
        poses.append(look_at(loc, focus_world, up))
    return poses


def pinhole_rays(c2w: np.ndarray, H: int, W: int, fx: float, fy: float, cx: float, cy: float):
    """All H*W rays of one view, row-major pixels, unit directions - the no-skew case of
    ``utils/rend_util.py:97-176`` (lift pixel (i,j,1) through K^-1, normalise, rotate by c2w)."""
    j, i = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing="ij")
    x = (i.reshape(-1) - np.float32(cx)) / np.float32(fx)
    y = (j.reshape(-1) - np.float32(cy)) / np.float32(fy)
    d = np.stack([x, y, np.ones_like(x)], -1).astype(np.float32)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    R = c2w[:3, :3].astype(np.float32)
    rays_d = d @ R.T
    rays_o = np.broadcast_to(c2w[:3, 3].astype(np.float32), rays_d.shape).copy()
    return torch.from_numpy(rays_o), torch.from_numpy(np.ascontiguousarray(rays_d))


def frame_rays(H: int = 800, W: int = 800, view: int = 0, n_views: int = 90, focal: float | None = None,
               radius: float = 2.5):
    """Rays of one spiral frame. Default intrinsics follow NeRF-synthetic (800x800, focal 1111.1) scaled to HxW."""
    if focal is None:
        focal = 1111.1 * W / 800.0
    pose = spiral_poses(n_views=n_views, radius=radius)[view % n_views]
    return pinhole_rays(pose, H, W, focal, focal, W / 2.0, H / 2.0)
