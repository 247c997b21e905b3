"""``MeshGrid`` / ``frnn`` drop-ins (reference: ``models/mesh_grid.py``; third-party ``frnn.frnn_grid_points``).

The spatial index is the library's Morton-ordered octree (``csrc/grid.cu``) instead of FRNN's uniform grid; the
Python surface - constructor arguments, attributes, return shapes / dtypes / ordering - is the reference's.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib


class GridHandle:
    """Owns an ``nmb_grid`` built over a ``[V,3]`` CUDA tensor (what FRNN returns as its opaque ``grid`` tuple)."""

    def __init__(self, vertices: torch.Tensor):
        _lib.require_cuda(vertices, "GridHandle")
        self.vertices = vertices.detach().float().contiguous()
        self.device = self.vertices.device
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().nmb_grid_create(_lib.ptr(self.vertices), self.vertices.shape[0],
                                                  _lib.stream_ptr(self.device), C.byref(h)))
        self.handle = h
        self.num_vertices = int(self.vertices.shape[0])

    def update(self, vertices: torch.Tensor):
        """``nmb_grid_update``: rebuild the octree over moved vertices (same count), reusing the grid's buffers.
        ``self.vertices`` takes the new positions in place; fields and edits packed before must be re-packed."""
        _lib.require_cuda(vertices, "GridHandle.update")
        if tuple(vertices.shape) != (self.num_vertices, 3):
            raise ValueError("GridHandle.update keeps the vertex count: expected [%d, 3], got %s"
                             % (self.num_vertices, tuple(vertices.shape)))
        if vertices.data_ptr() != self.vertices.data_ptr():
            self.vertices.copy_(vertices.detach())
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().nmb_grid_update(self.handle, _lib.ptr(self.vertices), self.num_vertices,
                                                  _lib.stream_ptr(self.device)))

    @property
    def generation(self) -> int:
        """Number of ``update`` calls so far (``nmb_grid_generation``): part of the packed fields' cache keys."""
        return int(_lib.lib().nmb_grid_generation(self.handle))

    def __del__(self):
        h, self.handle = getattr(self, "handle", None), None
        if h:
            try:
                _lib.lib().nmb_grid_destroy(h)
            except Exception:
                pass

    def knn(self, xyz: torch.Tensor, K: int, r: float = 100.0):
        """xyz [M,3] -> (d2 [M,K] ascending squared distances, idx [M,K] int64 original order)."""
        xyz = xyz.detach().float().contiguous()
        M = xyz.shape[0]
        d2 = torch.empty(M, K, dtype=torch.float32, device=self.device)
        idx = torch.empty(M, K, dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().nmb_knn(self.handle, _lib.ptr(xyz), M, K, float(r), _lib.ptr(d2), _lib.ptr(idx),
                                          _lib.stream_ptr(self.device)))
        return d2, idx

    def mesh_distance(self, xyz: torch.Tensor, indicator: torch.Tensor, w1: float, want_grad: bool = False):
        xyz = xyz.detach().float().contiguous()
        indicator = indicator.detach().float().contiguous()
        M = xyz.shape[0]
        ds = torch.empty(M, 1, dtype=torch.float32, device=self.device)
        idx = torch.empty(M, 8, dtype=torch.int64, device=self.device)
        w = torch.empty(M, 8, dtype=torch.float32, device=self.device)
        g = torch.empty(M, 3, dtype=torch.float32, device=self.device) if want_grad else None
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().nmb_mesh_distance(self.handle, _lib.ptr(indicator), float(w1), _lib.ptr(xyz), M,
                                                    _lib.ptr(ds), _lib.ptr(idx), _lib.ptr(w), _lib.ptr(g),
                                                    _lib.stream_ptr(self.device)))
        return (ds, idx, w, g) if want_grad else (ds, idx, w)


def frnn_grid_points(points1, points2, lengths1=None, lengths2=None, K=8, r=100.0, grid=None, return_nn=False,
                     return_sorted=True, radius_cell_ratio=2.0):
    """Drop-in for ``frnn.frnn_grid_points`` as called at ``models/mesh_grid.py:64-74,109-119`` (batch size 1):
    returns ``(dists [1,M,K] squared & ascending, idxs [1,M,K] int64, None, grid)``."""
    if points1.dim() != 3 or points1.shape[0] != 1 or points2.dim() != 3 or points2.shape[0] != 1:
        raise NotImplementedError("neumesh_b200.frnn_grid_points supports batch size 1 (all the reference uses)")
    if return_nn:
        raise NotImplementedError("return_nn=True is not used by the reference and not provided")
    if not isinstance(grid, GridHandle) or grid.vertices.data_ptr() != points2[0].detach().float().contiguous().data_ptr():
        if not isinstance(grid, GridHandle) or grid.num_vertices != points2.shape[1] \
                or not torch.equal(grid.vertices, points2[0].detach().float()):
            grid = GridHandle(points2[0])
    d2, idx = grid.knn(points1[0], int(K), float(r))
    return d2[None], idx[None], None, grid


class MeshPrimitive:
    """reference ``models/mesh_grid.py:8-42`` minus the Embree ray-caster (``cast_ray`` is a CPU utility of the
    painting tool, out of scope - SURVEY.md section 2 row 3)."""

    def __init__(self, mesh):
        self.mesh = mesh
        if hasattr(mesh, "compute_vertex_normals"):
            mesh.compute_vertex_normals()

    def cast_ray(self, rays_o, rays_d):
        raise NotImplementedError("cast_ray (Open3D/Embree, painting tool only) is outside the rendering hot path")

    def get_number_of_vertices(self):
        return len(self.mesh.vertices)


class MeshGrid(MeshPrimitive):
    def __init__(self, mesh, device, distance_method="frnn"):
        """``mesh``: anything with ``vertices`` / ``vertex_normals`` array-likes (an Open3D ``TriangleMesh`` or
        ``neumesh_b200.synth.SynthMesh``).  reference: ``models/mesh_grid.py:46-75``."""
        super().__init__(mesh)
        if isinstance(device, int):
            device = torch.device("cuda", device)
        self.vertices = torch.as_tensor(np.asarray(mesh.vertices), dtype=torch.float32).to(device)
        self.vertex_normals = torch.as_tensor(np.asarray(mesh.vertex_normals), dtype=torch.float32).to(device)
        self.grid = GridHandle(self.vertices)  # replaces the V x V K=32 FRNN self-query
        self.distance_method = distance_method

    def compute_distance(self, xyz, indicator_vector=None, indicator_weight=0.1, K=8):
        if self.distance_method == "frnn":
            return self.compute_distance_frnn(xyz, K, indicator_vector=indicator_vector,
                                              indicator_weight=indicator_weight)
        raise NotImplementedError

    def compute_distance_frnn(self, xyz, K=8, indicator_vector=None, indicator_weight=0.1):
        """xyz [N,3] -> (distance [N,1], indices [N,K] int64, weights [N,K]); reference ``mesh_grid.py:88-144``.

        No grad needed and K == 8: one fused CUDA kernel.  Otherwise the neighbour search runs in CUDA and the
        (differentiable) blend is expressed in torch ops exactly as the reference does, so gradients w.r.t. ``xyz``,
        ``indicator_vector`` and ``indicator_weight`` flow (indices / weights are detached, ``mesh_grid.py:121-122``).
        """
        ind = self.vertex_normals if indicator_vector is None else indicator_vector
        w1 = indicator_weight
        needs_grad = torch.is_grad_enabled() and (
            xyz.requires_grad or ind.requires_grad or (torch.is_tensor(w1) and w1.requires_grad))
        if not needs_grad and K == 8:
            return self.grid.mesh_distance(xyz, ind, float(w1))
        d2, idx = self.grid.knn(xyz, K)
        dist = d2.sqrt()
        w = 1.0 / (dist + 1e-7)
        w = w / w.sum(dim=-1, keepdim=True)
        v = xyz.unsqueeze(-2) - self.vertices[idx]
        rho = torch.norm(v, dim=-1, keepdim=True)
        mid = (ind[idx] * w1 + v * rho) / (w1 + rho)
        ds = (w.unsqueeze(-1) * (v * mid).sum(dim=-1, keepdim=True)).sum(dim=-2)
        return ds, idx, w

    def deform_(self, vertices, normals=None):
        """Move the mesh's vertices in place: ``vertices`` is a CUDA ``[V,3]`` tensor with the grid's vertex count.
        ``self.vertices`` is overwritten, the octree rebuilt in its buffers (``nmb_grid_update``), and
        ``vertex_normals`` becomes ``normals`` or, without them, the area-weighted normals of the moved mesh
        (``nmb_vertex_normals`` over ``mesh.triangles``, uploaded on the first call).  The previous ``vertex_normals``
        tensor is replaced, not overwritten, so a caller holding it keeps the old normals."""
        from .renderer import vertex_normals
        _lib.require_cuda(vertices, "MeshGrid.deform_")
        self.grid.update(vertices)   # checks the shape, copies into self.vertices (the grid's own tensor)
        if normals is None:
            if getattr(self, "_triangles", None) is None:
                tri = getattr(self.mesh, "triangles", None)
                if tri is None:
                    raise ValueError("MeshGrid.deform_ without normals needs mesh.triangles to compute them")
                self._triangles = torch.as_tensor(np.asarray(tri), dtype=torch.int32).to(self.vertices.device)
            normals = vertex_normals(self.vertices, self._triangles)
        elif tuple(normals.shape) != tuple(self.vertices.shape):
            raise ValueError("normals must be [V,3] like the vertices, got %s" % (tuple(normals.shape),))
        self.vertex_normals = normals.detach().to(self.vertices.device, torch.float32).contiguous()

    def get_vertex_normal_torch(self):
        return self.vertex_normals

    def get_vertices_torch(self):
        return self.vertices
