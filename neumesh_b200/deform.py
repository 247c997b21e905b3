"""Geometry editing: ``deform_model`` (reference ``editing/render_geometry_editing.py:37-67``) on the device.

The reference moves a NeuMesh model's mesh and keeps its codes: it builds a new ``MeshGrid`` from the deformed Open3D
mesh (normals on the CPU), rotates every vertex's indicator vector by the rotation between its old and new normal (kornia)
and swaps both in.  Here the same call also takes the deformed vertices as a CUDA tensor; the model's grid is then
rebuilt in place (``MeshGrid.deform_`` -> ``nmb_grid_update``), its normals come from ``nmb_vertex_normals`` and the
rotation from ``nmb_indicator_rotate``, so an animated or dragged mesh stays on the device from vertex positions to
pixels.  The next fused call re-packs the field (``nmb_field_update``: the grid's generation is in its cache key).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _lib
from .mesh_grid import MeshGrid


def indicator_rotate(n_old: torch.Tensor, n_new: torch.Tensor, indicator: torch.Tensor) -> torch.Tensor:
    """``nmb_indicator_rotate``: the reference's rotation of ``indicator`` [V,3] by the rotation taking ``n_old`` to
    ``n_new`` (formula and its quirks: ``oracle/deform.py``).  CUDA tensors; returns a new [V,3] fp32 tensor."""
    for t in (n_old, n_new, indicator):
        _lib.require_cuda(t, "indicator_rotate")
    a = n_old.detach().float().contiguous()
    b = n_new.detach().float().contiguous()
    v = indicator.detach().float().contiguous()
    if not (a.shape == b.shape == v.shape and a.dim() == 2 and a.shape[1] == 3):
        raise ValueError("indicator_rotate: n_old, n_new and indicator must all be [V,3], got %s, %s, %s"
                         % (tuple(a.shape), tuple(b.shape), tuple(v.shape)))
    out = torch.empty_like(v)
    with torch.cuda.device(v.device):
        _lib.check(_lib.lib().nmb_indicator_rotate(_lib.ptr(a), _lib.ptr(b), _lib.ptr(v), v.shape[0], _lib.ptr(out),
                                                   _lib.stream_ptr(v.device)))
    return out


def deform_model(deformed_mesh, model, device, fix_indicator=False):
    """Reference ``deform_model(deformed_mesh, model, device, fix_indicator=False)``.

    ``deformed_mesh``: an Open3D-like mesh (``vertices`` / ``vertex_normals``; a new ``MeshGrid`` is built from it, as
    the reference does) or a CUDA ``[V,3]`` tensor of moved vertex positions (``model.mesh_grid`` is deformed in place,
    normals from its mesh's triangles).  Unless ``fix_indicator``, ``model.indicator_vector`` becomes a new
    ``nn.Parameter`` holding the rotated vectors (``render_geometry_editing.py:65``)."""
    old_grid = model.mesh_grid
    old_normals = old_grid.get_vertex_normal_torch()
    if torch.is_tensor(deformed_mesh):
        old_grid.deform_(deformed_mesh)   # replaces vertex_normals: old_normals still holds the previous ones
        new_grid = old_grid
    else:
        new_grid = MeshGrid(deformed_mesh, device, distance_method=old_grid.distance_method)
    if not fix_indicator:
        with torch.no_grad():
            rotated = indicator_rotate(old_normals, new_grid.get_vertex_normal_torch(), model.indicator_vector)
        model.indicator_vector = nn.Parameter(rotated)
    model.mesh_grid = new_grid
