"""Exact K-nearest-neighbour restatement of ``frnn.frnn_grid_points`` - TEST INFRASTRUCTURE.

The reference's only native dependency on the hot path is the third-party package ``frnn``
(github.com/lxxue/FRNN; version unpinned - ``README.md:25`` gives a URL only; absent from ``environment.yml`` and
from the reference repository).  Its algorithm (published): counting-sort the points into a uniform grid of cell size
``r / radius_cell_ratio``, then, per query, scan the 3x3x3 neighbouring cells keeping the K closest points that lie
within ``r`` in a register min-K; results are squared Euclidean distances, optionally sorted ascending, padded with
-1 when fewer than K points lie within ``r``.

What the reference's two call sites (``models/mesh_grid.py:64-74`` and ``:109-119``) rely on - and therefore what is
restated here - is narrower: ``r = 100`` on a scene inside the unit sphere never binds, so the result is the exact
K nearest neighbours:

* ``dists``  [1, M, K] float32 - *squared* distances (caller takes ``.sqrt()`` at ``mesh_grid.py:123``),
* ``idxs``   [1, M, K] int64   - indices into ``points2`` in its original order (``mesh_grid.py:134``),
* ascending by distance (``return_sorted=True``), 4-tuple return whose last element is an opaque ``grid`` handle.

**parity unpinned**: the reference tree holds no golden vectors for this function and the package itself is not
available; tie order between exactly equidistant points is implementation-defined.
"""
from __future__ import annotations

import numpy as np
import torch

try:  # scipy is present in this image; the brute-force branch below needs nothing but torch
    from scipy.spatial import cKDTree
except Exception:  # pragma: no cover
    cKDTree = None

_TREE_CACHE: "dict[tuple, object]" = {}


def _sq_dist_f32(q: torch.Tensor, p: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """fp32 sum of squared coordinate differences (dx*dx + dy*dy + dz*dz, left to right)."""
    d = q[:, None, :] - p[idx]
    return d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]


def knn_exact(queries: torch.Tensor, points: torch.Tensor, K: int, method: str = "auto"):
    """queries [M,3], points [V,3] fp32 (CPU) -> (d2 [M,K] fp32 ascending, idx [M,K] int64)."""
    q = queries.detach().to(torch.float32).cpu().contiguous()
    p = points.detach().to(torch.float32).cpu().contiguous()
    M, V = q.shape[0], p.shape[0]
    if method == "auto":
        method = "kdtree" if (cKDTree is not None and M * V > (1 << 24)) else "brute"
    if method == "kdtree":
        key = (p.data_ptr(), V, float(p[0, 0]), float(p[-1, -1]))
        tree = _TREE_CACHE.get(key)
        if tree is None:
            _TREE_CACHE.clear()
            tree = cKDTree(p.numpy().astype(np.float64))
            _TREE_CACHE[key] = tree
        # take a few extra candidates, then re-rank in fp32 so that the selection is the fp32 one
        kq = min(V, K + 4)
        _, cand = tree.query(q.numpy().astype(np.float64), k=kq, workers=-1)
        cand = torch.from_numpy(np.ascontiguousarray(cand)).long().reshape(M, kq)
        d2 = _sq_dist_f32(q, p, cand)
        order = torch.argsort(d2, dim=1, stable=True)[:, :K]
        return torch.gather(d2, 1, order), torch.gather(cand, 1, order)
    # brute force, chunked over queries
    d2_out = torch.empty(M, K, dtype=torch.float32)
    idx_out = torch.empty(M, K, dtype=torch.int64)
    step = max(1, (1 << 24) // max(V, 1))
    for s in range(0, M, step):
        qq = q[s:s + step]
        dx = qq[:, None, 0] - p[None, :, 0]
        dy = qq[:, None, 1] - p[None, :, 1]
        dz = qq[:, None, 2] - p[None, :, 2]
        d2 = dx * dx + dy * dy + dz * dz
        v, i = torch.topk(d2, K, dim=1, largest=False, sorted=True)
        d2_out[s:s + step], idx_out[s:s + step] = v, i
    return d2_out, idx_out


def frnn_grid_points(points1, points2, lengths1=None, lengths2=None, K=8, r=100.0, grid=None, return_nn=False,
                     return_sorted=True, radius_cell_ratio=2.0):
    """Signature of ``frnn.frnn_grid_points`` as used at ``models/mesh_grid.py:64-74,109-119`` (batch size 1)."""
    assert points1.dim() == 3 and points2.dim() == 3 and points1.shape[0] == 1 and points2.shape[0] == 1
    d2, idx = knn_exact(points1[0], points2[0], K)
    out_of_r = d2 > float(r) * float(r)
    if out_of_r.any():  # FRNN pads with -1 outside the radius; never happens at r=100 in the unit sphere
        d2 = d2.masked_fill(out_of_r, -1.0)
        idx = idx.masked_fill(out_of_r, -1)
    dev = points1.device
    return d2[None].to(dev), idx[None].to(dev), None, ("oracle-grid", points2.shape[1])
