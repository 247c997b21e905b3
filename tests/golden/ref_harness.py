"""Import the UNMODIFIED reference (a checkout of zju3dv/NeuMesh named by ``NEUMESH_REFERENCE_ROOT``) on CPU, for
golden-vector generation.  No test, ``bench.py`` or ``smoke()`` imports this module: the tests compare against the
vectors it produced.

* plumbing dependencies that are absent here and irrelevant to the hot path (``addict``, ``imageio``,
  ``skimage``, ``kornia``, ``open3d``) are stubbed in ``sys.modules`` (SURVEY.md section 8c);
* ``frnn`` - the one third-party *native* dependency of the path (github.com/lxxue/FRNN, unpinned, absent) - is
  replaced by ``oracle.knn.frnn_grid_points``: an exact-KNN restatement of what the two call sites
  ``models/mesh_grid.py:64-74,109-119`` rely on.
"""
from __future__ import annotations

import os
import sys
import types

REF_ROOT = os.environ.get("NEUMESH_REFERENCE_ROOT", "")
REPO_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def available() -> bool:
    return os.path.isfile(os.path.join(REF_ROOT, "models", "renderer.py"))


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


_loaded = None


def load():
    """Returns a namespace with the reference's hot-path symbols (imported verbatim)."""
    global _loaded
    if _loaded is not None:
        return _loaded
    if not available():
        raise RuntimeError("reference tree not present at %s" % REF_ROOT)
    if REPO_ROOT not in sys.path:
        sys.path.insert(0, REPO_ROOT)
    from oracle import knn as oracle_knn

    class _Dict(dict):
        pass

    for name in ("addict", "imageio", "skimage", "skimage.transform", "kornia", "kornia.losses", "open3d"):
        if name not in sys.modules:
            _stub(name)
    sys.modules["addict"].Dict = _Dict
    sys.modules["skimage"].transform = sys.modules["skimage.transform"]
    sys.modules["skimage.transform"].rescale = lambda *a, **k: None
    sys.modules["kornia"].losses = sys.modules["kornia.losses"]
    sys.modules["kornia.losses"].ssim = lambda *a, **k: None
    o3d = sys.modules["open3d"]
    if not hasattr(o3d, "io"):
        o3d.io = types.SimpleNamespace(read_triangle_mesh=None)
    _stub("frnn", frnn_grid_points=oracle_knn.frnn_grid_points)

    # the reference uses top-level package names (models, utils, dataio): make them resolve to REF_ROOT
    # without shadowing this repo's own packages (none of which use those names).
    sys.path.insert(0, REF_ROOT)
    try:
        import models.renderer as renderer
        import models.mesh_grid as mesh_grid
        import models.base as base
        import models.frameworks.neumesh.neumesh as neumesh
        import utils.rend_util as rend_util
        import utils.train_util as train_util
        import editing.texture_neumesh.texture_neumesh as texture_neumesh   # empty package __init__: no Open3D import
        import models.frameworks.neus.neus as neus
        import models.ray_casting as ray_casting
    finally:
        sys.path.remove(REF_ROOT)

    import torch

    class HarnessMeshGrid(mesh_grid.MeshGrid):
        """``MeshGrid`` without the Open3D-dependent constructor (``models/mesh_grid.py:46-75``): sets the same
        attributes the constructor would."""

        def __init__(self, vertices, vertex_normals, distance_method="frnn"):
            self.mesh = None
            self.vertices = torch.as_tensor(vertices, dtype=torch.float32)
            self.vertex_normals = torch.as_tensor(vertex_normals, dtype=torch.float32)
            self.grid = None
            self.distance_method = distance_method

        def get_number_of_vertices(self):
            return self.vertices.shape[0]

    ns = types.SimpleNamespace(renderer=renderer, mesh_grid=mesh_grid, base=base, neumesh=neumesh,
                               rend_util=rend_util, train_util=train_util, texture_neumesh=texture_neumesh, neus=neus, ray_casting=ray_casting,
                               HarnessMeshGrid=HarnessMeshGrid)
    _loaded = ns
    return ns


def build_reference_model(mesh, cfg, state_dict):
    """Reference ``NeuMesh`` on CPU with the given parameters."""
    import contextlib
    import io

    ns = load()
    mg = ns.HarnessMeshGrid(mesh.vertices, mesh.vertex_normals)
    with contextlib.redirect_stdout(io.StringIO()):
        model = ns.neumesh.NeuMesh(mg, **cfg.model_kwargs())
    missing = model.load_state_dict(state_dict, strict=True)
    model.eval()
    return model
