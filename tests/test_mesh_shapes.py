"""The octree walks, the shell certificate and the bounded near / far scan on meshes other than the icosphere.

Every other GPU test queries ``synth.icosphere_mesh``: closed, star-shaped, centred, evenly tessellated and jittered
so that no two distances tie.  The code below depends on the mesh's shape (disc bounds that are safe only through fp32
margins, a (distance, slot) tie-break, per-node indicator statistics, the certificate's ``far_r`` rule), so it is held
here to exact oracles on open, non-convex, unevenly dense and exactly tied meshes (``synth.open_bowl``, ``torus``,
``double_sheet``, ``lattice_plane``, ``clustered``, ``fan_mesh``, ``far_bowl``):

* neighbours: bit-identical squared distances and, for the fused K = 8 path, the brute force's (d^2, slot) ranking;
* ds is computed with ``__f*_rn`` intrinsics in every kernel, so once the neighbours are exact the point query is
  exact, and it serves as ground truth for the certificate, the bounded near / far scan and the render's samples;
* the kernel's ``linspace01`` equals ``torch.linspace(0, 1, n)`` (CPU) bit for bit, so a torch scan reproduces the
  scan's sample depths exactly.

No bitwise assertion here has an outlier allowance.
"""
import functools
import math

import numpy as np
import pytest
import torch

import helpers
from neumesh_b200 import synth

SHAPES = {
    "bowl": lambda: synth.open_bowl(seed=3),
    "torus": lambda: synth.torus(seed=4),
    "double_sheet": lambda: synth.double_sheet(seed=5),
    "lattice": lambda: synth.lattice_plane(),
    "clustered": lambda: synth.clustered(seed=6),
}
KNN_SHAPES = dict(SHAPES, fan9=lambda: synth.fan_mesh(9, seed=7), fan33=lambda: synth.fan_mesh(33, seed=8),
                  far_bowl=lambda: synth.far_bowl(seed=3))


@functools.lru_cache(maxsize=None)
def _mesh(name):
    return KNN_SHAPES[name]()


def _dev():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (no CPU fallback exists)")
    return torch.device("cuda:0")


def _model(name, sd=None, cfg=None, seed=11):
    from neumesh_b200.neumesh import DEFAULT_MLP_ENGINE
    mesh = _mesh(name)
    cfg = cfg or synth.ModelConfig()
    sd = sd or synth.make_state_dict(mesh, cfg, seed=seed)
    return mesh, cfg, sd, helpers.cuda_model(mesh, cfg, sd, DEFAULT_MLP_ENGINE)


# ---------------------------------------------------------------------------------------------------------------
# the generators (CPU)
# ---------------------------------------------------------------------------------------------------------------
def test_mesh_family_generators():
    for name, make in KNN_SHAPES.items():
        a, b = make(), make()
        assert np.array_equal(a.vertices, b.vertices) and np.array_equal(a.triangles, b.triangles), name
        assert np.array_equal(a.vertex_normals, b.vertex_normals), name
        v = a.vertices
        assert np.array_equal(v, v.astype(np.float32).astype(np.float64)), f"{name}: vertices not rounded through fp32"
        assert a.triangles.min() >= 0 and a.triangles.max() < v.shape[0], name
        used = np.zeros(v.shape[0], dtype=bool)
        used[a.triangles.reshape(-1)] = True
        if name == "clustered":
            # the only unreferenced vertices are the exact copies of one vertex added on purpose
            extra = v[~used]
            assert extra.shape[0] == 200 and (extra == extra[0]).all() and (v[used] == extra[0]).all(axis=1).any()
        else:
            assert used.all(), f"{name}: unreferenced vertices"
        if name == "far_bowl":
            c = np.asarray(synth.FAR_BOWL_OFFSET)
            assert np.linalg.norm(v - c, axis=1).max() < 0.02
        else:
            assert np.linalg.norm(v, axis=1).max() < 1.0, name
    assert KNN_SHAPES["fan9"]().vertices.shape[0] == 9 and KNN_SHAPES["fan33"]().vertices.shape[0] == 33
    lat = synth.lattice_plane()
    assert lat.vertices.shape[0] == 257 * 257
    # every coordinate is an exact multiple of 1/256 (exact in fp32, hence exact squared-distance ties)
    assert np.array_equal(lat.vertices * 256, np.round(lat.vertices * 256)) and (lat.vertices[:, 2] == 0).all()
    # clustered: the octree's deepest cells (grid.cu build_grid: depth L with V / 4^L <= 2, cube of the bounding box's
    # largest side) hold far more than LEAF_MAX = 32 points, so max-depth leaves exceed LEAF_MAX
    for name, want_over in (("clustered", True), ("torus", False)):
        v = KNN_SHAPES[name]().vertices.astype(np.float32)
        L = 1
        while L < 10 and v.shape[0] / 4.0 ** L > 2.0:
            L += 1
        lo = v.min(0)
        side = float((v.max(0) - lo).max()) * 1.0001 + 1e-6
        q = np.clip(np.floor((v - lo) * np.float32(2 ** L / side)).astype(np.int64), 0, 2 ** L - 1)
        _, counts = np.unique((q[:, 0] << 20) | (q[:, 1] << 10) | q[:, 2], return_counts=True)
        assert (counts.max() > 32) == want_over, (name, L, counts.max())
    # double sheet: the two sheets lie within each other's 0.1 shell
    ds_ = KNN_SHAPES["double_sheet"]()
    half = ds_.vertices.shape[0] // 2
    a, b = ds_.vertices[:half], ds_.vertices[half:]
    assert np.allclose(np.abs(((a - b) * ds_.vertex_normals[:half]).sum(1)), 0.03, atol=1e-4)
    # different seeds give different meshes
    assert not np.array_equal(synth.torus(seed=1).vertices, synth.torus(seed=2).vertices)


# ---------------------------------------------------------------------------------------------------------------
# exact K nearest neighbours
# ---------------------------------------------------------------------------------------------------------------
def _queries(name, n_near=16000, n_far=4000, seed=0):
    """Near the surface, on vertices, on the 1/256 lattice (cell centres and edge midpoints of the lattice mesh: 2-, 4-
    and 8-way exact ties), and far away (radius up to 1.5).  The far bowl gets the open bowl's queries mapped through
    the same scale and offset."""
    base = "bowl" if name == "far_bowl" else name
    mesh = _mesh(base)
    g = torch.Generator().manual_seed(seed)
    v = torch.from_numpy(mesh.vertices).float()
    n = torch.from_numpy(mesh.vertex_normals).float()
    i = torch.randint(0, v.shape[0], (n_near,), generator=g)
    near = v[i] + n[i] * (0.03 * torch.randn(n_near, 1, generator=g)) + 0.004 * torch.randn(n_near, 3, generator=g)
    on = v[torch.randint(0, v.shape[0], (2000,), generator=g)]
    h = 1.0 / 256
    ij = torch.randint(-120, 120, (3000, 2), generator=g).float()
    kz = torch.randint(-3, 4, (3000, 1), generator=g).float()
    offs = torch.tensor([[0.5, 0.5], [0.5, 0.0], [0.0, 0.5], [0.0, 0.0]]).repeat(750, 1)
    lat = torch.cat([(ij + offs) * h, kz * h], 1)
    dirs = torch.nn.functional.normalize(torch.randn(n_far, 3, generator=g), dim=-1)
    far = dirs * (0.2 + 1.3 * torch.rand(n_far, 1, generator=g))
    q = torch.cat([near, on, lat, far, torch.zeros(1, 3)])
    if name == "far_bowl":
        q = (q.double() * synth.FAR_BOWL_SCALE + torch.tensor(synth.FAR_BOWL_OFFSET, dtype=torch.float64)).float()
        # ... and queries 0.05-40 away: from there the whole bowl lies within a relative 1e-3 in d^2, so the 8th
        # distance sits within fp32 rounding of many node bounds and only the bounds' margins keep the walk exact
        far_dirs = torch.nn.functional.normalize(torch.randn(4000, 3, generator=g, dtype=torch.float64), dim=-1)
        far_r = 0.05 * 800.0 ** torch.rand(4000, 1, generator=g, dtype=torch.float64)
        far_q = (torch.tensor(synth.FAR_BOWL_OFFSET, dtype=torch.float64) + far_dirs * far_r).float()
        q = torch.cat([q, torch.from_numpy(_mesh(name).vertices[:2000]).float(), far_q])
    return q


def _grid_order(grid, dev):
    """slot -> original vertex index (``nmb_grid_order``), as a tensor over the library's own device array."""
    from neumesh_b200 import _lib

    class _View:
        def __init__(self, p, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (p, False), "version": 3}

    p = _lib.lib().nmb_grid_order(grid.handle)
    return torch.as_tensor(_View(p, grid.num_vertices), device=dev).long().clone()


def _brute_knn(q, p, slot_of, K):
    """fp32 brute force on the GPU, every subtraction, square and sum rounded separately in the order of
    ``oracle/knn._sq_dist_f32``; ranked by the total order (d^2, slot).  -> (d2 [M,K], original index [M,K])."""
    out_d, out_i = [], []
    step = max(1, (1 << 26) // p.shape[0])
    for s in range(0, q.shape[0], step):
        qq = q[s:s + step]
        dx = qq[:, None, 0] - p[None, :, 0]
        dy = qq[:, None, 1] - p[None, :, 1]
        dz = qq[:, None, 2] - p[None, :, 2]
        d2 = dx * dx + dy * dy
        d2 = d2 + dz * dz
        key = (d2.view(torch.int32).long() << 32) | slot_of[None, :]    # d2 >= 0: its bits order like its value
        _, idx = torch.topk(key, K, dim=1, largest=False, sorted=True)
        out_d.append(torch.gather(d2, 1, idx))
        out_i.append(idx)
    return torch.cat(out_d), torch.cat(out_i)


def _sq_dist(q, p, idx):
    d = q[:, None, :] - p[idx]
    return d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]


def _distance_f32(q, p, ind, idx, w1):
    """mesh_grid.py:121-142 in fp32, each operation rounded separately in ``mesh_distance_point``'s order -> ds, w."""
    v = q[:, None, :] - p[idx]
    rho = ((v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1]) + v[..., 2] * v[..., 2]).sqrt()
    w = 1.0 / (rho + 1e-7)
    wsum = w[:, 0]
    for k in range(1, w.shape[1]):
        wsum = wsum + w[:, k]
    w = w / wsum[:, None]
    D = rho + w1
    m = (ind[idx] * w1 + v * rho[..., None]) / D[..., None]
    dot = (v[..., 0] * m[..., 0] + v[..., 1] * m[..., 1]) + v[..., 2] * m[..., 2]
    ds = w[:, 0] * dot[:, 0]
    for k in range(1, w.shape[1]):
        ds = ds + w[:, k] * dot[:, k]
    return ds, w


def _distance_f64(q, p, ind, idx, w1):
    """mesh_grid.py:121-142 in float64 on given neighbours (weights detached, as the reference does) -> ds, w, grad."""
    x = q.double().requires_grad_(True)
    pp = p.double()[idx]
    with torch.no_grad():
        dist = (q.double()[:, None, :] - pp).norm(dim=-1)
        w = 1.0 / (dist + 1e-7)
        w = w / w.sum(-1, keepdim=True)
    v = x[:, None, :] - pp
    rho = v.norm(dim=-1, keepdim=True)
    mid = (ind.double()[idx] * w1 + v * rho) / (w1 + rho)
    ds = (w * (v * mid).sum(-1)).sum(-1)
    (grad,) = torch.autograd.grad(ds.sum(), x)
    return ds.detach(), w, grad


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(KNN_SHAPES))
def test_knn_exact(shape):
    import neumesh_b200 as nb
    dev = _dev()
    mesh = _mesh(shape)
    p = torch.from_numpy(mesh.vertices).float().to(dev)
    V = p.shape[0]
    q = _queries(shape).to(dev)
    mg = nb.MeshGrid(mesh, dev)
    order = _grid_order(mg.grid, dev)
    assert torch.equal(torch.sort(order)[0], torch.arange(V, device=dev))
    slot_of = torch.empty_like(order)
    slot_of[order] = torch.arange(V, device=dev)
    d_ref, i_ref = _brute_knn(q, p, slot_of, min(32, V))

    # K = 8, the fused point kernel (knn_distance_kernel): the (d^2, slot) ranking, bit for bit
    sd = synth.make_state_dict(mesh, synth.ModelConfig(), seed=12)
    ind = sd["indicator_vector"].to(dev)
    ds, idx, w, grad = mg.grid.mesh_distance(q, ind, 0.1, want_grad=True)
    assert torch.equal(_sq_dist(q, p, idx), d_ref[:, :8]), "K = 8: squared distances differ from the brute force"
    n_tie = int((d_ref[:, 7] == d_ref[:, 8]).sum()) if V > 8 else 0
    assert torch.equal(idx, i_ref[:, :8]), "K = 8: neighbour lists differ from the (d^2, slot) ranking"
    # ds and w: every operation is an individually rounded intrinsic, so an fp32 restatement in the same order is exact
    ds32, w32 = _distance_f32(q, p, ind, idx, 0.1)
    assert torch.equal(ds[:, 0], ds32) and torch.equal(w, w32), "ds / w differ from the fp32 restatement"
    ds64, w64, g64 = _distance_f64(q, p, ind, idx, 0.1)
    e_ds = ((ds[:, 0].double() - ds64).abs() / ds64.abs().clamp_min(1.0)).max().item()
    e_w = (w.double() - w64).abs().max().item()
    e_g = ((grad.double() - g64).abs() / g64.abs().clamp_min(1.0)).max().item()
    # test_mesh_distance_vs_oracle's bars for ds and grad (relative where |ds| or |grad| exceed 1: queries reach radius
    # 1.5 here).  Its w bar (2e-7) is against the fp32 oracle; against float64 the four fp32 roundings of a weight in
    # [0, 1] give up to 2.75e-7 (measured on an H100), hence 4e-7.
    assert e_ds < 1e-6 and e_w < 4e-7 and e_g < 2e-5, (e_ds, e_w, e_g)

    # generic K (knn_generic_kernel, the frnn shim): no slot tie-break, so the index SETS agree below the K-th distance
    n_set = {}
    for K in (1, 8, 9, 32):
        if K > V:
            continue
        d2, ik = mg.grid.knn(q, K)
        assert torch.equal(d2, d_ref[:, :K]), f"K = {K}: squared distances differ from the brute force"
        assert torch.equal(_sq_dist(q, p, ik), d2), f"K = {K}: indices do not reproduce the distances"
        strict = d_ref[:, :K] < d_ref[:, K - 1:K]
        a = torch.sort(torch.where(strict, ik, -1), dim=1)[0]
        b = torch.sort(torch.where(strict, i_ref[:, :K], -1), dim=1)[0]
        assert torch.equal(a, b), f"K = {K}: neighbour sets differ below the K-th distance"
        n_set[K] = int((~strict).sum())
    print(f"[{shape}] V={V} {q.shape[0]} queries: K=8 lists bit-exact ({n_tie} with an 8th/9th distance tie); "
          f"entries at the K-th distance (set-compared only) {n_set}; float64: ds {e_ds:.2e} w {e_w:.2e} grad {e_g:.2e}")


# ---------------------------------------------------------------------------------------------------------------
# the shell certificate (csrc/shell.cu)
# ---------------------------------------------------------------------------------------------------------------
INDICATORS = ["default", "flipped", "scaled", "learned_w0.02", "learned_w0.6"]


def _indicator_case(shape, variant):
    cfg = synth.ModelConfig(learn_indicator_weight=variant.startswith("learned"))
    mesh = _mesh(shape)
    sd = synth.make_state_dict(mesh, cfg, seed=13)
    g = torch.Generator().manual_seed(14)
    ind = sd["indicator_vector"]
    if variant == "flipped":      # scans without a consistent orientation
        flip = torch.rand(ind.shape[0], generator=g) < 0.15
        sd["indicator_vector"] = torch.where(flip[:, None], -ind, ind)
    elif variant == "scaled":
        sd["indicator_vector"] = ind * (0.2 + 2.8 * torch.rand(ind.shape[0], 1, generator=g))
    elif variant.startswith("learned"):
        w1 = float(variant[len("learned_w"):])
        sd["indicator_weight_raw"] = torch.tensor([math.log(w1 / (1.0 - w1))], dtype=torch.float32)
    return _model(shape, sd=sd, cfg=cfg)


@pytest.mark.gpu
@pytest.mark.parametrize("indicator", INDICATORS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_shell_certificate_sound(shape, indicator):
    """Every point of a cell coded 1 has ds >= 0.1 and every point of a cell coded 2 has ds < 0.1, checked with the
    exact point query on random points of the coded cells and on every corner of every coded cell (the extreme points
    the certificate's bounds have to cover)."""
    dev = _dev()
    mesh, cfg, sd, model = _indicator_case(shape, indicator)
    cells, B = model.shell_free_grid()
    G = cells.shape[0]
    assert G > 1
    hs = torch.tensor(B, dtype=torch.float32) / G          # the kernel's half cell size, in fp32
    g = torch.Generator(device="cpu").manual_seed(15)
    report = []
    for code in (1, 2):
        zyx = torch.nonzero(cells == code)                   # [n, 3] cell indices (z, y, x)
        n = zyx.shape[0]
        if n == 0:
            report.append(f"code {code}: 0 cells")
            continue
        ijk = zyx.flip(1).float()                            # (x, y, z)
        pick = torch.randint(0, n, (min(2_000_000, 16 * n),), generator=g).to(dev)
        u = torch.rand(pick.shape[0], 3, generator=g).to(dev)
        inner = -B + (2 * ijk[pick] + 2 * u) * hs.to(dev)
        # the 8 corners of every coded cell, as the set of grid vertices they share
        corner_ids = torch.unique(((zyx[:, None, :] + torch.tensor(
            [[a, b, c] for a in (0, 1) for b in (0, 1) for c in (0, 1)], device=dev)[None]).reshape(-1, 3) *
            torch.tensor([(G + 1) ** 2, G + 1, 1], device=dev)).sum(-1))
        cz, cy, cx = corner_ids // (G + 1) ** 2, (corner_ids // (G + 1)) % (G + 1), corner_ids % (G + 1)
        corners = -B + 2 * torch.stack([cx, cy, cz], 1).float() * hs.to(dev)
        x = torch.cat([inner, corners])
        ds = torch.empty(x.shape[0], device=dev)
        with torch.no_grad():
            for s in range(0, x.shape[0], 1 << 22):
                ds[s:s + (1 << 22)] = model.compute_distance(x[s:s + (1 << 22)])[0][:, 0]
        if code == 1:
            bad = int((ds < 0.1).sum())
            report.append(f"code 1: {n} cells ({n / G ** 3:.3f}), {x.shape[0]} points, min ds {ds.min().item():.4f}")
        else:
            bad = int((ds >= 0.1).sum())
            report.append(f"code 2: {n} cells ({n / G ** 3:.4f}), {x.shape[0]} points, max ds {ds.max().item():.4f}")
        assert bad == 0, f"{shape}/{indicator}: {bad} points of code-{code} cells contradict the certificate"
    print(f"[{shape} / {indicator}] " + "; ".join(report))
    if indicator == "default" and shape in ("torus", "bowl"):
        # not vacuous where the certificate must hold: most of the cube is far from these surfaces
        assert (cells == 1).float().mean().item() > 0.2 and int((cells == 2).sum()) > 0
        near = torch.from_numpy(mesh.vertices).float().to(dev)
        ijk = ((near + B) * (0.5 * G / B)).long().clamp_(0, G - 1)
        assert not (cells[ijk[:, 2], ijk[:, 1], ijk[:, 0]] == 1).any()


# ---------------------------------------------------------------------------------------------------------------
# the bounded near / far scan (bound_dir_kernel<false / true> + certificate, bound_scan_kernel, bound_finish_kernel)
# ---------------------------------------------------------------------------------------------------------------
def _frame(view, H=256):
    """A spiral frame of H x H rays (>= 65 536: the certificate is used) plus three 32 x 32 cameras inside the unit
    sphere (near = 0), directions normalised once."""
    o, d = synth.frame_rays(H, H, view=view)
    os_, ds_ = [o], [d]
    for k, c in enumerate(([0.1, 0.2, -0.3], [-0.5, 0.0, 0.2], [0.0, -0.05, 0.0])):
        pose = synth.look_at(np.array(c), np.array([0.3, -0.2, 0.1]) * (k - 1))
        oi, di = synth.pinhole_rays(pose, 32, 32, 20.0, 20.0, 16.0, 16.0)
        os_.append(oi)
        ds_.append(di)
    o, d = torch.cat(os_), torch.cat(ds_)
    return o, torch.nn.functional.normalize(d, dim=-1)


class _PointQuery:
    """The exact CUDA point query (K = 8 point kernel) behind the oracle's field protocol.  It also counts how the scan's
    samples fall on the certificate: in cells coded 1 or 2 of the [-B, B]^3 grid, or outside that cube, where only the
    ``far_r`` rule can decide them; and keeps the ``ds < 0.1`` mask per sample."""

    def __init__(self, model, cells, B):
        self.model, self.cells, self.B = model, cells, B
        self.n_code = {1: 0, 2: 0}
        self.n_outside = 0
        self.inside = None

    def compute_distance(self, x):
        flat = x.reshape(-1, 3)
        ds = torch.empty(flat.shape[0], 1, device=flat.device)
        G, B = self.cells.shape[0], self.B
        with torch.no_grad():
            for s in range(0, flat.shape[0], 1 << 22):
                xs = flat[s:s + (1 << 22)]
                ds[s:s + (1 << 22)] = self.model.compute_distance(xs)[0]
                in_cube = (xs.abs() < B).all(1)
                ijk = ((xs[in_cube] + B) * (0.5 * G / B)).long().clamp_(0, G - 1)
                code = self.cells[ijk[:, 2], ijk[:, 1], ijk[:, 0]]
                for c in (1, 2):
                    self.n_code[c] += int((code == c).sum())
                self.n_outside += int((~in_cube).sum())
        self.inside = (ds < 0.1).reshape(x.shape[:-1])
        return ds.reshape(*x.shape[:-1], 1), None, None


@pytest.mark.gpu
@pytest.mark.parametrize("indicator", INDICATORS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_bounded_near_far_exact(shape, indicator):
    """Every indicator variant: they move the certificate's cells and its rho_safe / far_r rule outside the grid."""
    from neumesh_b200.renderer import render_fused
    from oracle import render as orender
    dev = _dev()
    mesh, cfg, sd, model = _indicator_case(shape, indicator)
    cells, B = model.shell_free_grid()
    assert int((cells == 1).sum()) > 0 and int((cells == 2).sum()) > 0
    o, d = _frame(view=list(SHAPES).index(shape) * 7 + 1)
    o, d = o.to(dev), d.to(dev)
    R = o.shape[0]
    kw = dict(normalize_dirs=False, sampling_only=True, N_upsample_iters=0)
    lines = []
    for radius in (1.0, 2.0):
        with torch.no_grad():
            plain = render_fused(o, d, model, obj_bounding_radius=radius, bounded_near_far=False, **kw)["near_far"]
            whole = render_fused(o, d, model, obj_bounding_radius=radius, chunk=R, **kw)["near_far"]
            small = render_fused(o, d, model, obj_bounding_radius=radius, chunk=8192, **kw)["near_far"]
        # 1. sphere near / far in the kernel's sum order
        mid = -((o[:, 0] * d[:, 0] + o[:, 1] * d[:, 1]) + o[:, 2] * d[:, 2])
        near, far = (mid - radius).clamp_min(0.0)[:, None], (mid + radius).clamp_min(radius)[:, None]
        assert torch.equal(plain, torch.cat([near, far], 1)), "sphere near / far differ"
        # 2.-5. depths (CPU linspace), points, ds at all 256 samples from the point query, the reference's min / max and
        # +-0.05 rules
        pq = _PointQuery(model, cells, B)
        lo, hi = orender.mesh_bounded_near_far(pq, o, d, near, far)
        ref = torch.cat([lo, hi], 1)
        n_bad_whole = int((whole != ref).any(1).sum())
        n_bad_small = int((small != ref).any(1).sum())
        n_near0 = int((near == 0).sum())
        hit = int(pq.inside.any(1).sum())
        m = pq.inside
        two = int(((m[:, 1:] & ~m[:, :-1]).sum(1) + m[:, 0].long() >= 2).sum())   # rays with >= 2 separate hit spans
        lines.append(f"radius {radius:g}: {R} rays x 256 samples, {hit} rays hit the shell ({two} twice), {n_near0} "
                     f"with near = 0; samples in code-1 / code-2 cells {pq.n_code[1]} / {pq.n_code[2]}, outside the "
                     f"cube {pq.n_outside}; mismatches whole frame {n_bad_whole}, 8192-ray chunks {n_bad_small}")
        assert n_bad_whole == 0, f"two-ended scan + certificate, radius {radius}: {n_bad_whole} rays differ"
        assert n_bad_small == 0, f"plain scan, radius {radius}: {n_bad_small} rays differ"
        # not vacuous: rays from inside the sphere, rays bounded by the mesh, samples the certificate decides, samples
        # outside the grid (radius 2), and on the torus rays that cross the shell twice
        assert n_near0 >= 3 * 1024 and hit > 1000 and pq.n_code[1] > 0 and pq.n_code[2] > 0
        assert radius < 2 or pq.n_outside > 0
        assert shape != "torus" or two > 100
    print(f"[{shape} / {indicator}] " + "; ".join(lines))


# ---------------------------------------------------------------------------------------------------------------
# the render's own samples against the point queries, and the composited outputs' invariances
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SHAPES))
def test_render_samples_equal_point_queries(shape):
    from neumesh_b200.renderer import render_fused
    dev = _dev()
    mesh, cfg, sd, model = _model(shape)
    o, d = synth.frame_rays(192, 192, view=list(SHAPES).index(shape) * 5 + 2)
    o, d = o.to(dev), torch.nn.functional.normalize(d, dim=-1).to(dev)
    R = o.shape[0]
    kw = dict(calc_normal=True, white_bkgd=True, bounded_near_far=True, normalize_dirs=False)
    summary = []
    for chunk in (R, 8192):           # the ray-ordered warm walks (>= 32 768 rays per chunk) and the per-point kernel
        with torch.no_grad():
            ex = render_fused(o, d, model, chunk=chunk, detailed_output=True, samples_output=True, **kw)
            z = ex["d_all"]
            x = o[:, None, :] + z[..., None] * d[:, None, :]
            s_pt = model.forward_density_only(x)[..., 0]
            s_n, n_pt = model.forward_with_nablas(x)
            xm = o[:, None, :] + ex["d_final"][..., None] * d[:, None, :]
            s_mid, c_mid = model.forward(xm, d[:, None, :].expand_as(xm))
        assert torch.equal(ex["implicit_surface"], s_pt), f"chunk {chunk}: sample sdf differs from the point query"
        assert torch.equal(ex["density"][..., 0], s_mid[..., 0]), f"chunk {chunk}: mid-point sdf differs"
        n_nab = int((ex["implicit_nablas"] != n_pt).any(-1).sum())
        n_rad = int((ex["radiance"] != c_mid).any(-1).sum())
        e_nab = (ex["implicit_nablas"] - n_pt).abs().max().item()
        e_rad = (ex["radiance"] - c_mid).abs().max().item()
        summary.append(f"chunk {chunk}: {z.numel()} samples + {xm.shape[0] * xm.shape[1]} mid-points sdf bitwise; "
                       f"nabla differs on {n_nab} (max {e_nab:.1e}), radiance on {n_rad} (max {e_rad:.1e})")
        assert n_nab == 0, f"chunk {chunk}: {n_nab} sample nablas differ from forward_with_nablas (max {e_nab:.2e})"
        assert n_rad == 0, f"chunk {chunk}: {n_rad} mid-point radiances differ from forward (max {e_rad:.2e})"
    print(f"[{shape}] " + "; ".join(summary))
    kw.pop("normalize_dirs")
    with torch.no_grad():
        a = render_fused(o, d, model, chunk=R, **kw)
        b = render_fused(o, d, model, chunk=8192, **kw)
        perm = torch.randperm(R, device=dev, generator=torch.Generator(device=dev).manual_seed(16))
        c = render_fused(o[perm], d[perm], model, chunk=R, **kw)
        e = render_fused(o, d, model, chunk=R, skip_dead_samples=False, **kw)
    for k in ("rgb", "depth_volume", "mask_volume", "normals_volume"):
        assert torch.isfinite(a[k]).all(), k
        assert torch.equal(a[k], b[k]), f"{k}: chunked render differs"
        assert torch.equal(a[k][perm], c[k]), f"{k}: permuted render differs"
        assert torch.equal(a[k], e[k]), f"{k}: live-sample path differs from the all-samples path"


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["torus", "bowl", "double_sheet"])
def test_render_teacher_forced(shape):
    _dev()
    mesh, cfg, sd, model = _model(shape)
    f = helpers.oracle_field(mesh, cfg, sd)
    o, d = synth.frame_rays(40, 40, view=list(SHAPES).index(shape) * 3 + 4)
    # the bowl: one solid ray's depth is ill-conditioned at fp32 - the fp32 oracle is itself 7.1e-6 from float64 on the
    # solid rays and the CUDA path 1.1e-5, so the two differ by 1.22e-5 in depth * acc there (measured on an H100); the
    # bar against float64 holds, the depth * acc bar against the fp32 oracle is pinned at 1.5e-5 for this mesh
    depth_acc_tol = 1.5e-5 if shape == "bowl" else helpers.DEPTH_TOL
    helpers.check_render_teacher_forced(model, mesh, cfg, sd, f, o, d, shape, ties_by_neighbours=True,
                                        depth_acc_tol=depth_acc_tol)
