"""Geometry editing on the device: ``nmb_grid_update``, ``nmb_indicator_rotate`` and ``deform_model``
(reference ``editing/render_geometry_editing.py:37-67``).

* the rotation's restatement (``oracle/deform.py``, kornia's ``angle_axis_to_rotation_matrix`` and the reference's
  ``|aa| = theta |axis|``) is pinned by hand-checked cases and by its float64 form (CPU);
* a grid updated in place equals a grid created on the moved vertices: the same slot order, and neighbours bit-identical
  to each other and to the fp32 brute force on the mesh family of ``test_mesh_shapes.py``;
* a model deformed in place renders bit for bit like a fresh model built on the deformed mesh, meets the teacher-forced
  bars, keeps its field and edit handles (re-packed, not re-created) and allocates nothing after the first deformation;
* a field or edit packed before an update is refused until it is re-packed.
"""
import ctypes
import math
import types

import numpy as np
import pytest
import torch

import helpers
from neumesh_b200 import synth
from oracle import deform as odeform


def _dev():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (no CPU fallback exists)")
    return torch.device("cuda:0")


# ---------------------------------------------------------------------------------------------------------------
# the rotation oracle (CPU)
# ---------------------------------------------------------------------------------------------------------------
def _rot1(n_old, n_new, ind, dtype=torch.float32):
    t = lambda x: torch.tensor([x], dtype=torch.float32)  # noqa: E731
    return odeform.indicator_rotate(t(n_old), t(n_new), t(ind), dtype)[0].double()


def _about_y(alpha, v):
    """Rotation of v by alpha about +y (right-handed)."""
    c, s = math.cos(alpha), math.sin(alpha)
    return torch.tensor([c * v[0] + s * v[2], v[1], -s * v[0] + c * v[2]], dtype=torch.float64)


def test_rotation_oracle_hand_cases():
    ind = (0.3, -0.2, 0.9)
    # identity: cross = 0 exactly, theta^2 = 0 -> I + [0]x
    assert torch.equal(_rot1((0, 0, 1), (0, 0, 1), ind), torch.tensor(ind, dtype=torch.float32).double())
    # exactly 180 degrees: c == -1 -> R = I (axis 0), then negated
    assert torch.equal(_rot1((0, 0, 1), (0, 0, -1), ind), -torch.tensor(ind, dtype=torch.float32).double())
    # a quarter turn about z: theta = pi/2 and w = (pi/2) / (pi/2 + 1e-6) < 1, so R[2,2] = w^2 (kornia's eps shows)
    wz = (math.pi / 2) / (math.pi / 2 + 1e-6)
    out = _rot1((1, 0, 0), (0, 1, 0), (1, 0, 1))
    assert torch.allclose(out, torch.tensor([0.0, wz, wz * wz], dtype=torch.float64), atol=2e-7, rtol=0), out
    # each side of the Taylor threshold theta^2 = |aa|^2 = 1e-6: n_old = z, n_new = z turned by phi about y, so
    # axis = (0, sin phi, 0) and aa = (0, phi sin phi, 0)
    for phi, rodrigues in ((0.04, True), (0.025, False)):
        n_new = (math.sin(phi), 0.0, math.cos(phi))
        nf = torch.tensor(n_new, dtype=torch.float32).double()
        ang = math.acos(float(nf[2]) / float(nf.norm()))
        alpha = float(nf[0]) * ang
        assert (alpha * alpha > 1e-6) == rodrigues
        out = _rot1((0, 0, 1), n_new, (1, 0, 0))
        if rodrigues:   # w_y = alpha / (alpha + 1e-6): (cos alpha, 0, -w_y sin alpha)
            want = torch.tensor([math.cos(alpha), 0.0, -alpha / (alpha + 1e-6) * math.sin(alpha)], dtype=torch.float64)
        else:           # first order: (1, 0, -alpha)
            want = torch.tensor([1.0, 0.0, -alpha], dtype=torch.float64)
        assert torch.allclose(out, want, atol=1e-7, rtol=0), (phi, out, want)
        # ... and the other branch's value is far outside that tolerance (the test tells the branches apart)
        other = _about_y(alpha * (alpha / (alpha + 1e-6)), (1, 0, 0)) if not rodrigues else \
            torch.tensor([1.0, 0.0, -alpha], dtype=torch.float64)
        assert (other - want).abs().max() > 5e-7
    # non-unit normals: |axis| = |n_old| |n_new| sin(theta) = 6, so |aa| = 3 pi - a rotation by 3 pi (~ pi), not the
    # quarter turn between the normals.  The reference computes this; so does the oracle.
    out = _rot1((2, 0, 0), (0, 3, 0), (1, 0, 0))
    assert torch.allclose(out, torch.tensor([-1.0, 0.0, 0.0], dtype=torch.float64), atol=3e-6, rtol=0), out


def _random_normals(n, seed):
    """Unit and non-unit normal pairs at every angle, with near-identical and near-opposite pairs."""
    g = torch.Generator().manual_seed(seed)
    a = torch.nn.functional.normalize(torch.randn(n, 3, generator=g, dtype=torch.float64), dim=-1)
    b = torch.nn.functional.normalize(torch.randn(n, 3, generator=g, dtype=torch.float64), dim=-1)
    k = n // 4
    b[:k] = torch.nn.functional.normalize(a[:k] + 10.0 ** (-6 * torch.rand(k, 1, generator=g, dtype=torch.float64))
                                          * torch.randn(k, 3, generator=g, dtype=torch.float64), dim=-1)
    b[k:2 * k] = torch.nn.functional.normalize(-a[k:2 * k] + 10.0 ** (-6 * torch.rand(k, 1, generator=g, dtype=torch.float64))
                                               * torch.randn(k, 3, generator=g, dtype=torch.float64), dim=-1)
    scale = torch.where(torch.rand(n, 1, generator=g) < 0.25, 0.5 + torch.rand(n, 1, generator=g), torch.ones(n, 1))
    ind = torch.randn(n, 3, generator=g, dtype=torch.float64) * 0.7
    return (a * scale).float(), b.float(), ind.float()


# |fp32 - float64| over the random set (same fp32 inputs): rounding of the cross product of two nearly opposite normals,
# of acos near +-1 and of the Rodrigues terms; the two forms may also pick different Taylor / Rodrigues branches within
# rounding of theta^2 = 1e-6, where the branches differ by ~5e-7.  Measured 4.4e-7 per unit |ind| (CPU).
ROT_F32_TOL = 1e-6


def _vs_float64(out, a, b, ind, tag):
    """max |out - float64 form| per unit |ind| over the rows whose c == -1 test agrees with float64's; the others
    (normals within fp32 rounding of opposite, where the reference's flip is a discontinuity) are counted and must all be
    within 1e-6 of c = -1."""
    r64 = odeform.indicator_rotate(a, b, ind, torch.float64)
    c64 = odeform.cos_between(a, b, torch.float64)
    same_flip = (odeform.cos_between(a, b, torch.float32) == -1) == (c64 == -1)
    assert bool(((c64 + 1).abs() < 1e-6)[~same_flip].all())
    scale = ind.double().norm(dim=-1, keepdim=True).clamp_min(1.0)
    err = ((out.double() - r64).abs() / scale)[same_flip].max().item()
    print(f"{tag} on {a.shape[0]} vertices: max error vs float64 {err:.2e} per unit |ind|; "
          f"{int((~same_flip).sum())} near-opposite rows flipped in one precision only")
    return err, r64


def test_rotation_oracle_fp32_vs_float64():
    a, b, ind = _random_normals(200000, seed=3)
    err, r64 = _vs_float64(odeform.indicator_rotate(a, b, ind, torch.float32), a, b, ind, "fp32 restatement")
    assert err < ROT_F32_TOL
    # |R ind| = |ind| up to kornia's eps (w = aa / (theta + 1e-6) is not quite a unit axis): R is a rotation
    assert torch.allclose(r64.norm(dim=-1), ind.double().norm(dim=-1), atol=1e-5, rtol=0)


class _RecordingGrid:
    """Stands in for a CUDA MeshGrid on a CPU host: records deform_ calls."""
    distance_method = "frnn"

    def __init__(self, V):
        self.V, self.calls = V, []

    def get_number_of_vertices(self):
        return self.V

    def get_vertex_normal_torch(self):
        return torch.zeros(self.V, 3)

    def deform_(self, vertices, normals=None):
        self.calls.append(vertices)


def test_deform_model_fix_indicator_touches_no_indicator(monkeypatch):
    import neumesh_b200 as nb
    from neumesh_b200 import deform

    def refuse(*a, **k):
        raise AssertionError("fix_indicator=True must not rotate the indicator vectors")

    monkeypatch.setattr(deform, "indicator_rotate", refuse)
    grid = _RecordingGrid(42)
    model = nb.NeuMesh(grid, **synth.ModelConfig().model_kwargs())
    param = model.indicator_vector
    before = param.detach().clone()
    v = torch.randn(42, 3)
    nb.deform_model(v, model, "cpu", fix_indicator=True)
    assert model.indicator_vector is param and torch.equal(param, before) and param._version == 0
    assert len(grid.calls) == 1 and grid.calls[0] is v and model.mesh_grid is grid


# ---------------------------------------------------------------------------------------------------------------
# nmb_grid_update on the mesh family (GPU)
# ---------------------------------------------------------------------------------------------------------------
def _affine():
    g = np.random.default_rng(5)
    A = np.array([[1.7, 0.4, -0.3], [-0.2, 0.6, 0.5], [0.3, -0.5, 1.2]]) @ np.linalg.qr(g.standard_normal((3, 3)))[0]
    return A, np.array([0.3, -0.2, 0.15])


def _deform_points(kind, p, phase=0.0, seed=0):
    """float64 [N,3] -> float64 [N,3]; `jitter` and `lattice` move vertices only (queries stay)."""
    if kind == "wave":
        s = p.std(axis=0).max()   # the far bowl is small: scale the wave to the mesh
        return p + np.stack([0 * p[:, 0], 0 * p[:, 0], 0.06 * s * np.sin(9.0 * p[:, 0] / s + 7.0 * p[:, 1] / s + phase)], 1)
    if kind == "jitter":
        s = p.std(axis=0).max()
        return p + 0.004 * s * np.random.default_rng(seed).standard_normal(p.shape)
    if kind == "affine":
        A, t = _affine()
        return p @ A.T + t
    if kind == "lattice":   # every coordinate on the 1/256 lattice: exact distance ties and coincident vertices
        return np.round(p * 256.0) / 256.0
    raise ValueError(kind)


DEFORMS = ["wave", "jitter", "affine", "lattice"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", DEFORMS)
@pytest.mark.parametrize("shape", ["bowl", "torus", "double_sheet", "lattice", "clustered", "fan9", "fan33", "far_bowl"])
def test_grid_update_equals_create(shape, kind):
    import neumesh_b200 as nb
    from test_mesh_shapes import _brute_knn, _grid_order, _mesh, _queries, _sq_dist
    dev = _dev()
    mesh = _mesh(shape)
    mg = nb.MeshGrid(mesh, dev)
    order_ptr = _lib_order_ptr(mg.grid)
    moved = torch.from_numpy(_deform_points(kind, mesh.vertices)).float().to(dev)
    mg.deform_(moved, normals=torch.zeros_like(moved))
    assert mg.grid.generation == 1 and _lib_order_ptr(mg.grid) == order_ptr, "the grid's buffers are reused"
    fresh = nb.GridHandle(moved)
    V = moved.shape[0]
    order_u, order_c = _grid_order(mg.grid, dev), _grid_order(fresh, dev)
    assert torch.equal(order_u, order_c), "nmb_grid_update's slot order differs from nmb_grid_create's"
    q = _queries(shape)
    if kind in ("wave", "affine"):
        q = torch.from_numpy(_deform_points(kind, q.double().numpy())).float()
    q = q.to(dev)
    slot_of = torch.empty_like(order_u)
    slot_of[order_u] = torch.arange(V, device=dev)
    d_ref, i_ref = _brute_knn(q, moved, slot_of, min(9, V))
    K = min(8, V)
    d_u, i_u = mg.grid.knn(q, K)
    d_c, i_c = fresh.knn(q, K)
    assert torch.equal(d_u, d_c) and torch.equal(i_u, i_c), "generic KNN differs between updated and created grid"
    assert torch.equal(d_u, d_ref[:, :K]), "generic KNN squared distances differ from the fp32 brute force"
    ind = torch.nn.functional.normalize(torch.randn(V, 3, generator=torch.Generator().manual_seed(2)), dim=-1).to(dev)
    a = mg.grid.mesh_distance(q, ind, 0.1, want_grad=True)
    b = fresh.mesh_distance(q, ind, 0.1, want_grad=True)
    for x, y in zip(a, b):
        assert torch.equal(x, y), "fused K = 8 query differs between updated and created grid"
    assert torch.equal(_sq_dist(q, moved, a[1]), d_ref[:, :8]), "K = 8 squared distances differ from the brute force"
    assert torch.equal(a[1], i_ref[:, :8]), "K = 8 neighbour lists differ from the (d^2, slot) ranking"
    ties = int((d_ref[:, 7] == d_ref[:, 8]).sum()) if V > 8 else 0
    print(f"[{shape}/{kind}] V={V}, {q.shape[0]} queries bit-identical to create and brute force; "
          f"{ties} queries with an 8th/9th tie")


def _lib_order_ptr(grid):
    from neumesh_b200 import _lib
    return _lib.lib().nmb_grid_order(grid.handle)


@pytest.mark.gpu
def test_grid_update_refuses_a_vertex_count_change():
    import neumesh_b200 as nb
    from neumesh_b200 import _lib
    dev = _dev()
    mesh = synth.icosphere_mesh(3, seed=1)
    mg = nb.MeshGrid(mesh, dev)
    V = mg.vertices.shape[0]
    bigger = torch.zeros(V + 1, 3, device=dev)
    with pytest.raises(ValueError, match="vertex count"):
        mg.deform_(bigger)
    rc = _lib.lib().nmb_grid_update(mg.grid.handle, _lib.ptr(bigger), V + 1, _lib.stream_ptr(dev))
    assert rc != 0 and b"V must equal" in _lib.lib().nmb_last_error()
    assert mg.grid.generation == 0


# ---------------------------------------------------------------------------------------------------------------
# nmb_indicator_rotate (GPU)
# ---------------------------------------------------------------------------------------------------------------
# kernel vs float64: twice the fp32 restatement's bound (the device's acosf / cosf / sinf are within 2 ulp, torch's CPU
# ones within 1)
ROT_KERNEL_TOL = 2 * ROT_F32_TOL


@pytest.mark.gpu
def test_indicator_rotate_kernel_vs_oracle():
    import neumesh_b200 as nb
    dev = _dev()
    a, b, ind = _random_normals(400000, seed=4)
    # rows that must come out exactly: identical normals (-> ind) and exactly opposite axis-aligned ones (-> -ind)
    e = torch.eye(3).repeat(200, 1)
    n0 = a.shape[0]
    a = torch.cat([a, e, e, a[:1000]])
    b = torch.cat([b, e, -e, a[:1000]])
    ind = torch.cat([ind, torch.randn(1600 + 600, 3, generator=torch.Generator().manual_seed(9))])
    n = a.shape[0]
    ident = torch.cat([torch.arange(n0, n0 + 600), torch.arange(n0 + 1200, n)])
    opp = torch.arange(n0 + 600, n0 + 1200)
    out = nb.indicator_rotate(a.to(dev), b.to(dev), ind.to(dev)).cpu()
    assert torch.equal(out[ident], ind[ident]), "identical normals must leave the indicator unchanged"
    assert torch.equal(out[opp], -ind[opp]), "exactly opposite normals must negate the indicator"
    err, _ = _vs_float64(out, a, b, ind, "nmb_indicator_rotate")
    r32 = odeform.indicator_rotate(a, b, ind, torch.float32)
    print(f"{int((out == r32).all(-1).sum())} of {n} rows bit-identical to the fp32 restatement")
    assert err < ROT_KERNEL_TOL
    # in place (ind_out == ind_in) gives the same result
    from neumesh_b200 import _lib
    x, ad, bd = ind.to(dev).contiguous(), a.to(dev), b.to(dev)   # kept alive across the call
    _lib.check(_lib.lib().nmb_indicator_rotate(_lib.ptr(ad), _lib.ptr(bd), _lib.ptr(x), n, _lib.ptr(x),
                                               _lib.stream_ptr(dev)))
    assert torch.equal(x.cpu(), out)


# ---------------------------------------------------------------------------------------------------------------
# deform_model: in place vs a fresh model (GPU)
# ---------------------------------------------------------------------------------------------------------------
def _wave(v, phase):
    """Per-frame wave displacement of the icosphere (float32 on the device)."""
    r = v.norm(dim=-1, keepdim=True)
    return v + 0.04 * torch.sin(8.0 * v[:, 0:1] + 6.0 * v[:, 1:2] + phase) * v / r


def _host_mesh(vertices, triangles, normals):
    """A host mesh with exactly these fp32 vertices and normals (no compute_vertex_normals: MeshGrid keeps them)."""
    return types.SimpleNamespace(vertices=vertices.double().cpu().numpy(), triangles=triangles,
                                 vertex_normals=normals.double().cpu().numpy())


def _deformed_pair(level=5, phase=0.7, engine=None, seed=21):
    """(in-place deformed model, fresh model on MeshGrid(deformed mesh) with the same normals and rotated indicator,
    deformed SynthMesh, cfg, deformed state dict)."""
    import neumesh_b200 as nb
    from neumesh_b200.neumesh import DEFAULT_MLP_ENGINE
    dev = _dev()
    engine = engine or DEFAULT_MLP_ENGINE
    cfg = synth.ModelConfig()
    mesh = synth.icosphere_mesh(level, seed=seed)
    sd = synth.make_state_dict(mesh, cfg, seed=seed + 1)
    model = helpers.cuda_model(mesh, cfg, sd, engine)
    o, d = synth.frame_rays(48, 48, view=3)
    with torch.no_grad():   # pack the field and build its certificate before the deformation
        nb.volume_render(o.to(dev), d.to(dev), model, calc_normal=True, white_bkgd=True)
    field = model._field.value
    moved = _wave(model.mesh_grid.vertices.clone(), phase)
    nb.deform_model(moved, model, dev)
    assert isinstance(model.indicator_vector, torch.nn.Parameter) and model.indicator_vector.requires_grad
    mesh_d = _host_mesh(moved, mesh.triangles, model.mesh_grid.vertex_normals)
    sd_d = dict(sd)
    sd_d["indicator_vector"] = model.indicator_vector.detach().cpu().clone()
    fresh = helpers.cuda_model(mesh_d, cfg, sd_d, engine)
    assert torch.equal(fresh.mesh_grid.vertex_normals, model.mesh_grid.vertex_normals)
    return model, fresh, mesh_d, cfg, sd_d, field


@pytest.mark.gpu
@pytest.mark.parametrize("calc_normal", [True, False])
def test_deformed_model_renders_like_a_fresh_model(calc_normal):
    from neumesh_b200.renderer import render_fused
    model, fresh, _, _, _, field = _deformed_pair()
    dev = _dev()
    o, d = synth.frame_rays(200, 200, view=5)
    o, d = o.to(dev), d.to(dev)
    R = o.shape[0]
    keys = ("rgb", "depth_volume", "mask_volume") + (("normals_volume",) if calc_normal else ())
    for chunk in (R, 8192):
        with torch.no_grad():
            a = render_fused(o, d, model, chunk=chunk, calc_normal=calc_normal, white_bkgd=True, bounded_near_far=True)
            b = render_fused(o, d, fresh, chunk=chunk, calc_normal=calc_normal, white_bkgd=True, bounded_near_far=True)
        for k in keys:
            assert torch.isfinite(a[k]).all(), k
            assert torch.equal(a[k], b[k]), f"chunk {chunk}: {k} of the deformed model differs from the fresh model"
    assert model._field.value == field, "the deformed model's field was re-created instead of re-packed"
    ca, Ba = model.shell_free_grid()
    cb, Bb = fresh.shell_free_grid()
    assert Ba == Bb and torch.equal(ca, cb), "shell certificate differs from the fresh model's"
    print(f"calc_normal={calc_normal}: {R} rays bit-identical in 1 and {math.ceil(R / 8192)} chunks; certificate cells "
          f"{int((ca == 1).sum())} outside / {int((ca == 2).sum())} inside")


@pytest.mark.gpu
def test_deformed_model_teacher_forced():
    model, _, mesh_d, cfg, sd_d, _ = _deformed_pair(level=4, phase=1.9, seed=23)
    f = helpers.oracle_field(mesh_d, cfg, sd_d)
    o, d = synth.frame_rays(40, 40, view=2)
    helpers.check_render_teacher_forced(model, mesh_d, cfg, sd_d, f, o, d, "deformed", ties_by_neighbours=True)


@pytest.mark.gpu
def test_texture_edit_on_a_deformed_main_model():
    import neumesh_b200 as nb
    from neumesh_b200 import texture_neumesh as tn
    dev = _dev()
    case = helpers.texture_edit_case()
    cfg = case["cfg"]

    def refs():
        return [helpers.cuda_model(m, cfg, sd, "tcgen05_f16") for m, sd in case["refs"]]

    main = helpers.cuda_model(case["main_mesh"], cfg, case["main_sd"], "tcgen05_f16")
    T = [t.to(dev) for t in case["T"]]
    edit = nb.TextureEditableNeuMesh(main, refs(), case["masks"].to(dev), case["codes"].to(dev), T).to(dev).eval()
    o, d = synth.frame_rays(160, 160, view=4)
    o, d = o.to(dev), d.to(dev)
    kw = dict(calc_normal=True, white_bkgd=True, bounded_near_far=True)
    with torch.no_grad():
        nb.volume_render(o, d, edit, **kw)
    handle = tn.packed_edit(edit).value
    moved = _wave(main.mesh_grid.vertices.clone(), 0.4)
    nb.deform_model(moved, main, dev)
    # the stale edit is refused until it is re-packed ...
    _check_refused_edit(main, tn._EDITS[edit].handle, dev)
    with torch.no_grad():
        rgb_a, depth_a, ex_a = nb.volume_render(o, d, edit, **kw)
    assert tn.packed_edit(edit).value == handle, "the edit was re-created instead of re-packed"
    mesh_d = _host_mesh(moved, case["main_mesh"].triangles, main.mesh_grid.vertex_normals)
    sd_d = dict(case["main_sd"])
    sd_d["indicator_vector"] = main.indicator_vector.detach().cpu().clone()
    main_f = helpers.cuda_model(mesh_d, cfg, sd_d, "tcgen05_f16")
    fresh = nb.TextureEditableNeuMesh(main_f, refs(), case["masks"].to(dev), case["codes"].to(dev), T).to(dev).eval()
    with torch.no_grad():
        rgb_b, depth_b, ex_b = nb.volume_render(o, d, fresh, **kw)
    assert torch.equal(rgb_a, rgb_b) and torch.equal(depth_a, depth_b)
    for k in ("mask_volume", "normals_volume"):
        assert torch.equal(ex_a[k], ex_b[k]), k


def _check_refused_edit(main, edit_handle, dev):
    """nmb_render_edit refuses an edit packed before the main grid's last update (the main field re-packed first)."""
    from neumesh_b200 import _lib
    field = main.packed_field()
    cfg = _lib.RenderCfg(obj_bounding_radius=1.0, N_samples=64, N_importance=64, N_upsample_iters=4)
    x = torch.zeros(1, 3, device=dev)
    y = torch.zeros(1, 3, device=dev)
    one = torch.zeros(1, device=dev)
    rc = _lib.lib().nmb_render_edit(field, edit_handle, ctypes.byref(cfg), _lib.ptr(x), _lib.ptr(x), 1, 1, _lib.ptr(y),
                                    _lib.ptr(one), _lib.ptr(one), None, None, None, 0, _lib.stream_ptr(dev))
    assert rc != 0 and b"nmb_edit_update" in _lib.lib().nmb_last_error(), _lib.lib().nmb_last_error()


@pytest.mark.gpu
def test_stale_field_is_refused():
    import neumesh_b200 as nb
    from neumesh_b200 import _lib
    dev = _dev()
    cfg = synth.ModelConfig()
    mesh = synth.icosphere_mesh(4, seed=2)
    sd = synth.make_state_dict(mesh, cfg, seed=3)
    model = helpers.cuda_model(mesh, cfg, sd, "tcgen05_f16")
    field = model.packed_field()
    mg = model.mesh_grid
    mg.deform_(_wave(mg.vertices.clone(), 0.3))   # the grid moves; the field is not re-packed
    L = _lib.lib()
    x = torch.zeros(4, 3, device=dev)
    s = torch.zeros(4, device=dev)
    rc = L.nmb_field_sdf(field, _lib.ptr(x), 4, _lib.ptr(s), None, _lib.stream_ptr(dev))
    assert rc != 0 and b"nmb_field_update" in L.nmb_last_error(), L.nmb_last_error()
    G, B = ctypes.c_int32(0), ctypes.c_float(0)
    assert L.nmb_field_shell_grid(field, None, ctypes.byref(G), ctypes.byref(B), _lib.stream_ptr(dev)) != 0
    idx = torch.zeros(4, 8, dtype=torch.int64, device=dev)
    w = torch.zeros(4, 8, device=dev)
    rgb = torch.zeros(4, 3, device=dev)
    rc = L.nmb_field_color(field, None, 0, _lib.ptr(s), _lib.ptr(idx), _lib.ptr(w), _lib.ptr(x), _lib.ptr(x), 4,
                           _lib.ptr(rgb), _lib.stream_ptr(dev))
    assert rc != 0 and b"nmb_field_update" in L.nmb_last_error()
    rcfg = _lib.RenderCfg(obj_bounding_radius=1.0, N_samples=64, N_importance=64, N_upsample_iters=4)
    rc = L.nmb_render(field, ctypes.byref(rcfg), _lib.ptr(x), _lib.ptr(x), 4, 4, _lib.ptr(rgb), _lib.ptr(s),
                      _lib.ptr(s), None, None, None, 0, _lib.stream_ptr(dev))
    assert rc != 0 and b"nmb_field_update" in L.nmb_last_error()
    # the Python layer re-packs: the same handle serves again
    with torch.no_grad():
        sdf = model.forward_density_only(x)
    assert model.packed_field().value == field.value and torch.isfinite(sdf).all()


@pytest.mark.gpu
def test_ten_deformations_allocate_nothing_after_the_first():
    import neumesh_b200 as nb
    from neumesh_b200 import _lib
    from neumesh_b200.renderer import render_fused
    dev = _dev()
    cfg = synth.ModelConfig()
    mesh = synth.icosphere_mesh(5, seed=4)
    model = helpers.cuda_model(mesh, cfg, synth.make_state_dict(mesh, cfg, seed=5), "tcgen05_f16")
    base = model.mesh_grid.vertices.clone()
    o, d = synth.frame_rays(256, 256, view=1)
    o, d = o.to(dev), d.to(dev)
    seen = []
    for frame in range(10):
        nb.deform_model(_wave(base, 0.3 * frame), model, dev)
        with torch.no_grad():
            out = render_fused(o, d, model, chunk=o.shape[0], calc_normal=True, white_bkgd=True, bounded_near_far=True)
        assert torch.isfinite(out["rgb"]).all()
        del out
        torch.cuda.synchronize()
        seen.append((torch.cuda.memory_allocated(dev), _lib.alloc_count(), model._field.value,
                     model.mesh_grid.grid.generation))
    print("per frame (torch bytes, library allocations):", [(s[0], s[1]) for s in seen])
    assert all(s[2] == seen[0][2] for s in seen), "the field handle changed: re-created instead of re-packed"
    assert [s[3] for s in seen] == list(range(1, 11))
    assert all(s[:2] == seen[0][:2] for s in seen[1:]), "a deformation after the first allocated device memory"
