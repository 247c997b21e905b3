"""CPU tests: the oracle is pinned, bit for bit, against the committed golden vectors that the UNMODIFIED reference
produced (``tests/golden/make_golden.py``)."""
import os

import numpy as np
import pytest
import torch

import helpers
from neumesh_b200 import synth
from oracle import knn as oknn
from oracle import render as orender

GOLDEN = ["scan63like_small.npz", "nonabla_unbounded.npz"]


@pytest.mark.parametrize("name", GOLDEN)
def test_oracle_field_matches_reference_golden(golden_dir, name):
    g, mesh, cfg, sd, kw = helpers.golden_case(os.path.join(golden_dir, name))
    f = helpers.oracle_field(mesh, cfg, sd)
    xyz, view = torch.from_numpy(g["xyz"]), torch.from_numpy(g["view_dirs"])
    ds, idx, w = f.compute_distance(xyz)
    assert torch.equal(idx, torch.from_numpy(g["idx"]))
    assert torch.equal(ds, torch.from_numpy(g["ds"]))
    assert torch.equal(w, torch.from_numpy(g["w"]))
    assert torch.equal(f.forward_density_only(xyz), torch.from_numpy(g["sdf"]))
    sdf, nabla = f.forward_with_nablas(xyz)
    assert torch.equal(nabla, torch.from_numpy(g["nabla"]))
    sdf2, rgb = f.forward(xyz, view)
    assert torch.equal(rgb, torch.from_numpy(g["rgb_pts"]))
    assert torch.equal(sdf2, torch.from_numpy(g["sdf_forward"]))


@pytest.mark.parametrize("name", GOLDEN)
def test_oracle_render_matches_reference_golden(golden_dir, name):
    g, mesh, cfg, sd, kw = helpers.golden_case(os.path.join(golden_dir, name))
    f = helpers.oracle_field(mesh, cfg, sd)
    rgb, depth, ex = orender.volume_render(torch.from_numpy(g["rays_o"]), torch.from_numpy(g["rays_d"]), f,
                                           detailed_output=True, **kw)
    # bit-exact: same torch ops in the same order on the same platform
    assert torch.equal(rgb, torch.from_numpy(g["render_rgb"]))
    assert torch.equal(depth, torch.from_numpy(g["render_depth"]))
    assert torch.equal(ex["mask_volume"], torch.from_numpy(g["render_acc"]))
    assert torch.equal(ex["d_final"], torch.from_numpy(g["render_d_final"]))
    if "render_normals" in g:
        assert torch.equal(ex["normals_volume"], torch.from_numpy(g["render_normals"]))


def test_knn_oracle_brute_vs_kdtree():
    mesh = synth.icosphere_mesh(4, seed=3)
    p = torch.from_numpy(mesh.vertices).float()
    q, _ = helpers.sample_points(3000, seed=7)
    d_b, i_b = oknn.knn_exact(q, p, 8, method="brute")
    d_k, i_k = oknn.knn_exact(q, p, 8, method="kdtree")
    assert torch.equal(i_b, i_k) and torch.equal(d_b, d_k)
    assert (d_b[:, 1:] >= d_b[:, :-1]).all()
    # frnn call-site contract (mesh_grid.py:109-119): batch dim 1, squared distances, int64, 4-tuple
    dists, idxs, nn_, grid = oknn.frnn_grid_points(q[None], p[None], None, None, K=8, r=100.0, grid=None)
    assert dists.shape == (1, 3000, 8) and idxs.dtype == torch.int64 and nn_ is None and grid is not None
    assert torch.allclose(dists[0, :, 0], ((q - p[idxs[0, :, 0]]) ** 2).sum(-1), atol=1e-7)


def _pin_case(golden_dir):
    g = dict(np.load(os.path.join(golden_dir, "oracle_pin_small.npz"), allow_pickle=False))
    cfg = synth.ModelConfig()
    mesh = synth.icosphere_mesh(int(g["level"]), seed=int(g["seed"]))
    sd = synth.make_state_dict(mesh, cfg, seed=int(g["seed"]) + 1)
    assert helpers.state_digest(sd) == str(g["state_digest"]), "synthetic state_dict is not reproducible on this platform"
    return g, mesh, cfg, sd


def test_oracle_vs_unmodified_reference(golden_dir):
    """Bit for bit against the outputs of the unmodified reference (``tests/golden/make_golden.py oracle_pin``)."""
    g, mesh, cfg, sd = _pin_case(golden_dir)
    f = helpers.oracle_field(mesh, cfg, sd)
    x, v = helpers.sample_points(500, seed=1)
    assert torch.equal(f.forward_density_only(x), torch.from_numpy(g["pts_density_only"]))
    s_o, n_o = f.forward_with_nablas(x)
    assert torch.equal(n_o, torch.from_numpy(g["pts_nabla"])) and torch.equal(s_o, torch.from_numpy(g["pts_sdf_with_nabla"]))
    _, c_o = f.forward(x, v)
    assert torch.equal(c_o, torch.from_numpy(g["pts_rgb"]))
    o, d = synth.frame_rays(10, 10, view=1)
    kw = dict(calc_normal=True, white_bkgd=True, bounded_near_far=True)
    rgb_o, dep_o, ex_o = orender.volume_render(o, d, f, detailed_output=True, rayschunk=64, **kw)
    for k in ("rgb", "depth_volume", "mask_volume", "normals_volume", "d_final", "implicit_surface", "radiance"):
        assert torch.equal(torch.from_numpy(g["render_" + k]), ex_o[k]), k
    # sample_pdf on its own, incl. the u = 0 / u = 1 ends (SURVEY.md section 8a')
    bins, wts = torch.from_numpy(g["pdf_bins"]), torch.from_numpy(g["pdf_weights"])
    assert torch.equal(torch.from_numpy(g["pdf_samples"]), orender.inverse_cdf_samples(bins, wts, 16))


def test_dropin_render_and_trainer_loss_match_reference_golden(golden_dir):
    """INTEGRATION.md section 3 end to end, as far as a CPU allows: the drop-in renderer and ``neumesh_b200.NeuMesh``
    (over the CPU mesh grid) reproduce the unmodified reference's render and its output keys, no-grad and under autograd
    with ``perturb=True``, and the training losses back-propagate to every parameter."""
    import neumesh_b200 as nb
    g, mesh, cfg, sd = _pin_case(golden_dir)
    ours = nb.NeuMesh(helpers.OracleMeshGrid(mesh), **cfg.model_kwargs())
    ours.load_state_dict(sd, strict=True)      # identical state_dict keys
    ours.eval()
    o, d = synth.frame_rays(8, 8, view=2)
    kw = dict(calc_normal=True, white_bkgd=True, bounded_near_far=True, detailed_output=True, rayschunk=64)
    with torch.no_grad():
        rgb_n, dep_n, ex_n = nb.volume_render(o, d, ours, **kw)
    assert set(str(k) for k in g["small_keys"]) <= set(ex_n.keys()) | {"near_far"}
    assert (rgb_n - torch.from_numpy(g["small_rgb"])).abs().max() < 1e-5
    assert (dep_n - torch.from_numpy(g["small_depth"])).abs().max() < 1e-5
    # training-style call: grad enabled, perturb=True (the reference's default), samples_output for the distillation loss
    ours.train()
    ours.fused_train = False
    torch.manual_seed(3)
    rgb_t, dep_t, ex_t = nb.volume_render(o, d, ours, calc_normal=True, detailed_output=True, samples_output=True,
                                          perturb=True, rayschunk=64)
    assert set(str(k) for k in g["train_keys"]) <= set(ex_t.keys()) | {"near_far"}
    assert {"xyz", "dirs", "density", "colors", "implicit_nablas"} <= set(ex_t.keys())
    loss = helpers.train_loss(rgb_t, dep_t, ex_t) + ex_t["density"].abs().mean() + ex_t["colors"].mean()
    loss.backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for n, p in ours.named_parameters()
               if n != "indicator_weight_raw")


def test_oracle_perturb_with_injected_uniforms_equals_reference_with_patched_rand(golden_dir):
    """perturb=True (rend_util.py:292-295) draws ``torch.rand`` once per up-sampling iteration; the oracle takes the draws
    as ``perturb_u``.  The reference rendered with ``torch.rand`` patched to hand it the same draws: both renders are
    bit-identical."""
    g, mesh, cfg, sd = _pin_case(golden_dir)
    f = helpers.oracle_field(mesh, cfg, sd)
    o, d = synth.frame_rays(9, 9, view=4)
    u = torch.rand(4, o.shape[0], 16, generator=torch.Generator().manual_seed(11))
    assert torch.equal(u, torch.from_numpy(g["perturb_u"]))
    kw = dict(calc_normal=True, white_bkgd=False, bounded_near_far=True)
    rgb_o, dep_o, ex_o = orender.volume_render(o, d, f, detailed_output=True, perturb_u=u, **kw)
    assert torch.equal(torch.from_numpy(g["perturb_rgb"]), rgb_o) and torch.equal(torch.from_numpy(g["perturb_depth"]), dep_o)
    assert torch.equal(torch.from_numpy(g["perturb_d_final"]), ex_o["d_final"])
    # and it differs from the deterministic render (the draws are used)
    rgb_d, _, _ = orender.volume_render(o, d, f, **kw)
    assert not torch.equal(rgb_d, rgb_o)
