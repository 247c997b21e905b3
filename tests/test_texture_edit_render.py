"""Fused render of texture-edited models (``nmb_render_edit``; ``editing/texture_neumesh/texture_neumesh.py:81-121``).

GPU: teacher-forced against the oracle (``oracle.texture.TextureEditOracle`` + the reference's compositing), per-sample
colours against the drop-in's point path, the reference's golden render, bit-for-bit properties at full size,
configurations the edit must cover, routing and re-packing.  CPU: eligibility decisions that need no device."""
import os

import numpy as np
import pytest
import torch

import helpers
from neumesh_b200 import synth

ENGINES = ["fp32", "tcgen05", "tcgen05_f16"]
RGB_TOL, DEPTH_TOL = 1e-4, 1e-5
TF_KW = dict(calc_normal=True, white_bkgd=True, bounded_near_far=True)
PROPS = ("rgb", "depth_volume", "mask_volume", "normals_volume")


def _dev():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (no CPU fallback exists)")
    return torch.device("cuda:0")


def _case(main_cfg=None, ref_cfgs=None, n_ref=2, rot=True, masks=None, main_level=4, seed=40):
    """helpers.texture_edit_case with every knob the configuration tests need (the defaults give the same inputs)."""
    main_cfg = main_cfg or synth.ModelConfig()
    ref_cfgs = ref_cfgs or [synth.ModelConfig()] * n_ref
    g = torch.Generator().manual_seed(seed)
    main_mesh = synth.icosphere_mesh(main_level, seed=seed)
    main_sd = synth.make_state_dict(main_mesh, main_cfg, seed=seed + 1)
    refs = []
    for j, (level, c) in enumerate(zip((3, 2), ref_cfgs)):
        m = synth.icosphere_mesh(level, seed=seed + 10 + j)
        refs.append((m, synth.make_state_dict(m, c, seed=seed + 20 + j), c))
    v = torch.from_numpy(main_mesh.vertices).float()
    mk = torch.stack([v[:, 0] > 0.1, v[:, 2] > 0.25])[:n_ref] if masks is None else masks(v)[:n_ref]
    codes = torch.randn(v.shape[0], ref_cfgs[0].color_dim, generator=g)
    T = []
    for _ in range(2):
        q, _r = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
        if torch.det(q) < 0:
            q[:, 0] = -q[:, 0]
        t = torch.eye(4)
        t[:3, :3] = q.float()
        t[:3, 3] = torch.randn(3, generator=g) * 0.1
        T.append(t)
    return dict(main_cfg=main_cfg, main_mesh=main_mesh, main_sd=main_sd, refs=refs, masks=mk, codes=codes,
                T=T[:n_ref] if rot else None)


def _oracle(case):
    from oracle.field import FieldOracle
    from oracle.texture import TextureEditOracle
    main = FieldOracle(case["main_mesh"].vertices, case["main_sd"], case["main_cfg"])
    refs = [FieldOracle(m.vertices, sd, c) for m, sd, c in case["refs"]]
    rot = torch.stack([t[:3, :3] for t in case["T"]]) if case["T"] is not None else None
    return TextureEditOracle(main, refs, case["masks"], case["codes"], rot)


def _models(case, engine="tcgen05_f16", dev="cuda:0", cls=None):
    import neumesh_b200 as nb
    main = helpers.cuda_model(case["main_mesh"], case["main_cfg"], case["main_sd"], engine, dev)
    refs = [helpers.cuda_model(m, c, sd, engine, dev) for m, sd, c in case["refs"]]
    T = [t.to(dev) for t in case["T"]] if case["T"] is not None else None
    cls = cls or nb.TextureEditableNeuMesh
    return cls(main, refs, case["masks"].to(dev), case["codes"].to(dev), T).to(dev).eval()


def _oracle_render(f, o, d, z_all):
    """Oracle field + the reference's compositing at the render's own sample depths (renderer.py:264-333)."""
    from oracle import render as orender
    dn = torch.nn.functional.normalize(d, dim=-1)
    pts = o[:, None, :] + z_all[..., None] * dn[:, None, :]
    z_mid = 0.5 * (z_all[..., 1:] + z_all[..., :-1])
    pm = o[:, None, :] + z_mid[..., None] * dn[:, None, :]
    N, P = z_all.shape
    sdf, nab = f.forward_with_nablas(pts.reshape(-1, 3))
    sdf, nab = sdf.reshape(N, P), nab.reshape(N, P, 3)
    cdf = torch.sigmoid(sdf * f.forward_s())
    alpha = ((cdf[..., :-1] - cdf[..., 1:]) / (cdf[..., :-1] + 1e-10)).clamp_min(0)
    _, rad = f.forward(pm.reshape(-1, 3), dn[:, None, :].expand_as(pm).reshape(-1, 3))
    rad = rad.reshape(N, P - 1, 3)
    w = orender.transmittance_weights(alpha)
    acc = w.sum(-1)
    rgb = (w[..., None] * rad).sum(-2) + (1 - acc[..., None])
    depth = (w / (acc[..., None] + 1e-10) * z_mid).sum(-1)
    normals = (torch.nn.functional.normalize(nab, dim=-1)[..., :-1, :] * w[..., None]).sum(-2)
    return rgb, depth, acc, normals, rad


def _check_teacher_forced(case, engine, rays=40, view=5, rays_od=None, tag=""):
    """Test 1's bars; returns the render's extras."""
    import neumesh_b200 as nb
    from neumesh_b200 import texture_neumesh
    dev = _dev()
    model = _models(case, engine)
    f = _oracle(case)
    o, d = rays_od if rays_od is not None else synth.frame_rays(rays, rays, view=view)
    with torch.no_grad():
        rgb, depth, ex = nb.volume_render(o.to(dev), d.to(dev), model, detailed_output=True, **TF_KW)
    assert model in texture_neumesh._EDITS, "the edit must render on the fused path"
    z_all = ex["d_all"].cpu()
    r_rgb, r_depth, r_acc, r_n, r_rad = _oracle_render(f, o, d, z_all)
    acc = ex["mask_volume"].cpu()
    solid = acc >= 0.5
    e_rgb = (rgb.cpu() - r_rgb).abs().max().item()
    dd = (depth.cpu() - r_depth).abs()
    e_nrm = (ex["normals_volume"].cpu() - r_n).abs().max().item()
    e_rad = (ex["radiance"].cpu() - r_rad).abs().amax(-1)
    # an exact fp32 distance tie between the 8th and 9th neighbour picks an implementation-defined vertex (see
    # test_gpu_parity.test_render_teacher_forced): a handful of samples may differ there
    n_bad = int((e_rad > 5e-6).sum())
    print(f"[{engine}{tag}] edit teacher-forced: rgb {e_rgb:.3e} depth(solid, {int(solid.sum())} rays) "
          f"max {dd[solid].max() if solid.any() else 0:.3e} normals {e_nrm:.3e}; per-sample radiance max "
          f"{e_rad.max():.3e}, {n_bad} of {e_rad.numel()} samples above 5e-6")
    assert e_rgb <= RGB_TOL
    if solid.any():
        assert dd[solid].quantile(0.99).item() <= DEPTH_TOL and dd[solid].max().item() <= 2 * DEPTH_TOL
    assert (dd * acc.clamp_min(1e-6)).max().item() <= DEPTH_TOL
    assert e_nrm <= 2.5e-4
    assert n_bad <= 16
    assert set(ex) >= {"rgb", "depth_volume", "mask_volume", "normals_volume", "implicit_nablas", "implicit_surface",
                       "radiance", "alpha", "cdf", "visibility_weights", "d_final", "d_all", "near_far"}
    return model, rgb, ex


# ---------------------------------------------------------------------------------------------------------------
# 1. teacher-forced against the oracle
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
def test_edit_render_teacher_forced(engine):
    import neumesh_b200 as nb
    case = _case()
    model, rgb, ex = _check_teacher_forced(case, engine)
    o, d = synth.frame_rays(40, 40, view=5)
    dev = _dev()
    with torch.no_grad():
        plain, _, _ = nb.volume_render(o.to(dev), d.to(dev), model.main_model, detailed_output=False, **TF_KW)
    changed = int(((rgb - plain).abs().amax(-1) > 1e-3).sum())
    hit = int((ex["mask_volume"] >= 0.5).sum())
    print(f"[{engine}] rays recoloured by the edit: {changed} of {hit} rays with acc >= 0.5")
    assert changed >= 0.2 * hit   # the caps cover 26 % of the object's rays in this view


# ---------------------------------------------------------------------------------------------------------------
# 2. against the drop-in's point path (TextureEditableNeuMesh.forward)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
def test_edit_radiance_matches_point_path(engine):
    import neumesh_b200 as nb
    dev = _dev()
    case = _case()
    model = _models(case, engine)
    o, d = synth.frame_rays(32, 32, view=5)
    with torch.no_grad():
        _, _, ex = nb.volume_render(o.to(dev), d.to(dev), model, detailed_output=True, **TF_KW)
    # the mid-points exactly as the kernels form them: F.normalize with separately rounded products / sums, then
    # o + z_mid * d (torch CPU elementwise ops round every step, as the kernels do)
    n = ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).sqrt().clamp_min(1e-12)
    dn = d / n[:, None]
    z = ex["d_all"].cpu()
    zm = 0.5 * (z[:, 1:] + z[:, :-1])
    xyz = (o[:, None, :] + zm[..., None] * dn[:, None, :]).reshape(-1, 3)
    dirs = dn[:, None, :].expand(-1, zm.shape[1], -1).reshape(-1, 3).contiguous()
    with torch.no_grad():
        _, c_pt = model.forward(xyz.to(dev), dirs.to(dev))
        _, _, _, idx, _ = model.main_model.forward(xyz.to(dev), dirs.to(dev), nablas_only=True, return_ds=True)
    painted = model.main_editing_masks[:, idx].any(-1).any(0).cpu()      # any reference paints any neighbour
    rad = ex["radiance"].reshape(-1, 3).cpu()
    c_pt = c_pt.cpu()
    err = (rad - c_pt).abs().amax(-1)
    print(f"[{engine}] radiance vs point path: {int(painted.sum())} of {painted.numel()} samples painted, max "
          f"{err[painted].max():.3e}; unpainted max {err[~painted].max():.3e}")
    assert painted.sum() > 1000 and (~painted).sum() > 1000
    assert torch.equal(rad[~painted], c_pt[~painted]), "same kernels, same neighbours -> same bits"
    assert err[painted].max().item() <= 1e-6


# ---------------------------------------------------------------------------------------------------------------
# 3. free-running against the reference's golden render
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_edit_render_vs_reference_golden(golden_dir):
    import neumesh_b200 as nb
    from neumesh_b200 import texture_neumesh
    dev = _dev()
    g = dict(np.load(os.path.join(golden_dir, "texture_edit_small.npz"), allow_pickle=False))
    case = _case(seed=int(g["seed"]))
    assert helpers.state_digest(case["main_sd"]) == str(g["digest_main"])
    model = _models(case)
    with torch.no_grad():
        r, d, _ = nb.volume_render(torch.from_numpy(g["rays_o"]).to(dev), torch.from_numpy(g["rays_d"]).to(dev), model,
                                   detailed_output=False, calc_normal=False, white_bkgd=True, bounded_near_far=True)
    assert model in texture_neumesh._EDITS
    dr = (r.cpu() - torch.from_numpy(g["render_rgb"])).abs().max(-1)[0]
    dd = (d.cpu() - torch.from_numpy(g["render_depth"])).abs()
    ok = ((dr <= RGB_TOL) & (dd <= DEPTH_TOL)).float().mean().item()
    print(f"edit render: rays within (1e-4, 1e-5) of the reference's golden: {ok:.3f}")
    assert 1.0 - ok <= 0.0565 + 3.0 * (0.0565 * 0.9435 / dr.numel()) ** 0.5 and dr.median() <= 1e-6


# ---------------------------------------------------------------------------------------------------------------
# 4. properties at full size, bit for bit
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_edit_full_size_properties():
    import neumesh_b200 as nb
    from neumesh_b200 import parallel
    from neumesh_b200.renderer import render_fused
    dev = _dev()
    case = _case(main_level=7, masks=lambda v: torch.stack([v[:, 0] > 0.2, v[:, 2] > 0.3]))
    model = _models(case)
    o, d = synth.frame_rays(256, 256, view=0)
    o, d = o.to(dev), d.to(dev)
    kw = dict(calc_normal=True, white_bkgd=True, bounded_near_far=True, detailed_output=False)
    with torch.no_grad():
        a = render_fused(o, d, model, chunk=o.shape[0], **kw)
        b = render_fused(o, d, model, chunk=8192, **kw)
        perm = torch.randperm(o.shape[0], device=dev)
        c = render_fused(o[perm], d[perm], model, chunk=32768, **kw)
        e = render_fused(o, d, model, chunk=o.shape[0], skip_dead_samples=False, **kw)
        plain = render_fused(o, d, model.main_model, **kw)
        _, _, vr = nb.volume_render(o, d, model, **kw)
        sh = parallel.render_sharded(o, d, model, **kw)
        zero = nb.TextureEditableNeuMesh(model.main_model, list(model.ref_models),
                                         torch.zeros_like(model.main_editing_masks), model.main_editing_colorfeats,
                                         [t.to(dev) for t in case["T"]])
        z = render_fused(o, d, zero, **kw)
    for k in PROPS:
        assert torch.isfinite(a[k]).all(), k
        assert torch.equal(a[k], b[k]), f"{k}: chunked render differs"
        assert torch.equal(a[k][perm], c[k]), f"{k}: permuted render differs"
        assert torch.equal(a[k], e[k]), f"{k}: live-sample path differs from the all-samples path"
        assert torch.equal(z[k], plain[k]), f"{k}: an edit that paints nothing differs from the plain render"
        assert torch.equal(sh[k], vr[k]), f"{k}: render_sharded (world size 1) differs from volume_render"
    assert int(((a["rgb"] - plain["rgb"]).abs().amax(-1) > 1e-3).sum()) > 1000


# ---------------------------------------------------------------------------------------------------------------
# 5. configurations
# ---------------------------------------------------------------------------------------------------------------
def _cfg(**kw):
    return synth.ModelConfig(**kw)


CONFIGS = {
    "ref_colour_config": dict(ref_cfgs=[_cfg(multires_view=2, D_color=3, multires_d=6), _cfg()]),
    "main_nonabla_ref_nabla": dict(main_cfg=_cfg(enable_nablas_input=False)),
    "main_nabla_ref_nonabla": dict(ref_cfgs=[_cfg(enable_nablas_input=False)] * 2),
    "color_dim_64": dict(main_cfg=_cfg(color_dim=64), ref_cfgs=[_cfg(color_dim=64)] * 2),
    "no_rotation": dict(rot=False),
    "one_reference": dict(n_ref=1),
    "all_true_mask": dict(masks=lambda v: torch.stack([torch.ones_like(v[:, 0], dtype=torch.bool), v[:, 2] > 0.25])),
    "reference_paints_nothing": dict(masks=lambda v: torch.stack([v[:, 0] > 0.1, torch.zeros_like(v[:, 0],
                                                                                                  dtype=torch.bool)])),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_edit_configurations_vs_oracle(name):
    _check_teacher_forced(_case(**CONFIGS[name]), "tcgen05_f16", rays=24, tag=" " + name)


@pytest.mark.gpu
def test_edit_all_rays_miss_vs_oracle():
    o = torch.tensor([[0.0, 0.0, 2.5]]).expand(400, 3).contiguous()
    g = torch.Generator().manual_seed(3)
    d = torch.nn.functional.normalize(torch.tensor([0.0, 0.0, 1.0]) + 0.2 * torch.randn(400, 3, generator=g), dim=-1)
    _, _, ex = _check_teacher_forced(_case(), "tcgen05_f16", rays_od=(o, d), tag=" miss")
    assert ex["mask_volume"].max().item() <= 1e-6


# ---------------------------------------------------------------------------------------------------------------
# 6. routing
# ---------------------------------------------------------------------------------------------------------------
def _todays_route(model, o, d, **kw):
    """The route volume_render keeps for edits outside nmb_render_edit: fused cascade on the main model, then the
    generic torch-op evaluation of the edit model in rayschunk pieces."""
    from neumesh_b200 import renderer as R
    d = torch.nn.functional.normalize(d, dim=-1)
    z = R.render_fused(o, d, model.main_model, normalize_dirs=False, min_chunk=4096, sampling_only=True,
                       bounded_near_far=kw["bounded_near_far"])["d_all"]
    pieces = []
    for s in range(0, o.shape[0], 4096):
        pieces.append(R._render_generic(
            o[s:s + 4096], d[s:s + 4096], model, dim_batchify=0, obj_bounding_radius=1.0,
            calc_normal=kw["calc_normal"], use_view_dirs=True, netchunk=1048576, white_bkgd=kw["white_bkgd"],
            near_bypass=None, far_bypass=None, detailed_output=False, perturb=False, N_samples=64, N_importance=64,
            N_upsample_iters=4, samples_output=False, bounded_near_far=kw["bounded_near_far"],
            random_color_direction=False, z_samples=z[s:s + 4096]))
    return {k: torch.cat([p[k] for p in pieces]) for k in pieces[0]}


@pytest.mark.gpu
def test_edit_routing():
    import torch.nn as nn

    import neumesh_b200 as nb
    from neumesh_b200 import texture_neumesh
    dev = _dev()
    o, d = synth.frame_rays(24, 24, view=5)
    o, d = o.to(dev), d.to(dev)
    kw = dict(calc_normal=True, white_bkgd=True, bounded_near_far=True)

    def check_generic(model):
        with torch.no_grad():
            _, _, out = nb.volume_render(o, d, model, detailed_output=False, rayschunk=4096, **kw)
            ref = _todays_route(model, o, d, **kw)
        assert model not in texture_neumesh._EDITS
        for k in PROPS:
            assert torch.equal(out[k], ref[k]), k
        return out

    # a reference model outside the fused kernels' specialisation
    wide = _case(ref_cfgs=[_cfg(W=128), _cfg()])
    check_generic(_models(wide))
    # fused_render = False
    m = _models(_case())
    m.fused_render = False
    slow = check_generic(m)

    # a stand-in with the five attributes (e.g. the reference's own class) takes the fused path
    class Standin(nn.Module):
        def __init__(self, main, refs, masks, codes, T):
            super().__init__()
            self.main_model, self.ref_models = main, nn.ModuleList(refs)
            self.main_editing_masks, self.main_editing_colorfeats = masks, codes
            self.rot_s_m = torch.stack([t[:3, :3] for t in T])

        def forward_s(self):
            return self.main_model.forward_s()

    s = _models(_case(), cls=Standin)
    m.fused_render = True
    with torch.no_grad():
        _, _, a = nb.volume_render(o, d, s, detailed_output=False, **kw)
        _, _, b = nb.volume_render(o, d, m, detailed_output=False, **kw)
    assert s in texture_neumesh._EDITS and m in texture_neumesh._EDITS
    for k in PROPS:
        assert torch.equal(a[k], b[k]), k
    assert (a["rgb"] - slow["rgb"]).abs().max().item() <= RGB_TOL


# ---------------------------------------------------------------------------------------------------------------
# 7. re-packing
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_edit_repacks_after_in_place_changes():
    import neumesh_b200 as nb
    dev = _dev()
    case = _case()
    model = _models(case)
    o, d = synth.frame_rays(24, 24, view=5)
    o, d = o.to(dev), d.to(dev)
    kw = dict(calc_normal=True, white_bkgd=True, bounded_near_far=True, detailed_output=False)

    def render(m):
        with torch.no_grad():
            return nb.volume_render(o, d, m, **kw)[2]

    def fresh():
        c = dict(case)
        c["main_sd"] = {k: v.cpu() for k, v in model.main_model.state_dict().items()}
        c["refs"] = [(mesh, {k: v.cpu() for k, v in r.state_dict().items()}, cfg)
                     for (mesh, _, cfg), r in zip(case["refs"], model.ref_models)]
        c["masks"], c["codes"] = model.main_editing_masks.cpu(), model.main_editing_colorfeats.cpu()
        return _models(c)

    before = render(model)
    steps = {
        "masks": lambda: model.main_editing_masks[0, :800].logical_not_(),
        "codes": lambda: model.main_editing_colorfeats.mul_(1.5),
        "reference colour weights": lambda: model.ref_models[0].color_linear[0].bias.add_(0.2),
    }
    for name, step in steps.items():
        with torch.no_grad():
            step()
        got, want = render(model), render(fresh())
        assert not torch.equal(got["rgb"], before["rgb"]), f"{name}: the change did not reach the render"
        for k in PROPS:
            assert torch.equal(got[k], want[k]), f"{name}: {k}"
        before = got
    # hot-swapped main mesh grid (same vertex count, moved vertices)
    mesh2 = synth.icosphere_mesh(4, seed=41)
    model.main_model.mesh_grid = nb.MeshGrid(mesh2, dev)
    case["main_mesh"] = mesh2
    got, want = render(model), render(fresh())
    assert not torch.equal(got["depth_volume"], before["depth_volume"])
    for k in PROPS:
        assert torch.equal(got[k], want[k]), f"mesh grid: {k}"


# ---------------------------------------------------------------------------------------------------------------
# CPU: eligibility
# ---------------------------------------------------------------------------------------------------------------
def _cpu_models(case):
    import neumesh_b200 as nb

    def build(mesh, cfg, sd):
        m = nb.NeuMesh(helpers.OracleMeshGrid(mesh), **cfg.model_kwargs())
        m.load_state_dict(sd, strict=True)
        return m.eval()

    main = build(case["main_mesh"], case["main_cfg"], case["main_sd"])
    refs = [build(m, c, sd) for m, sd, c in case["refs"]]
    return main, refs


def test_edit_eligibility_cpu():
    import neumesh_b200 as nb
    from neumesh_b200 import renderer as R
    from neumesh_b200 import texture_neumesh as tn
    case = _case()
    main, refs = _cpu_models(case)
    model = nb.TextureEditableNeuMesh(main, refs, case["masks"], case["codes"], case["T"])
    assert tn.is_edit_model(model) and model.fused_render is True
    assert not tn.is_edit_model(main)
    # a CPU edit model is never fused
    assert not tn.edit_fused_supported(model)
    assert not R.fused_eligible(model, torch.zeros(4, 3), batched=False, random_color_direction=False,
                                use_view_dirs=True, N_samples=64, N_importance=64, N_upsample_iters=4)
    with pytest.raises(ValueError, match="fused kernels"):
        tn.packed_edit(model)
    # shape errors are reported before anything touches a device
    wide = nb.TextureEditableNeuMesh(main, refs, case["masks"], torch.zeros(case["codes"].shape[0], 64), case["T"])
    with pytest.raises(ValueError, match="color_dim 32 but main_editing_colorfeats is 64 wide"):
        tn.packed_edit(wide)
    bad = nb.TextureEditableNeuMesh(main, refs, case["masks"][:1], case["codes"], case["T"])
    with pytest.raises(ValueError, match=r"expected \[n_ref, V_main\]"):
        tn.packed_edit(bad)
