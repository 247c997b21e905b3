"""Texture-editing blend path (SURVEY.md section 8f item 2; ``editing/texture_neumesh/texture_neumesh.py``).

CPU: the oracle restatement and this package's drop-in class (torch-op path over the test-only CPU mesh grid) against
``tests/golden/texture_edit_small.npz``, which the UNMODIFIED reference class produced.  GPU: the drop-in over CUDA
``NeuMesh`` models (``nmb_field_forward_ex`` + ``nmb_field_color``) against the oracle and the golden file."""
import os

import numpy as np
import pytest
import torch

import helpers
from neumesh_b200 import synth
from oracle import render as orender

NAME = "texture_edit_small.npz"
RKW = dict(calc_normal=False, white_bkgd=True, bounded_near_far=True)


def _golden(golden_dir):
    g = dict(np.load(os.path.join(golden_dir, NAME), allow_pickle=False))
    case = helpers.texture_edit_case(int(g["seed"]))
    assert helpers.state_digest(case["main_sd"]) == str(g["digest_main"])
    assert helpers.state_digest({"codes": case["codes"], "masks": case["masks"].float()}) == str(g["digest_codes"]), \
        "synthetic edit inputs are not reproducible on this platform"
    return g, case


def test_texture_oracle_matches_reference_golden(golden_dir):
    g, case = _golden(golden_dir)
    f = helpers.texture_edit_oracle(case)
    xyz, view = torch.from_numpy(g["xyz"]), torch.from_numpy(g["view_dirs"])
    sdf, rgb = f.forward(xyz, view)
    assert torch.equal(sdf, torch.from_numpy(g["sdf"]))
    assert torch.equal(rgb, torch.from_numpy(g["rgb"])), (rgb - torch.from_numpy(g["rgb"])).abs().max()
    # the edit really recolours a good part of the probe points
    assert ((torch.from_numpy(g["rgb"]) - torch.from_numpy(g["rgb_unedited"])).abs().max(-1)[0] > 1e-6).sum() > 100
    r, d, _ = orender.volume_render(torch.from_numpy(g["rays_o"]), torch.from_numpy(g["rays_d"]), f,
                                    detailed_output=False, **RKW)
    assert torch.equal(r, torch.from_numpy(g["render_rgb"])) and torch.equal(d, torch.from_numpy(g["render_depth"]))


def _dropin(case, device, engine="tcgen05"):
    import neumesh_b200 as nb
    kw = case["cfg"].model_kwargs()

    def build(mesh, sd):
        if device.type == "cuda":
            mg = nb.MeshGrid(mesh, device)
        else:
            mg = helpers.OracleMeshGrid(mesh)
        m = nb.NeuMesh(mg, mlp_engine=engine, **kw)
        m.load_state_dict(sd, strict=True)
        return m.to(device).eval()

    main = build(case["main_mesh"], case["main_sd"])
    refs = [build(m, sd) for m, sd in case["refs"]]
    model = nb.TextureEditableNeuMesh(main, refs, case["masks"].to(device), case["codes"].to(device),
                                      T_r_m_list=[T.to(device) for T in case["T"]])
    return model.to(device).eval()


def test_texture_dropin_torch_path_cpu(golden_dir):
    """Same constructor / protocol as the reference class; on CPU every call takes the torch-op path."""
    g, case = _golden(golden_dir)
    model = _dropin(case, torch.device("cpu"))
    xyz, view = torch.from_numpy(g["xyz"]), torch.from_numpy(g["view_dirs"])
    sdf, rgb = model.forward(xyz.clone(), view)
    assert (sdf.detach() - torch.from_numpy(g["sdf"])).abs().max() < 2e-6
    assert (rgb.detach() - torch.from_numpy(g["rgb"])).abs().max() < 2e-6
    for name in ("compute_distance", "forward_s", "forward_density_only", "forward_with_nablas"):
        assert hasattr(model, name)


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ["tcgen05", "fp32", "tcgen05_f16"])
def test_texture_dropin_fused_vs_oracle_and_golden(golden_dir, engine):
    import neumesh_b200 as nb
    from neumesh_b200 import _lib
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (no CPU fallback exists)")
    dev = torch.device("cuda:0")
    g, case = _golden(golden_dir)
    model = _dropin(case, dev, engine)
    f = helpers.texture_edit_oracle(case)
    xyz, view = torch.from_numpy(g["xyz"]), torch.from_numpy(g["view_dirs"])
    n0 = _lib.launch_count()
    with torch.no_grad():
        sdf, rgb = model.forward(xyz.to(dev), view.to(dev))
    assert _lib.launch_count() - n0 >= 8, "the edit path must run in the CUDA library, not in torch ops"
    e_sdf = (sdf.cpu() - torch.from_numpy(g["sdf"])).abs().max().item()
    e_rgb = (rgb.cpu() - torch.from_numpy(g["rgb"])).abs().max().item()
    print(f"[{engine}] texture edit, max-abs vs the reference's golden: sdf {e_sdf:.2e} rgb {e_rgb:.2e}")
    assert e_sdf < 5e-6 and e_rgb < 5e-6
    # bigger probe against the oracle, incl. points with no painted neighbour at all
    x2, v2 = helpers.sample_points(4000, seed=77)
    with torch.no_grad():
        s2, c2 = model.forward(x2.to(dev), v2.to(dev))
    s_ref, c_ref = f.forward(x2, v2)
    assert (s2.cpu() - s_ref).abs().max() < 5e-6 and (c2.cpu() - c_ref).abs().max() < 5e-6
    # forward_color on the model's own table == the colour forward() returns; and on a foreign table
    main = model.main_model
    with torch.no_grad():
        sdf_m, nab, ds, idx, w = main.forward(x2.to(dev), v2.to(dev), nablas_only=True, return_ds=True)
        own = main.forward_color(ds, v2.to(dev), main.color_features, indices=idx, weights=w, nabla=nab)
        _, direct = main.forward(x2.to(dev), v2.to(dev))
        foreign = main.forward_color(ds, v2.to(dev), case["codes"].to(dev), indices=idx, weights=w, nabla=nab)
    assert idx.dtype == torch.int64 and ds.shape == (4000, 1) and w.shape == (4000, 8)
    assert torch.equal(own, direct), "same inputs through either entry point -> same bits"
    fm = f.main
    s_o, n_o, d_emb, ds_o, idx_o, w_o = fm._sdf_nabla(x2)
    assert torch.equal(idx.cpu(), idx_o) and (ds.cpu() - ds_o).abs().max() < 1e-6
    c_foreign = fm._color_from(d_emb, v2, idx_o, w_o, n_o, table=case["codes"])
    assert (foreign.cpu() - c_foreign).abs().max() < 5e-6
    # render through the generic renderer (the model is not a NeuMesh): free-running against the golden render
    with torch.no_grad():
        r, d, ex = nb.volume_render(torch.from_numpy(g["rays_o"]).to(dev), torch.from_numpy(g["rays_d"]).to(dev), model,
                                    detailed_output=False, **RKW)
    dr = (r.cpu() - torch.from_numpy(g["render_rgb"])).abs().max(-1)[0]
    dd = (d.cpu() - torch.from_numpy(g["render_depth"])).abs()
    ok = ((dr <= 1e-4) & (dd <= 1e-5)).float().mean().item()
    print(f"[{engine}] texture edit render: rays within (1e-4, 1e-5) of the reference's golden: {ok:.3f}")
    # 100 rays: floor of the unmodified reference on a full frame (0.0565, tests/golden/frame_config1.npz) + 3 binomial sigmas
    assert 1.0 - ok <= 0.0565 + 3.0 * (0.0565 * 0.9435 / dr.numel()) ** 0.5 and dr.median() <= 1e-6
