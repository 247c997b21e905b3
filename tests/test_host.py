"""CPU tests of the host-side logic: C-ABI exports, state_dict compatibility, generic renderer path, synthetic data."""
import ctypes
import os
import re
import types

import numpy as np
import pytest
import torch

import helpers
from neumesh_b200 import _lib, synth
from neumesh_b200 import renderer as nbr
from oracle import render as orender

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# reference NeuMesh.state_dict() keys (SURVEY.md section 5; verified there by instantiating the reference class)
REFERENCE_KEYS = ["ln_s", "geometry_features", "color_features", "indicator_vector"] + \
    [f"pts_linears.{p}.{s}" for p in ("0", "2.0", "3.0") for s in ("bias", "weight_g", "weight_v")] + \
    [f"density_linear.{s}" for s in ("bias", "weight_g", "weight_v")] + \
    [f"views_linears.{p}.{s}" for p in ("0", "2.0", "3.0", "4.0") for s in ("weight", "bias")] + \
    ["color_linear.0.weight", "color_linear.0.bias"]


def test_library_loads_and_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "neumesh_b200.h")).read()
    declared = set(re.findall(r"\b(nmb_[a-z_0-9]+)\s*\(", header))
    declared -= {"nmb_render_workspace_bytes"} - declared  # no-op, keeps the set explicit
    lib = _lib.lib()
    assert lib.nmb_version() == 100
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/neumesh_b200.h but not exported"
        assert name in _lib.SIGNATURES, f"{name} has no ctypes signature in neumesh_b200/_lib.py"
    assert set(_lib.SIGNATURES) <= declared
    assert lib.nmb_launch_count() == 0 or lib.nmb_launch_count() > 0


def test_no_cpu_fallback_without_cuda():
    if torch.cuda.is_available():
        pytest.skip("this check is for CPU-only hosts")
    out = ctypes.c_void_p()
    v = (ctypes.c_float * 30)()
    rc = _lib.lib().nmb_grid_create(ctypes.cast(v, ctypes.c_void_p), 10, None, ctypes.byref(out))
    assert rc != 0 and b"no CUDA device" in _lib.lib().nmb_last_error()
    import neumesh_b200 as nb
    with pytest.raises(RuntimeError):
        nb.MeshGrid(synth.icosphere_mesh(1), torch.device("cpu"))


class _FakeGrid:  # the NeuMesh constructor only needs the vertex count and normals
    def get_number_of_vertices(self):
        return 42

    def get_vertex_normal_torch(self):
        return torch.zeros(42, 3)


class _FakeCudaGrid(_FakeGrid):  # passes where only a CUDA MeshGrid's presence is checked (NeuMesh.fused_supported)
    grid = types.SimpleNamespace(handle=None)


def test_state_dict_keys_match_reference():
    import neumesh_b200 as nb
    cfg = synth.ModelConfig()
    m = nb.NeuMesh(_FakeGrid(), **cfg.model_kwargs())
    assert sorted(m.state_dict().keys()) == sorted(REFERENCE_KEYS)
    mesh = synth.icosphere_mesh(1)
    sd = synth.make_state_dict(mesh, cfg)
    assert sorted(sd.keys()) == sorted(REFERENCE_KEYS)
    m.load_state_dict(sd, strict=True)
    cfg2 = synth.ModelConfig(learn_indicator_weight=True)
    m2 = nb.NeuMesh(_FakeGrid(), **cfg2.model_kwargs())
    assert "indicator_weight_raw" in m2.state_dict()


def test_fused_supported_asks_the_library():
    """``fused_supported()`` agrees with the limits the field engine tests state (``helpers.inside``) on every row of
    their configuration matrix and limit cases, on every engine, on a host without a GPU.  One model per configuration:
    ``mlp_engine`` is re-assigned between the engines."""
    import neumesh_b200 as nb
    engines = ["tcgen05_f16", "tcgen05", "fp32"]
    for name, kw in list(helpers.ROWS.items()) + list(helpers.LIMITS.items()):
        cfg = synth.ModelConfig(**kw)
        m = nb.NeuMesh(_FakeCudaGrid(), **cfg.model_kwargs())
        for i, engine in enumerate(engines):
            m.mlp_engine = engine
            assert m.fused_supported() == helpers.inside(engine, cfg), (name, engine)
            if name in helpers.EXPECT_INSIDE:
                assert m.fused_supported() == bool(helpers.EXPECT_INSIDE[name][i]), (name, engine)
    # what the descriptor does not carry is decided before the library is asked
    assert not nb.NeuMesh(_FakeGrid(), **synth.ModelConfig().model_kwargs()).fused_supported()
    assert not nb.NeuMesh(_FakeCudaGrid(), input_view_dim=2, **synth.ModelConfig().model_kwargs()).fused_supported()
    # the library names the limit; packed_field raises with it before touching a device
    wide = nb.NeuMesh(_FakeCudaGrid(), **synth.ModelConfig(W=128).model_kwargs())
    assert not wide.fused_supported()
    d = wide._field_desc()
    assert _lib.lib().nmb_field_check(ctypes.byref(d), 2) == 2
    assert b"W = 256" in _lib.lib().nmb_last_error()
    with pytest.raises(RuntimeError, match="W = 256"):
        wide.packed_field()


def test_volume_render_routing(monkeypatch):
    """The fused route ``volume_render`` takes, over models x grad mode x every argument its conditions read.
    R: ``nmb_render`` renders the whole call (``fused_eligible``); M / S: the fused sampling cascade runs on the edit's
    main model / on the model itself, the generic path evaluates the samples (``fused_cascade_model``); G: the generic
    path throughout.  Stand-ins replace the CUDA tensors; the expected routes are written out by hand."""
    import neumesh_b200 as nb
    cuda = types.SimpleNamespace(is_cuda=True)

    def neumesh(cuda_tables, W=256):
        m = nb.NeuMesh(_FakeCudaGrid(), **synth.ModelConfig(W=W).model_kwargs())
        if cuda_tables:
            m.__dict__["geometry_features"] = cuda   # shadows the CPU parameter where .is_cuda is read
        return m

    class Edit:   # the attributes of a texture-edit model; `eligible` stands for what edit_fused_supported checks
        def __init__(self, main, eligible=True, fused_render=True):
            self.main_model, self.ref_models = main, [main]
            self.main_editing_masks = self.main_editing_colorfeats = self.rot_s_m = None
            self.eligible, self.fused_render = eligible, fused_render

    monkeypatch.setattr(nbr, "edit_fused_supported", lambda m: m.eligible and m.main_model.geometry_features.is_cuda)

    def models(cuda_tables=True):
        # NeuMesh, NeuMesh with W = 128, eligible edit, ineligible edit, edit with fused_render = False, foreign model
        return [neumesh(cuda_tables), neumesh(cuda_tables, W=128), Edit(neumesh(cuda_tables)),
                Edit(neumesh(cuda_tables), eligible=False), Edit(neumesh(cuda_tables), fused_render=False),
                torch.nn.Linear(1, 1)]

    def rays(batch=None, on_cuda=True):
        return types.SimpleNamespace(is_cuda=on_cuda, shape=(4, 3) if batch is None else (batch, 4, 3))

    # name: (keyword changes, routes of the six models without grad, routes in grad mode)
    table = {
        "defaults": (dict(), "RGRMMG", "SGGGGG"),
        "random_color_direction": (dict(random_color_direction=True), "GGGGGG", "SGGGGG"),
        "no view dirs": (dict(use_view_dirs=False), "GGGGGG", "GGGGGG"),
        "batched, B = 1": (dict(batched=True, rays_o=rays(1)), "RGRMMG", "SGGGGG"),
        "batched, B = 2": (dict(batched=True, rays_o=rays(2)), "GGGGGG", "GGGGGG"),
        "N_samples = 2": (dict(N_samples=2), "RGRMMG", "SGGGGG"),
        "N_samples = 1": (dict(N_samples=1), "GGGGGG", "GGGGGG"),
        "no up-sampling": (dict(N_upsample_iters=0), "RGRMMG", "SGGGGG"),
        "N_importance not divisible": (dict(N_upsample_iters=3), "GGGGGG", "GGGGGG"),
        # nmb_render rejects a negative count, so neither fused route may take it
        "N_upsample_iters < 0": (dict(N_upsample_iters=-1), "GGGGGG", "GGGGGG"),
        "z_samples given": (dict(z_samples=torch.zeros(4, 128)), "RGRGGG", "GGGGGG"),
        "rays on the CPU": (dict(rays_o=rays(on_cuda=False)), "GGGGGG", "GGGGGG"),
        "tables on the CPU": (dict(cuda_tables=False), "GGGGGG", "GGGGGG"),
    }
    for name, (change, want_nograd, want_grad) in table.items():
        kw = dict(rays_o=rays(), batched=False, random_color_direction=False, use_view_dirs=True, N_samples=64,
                  N_importance=64, N_upsample_iters=4, z_samples=None, cuda_tables=True)
        kw.update(change)
        rays_o, z_samples, ms = kw.pop("rays_o"), kw.pop("z_samples"), models(kw.pop("cuda_tables"))
        for grad, want in ((False, want_nograd), (True, want_grad)):
            got = ""
            for m in ms:
                with torch.set_grad_enabled(grad):
                    if nbr.fused_eligible(m, rays_o, **kw):
                        got += "R"
                        continue
                    geo = nbr.fused_cascade_model(m, rays_o, z_samples=z_samples, **kw)
                got += "G" if geo is None else "S" if geo is m else "M" if geo is m.main_model else "?"
            assert got == want, (name, "grad" if grad else "no grad", got, want)


def test_generic_renderer_path_equals_oracle(golden_dir):
    """volume_render's torch-op path (used for arbitrary models / training) driven by the oracle field on CPU."""
    g, mesh, cfg, sd, kw = helpers.golden_case(os.path.join(golden_dir, "scan63like_small.npz"))
    f = helpers.oracle_field(mesh, cfg, sd)
    o, d = torch.from_numpy(g["rays_o"]), torch.from_numpy(g["rays_d"])
    with torch.no_grad():
        rgb, depth, ex = nbr.volume_render(o, d, f, detailed_output=True, rayschunk=50, **kw)
    assert torch.equal(rgb, torch.from_numpy(g["render_rgb"]))
    assert torch.equal(depth, torch.from_numpy(g["render_depth"]))
    assert torch.equal(ex["normals_volume"], torch.from_numpy(g["render_normals"]))
    # batched [1, N, 3] form used by train.py / render.py
    with torch.no_grad():
        rgb_b, depth_b, _ = nbr.volume_render(o[None], d[None], f, batched=True, detailed_output=False, **kw)
    assert rgb_b.shape == (1, o.shape[0], 3) and torch.equal(rgb_b[0], rgb)


def test_batchify_query_shapes():
    fn = lambda x, y: (x.sum(-1, keepdim=True), {"a": y * 2})  # noqa: E731
    x, y = torch.rand(7, 5, 3), torch.rand(7, 5, 2)
    s, d = nbr.batchify_query(fn, x, y, chunk=4, dim_batchify=0)
    assert s.shape == (7, 5, 1) and d["a"].shape == (7, 5, 2) and torch.equal(d["a"], y * 2)


def test_synthetic_mesh_and_rays():
    mesh = synth.icosphere_mesh(3, seed=0)
    assert mesh.vertices.shape == (642, 3) and mesh.triangles.shape == (1280, 3)
    n = mesh.vertex_normals
    assert np.allclose(np.linalg.norm(n, axis=1), 1.0, atol=1e-9)
    assert ((n * mesh.vertices).sum(1) > 0.3).all()  # outward
    o, d = synth.frame_rays(16, 16)
    assert o.shape == (256, 3) and torch.allclose(d.norm(dim=-1), torch.ones(256), atol=1e-6)
    # the centre ray points at the origin
    c = d.reshape(16, 16, 3)[8, 8]
    assert torch.allclose(torch.nn.functional.normalize(-o[0], dim=0), c, atol=0.05)


def test_trained_like_fixture_is_sdf_like():
    cfg = synth.ModelConfig()
    mesh = synth.icosphere_mesh(3, seed=0)
    f = helpers.oracle_field(mesh, cfg, synth.make_state_dict(mesh, cfg))
    x, _ = helpers.sample_points(400, seed=2)
    ds, _, _ = f.compute_distance(x)
    sdf = f.forward_density_only(x)
    assert (sdf - ds).abs().max() < 0.05


def test_render_fused_empty_shard_needs_no_library_call():
    """A rank whose block-cyclic shard is empty (n_rays < 128 * world) must return empty outputs instead of handing
    null pointers to ``nmb_render`` - the other ranks would otherwise hang in the image all-gather."""
    from neumesh_b200 import parallel
    from neumesh_b200.renderer import render_fused
    assert parallel.shard_count(512, 5, 8) == 0 and parallel.shard_count(512, 3, 8) == 128
    e = torch.empty(0, 3)
    out = render_fused(e, e, model=None, calc_normal=True, detailed_output=True, samples_output=True)
    assert out["rgb"].shape == (0, 3) and out["depth_volume"].shape == (0,) and out["normals_volume"].shape == (0, 3)
    assert out["implicit_nablas"].shape == (0, 128, 3) and out["colors"].shape == (0, 127, 3)
    full = parallel.gather_image({k: out[k] for k in ("rgb", "depth_volume", "mask_volume", "normals_volume")}, 0, 0, 1)
    assert full["rgb"].shape == (0, 3)
    # the sampling cascade alone (volume_render's route for texture edits and training steps) keeps its own keys
    out = render_fused(e, e, model=None, sampling_only=True)
    assert list(out) == ["d_all", "implicit_surface", "near_far"]
    assert out["d_all"].shape == (0, 128) and out["implicit_surface"].shape == (0, 128) and out["near_far"].shape == (0, 2)


def test_clock_sampler_reports_only_samples_of_the_timed_region():
    """bench.py starts `nvidia-smi -lms` before the warm-up (its start-up stalls driver calls) and must report only the
    samples taken after `mark()`: the warm-up clocks and throttle reasons do not describe the timed steps."""
    import bench

    class _Proc:
        def terminate(self):
            pass

        def wait(self, timeout=None):
            return 0

    s = bench.ClockSampler(0)
    s.proc = _Proc()
    s.lines = ["0, 1200, 1965, 300.0, Not Active, Active, Not Active, Not Active\n"] * 3     # start-up / warm-up
    s.mark()
    s.lines += ["0, 1950, 1965, 800.0, Not Active, Not Active, Not Active, Active\n",
                "0, 1920, 1965, 790.0, Not Active, Not Active, Not Active, Active\n",
                "garbage line\n"]
    out = s.stop()
    assert out["samples"] == 2 and out["sm_mhz"] == 1935.0 and out["sm_max_mhz"] == 1965.0
    assert out["reasons"] == ["sw_power_cap"]          # the warm-up's hw_thermal_slowdown is not reported
    # without nvidia-smi the bench still prints a line
    t = bench.ClockSampler(0)
    t.wait_ready(0.01)
    t.mark()
    assert t.stop()["reasons"] == ["nvidia-smi unavailable"]
