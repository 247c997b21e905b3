"""Frame-scale golden renders of the UNMODIFIED reference (the checkout named by ``NEUMESH_REFERENCE_ROOT`` imported verbatim on CPU through
``ref_harness``) for BASELINE.json configs 1 / 3 / 5, together with the reference's OWN noise floor.

For each config a strided subset of the rays of a real 800 x 800 spiral frame is rendered twice by the reference
renderer (``models/renderer.py::volume_render``) over the reference ``NeuMesh``:

* ``clean``  - as is;
* ``noisy``  - with ``forward_density_only`` (the no-grad sampling cascade's only input) perturbed by Gaussian noise of
  sigma = 4e-7, the level at which two fp32 evaluations of the same sdf network differ (MKL sgemm vs the CUDA kernels:
  max 1.1e-6 over 5 000 points, ``tests/test_gpu_parity.py::test_field_vs_oracle``).

``tests/test_gpu_parity.py::test_frame_parity_vs_reference_noise_floor`` then asserts that the CUDA path's outlier rate
(rays outside 1e-4 RGB / 1e-5 depth of ``clean``) does not exceed the reference's self-noise outlier rate
(``noisy`` vs ``clean``) by more than 3 binomial sigmas.

Run with the reference checkout present (minutes of CPU):  ``NEUMESH_REFERENCE_ROOT=... python tests/golden/make_frame_golden.py [config1|config3|config5]``.
"""
from __future__ import annotations

import os
import sys
import time
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
warnings.filterwarnings("ignore")

import ref_harness  # noqa: E402
from make_golden import state_digest  # noqa: E402
from neumesh_b200 import synth  # noqa: E402

NOISE_SIGMA = 4e-7

# name -> (mesh level, ModelConfig kwargs, render kwargs, number of rays, view)
CASES = {
    "config1": (7, {}, dict(calc_normal=True, white_bkgd=True, bounded_near_far=True), 20000, 0),
    "config3": (7, dict(geometry_dim=256, color_dim=256), dict(calc_normal=True, white_bkgd=True, bounded_near_far=True),
                6000, 11),
    "config5": (9, {}, dict(calc_normal=True, white_bkgd=True, bounded_near_far=True, N_samples=128, N_importance=128,
                            N_upsample_iters=4), 4000, 0),
}


def frame_subset(n_rays, view):
    o, d = synth.frame_rays(800, 800, view=view)
    # a strided subset that covers the whole frame; odd stride so that every image column is visited
    stride = max(1, (640000 // n_rays) | 1)
    sel = torch.arange(0, 640000, stride)[:n_rays]
    return sel, o[sel].contiguous(), d[sel].contiguous()


class NoisyDensity:
    """Wraps a reference model: the sampling cascade sees sdf + N(0, sigma^2); everything else is untouched."""

    def __init__(self, base, sigma, seed):
        self.b, self.sigma, self.g = base, sigma, torch.Generator().manual_seed(seed)

    def __getattr__(self, k):
        return getattr(self.b, k)

    def forward_density_only(self, x):
        y = self.b.forward_density_only(x)
        return y + self.sigma * torch.randn(y.shape, generator=self.g)


def make(name):
    level, cfg_kw, kw, n_rays, view = CASES[name]
    ns = ref_harness.load()
    cfg = synth.ModelConfig(**cfg_kw)
    mesh = synth.icosphere_mesh(level, seed=0)
    sd = synth.make_state_dict(mesh, cfg, seed=1)
    model = ref_harness.build_reference_model(mesh, cfg, sd)
    sel, o, d = frame_subset(n_rays, view)
    out = dict(level=np.int64(level), view=np.int64(view), sel=sel.numpy().astype(np.int32),
               state_digest=np.array(state_digest(sd)), sigma=np.float64(NOISE_SIGMA))
    for k, v in cfg_kw.items():
        out["cfg_" + k] = np.int64(v)
    for k, v in kw.items():
        out["kw_" + k] = np.array(v)
    for tag, m in (("clean", model), ("noisy", NoisyDensity(model, NOISE_SIGMA, seed=9))):
        t0 = time.time()
        with torch.no_grad():
            rgb, depth, ex = ns.renderer.volume_render(o, d, m, detailed_output=False, rayschunk=1024, **kw)
        print(f"{name} {tag}: {n_rays} rays in {time.time() - t0:.0f} s", flush=True)
        out[tag + "_rgb"] = rgb.numpy()
        out[tag + "_depth"] = depth.numpy()
        out[tag + "_acc"] = ex["mask_volume"].numpy()
        if "normals_volume" in ex:
            out[tag + "_normals"] = ex["normals_volume"].numpy()
    dr = np.abs(out["noisy_rgb"] - out["clean_rgb"]).max(-1)
    dd = np.abs(out["noisy_depth"] - out["clean_depth"])
    floor = 1.0 - ((dr <= 1e-4) & (dd <= 1e-5)).mean()
    print(f"{name}: reference self-noise floor (sigma {NOISE_SIGMA:g}): {floor:.4f} of {n_rays} rays outside (1e-4, 1e-5)")
    path = os.path.join(HERE, f"frame_{name}.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes", flush=True)


def add_noise_level(name, sigma, tag):
    """Append a second self-noise render (other sigma) to an existing golden file."""
    level, cfg_kw, kw, n_rays, view = CASES[name]
    path = os.path.join(HERE, f"frame_{name}.npz")
    out = dict(np.load(path, allow_pickle=False))
    ns = ref_harness.load()
    cfg = synth.ModelConfig(**cfg_kw)
    mesh = synth.icosphere_mesh(level, seed=0)
    sd = synth.make_state_dict(mesh, cfg, seed=1)
    model = ref_harness.build_reference_model(mesh, cfg, sd)
    sel, o, d = frame_subset(n_rays, view)
    with torch.no_grad():
        rgb, depth, ex = ns.renderer.volume_render(o, d, NoisyDensity(model, sigma, seed=9), detailed_output=False,
                                                   rayschunk=1024, **kw)
    out[tag + "_rgb"], out[tag + "_depth"], out[tag + "_acc"] = rgb.numpy(), depth.numpy(), ex["mask_volume"].numpy()
    out[tag + "_sigma"] = np.float64(sigma)
    dr = np.abs(out[tag + "_rgb"] - out["clean_rgb"]).max(-1)
    dd = np.abs(out[tag + "_depth"] - out["clean_depth"])
    print(f"{name}: reference self-noise floor (sigma {sigma:g}): {1.0 - ((dr <= 1e-4) & (dd <= 1e-5)).mean():.4f}")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes", flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "noisy8":
        add_noise_level("config1", 8e-7, "noisy8")     # yardstick of the CUDA-core verification engine
    else:
        for n in (sys.argv[1:] or list(CASES)):
            make(n)
