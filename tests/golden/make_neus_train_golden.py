"""Golden NeuS stage-1 training step of the UNMODIFIED reference (the checkout named by ``NEUMESH_REFERENCE_ROOT``
imported verbatim on CPU through ``ref_harness``): ``tests/golden/neus_train_step_small.npz``.

One step of ``configs/neus_dtu_scan63.yaml`` (image L1 over the masked rays, mask BCE, eikonal 0.1) through the
reference's ``models/renderer.py::volume_render`` and ``NeuS`` under autograd, with ``perturb=False`` so that the sample
depths are deterministic.  Recorded: the final sample depths (spied at ``forward_with_nablas``), the loss and every
parameter's gradient, ``ln_s`` included (large ones subsampled).  ``tests/test_neus_train.py`` holds the drop-in's torch
path (CPU) and the fused ops (GPU) against it.

``NEUMESH_REFERENCE_ROOT=<reference checkout> python tests/golden/make_neus_train_golden.py``
"""
from __future__ import annotations

import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))
warnings.filterwarnings("ignore")

import ref_harness  # noqa: E402
from make_golden import state_digest  # noqa: E402
from neumesh_b200 import synth  # noqa: E402

NEUS_TRAIN_KW = dict(perturb=False, calc_normal=True, bounded_near_far=False, white_bkgd=False, N_samples=64,
                     N_importance=64, N_upsample_iters=4)


NEUS_GRAD_STRIDE = 37   # gradients with 4096 or more entries are recorded at every 37th entry


def make_neus_train_case(name, n_rays, seed):
    """One NeuS stage-1 step (configs/neus_dtu_scan63.yaml: image L1, mask BCE, eikonal 0.1) through the UNMODIFIED
    reference renderer and NeuS under autograd; perturb=False so that the sample depths are deterministic."""
    import contextlib
    import io
    import helpers
    from neus_train_common import neus_loss
    ns = ref_harness.load()
    with contextlib.redirect_stdout(io.StringIO()):
        model = ns.neus.NeuS(**helpers.NEUS_KW)
    sd = helpers.neus_state_dict(model, seed)
    model.load_state_dict(sd, strict=True)
    model.train()
    o, d = synth.frame_rays(24, 24, view=2)
    sel = torch.linspace(0, o.shape[0] - 1, n_rays).long()
    o, d = o[sel].contiguous(), d[sel].contiguous()
    g = torch.Generator().manual_seed(seed)
    target_rgb = torch.rand(n_rays, 3, generator=g)
    target_mask = torch.rand(n_rays, generator=g) > 0.3
    seen = {}
    fwn = model.forward_with_nablas

    def spy(xyz, *a, **k):
        seen["pts"] = xyz.detach().clone()
        return fwn(xyz, *a, **k)

    model.forward_with_nablas = spy
    rgb, depth, ex = ns.renderer.volume_render(o, d, model, rayschunk=4096, detailed_output=True, **NEUS_TRAIN_KW)
    model.forward_with_nablas = fwn
    dn = torch.nn.functional.normalize(d, dim=-1)
    d_all = ((seen["pts"].reshape(o.shape[0], -1, 3) - o[:, None, :]) * dn[:, None, :]).sum(-1)
    loss = neus_loss(rgb, target_rgb, target_mask, ex)
    loss.backward()
    out = dict(seed=np.int64(seed), state_digest=np.array(state_digest(sd)), rays_o=o.numpy(), rays_d=d.numpy(),
               target_rgb=target_rgb.numpy(), target_mask=target_mask.numpy(), loss=np.float64(loss.item()),
               d_all=d_all.numpy())
    for k, v in NEUS_TRAIN_KW.items():
        out["kw_" + k] = np.array(v)
    for k, p in model.named_parameters():
        gr = p.grad.reshape(-1)
        out["grad_" + k] = (gr if gr.numel() < 4096 else gr[::NEUS_GRAD_STRIDE]).numpy()
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes; loss", loss.item(), "; samples per ray", d_all.shape[1])


if __name__ == "__main__":
    make_neus_train_case("neus_train_step_small", 48, seed=70)
