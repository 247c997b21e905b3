"""Training-path semantics (config 4): gradients of a trainer-style loss through ``neumesh_b200.volume_render`` +
``neumesh_b200.NeuMesh`` (differentiable torch-op path) against the gradients the UNMODIFIED reference produced
(``tests/golden/train_step_small.npz``).  CPU: neighbour search by the oracle; GPU: by the CUDA octree."""
import os

import numpy as np
import pytest
import torch

import helpers
import neumesh_b200 as nb
from neumesh_b200 import synth


def _load(golden_dir):
    g = dict(np.load(os.path.join(golden_dir, "train_step_small.npz"), allow_pickle=False))
    cfg = synth.ModelConfig()
    mesh = synth.icosphere_mesh(int(g["level"]), seed=int(g["seed"]))
    sd = synth.make_state_dict(mesh, cfg, seed=int(g["seed"]) + 1)
    assert helpers.state_digest(sd) == str(g["state_digest"])
    return g, cfg, mesh, sd


def _grads(model, o, d):
    rgb, depth, ex = nb.volume_render(o, d, model, rayschunk=4096, **helpers.TRAIN_KW)
    loss = helpers.train_loss(rgb, depth, ex)
    loss.backward()
    return loss.item(), dict(model.named_parameters())


def _check(g, loss, params, rtol, l2tol):
    assert abs(loss - float(g["loss"])) <= 1e-5 * max(1.0, abs(float(g["loss"])))
    worst = 0.0
    for k in helpers.GRAD_KEYS:
        got = params[k].grad.detach().cpu()
        ref_norm = float(g["gnorm_" + k])
        assert torch.isfinite(got).all(), k
        assert abs(got.double().norm().item() - ref_norm) <= rtol * ref_norm + 1e-9, k
        ref = torch.from_numpy(g["grad_" + k])
        sub = got if got.numel() < 20000 else got[::7]
        rel = ((sub - ref).double().norm() / ref.double().norm().clamp_min(1e-12)).item()
        worst = max(worst, rel)
        assert rel <= l2tol, (k, rel)
    print(f"loss {loss:.8f} (reference {float(g['loss']):.8f}); worst relative L2 gradient error {worst:.2e}")


def test_train_step_gradients_cpu(golden_dir):
    g, cfg, mesh, sd = _load(golden_dir)
    model = nb.NeuMesh(helpers.OracleMeshGrid(mesh), **cfg.model_kwargs())
    model.load_state_dict(sd)
    model.train()
    loss, params = _grads(model, torch.from_numpy(g["rays_o"]), torch.from_numpy(g["rays_d"]))
    _check(g, loss, params, rtol=2e-5, l2tol=1e-4)


@pytest.mark.gpu
def test_train_step_gradients_gpu(golden_dir):
    assert torch.cuda.is_available()
    dev = torch.device("cuda:0")
    g, cfg, mesh, sd = _load(golden_dir)
    model = helpers.cuda_model(mesh, cfg, sd, "tcgen05").train()
    model.fused_train = False   # this file covers the torch-op path; tests/test_train_ops.py covers the fused CUDA op
    o, d = torch.from_numpy(g["rays_o"]).to(dev), torch.from_numpy(g["rays_d"]).to(dev)
    # sample depths teacher-forced to the reference's (the discrete cascade is compared separately): with identical
    # samples the gradients agree to fp32 rounding (cuBLAS / elementwise kernels vs MKL)
    rgb, depth, ex = nb.volume_render(o, d, model, rayschunk=4096, z_samples=torch.from_numpy(g["d_all"]).to(dev),
                                      **helpers.TRAIN_KW)
    loss_t = helpers.train_loss(rgb, depth, ex)
    loss_t.backward()
    loss, params = loss_t.item(), dict(model.named_parameters())
    # torch-op path on the GPU: cuBLAS / ATen kernels, atomics in index_add, hence the wider bar than the fused CUDA op
    # is held to (tests/test_train_ops.py) against the same golden gradients
    _check(g, loss, params, rtol=2e-2, l2tol=2e-2)
    # an optimiser step changes the parameters in place: the fused no-grad path must pick the new values up
    x = torch.rand(64, 3, device=dev) - 0.5
    with torch.no_grad():
        a = model.forward_density_only(x)
        for p in model.parameters():
            if p.grad is not None:
                p.add_(p.grad, alpha=-1e-2)
        b = model.forward_density_only(x)
    assert not torch.equal(a, b)
