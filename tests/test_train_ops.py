"""The fused training op (``neumesh_b200/train_ops.py``; config 4).

CPU (``-m "not gpu"``): the SEQUENCING of ``field_forward`` / ``field_backward`` / ``FusedFieldFn`` is run with a torch
implementation of the kernel interface (``tests/train_prims_torch.py``) and compared with (a) autograd through this
package's torch-op field and (b) the gradients the UNMODIFIED reference produced (``tests/golden/train_step_small.npz``).
GPU (``-m gpu``): every ``nmb_tr_*`` kernel against the same torch primitive on random inputs, then the whole training
step on the CUDA kernels against the reference's golden gradients."""
import os

import numpy as np
import pytest
import torch

import helpers
import neumesh_b200 as nb
from neumesh_b200 import synth, train_ops
from train_prims_torch import TorchPrims


def _model_cpu(mesh, cfg, sd, fused):
    model = nb.NeuMesh(helpers.OracleMeshGrid(mesh), **cfg.model_kwargs())
    model.load_state_dict(sd)
    model.train()
    model.fused_train = fused
    model._train_prims = TorchPrims("cpu") if fused else None
    return model


@pytest.mark.parametrize("cfg_kw", [dict(), dict(enable_nablas_input=False, learn_indicator_weight=True),
                                    dict(geometry_dim=64, color_dim=96)])
def test_fused_field_sequencing_equals_autograd_cpu(cfg_kw):
    cfg = synth.ModelConfig(**cfg_kw)
    mesh = synth.icosphere_mesh(2, seed=3)
    sd = synth.make_state_dict(mesh, cfg, seed=4)
    x, v = helpers.sample_points(96, seed=5)
    x = x * 0.9
    g = torch.Generator().manual_seed(1)
    cs, cn, cr = torch.randn(96, 1, generator=g), torch.randn(96, 3, generator=g), torch.randn(96, 3, generator=g)
    grads = {}
    for fused in (False, True):
        model = _model_cpu(mesh, cfg, sd, fused)
        sdf, rgb = model.forward(x.clone(), v)
        sdf2, nabla = model.forward_with_nablas(x.clone())
        loss = (sdf * cs).sum() + (rgb * cr).sum() + (nabla * cn).sum() + 0.3 * (sdf2 * cs).sum()
        loss.backward()
        grads[fused] = (loss.item(), {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None})
    (l0, g0), (l1, g1) = grads[False], grads[True]
    assert abs(l0 - l1) <= 1e-4 * max(1.0, abs(l0))
    assert set(g0) == set(g1)
    worst = 0.0
    for k in g0:
        rel = ((g0[k] - g1[k]).double().norm() / g0[k].double().norm().clamp_min(1e-12)).item()
        worst = max(worst, rel)
        assert rel < 2e-4, (k, rel)
    print(f"{cfg_kw}: fused sequencing vs autograd, worst relative L2 gradient difference {worst:.2e}")


def _load(golden_dir):
    g = dict(np.load(os.path.join(golden_dir, "train_step_small.npz"), allow_pickle=False))
    cfg = synth.ModelConfig()
    mesh = synth.icosphere_mesh(int(g["level"]), seed=int(g["seed"]))
    sd = synth.make_state_dict(mesh, cfg, seed=int(g["seed"]) + 1)
    assert helpers.state_digest(sd) == str(g["state_digest"])
    return g, cfg, mesh, sd


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
    return worst


def test_train_step_fused_sequencing_vs_reference_golden_cpu(golden_dir):
    """Whole training step through ``volume_render`` with the fused op's sequencing (torch primitives) on CPU against
    the UNMODIFIED reference's gradients."""
    g, cfg, mesh, sd = _load(golden_dir)
    model = _model_cpu(mesh, cfg, sd, True)
    rgb, depth, ex = nb.volume_render(torch.from_numpy(g["rays_o"]), torch.from_numpy(g["rays_d"]), model,
                                      rayschunk=4096, **helpers.TRAIN_KW)
    loss = helpers.train_loss(rgb, depth, ex)
    loss.backward()
    worst = _check(g, loss.item(), dict(model.named_parameters()), rtol=3e-4, l2tol=1e-3)
    print(f"fused sequencing (CPU torch primitives) vs reference golden gradients: worst relative L2 {worst:.2e}")
    # teacher-forced sample depths (the hook the GPU test uses): same gradients
    model.zero_grad()
    rgb, depth, ex = nb.volume_render(torch.from_numpy(g["rays_o"]), torch.from_numpy(g["rays_d"]), model,
                                      rayschunk=4096, z_samples=torch.from_numpy(g["d_all"]), **helpers.TRAIN_KW)
    loss = helpers.train_loss(rgb, depth, ex)
    loss.backward()
    _check(g, loss.item(), dict(model.named_parameters()), rtol=3e-4, l2tol=1e-3)


# ------------------------------------------------------------------------------------------------------------------
# GPU: every nmb_tr_* kernel against the torch primitive, then the training step on the CUDA kernels
# ------------------------------------------------------------------------------------------------------------------
def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-20)).item()


@pytest.mark.gpu
def test_tr_gemm_vs_torch():
    dev = torch.device("cuda:0")
    P, T = train_ops.CudaPrims(dev), TorchPrims(dev)
    g = torch.Generator(device="cpu").manual_seed(0)
    worst = 0.0
    # (M, N, K): forward layer, tangent first layer (K = 17), input gradient (N = 177), weight gradients (split-K)
    for (M, N, K) in [(1000, 256, 177), (777, 256, 17), (1500, 177, 256), (256, 207, 40000), (256, 17, 9000), (130, 3, 5)]:
        for a_kc in (True, False):
            for b_kc in (True, False):
                lda = (K if a_kc else M) + 3
                ldb = (K if b_kc else N) + 5
                A = torch.randn((M if a_kc else K) * lda, generator=g).to(dev)
                B = torch.randn((N if b_kc else K) * ldb, generator=g).to(dev)
                bias = torch.randn(N, generator=g).to(dev)
                mask = torch.randn(M, N + 2, generator=g).to(dev)
                for (use_bias, epi, acc) in [(False, 0, False), (True, 1, False), (False, 2, False), (False, 0, True)]:
                    C0 = torch.randn(M, N + 1, generator=g).to(dev)
                    C1, C2 = C0.clone(), C0.clone()
                    kw = dict(bias=bias if use_bias else None, epilogue=epi, mask=mask if epi == 2 else None,
                              ldmask=N + 2 if epi == 2 else 0, accumulate=acc)
                    P.gemm(A, lda, a_kc, B, ldb, b_kc, C1, N + 1, M, N, K, **kw)
                    T.gemm(A, lda, a_kc, B, ldb, b_kc, C2, N + 1, M, N, K, **kw)
                    assert torch.equal(C1[:, N], C0[:, N]), "wrote outside the N columns"
                    e = _rel(C1[:, :N], C2[:, :N])
                    worst = max(worst, e)
                    assert e < 2e-5, ((M, N, K), a_kc, b_kc, use_bias, epi, acc, e)
    print(f"nmb_tr_gemm vs torch.matmul (fp32): worst relative L2 difference {worst:.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_kw", [
    dict(), dict(enable_nablas_input=False, geometry_dim=64, color_dim=96),
    # rows B, C, E of tests/test_field_envelope.py: one hidden geometry layer and raw codes only; the deepest geometry
    # net with 64-d colour codes (multires_d 8 instead of 16: the kernels and the float64 torch sequence compute ds
    # independently, and a 2^15 band turns their fp32 / float64 difference in ds into a 1e-3 one in the encoding);
    # one colour layer with 96-d / 160-d codes and 6 view bands
    dict(D_density=1, D_color=4, multires_d=4, multires_fg=0, multires_ft=2, multires_view=4,
         learn_indicator_weight=True),
    dict(D_density=7, D_color=2, color_dim=64, multires_d=8, multires_fg=3, multires_ft=1, multires_view=2,
         learn_indicator_weight=True),
    dict(D_density=2, D_color=1, geometry_dim=96, color_dim=160, multires_d=8, multires_fg=1, multires_ft=0,
         multires_view=6, learn_indicator_weight=True),
])
def test_tr_kernels_and_field_op_vs_torch_primitives(cfg_kw):
    """field_forward / field_backward on the CUDA kernels vs the same sequencing on torch primitives (same device, in
    float64, so that the reference's own rounding cannot decide the result): every intermediate the kernels produce is
    compared, so a wrong kernel is named by the first mismatch.  An fp32 torch sequence is not accurate enough to be the
    reference: on an H100 its colour-code gradient (64-d / 96-d codes) is 3.0e-4 from float64 (relative L2) while the
    CUDA kernels' is 4.2e-7."""
    dev = torch.device("cuda:0")
    cfg = synth.ModelConfig(**cfg_kw)
    mesh = synth.icosphere_mesh(4, seed=3)
    sd = synth.make_state_dict(mesh, cfg, seed=4)
    model = helpers.cuda_model(mesh, cfg, sd, "tcgen05").train()
    c = model._cfg
    spec = train_ops.FieldSpec(c["geometry_dim"], c["color_dim"], c["multires_d"], c["multires_fg"], c["multires_ft"],
                               c["multires_view"], model.enable_nablas_input, c["D_density"], c["D_color"])
    x, v = helpers.sample_points(3001, seed=5)
    x[0] = torch.from_numpy(mesh.vertices[7]).float()          # rho = 0 branch
    x, v = x.to(dev), v.to(dev)
    with torch.no_grad():
        _, idx, w = model.mesh_grid.compute_distance(x, indicator_vector=model.indicator_vector.detach(),
                                                     indicator_weight=0.1)
        geo_l = model._geo_linears()
        geo = [(torch._weight_norm(l.weight_v, l.weight_g, 0).contiguous(), l.bias.detach()) for l in geo_l[:-1]]
        geo_out = (torch._weight_norm(geo_l[-1].weight_v, geo_l[-1].weight_g, 0).contiguous(), geo_l[-1].bias.detach())
        col_l = model._col_linears()
        col = [(l.weight.detach().contiguous(), l.bias.detach()) for l in col_l[:-1]]
        col_out = (col_l[-1].weight.detach().contiguous(), col_l[-1].bias.detach())
    t = dict(xyz=x, dirs=v, idx=idx.contiguous(), w=w.contiguous(), vertices=model.mesh_grid.get_vertices_torch().contiguous(),
             indicator_vector=model.indicator_vector.detach().contiguous(),
             geometry_features=model.geometry_features.detach().contiguous(),
             color_features=model.color_features.detach().contiguous(), w1=0.1)
    g = torch.Generator().manual_seed(2)
    b_sdf, b_nab, b_rgb = (torch.randn(3001, generator=g).to(dev), torch.randn(3001, 3, generator=g).to(dev),
                           torch.randn(3001, 3, generator=g).to(dev))
    res = {}
    for name, P, dt in (("cuda", train_ops.CudaPrims(dev), torch.float32), ("torch", TorchPrims(dev, torch.float64), torch.float64)):
        cast = lambda z: z.to(dt) if torch.is_tensor(z) and z.is_floating_point() else z   # noqa: E731
        cl = lambda layers: [(cast(wt), cast(bs)) for wt, bs in layers]                      # noqa: E731
        sdf, nabla, rgb, S = train_ops.field_forward(P, spec, {k: cast(vv) for k, vv in t.items()}, cl(geo),
                                                     tuple(map(cast, geo_out)), cl(col), tuple(map(cast, col_out)))
        G = train_ops.field_backward(P, spec, S, cl(geo), tuple(map(cast, geo_out)), cl(col), tuple(map(cast, col_out)),
                                     cast(b_sdf), cast(b_nab), cast(b_rgb))
        res[name] = (sdf, nabla, rgb, S, G)
    torch.cuda.synchronize()
    a, b = res["cuda"], res["torch"]
    worst = 0.0
    for k in ("ds", "G", "Xg", "T0", "Xc", "g", "rgb"):
        e = _rel(a[3][k], b[3][k])
        worst = max(worst, e)
        assert e < 2e-5, ("saved " + k, e)
    for k in ("hs", "ts", "zs", "as_", "cs"):
        for i, (u, vv) in enumerate(zip(a[3][k], b[3][k])):
            e = _rel(u, vv)
            worst = max(worst, e)
            assert e < 5e-5, (f"saved {k}[{i}]", e)
    for i, k in enumerate(("sdf", "nabla", "rgb")):
        e = _rel(a[i], b[i])
        assert e < 2e-5, (k, e)
    Ga, Gb = a[4], b[4]
    for k in ("geometry_features", "color_features", "indicator_vector", "w1"):
        e = _rel(Ga[k], Gb[k])
        worst = max(worst, e)
        assert e < 2e-4, ("grad " + k, e)
    for k in ("geo", "col"):
        for i, ((dW, db), (rW, rb)) in enumerate(zip(Ga[k], Gb[k])):
            e = max(_rel(dW, rW), _rel(db, rb))
            worst = max(worst, e)
            assert e < 2e-4, (f"grad {k}[{i}]", e)
    for k in ("geo_out", "col_out"):
        e = max(_rel(Ga[k][0], Gb[k][0]), _rel(Ga[k][1], Gb[k][1]))
        worst = max(worst, e)
        assert e < 2e-4, ("grad " + k, e)
    print(f"{cfg_kw}: CUDA training kernels vs torch primitives, worst relative L2 difference {worst:.2e}")


@pytest.mark.gpu
def test_train_step_fused_cuda_vs_reference_golden(golden_dir):
    """The training step of config 4 on the CUDA kernels (fused sampling cascade + FusedFieldFn forward / backward)
    against the gradients of the UNMODIFIED reference.  The sample depths are teacher-forced to the reference's
    (``d_all`` of the golden file) for the tight comparison - the discrete cascade is compared separately - and the
    free-running step (own CUDA cascade) is checked for agreement of the loss."""
    dev = torch.device("cuda:0")
    g, cfg, mesh, sd = _load(golden_dir)
    o, d = torch.from_numpy(g["rays_o"]).to(dev), torch.from_numpy(g["rays_d"]).to(dev)
    model = helpers.cuda_model(mesh, cfg, sd, "tcgen05").train()
    assert model._fused_train_ok(o)
    n0 = nb._lib.launch_count()
    rgb, depth, ex = nb.volume_render(o, d, model, rayschunk=4096, z_samples=torch.from_numpy(g["d_all"]).to(dev),
                                      **helpers.TRAIN_KW)
    loss = helpers.train_loss(rgb, depth, ex)
    loss.backward()
    torch.cuda.synchronize()
    assert nb._lib.launch_count() - n0 > 50, "the training step did not run on the library's kernels"
    worst = _check(g, loss.item(), dict(model.named_parameters()), rtol=1e-3, l2tol=1e-3)
    print(f"CUDA training step (teacher-forced samples) vs reference golden gradients: worst relative L2 {worst:.2e}")
    # free-running: fused CUDA sampling cascade + fused field op
    model.zero_grad()
    rgb2, depth2, ex2 = nb.volume_render(o, d, model, rayschunk=4096, **helpers.TRAIN_KW)
    loss2 = helpers.train_loss(rgb2, depth2, ex2)
    loss2.backward()
    assert abs(loss2.item() - float(g["loss"])) <= 2e-3 * abs(float(g["loss"]))
    assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.grad is not None)
    # perturb=True runs the same kernels with injected / drawn uniforms
    model.zero_grad()
    kw = dict(helpers.TRAIN_KW)
    kw["perturb"] = True
    rgb3, _, ex3 = nb.volume_render(o, d, model, rayschunk=4096, **kw)
    assert torch.isfinite(rgb3).all() and ex3["implicit_nablas"].shape == (o.shape[0], 128, 3)
