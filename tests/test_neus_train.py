"""NeuS training on the library's kernels: ``neus_ops.FusedSurfaceFn`` (value + reverse-mode adjoint through the softplus
MLP, the ``nmb_ns_*`` kernels of ``csrc/train_neus.cu`` and the training GEMMs) and ``FusedRadianceFn``, behind the
grad-enabled calls of ``neus.NeuS``.

The reference is the module's own torch-op path: the nabla by ``autograd.grad(..., create_graph=True)`` and every
parameter gradient by a real double backward, in float64; the yardstick is that path in fp32 (bars of
``test_train_envelope._compare``).  The whole step is also held against ``tests/golden/neus_train_step_small.npz``,
gradients of the UNMODIFIED reference's NeuS stage-1 loss (``tests/golden/make_neus_train_golden.py``).

CPU: the op's sequencing on torch primitives over ``test_train_envelope.NEUS_CASES`` and the upstream patterns, which
calls each route accepts, and the drop-in's torch path against the golden file.  GPU: every ``nmb_ns_*`` kernel, the
ops on both GEMM engines, the whole step against the golden file, bit-reproducibility under
``torch.use_deterministic_algorithms(True)``, M = 0, and ``fused_train = False``."""
from __future__ import annotations

import numpy as np
import pytest
import torch

import helpers
import neumesh_b200 as nb
from neumesh_b200 import neus_ops, train_ops
from neumesh_b200.neus import NeuS
from neus_train_common import NeusTorchPrims, neus_loss
from test_train_envelope import NEUS_CASES, _compare, _neus, _neus_points, _rel

ENGINES = ("fp32", "tf32x3")
# which outputs carry an upstream gradient: sdf (s), nabla (n), feature (f), rgb (r)
PATTERNS = {"all": "snfr", "sdf_only": "s", "nabla_only": "n", "rgb_only": "r", "feature_only": "f"}


def _upstream(M, F, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(*s, generator=g).to(dtype) for s in ((M,), (M, 3), (M, F), (M, 3))]


def _run(m, x, v, up, pattern):
    """sdf, nabla, feature (grad-enabled forward_with_nablas), rgb (radiance net on them); a loss that puts the
    pattern's upstream gradients on them; -> outputs and every parameter gradient by name."""
    m.zero_grad(set_to_none=True)
    x = x.clone()      # the torch-op path sets requires_grad on the caller's tensor, as the reference does
    sdf, nabla, feat = m.implicit_surface.forward_with_nablas(x)
    rgb = m.radiance_net.forward(x, v, nabla, feat)
    terms = dict(s=(sdf, up[0]), n=(nabla, up[1]), f=(feat, up[2]), r=(rgb, up[3]))
    loss = sum((terms[k][0] * terms[k][1].to(terms[k][0])).sum() for k in pattern)
    loss.backward()
    out = {"sdf": sdf, "nabla": nabla, "feature": feat, "rgb": rgb}
    out.update({k: (p.grad if p.grad is not None else torch.zeros_like(p)) for k, p in m.named_parameters()
                if k != "ln_s"})
    return out, (sdf, nabla, feat, rgb)


def _grad_fns(t):
    """Class names of every node of the graph behind t."""
    seen, stack, names = set(), [t.grad_fn], set()
    while stack:
        f = stack.pop()
        if f is None or f in seen:
            continue
        seen.add(f)
        names.add(type(f).__name__)
        stack.extend(nf for nf, _ in f.next_functions)
    return names


def _off_radiance_kinks(case, x, v, seed, margin=1e-4):
    """Moves the points whose radiance-net pre-activations come within ``margin`` of a ReLU kink (in float64): there
    fp32 and float64 may take different sides, and a gradient then differs by a whole point's term."""
    m = _neus(case).double()
    net = m.radiance_net
    g = torch.Generator().manual_seed(seed)
    for _ in range(50):
        sdf, nabla, feat = m.implicit_surface.forward_with_nablas(x.double().clone(), has_grad_bypass=False)
        h = net._input(x.double(), v.double(), nabla, feat)
        near = torch.zeros(x.shape[0], dtype=torch.bool)
        with torch.no_grad():
            for lin in net.layers[:-1]:
                z = torch.nn.functional.linear(h, torch._weight_norm(lin.weight_v, lin.weight_g, 0), lin.bias)
                near |= (z.abs() < margin).any(-1)
                h = z.clamp_min(0)
        if not near.any():
            return x, v
        n = int(near.sum())
        x, v = x.clone(), v.clone()
        x[near] = torch.rand(n, 3, generator=g) * 1.6 - 0.8
        v[near] = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    raise AssertionError("could not move the points off the radiance net's ReLU kinks")


def _check_case(case, M, pattern, dev, engine, prims=None, floor_fwd=2e-6, floor_grad=2e-5):
    m = _neus(case)
    F = m.implicit_surface.W_geo_feat
    x, v = _off_radiance_kinks(case, *_neus_points(M, seed=81), seed=86)
    up = _upstream(M, F, seed=82)
    ref, _ = _run(m.double().train(), x.double(), v.double(), up, pattern)
    m.fused_train = False
    yard, _ = _run(m.float(), x, v, up, pattern)
    m.fused_train = True
    m = m.to(dev)
    m.train_engine = engine
    m._train_prims = prims
    got, (sdf, nabla, feat, rgb) = _run(m, x.to(dev), v.to(dev), up, pattern)
    assert "FusedSurfaceFnBackward" in _grad_fns(sdf) and "FusedRadianceFnBackward" in _grad_fns(rgb)
    # bands: the nabla's Jacobian scales the fp32 rounding of the input adjoint by up to 2^(L-1) (the envelope's rule)
    _compare(f"{dev} {engine} {case} M={M} {pattern}", got, ref, yard, floor_fwd, floor_grad,
             bands=max(m.implicit_surface.embed_multires, 0))


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(NEUS_CASES))
def test_ops_sequencing_vs_float64_cpu(case):
    _check_case(case, 97, PATTERNS["all"], "cpu", "fp32", prims=NeusTorchPrims("cpu"))


@pytest.mark.parametrize("pattern", list(PATTERNS))
def test_upstream_patterns_sequencing_cpu(pattern):
    _check_case("D8_skip4_em6_W256", 97, PATTERNS[pattern], "cpu", "fp32", prims=NeusTorchPrims("cpu"))


def test_value_only_mode_sequencing_cpu():
    """Grad-enabled ``ImplicitSurface.forward`` (``forward_density_only``) is the op without the adjoint."""
    m = _neus("D8_skip4_em6_W256").train()
    x, _ = _neus_points(61, seed=83)
    w = torch.randn(61, generator=torch.Generator().manual_seed(84))
    res = {}
    for fused in (False, True):
        m.zero_grad(set_to_none=True)
        m.fused_train, m._train_prims = fused, (NeusTorchPrims("cpu") if fused else None)
        sdf = m.forward_density_only(x)
        assert ("FusedSurfaceFnBackward" in _grad_fns(sdf)) == fused
        (sdf * w).sum().backward()
        res[fused] = {"sdf": sdf, **{k: p.grad for k, p in m.named_parameters() if p.grad is not None}}
    assert set(res[True]) == set(res[False])
    for k in res[False]:
        assert _rel(res[True][k], res[False][k]) < 2e-5, k


def test_routes_cpu():
    """Which calls take the ops (CPU with injected torch primitives stands in for CUDA)."""
    m = _neus("D8_skip4_em6_W256").train()
    m._train_prims = NeusTorchPrims("cpu")
    x, v = _neus_points(9, seed=85)
    fused = lambda t: "FusedSurfaceFnBackward" in _grad_fns(t)   # noqa: E731
    sdf, nabla, feat = m.implicit_surface.forward_with_nablas(x)
    assert fused(sdf) and fused(nabla) and not x.requires_grad, "the fused route must not touch the caller's x"
    assert "FusedRadianceFnBackward" in _grad_fns(m.radiance_net(x, v, nabla, feat))
    assert fused(m.forward_density_only(x))
    sdf, rad = m.forward(x, v)
    assert fused(sdf) and "FusedRadianceFnBackward" in _grad_fns(rad)
    # grad mode off: no graph at all
    with torch.no_grad():
        assert m.forward_density_only(x).grad_fn is None
    # an x that needs a gradient keeps the torch path, and gets its gradient
    xg = x.clone().requires_grad_(True)
    sdf, nabla, _ = m.implicit_surface.forward_with_nablas(xg * 1.0)
    assert not fused(sdf)
    sdf.sum().backward()
    assert xg.grad is not None and xg.grad.abs().sum() > 0
    # fused_train = False, float64 models, no primitives on CPU
    m.fused_train = False
    assert not fused(m.forward_density_only(x)) and not fused(m.forward_with_nablas(x.clone())[0])
    m.fused_train = True
    assert m.implicit_surface.fused_train and m.radiance_net.fused_train
    md = _neus("D8_skip4_em6_W256").double().train()
    md._train_prims = NeusTorchPrims("cpu")
    assert not fused(md.forward_density_only(x.double()))
    mc = _neus("D8_skip4_em6_W256").train()
    assert not fused(mc.forward_density_only(x))
    # radiance net with skips; surface without a geometry feature
    ms = NeuS(**dict(helpers.NEUS_KW, radiance_cfg=dict(helpers.NEUS_KW["radiance_cfg"], skips=[2]))).train()
    ms._train_prims = NeusTorchPrims("cpu")
    _, rad = ms.forward(x, v)
    assert fused(ms.forward_density_only(x)) and "FusedRadianceFnBackward" not in _grad_fns(rad)
    m0 = NeuS(**dict(helpers.NEUS_KW, W_geo_feat=0)).train()
    m0._train_prims = NeusTorchPrims("cpu")
    assert not fused(m0.forward_density_only(x))
    # not part of the state_dict
    assert set(m.state_dict()) == set(_neus("D8_skip4_em6_W256").state_dict())


def _golden(golden_dir):
    g = dict(np.load(f"{golden_dir}/neus_train_step_small.npz", allow_pickle=False))
    m = NeuS(**helpers.NEUS_KW)
    sd = helpers.neus_state_dict(m, int(g["seed"]))
    assert helpers.state_digest(sd) == str(g["state_digest"])
    m.load_state_dict(sd, strict=True)
    return g, m.train()


def _golden_step(m, g, dev):
    t = lambda k: torch.from_numpy(g[k]).to(dev)   # noqa: E731
    m.zero_grad(set_to_none=True)
    kw = {k[3:]: (bool(v) if v.dtype == bool else int(v)) for k, v in g.items() if k.startswith("kw_")}
    rgb, depth, ex = nb.volume_render(t("rays_o"), t("rays_d"), m, z_samples=t("d_all"), detailed_output=True,
                                      rayschunk=4096, **kw)
    loss = neus_loss(rgb, t("target_rgb"), t("target_mask"), ex)
    loss.backward()
    params = dict(m.named_parameters())
    return loss, params, ex


def _golden_errors(g, loss, params):
    errs = {"loss": abs(loss.item() - float(g["loss"])) / abs(float(g["loss"]))}
    for k in params:
        ref = torch.from_numpy(g["grad_" + k]).double()
        got = params[k].grad.detach().double().cpu().reshape(-1)
        got = got if got.numel() < 4096 else got[::37]   # make_neus_train_golden.NEUS_GRAD_STRIDE
        errs[k] = (got - ref.reshape(-1)).norm().item() / max(ref.norm().item(), 1e-30)
    return errs


def test_torch_path_step_reproduces_reference_golden_cpu(golden_dir):
    """The drop-in's torch-op path (CPU) through ``nb.volume_render`` at the reference's sample depths reproduces the
    reference's loss and every parameter gradient, ``ln_s`` included."""
    g, m = _golden(golden_dir)
    loss, params, _ = _golden_step(m, g, "cpu")
    errs = _golden_errors(g, loss, params)
    print("torch path vs the unmodified reference, relative L2:", {k: f"{e:.1e}" for k, e in errs.items()})
    assert max(errs.values()) < 1e-4, errs


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _dev():
    return torch.device("cuda:0")


KERNEL_M = [0, 1, 127, 4099, 130560]


@pytest.mark.gpu
@pytest.mark.parametrize("L", [0, 6, 10])
@pytest.mark.parametrize("M", KERNEL_M)
def test_ns_kernels_vs_float64(M, L):
    dev = _dev()
    P, R = train_ops.CudaPrims(dev), NeusTorchPrims(dev, torch.float64)
    g = torch.Generator().manual_seed(90 + L)
    C, N = 3 * (1 + 2 * L), 217
    x = (torch.rand(M, 3, generator=g) * 1.6 - 0.8)
    z = torch.randn(M, N, generator=g) * 0.05        # straddles the softplus threshold z = 0.2 and its curved part
    if M:
        z[:, :8] = torch.tensor([0.2, 0.19999999, 0.20000001, -0.3, 0.5, 0.0, -0.05, 0.05])
    gm, row = torch.randn(M, N, generator=g), torch.randn(N, generator=g)
    ebar, bn = torch.randn(M, C, generator=g), torch.randn(M, 3, generator=g)
    f32 = lambda t: t.to(dev).float().contiguous()   # noqa: E731
    f64 = lambda t: t.to(dev).double().contiguous()  # noqa: E731
    n0 = nb._lib.launch_count()
    out = {}
    # PE into the tail of a wider buffer (the skip layer's e columns); the head must stay untouched
    buf = torch.full((M, N + C), 7.0, device=dev)
    P.pe(f32(x), L, neus_ops._at(buf, N), N + C)
    refb = torch.empty(M, C, device=dev, dtype=torch.float64)
    R.pe(f64(x), L, refb, C)
    out["pe"] = (buf[:, N:], refb)
    assert bool((buf[:, :N] == 7.0).all())
    for name, args32, shape in (("pe_jt", (f32(ebar),), (M, 3)), ("pe_j", (f32(bn),), (M, C))):
        o, r = torch.empty(*shape, device=dev), torch.empty(*shape, device=dev, dtype=torch.float64)
        getattr(P, name)(f32(x), L, *args32, o)
        getattr(R, name)(f64(x), L, *(f64(a) for a in args32), r)
        out[name] = (o, r)
    h = torch.full((M, N + 5), 7.0, device=dev)
    P.softplus(f32(z), h, N + 5)
    rh = torch.empty(M, N, device=dev, dtype=torch.float64)
    R.softplus(f64(z), rh, N)
    out["softplus"] = (h[:, :N], rh)
    assert bool((h[:, N:] == 7.0).all())
    for name, (gg, rr, zz) in {"gate": (gm, None, z), "gate_row": (None, row, z), "broadcast": (None, row, None)}.items():
        o, r = torch.empty(M, N, device=dev), torch.empty(M, N, device=dev, dtype=torch.float64)
        P.gate(None if gg is None else f32(gg), None if rr is None else f32(rr), None if zz is None else f32(zz), o)
        R.gate(None if gg is None else f64(gg), None if rr is None else f64(rr), None if zz is None else f64(zz), r)
        out[name] = (o, r)
    torch.cuda.synchronize()
    assert nb._lib.launch_count() - n0 == (0 if M == 0 else 7)
    for k, (o, r) in out.items():
        e = (o.double() - r).abs()
        # softplus / gate: a few ulps of the value; PE: of 1 (sin / cos); J contractions: of the largest term 2^(L-1)
        floor = {"pe": 1.0, "pe_jt": 2.0 ** max(L - 1, 0) * 8, "pe_j": 2.0 ** max(L - 1, 0) * 4}.get(k, 1e-30)
        worst = (e / (r.abs() + floor)).max().item() if M else 0.0
        assert worst < 4e-6, (k, worst)


def _gpu_cases():
    return [(c, M) for c in NEUS_CASES for M in (1, 127, 4099)]


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case,M", _gpu_cases())
def test_ops_vs_float64(case, M, engine):
    _check_case(case, M, PATTERNS["all"], _dev(), engine)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", list(PATTERNS))
def test_upstream_patterns_vs_float64(pattern):
    _check_case("D8_skip4_em6_W256", 4099, PATTERNS[pattern], _dev(), "fp32")


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
def test_ops_large_batch_vs_float64(engine):
    _check_case("D8_skip4_em6_W256", 130560, PATTERNS["all"], _dev(), engine)


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
def test_step_vs_reference_golden(engine, golden_dir):
    """The whole NeuS stage-1 step through ``nb.volume_render`` on the fused ops at the reference's depths, against the
    reference's loss and gradients (``ln_s`` included)."""
    g, m = _golden(golden_dir)
    m = m.to(_dev())
    m.train_engine = engine
    n0 = nb._lib.launch_count()
    loss, params, ex = _golden_step(m, g, _dev())
    torch.cuda.synchronize()
    assert nb._lib.launch_count() - n0 > 100, "the step did not run on the library's kernels"
    fns = _grad_fns(loss)
    assert {"FusedSurfaceFnBackward", "FusedRadianceFnBackward"} <= fns, fns
    errs = _golden_errors(g, loss, params)
    print(f"[{engine}] fused step vs the unmodified reference, relative L2:", {k: f"{e:.1e}" for k, e in errs.items()})
    assert max(errs.values()) <= 1e-3, errs


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
def test_adam_steps_bit_reproducible_deterministic(engine, golden_dir):
    g, _ = _golden(golden_dir)
    runs = []
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            _, m = _golden(golden_dir)
            m = m.to(_dev())
            m.train_engine = engine
            opt = torch.optim.Adam(m.parameters(), lr=5e-4)
            losses = []
            for _ in range(3):
                loss, _, _ = _golden_step(m, g, _dev())
                opt.step()
                losses.append(loss.detach())
            runs.append((losses, [p.detach().clone() for p in m.parameters()]))
    finally:
        torch.use_deterministic_algorithms(was)
    for a, b in zip(runs[0][0] + runs[0][1], runs[1][0] + runs[1][1]):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_empty_batch_launches_nothing():
    m = _neus("D8_skip4_em6_W256").to(_dev()).train()
    x = torch.empty(0, 3, device=_dev())
    n0 = nb._lib.launch_count()
    sdf, nabla, feat = m.implicit_surface.forward_with_nablas(x)
    rgb = m.radiance_net(x, x, nabla, feat)
    (sdf.sum() + nabla.sum() + rgb.sum()).backward()
    dens = m.forward_density_only(x)
    dens.sum().backward()
    torch.cuda.synchronize()
    assert nb._lib.launch_count() == n0
    assert sdf.shape == (0,) and nabla.shape == (0, 3) and rgb.shape == (0, 3) and feat.shape == (0, 256)


@pytest.mark.gpu
def test_fused_train_off_is_the_torch_path():
    """``fused_train = False`` launches nothing of the library and gives exactly the torch-op path's outputs and
    gradients: those of a call whose x requires a gradient, which takes that path whatever ``fused_train`` says."""
    m = _neus("D8_skip4_em6_W256").to(_dev()).train()
    x, _ = (t.to(_dev()) for t in _neus_points(513, seed=87))
    res = []
    for off in (True, False):
        m.fused_train = not off
        m.zero_grad(set_to_none=True)
        xi = x.clone().requires_grad_(not off)
        n0 = nb._lib.launch_count()
        sdf, nabla = m.forward_with_nablas(xi)
        dens = m.forward_density_only(xi)
        (sdf.sum() + (nabla ** 2).sum() + dens.sum()).backward()
        torch.cuda.synchronize()
        assert nb._lib.launch_count() == n0
        assert "FusedSurfaceFnBackward" not in _grad_fns(sdf)
        res.append([sdf.detach(), nabla.detach(), dens.detach()] + [p.grad.clone() for p in m.parameters()
                                                                    if p.grad is not None])
    m.fused_train = True
    assert len(res[0]) == len(res[1]) and all(torch.equal(a, b) for a, b in zip(*res))
