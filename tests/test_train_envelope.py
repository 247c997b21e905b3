"""Envelope of the training half of the field: the fused training op (``train_ops.FusedFieldFn`` on the ``nmb_tr_*``
kernels of ``csrc/train.cu``) and the NeuS distillation teacher (``neus.py``), each against float64.

The reference of the field op is written here from the model's definition, not from the op: the mesh distance of
``oracle.field.mesh_distance`` at the neighbours (``idx``, ``w``) the op itself used, the encodings of
``oracle.field.positional_encoding`` / ``blend_rows``, the weight-normed softplus MLP and the colour MLP in torch ops,
the nabla by ``autograd.grad(..., create_graph=True)`` and every parameter gradient by a real double backward.  Nothing
of ``train_ops``, ``TorchPrims`` or ``tools/train_math_proto.py`` is in it, so a wrong backward formula cannot hide
behind a reference that shares it.

Bars are relative L2 errors per tensor.  The yardstick of a comparison is the same reference evaluated in fp32: the
kernels may be at most twice as far from float64 as that plus a floor.  The high-band rows (multires_d 16 and 28)
amplify the fp32 rounding of ds by 2^(L-1), so only the yardstick rule is meaningful there; on the rows the per-kernel
test ``test_tr_kernels_and_field_op_vs_torch_primitives`` covers (A, B, E) the fixed bars 2e-5 (forward) and 2e-4
(gradients) apply as well.

CPU (``-m "not gpu"``): the op's sequencing on torch primitives over the whole configuration matrix, the upstream-gradient
patterns and the whole training step against float64, and which rows each route accepts.
GPU (``-m gpu``): the CUDA kernels over the matrix, the batch sizes the kernels' geometry makes interesting, every
upstream-gradient pattern, the kernels' edges, the whole step and the NeuS teacher; about 30 s on an H100 80GB HBM3
(132 SMs, 400 W power limit).
"""
from __future__ import annotations

import functools
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import helpers
import neumesh_b200 as nb
from neumesh_b200 import synth, train_ops
from neumesh_b200.neus import NeuS, RadianceNet
from oracle.field import blend_rows, positional_encoding
from train_prims_torch import TorchPrims

# ------------------------------------------------------------------------------------------------------------------
# configuration matrix
# ------------------------------------------------------------------------------------------------------------------
# Rows the fused inference path refuses but the training op takes (W = 256, non-negative bands)
OUTSIDE = {
    "D_density_8": dict(D_density=8),
    "D_color_8": dict(D_color=8),
    "codes_48_40": dict(geometry_dim=48, color_dim=40),    # code widths that are not multiples of 32
    # 65-column colour head on the tensor-core engines; 64-d colour codes keep the fp32 engine out as well
    "multires_view_7": dict(multires_view=7, color_dim=64),
}
# Degenerate encodings: a raw ds only; raw codes and raw view directions only
DEGENERATE = {
    "multires_d_0": dict(multires_d=0, learn_indicator_weight=True),
    "raw_codes_and_view": dict(multires_fg=0, multires_ft=0, multires_view=0),
}
MATRIX = {**helpers.ROWS, **OUTSIDE, **DEGENERATE}
# rows where the per-kernel test's fixed bars (2e-5 forward, 2e-4 gradients) also hold
FIXED_BAR_ROWS = ("A", "B", "E")
FWD = ("sdf", "nabla", "rgb")


def _rel(a, b, scale=0.0, den_floor=0.0):
    """Relative L2 difference; ``scale`` floors the denominator at scale * sqrt(numel) (outputs that pass through 0),
    ``den_floor`` at an absolute value."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    den = max(b.norm().item(), scale * math.sqrt(max(b.numel(), 1)), den_floor, 1e-30)
    return (a - b).norm().item() / den


def _compare(tag, got, ref, yard, floor_fwd, floor_grad, fixed=False, bands=0):
    """Every tensor of ``ref``: the error of ``got`` at most 2 x the yardstick's (``yard``: fp32 reference) + floor.
    A weight-norm gain's gradient is the projection (dW . v) / |v| of its layer's weight gradient, which cancels to a
    small part of dW: its error is measured relative to the layer's ``weight_v`` gradient when that is larger.
    ``bands``: multires_d; the gradient floor is at least the fp32 rounding of ds amplified by the top band, 2^-24 x
    2^(bands - 1) (1e-5 at multires_d 8, 2e-3 at 16)."""
    floor_grad = max(floor_grad, 2.0 ** (bands - 25))
    lines, bad, worst = [], [], (0.0, "")
    for k in ref:
        fwd = k in FWD
        scale = 1e-3 if fwd else 0.0
        vk = k[:-1] + "v" if k.endswith("weight_g") else None
        den_floor = ref[vk].double().norm().item() if vk in ref else 0.0
        e, y = _rel(got[k], ref[k], scale, den_floor), _rel(yard[k], ref[k], scale, den_floor)
        bar = 2 * y + (floor_fwd if fwd else floor_grad)
        if fixed:
            bar = min(bar, 2e-5 if fwd else 2e-4)
        lines.append(f"{k} {e:.1e}/{y:.1e}")
        worst = max(worst, (e, k))
        if not (e <= bar):
            bad.append((k, e, y, bar))
    print(f"[{tag}] worst relative L2 {worst[0]:.2e} ({worst[1]});  error / fp32 yardstick: " + ", ".join(lines))
    assert not bad, bad


@functools.lru_cache(maxsize=None)
def _case(row):
    cfg = synth.ModelConfig(**MATRIX[row])
    mesh = synth.icosphere_mesh(4, seed=3)
    sd = synth.make_state_dict(mesh, cfg, seed=4)
    return cfg, mesh, sd


def _cpu_model(row, dtype=torch.float32, fused=False):
    cfg, mesh, sd = _case(row)
    m = nb.NeuMesh(helpers.OracleMeshGrid(mesh), **cfg.model_kwargs())
    m.load_state_dict(sd)
    m.train()
    m.fused_train = fused
    m._train_prims = TorchPrims("cpu") if fused else None
    return m.to(dtype)


def _vertex_slots(M):
    return ([0, M // 2] + ([M - 1] if M >= 9 else [])) if M >= 7 else []


def _points(M, mesh, seed):
    """M query points around the surface; from M = 7 on, two or three of them exactly on vertices (rho = 0)."""
    x, v = helpers.sample_points(M, seed=seed)
    x = x * 0.9
    pv = torch.from_numpy(mesh.vertices).float()
    for j, i in enumerate(_vertex_slots(M)):
        x[i] = pv[(97 * j + 11) % pv.shape[0]]
    return x, v


def _ref_module(row, dtype, dev):
    cfg, mesh, sd = _case(row)
    m = nb.NeuMesh(helpers.OracleMeshGrid(mesh), **cfg.model_kwargs())
    m.load_state_dict(sd)
    return m.to(device=dev, dtype=dtype)


# ------------------------------------------------------------------------------------------------------------------
# the float64 reference of the field op
# ------------------------------------------------------------------------------------------------------------------
def _wn(lin):
    return torch._weight_norm(lin.weight_v, lin.weight_g, 0), lin.bias


def reference_field(m, vertices, xyz, dirs, idx, w, with_color=True, kinks=None):
    """The field of NeuMesh module ``m`` in its own dtype at the given neighbours: (sdf [M,1], nabla [M,3], rgb [M,3] |
    None, named) where ``named`` holds the tensors FusedFieldFn takes as parameters (effective weights included), for
    gradients with respect to them.  Parameter gradients of ``m`` itself flow through ``torch._weight_norm``.
    ``kinks``: a list that receives the colour MLP's pre-activations (the inputs of its ReLUs)."""
    c = m._cfg
    dt, dev = m.geometry_features.dtype, m.geometry_features.device
    x = xyz.detach().to(dev, dt).requires_grad_(True)
    idx = idx.reshape(-1, 8).to(dev)
    w = w.detach().reshape(-1, 8).to(dev, dt)
    verts = vertices.to(dev, dt)
    named = {"indicator_vector": m.indicator_vector}
    with torch.enable_grad():
        if m.learn_indicator_weight:
            w1 = torch.sigmoid(m.indicator_weight_raw).reshape(())
        else:
            w1 = torch.tensor(0.1, dtype=dt, device=dev, requires_grad=True)
        named.update(w1=w1, geometry_features=m.geometry_features, color_features=m.color_features)
        # mesh_grid.py:121-144 (oracle.field.mesh_distance) at the supplied neighbours; rho is 0 with zero derivative
        # on a vertex, the limit the closed form takes there
        v = x[:, None, :] - verts[idx]
        r2 = (v * v).sum(-1, keepdim=True)
        rho = torch.where(r2 > 0, r2.clamp_min(torch.finfo(dt).tiny ** 0.5).sqrt(), torch.zeros_like(r2))
        ind_rows = m.indicator_vector[idx]
        mid = (ind_rows * w1 + v * rho) / (w1 + rho)
        ds = (w[..., None] * (v * mid).sum(-1, keepdim=True)).sum(-2)
        d_emb = positional_encoding(ds, c["multires_d"])
        fg = blend_rows(m.geometry_features, idx, w)
        named["_ind_rows"], named["_fg"] = ind_rows, fg     # per-point terms of the scatter-adds (not parameters)
        h = torch.cat([d_emb, positional_encoding(fg, c["multires_fg"])], -1)
        geo = m._geo_linears()
        for i, lin in enumerate(geo[:-1]):
            W, b = _wn(lin)
            named[f"geo.{i}.W"], named[f"geo.{i}.b"] = W, b
            h = F.softplus(F.linear(h, W, b), beta=100)
        W, b = _wn(geo[-1])
        named["geo_out.W"], named["geo_out.b"] = W, b
        sdf = F.linear(h, W, b)
        (nabla,) = torch.autograd.grad(sdf, x, torch.ones_like(sdf), create_graph=True)
        col = m._col_linears()
        for i, lin in enumerate(col[:-1]):
            named[f"col.{i}.W"], named[f"col.{i}.b"] = lin.weight, lin.bias
        named["col_out.W"], named["col_out.b"] = col[-1].weight, col[-1].bias
        rgb = None
        if with_color:
            fc = blend_rows(m.color_features, idx, w)
            named["_fc"] = fc
            parts = [nabla] if m.enable_nablas_input else []
            parts += [d_emb, positional_encoding(dirs.to(dev, dt), c["multires_view"]),
                      positional_encoding(fc, c["multires_ft"])]
            h = torch.cat(parts, -1)
            for lin in col[:-1]:
                z = F.linear(h, lin.weight, lin.bias)
                if kinks is not None:
                    kinks.append(z.detach())
                h = torch.relu(z)
            rgb = torch.sigmoid(F.linear(h, col[-1].weight, col[-1].bias))
    return sdf, nabla, rgb, named


def _neighbours(model, x):
    with torch.no_grad():
        _, idx, w = model.mesh_grid.compute_distance(x, indicator_vector=model.indicator_vector.detach(),
                                                     indicator_weight=model.indicator_weight_value())
    return idx, w


def _off_relu_kinks(row, model, x, v, seed, margin=3e-5):
    """Replace the points at which a colour pre-activation of the float64 field lies within ``margin`` x its layer's RMS
    of 0: there fp32 and float64 may take different sides of the ReLU, and the gradient jumps (about one such point in
    40 at this margin; a flipped unit moves the colour-weight gradients by ~1e-3 at M ~ 1e4, with the fp32 reference
    flipping other units).  Points on vertices are replaced by other vertices."""
    cfg, mesh, sd = _case(row)
    dev = model.geometry_features.device
    m = _ref_module(row, torch.float64, dev)
    verts = torch.from_numpy(mesh.vertices)
    pv = verts.float()
    g = torch.Generator().manual_seed(seed + 1000)
    x, v = x.clone(), v.clone()
    on_vertex = torch.zeros(x.shape[0], dtype=torch.bool)
    on_vertex[_vertex_slots(x.shape[0])] = True
    for _ in range(10):
        idx, w = _neighbours(model, x.to(dev))
        kinks = []
        reference_field(m, verts, x, v, idx, w, kinks=kinks)
        near = torch.zeros(x.shape[0], dtype=torch.bool)
        for z in kinks:
            near |= (z.abs() < margin * z.pow(2).mean().sqrt()).any(-1).cpu()
        if not near.any():
            return x, v
        n = int(near.sum())
        xn, vn = helpers.sample_points(n, seed=int(torch.randint(1 << 30, (1,), generator=g)))
        xn = xn * 0.9
        nv = near & on_vertex
        if nv.any():
            xn[nv[near]] = pv[torch.randint(pv.shape[0], (int(nv.sum()),), generator=g)]
        x[near], v[near] = xn, vn
    raise AssertionError("could not move the points off the colour MLP's ReLU kinks")


def _loss(sdf, nabla, rgb, up, pattern):
    bs, bn, br = up
    loss = sdf.new_zeros(())
    if "s" in pattern:
        loss = loss + (sdf.reshape(-1, 1) * bs.to(sdf)).sum()
    if "n" in pattern:
        loss = loss + (nabla.reshape(-1, 3) * bn.to(nabla)).sum()
    if "r" in pattern:
        loss = loss + (rgb.reshape(-1, 3) * br.to(rgb)).sum()
    return loss


def _upstream(M, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(M, 1, generator=g), torch.randn(M, 3, generator=g), torch.randn(M, 3, generator=g)


def _reference_run(row, dtype, dev, x, v, idx, w, up, pattern="snr", with_color=True):
    """-> {sdf, nabla, rgb, every parameter gradient by name} of the reference module in ``dtype`` on ``dev``."""
    cfg, mesh, sd = _case(row)
    m = nb.NeuMesh(helpers.OracleMeshGrid(mesh), **cfg.model_kwargs())
    m.load_state_dict(sd)
    m = m.to(device=dev, dtype=dtype)
    sdf, nabla, rgb, _ = reference_field(m, torch.from_numpy(mesh.vertices), x, v, idx, w, with_color)
    _loss(sdf, nabla, rgb, up, pattern).backward()
    out = {"sdf": sdf, "nabla": nabla}
    if with_color:
        out["rgb"] = rgb
    out.update({k: p.grad if p.grad is not None else torch.zeros_like(p) for k, p in m.named_parameters()
                if k != "ln_s"})
    return out


def _fused_run(model, x, v, up, pattern="snr"):
    """All three outputs through ``NeuMesh._train_field`` (FusedFieldFn) -> (results by name, idx, w)."""
    model.zero_grad(set_to_none=True)
    sdf, nabla, rgb, (idx, w) = model._train_field(x, v, with_color=True)
    _loss(sdf, nabla, rgb, up, pattern).backward()
    out = {"sdf": sdf, "nabla": nabla, "rgb": rgb}
    out.update({k: p.grad if p.grad is not None else torch.zeros_like(p) for k, p in model.named_parameters()
                if k != "ln_s"})
    return out, idx, w


# ------------------------------------------------------------------------------------------------------------------
# CPU: row membership, the sequencing over the whole matrix, the upstream-gradient patterns
# ------------------------------------------------------------------------------------------------------------------
class _FakeCudaGrid:   # passes where fused_supported() only checks that a CUDA MeshGrid is present
    grid = type("G", (), {"handle": None})()

    def get_number_of_vertices(self):
        return 42

    def get_vertex_normal_torch(self):
        return torch.zeros(42, 3)


def test_rows_cover_what_they_claim_cpu():
    """Each out-of-envelope row is refused by the library (``nmb_field_check`` via ``fused_supported()``, stated by
    ``helpers.inside``) on every engine, the other rows are accepted by at least one, and the training op takes all."""
    engines = ["tcgen05_f16", "tcgen05", "fp32"]
    for name, kw in MATRIX.items():
        cfg = synth.ModelConfig(**kw)
        m = nb.NeuMesh(_FakeCudaGrid(), **cfg.model_kwargs())
        seen = []
        for engine in engines:
            m.mlp_engine = engine
            assert m.fused_supported() == helpers.inside(engine, cfg), (name, engine)
            seen.append(m.fused_supported())
        assert any(seen) == (name not in OUTSIDE), (name, seen)
        m.train()
        m._train_prims = TorchPrims("cpu")
        with torch.enable_grad():
            assert m._fused_train_ok(), name


@pytest.mark.parametrize("row", list(MATRIX))
def test_fused_sequencing_vs_float64_reference_cpu(row):
    """FusedFieldFn on torch primitives (fp32, CPU) against the float64 reference, all three outputs, ~200 points."""
    cfg, mesh, sd = _case(row)
    model = _cpu_model(row, fused=True)
    x, v = _off_relu_kinks(row, model, *_points(203, mesh, seed=5), seed=5)
    up = _upstream(203, seed=6)
    got, idx, w = _fused_run(model, x, v, up)
    ref = _reference_run(row, torch.float64, "cpu", x, v, idx, w, up)
    yard = _reference_run(row, torch.float32, "cpu", x, v, idx, w, up)
    # measured: worst 1.5e-5 (raw_codes_and_view, geometry_features), 7.8e-6 on the fixed-bar rows
    _compare(f"cpu {row}", got, ref, yard, 2e-6, 2e-5, fixed=row in FIXED_BAR_ROWS, bands=cfg.multires_d)


def _op_inputs(model, x, v, idx, w, dt=torch.float32):
    """field_forward / field_backward arguments from a NeuMesh model (effective weights as FusedFieldFn sees them)."""
    c = model._cfg
    spec = train_ops.FieldSpec(c["geometry_dim"], c["color_dim"], c["multires_d"], c["multires_fg"], c["multires_ft"],
                               c["multires_view"], model.enable_nablas_input, c["D_density"], c["D_color"])
    cast = lambda z: z.detach().to(dt).contiguous()   # noqa: E731
    with torch.no_grad():
        geo_l, col_l = model._geo_linears(), model._col_linears()
        geo = [(cast(torch._weight_norm(l.weight_v, l.weight_g, 0)), cast(l.bias)) for l in geo_l]
        col = [(cast(l.weight), cast(l.bias)) for l in col_l]
    t = dict(xyz=cast(x), dirs=cast(v), idx=idx.reshape(-1, 8).contiguous(), w=cast(w.reshape(-1, 8)),
             vertices=cast(model.mesh_grid.get_vertices_torch()), indicator_vector=cast(model.indicator_vector),
             geometry_features=cast(model.geometry_features), color_features=cast(model.color_features),
             w1=model.indicator_weight_value())
    return spec, t, geo[:-1], geo[-1], col[:-1], col[-1]


def _direct_run(P, model, x, v, idx, w, up, pattern, with_color=True):
    """field_forward + field_backward with None for every upstream gradient the pattern leaves out -> results by the
    names of ``reference_field``'s ``named``."""
    spec, t, geo, geo_out, col, col_out = _op_inputs(model, x, v, idx, w)
    dev = t["xyz"].device
    sdf, nabla, rgb, S = train_ops.field_forward(P, spec, t, geo, geo_out, col, col_out, with_color=with_color)
    bs, bn, br = (u.to(dev).contiguous() for u in up)
    G = train_ops.field_backward(P, spec, S, geo, geo_out, col, col_out, bs.reshape(-1) if "s" in pattern else None,
                                 bn if "n" in pattern else None, br if "r" in pattern else None)
    out = {"sdf": sdf.reshape(-1, 1), "nabla": nabla}
    if with_color:
        out["rgb"] = rgb
    out.update(indicator_vector=G["indicator_vector"], w1=G["w1"].reshape(()), geometry_features=G["geometry_features"],
               color_features=G["color_features"])
    for i, (dW, db) in enumerate(G["geo"]):
        out[f"geo.{i}.W"], out[f"geo.{i}.b"] = dW, db
    out["geo_out.W"], out["geo_out.b"] = G["geo_out"]
    for i, (dW, db) in enumerate(G["col"]):
        out[f"col.{i}.W"], out[f"col.{i}.b"] = dW, db
    out["col_out.W"], out["col_out.b"] = G["col_out"]
    return out


def _reference_named(row, dtype, dev, x, v, idx, w, up, pattern, with_color=True, terms=False):
    """Reference outputs and gradients with respect to the op's own parameters (effective weights, w1); ``terms``:
    also with respect to the gathered indicator rows and the blended codes (the scatter-adds' per-point terms)."""
    cfg, mesh, sd = _case(row)
    m = nb.NeuMesh(helpers.OracleMeshGrid(mesh), **cfg.model_kwargs())
    m.load_state_dict(sd)
    m = m.to(device=dev, dtype=dtype)
    sdf, nabla, rgb, named = reference_field(m, torch.from_numpy(mesh.vertices), x, v, idx, w, with_color)
    loss = _loss(sdf, nabla, rgb, up, pattern)
    keys = [k for k in named if terms or not k.startswith("_")]
    grads = torch.autograd.grad(loss, [named[k] for k in keys], allow_unused=True)
    out = {"sdf": sdf, "nabla": nabla}
    if with_color:
        out["rgb"] = rgb
    out.update({k: (gr if gr is not None else torch.zeros_like(named[k])) for k, gr in zip(keys, grads)})
    return out


# pattern: which of sdf (s), nabla (n), rgb (r) carry an upstream gradient; None for the others
PATTERNS = {"all": ("A", "snr"), "sdf_only": ("A", "s"), "nabla_only": ("A", "n"), "rgb_only_nabla_input": ("A", "r"),
            "rgb_only_no_nabla_input": ("F", "r"), "sdf_nabla_no_colour": ("A", "sn")}


def _pattern_check(name, P, dev, M, floor_fwd, floor_grad):
    row, pattern = PATTERNS[name]
    with_color = name != "sdf_nabla_no_colour"
    cfg, mesh, sd = _case(row)
    model = _cpu_model(row) if dev == "cpu" else helpers.cuda_model(mesh, cfg, sd, "tcgen05").train()
    x, v = _off_relu_kinks(row, model, *_points(M, mesh, seed=8), seed=8)
    x, v = x.to(dev), v.to(dev)
    with torch.no_grad():
        _, idx, w = model.mesh_grid.compute_distance(x, indicator_vector=model.indicator_vector.detach(),
                                                     indicator_weight=model.indicator_weight_value())
    up = _upstream(M, seed=9)
    got = _direct_run(P, model, x, v, idx, w, up, pattern, with_color)
    ref = _reference_named(row, torch.float64, dev, x, v, idx, w, up, pattern, with_color)
    yard = _reference_named(row, torch.float32, dev, x, v, idx, w, up, pattern, with_color)
    # a gradient the pattern cannot reach is exactly zero in the reference and must be exactly zero here
    for k in ref:
        if k not in FWD and ref[k].abs().max().item() == 0:
            assert got[k].abs().max().item() == 0, (name, k)
    _compare(f"{dev} pattern {name} M={M}", got, ref, yard, floor_fwd, floor_grad, fixed=row in FIXED_BAR_ROWS,
             bands=cfg.multires_d)


@pytest.mark.parametrize("name", list(PATTERNS))
def test_upstream_patterns_sequencing_cpu(name):
    _pattern_check(name, TorchPrims("cpu"), "cpu", 157, 2e-6, 2e-5)


ENTRIES = ["forward_density_only", "forward_with_nablas", "empty", "leading_dims"]


def _api_patterns(entry, model, ref_model, mesh, dev):
    """The grad-mode entry points of NeuMesh (FusedFieldFn with with_color False, empty batch, [R,S,3] inputs) against
    the reference module ``ref_model`` (float64) at the neighbours the model's grid returns."""
    verts = torch.from_numpy(mesh.vertices)
    R, S = (0, 5) if entry == "empty" else ((3, 41) if entry == "leading_dims" else (1, 123))
    x, v = _points(max(R * S, 1), mesh, seed=12)
    x, v = x[:R * S].reshape(R, S, 3).to(dev), v[:R * S].reshape(R, S, 3).to(dev)
    g = torch.Generator().manual_seed(13)
    bs, bn, br = torch.randn(R, S, 1, generator=g), torch.randn(R, S, 3, generator=g), torch.randn(R, S, 3, generator=g)
    model.zero_grad(set_to_none=True)
    if entry == "forward_density_only":
        sdf = model.forward_density_only(x)
        nabla = rgb = None
        loss = (sdf * bs.to(dev)).sum()
    elif entry == "forward_with_nablas":
        sdf, nabla = model.forward_with_nablas(x)
        rgb = None
        loss = (sdf * bs.to(dev)).sum() + (nabla * bn.to(dev)).sum()
    else:
        sdf, rgb = model.forward(x, v)
        _, nabla = model.forward_with_nablas(x)
        loss = (sdf * bs.to(dev)).sum() + (nabla * bn.to(dev)).sum() + (rgb * br.to(dev)).sum()
    assert sdf.shape == (R, S, 1)
    if loss.requires_grad:      # an empty batch returns empty outputs without a graph
        loss.backward()
    got = {"sdf": sdf}
    if nabla is not None:
        got["nabla"] = nabla
    if rgb is not None:
        got["rgb"] = rgb
    got.update({k: p.grad if p.grad is not None else torch.zeros_like(p) for k, p in model.named_parameters()
                if k != "ln_s"})
    if R * S == 0:
        assert all(t.abs().sum().item() == 0 for k, t in got.items() if k not in FWD)
        return None
    with torch.no_grad():
        _, idx, w = model.mesh_grid.compute_distance(x.reshape(-1, 3), indicator_vector=model.indicator_vector.detach(),
                                                     indicator_weight=model.indicator_weight_value())
    out = {}
    for dt in (torch.float64, torch.float32):
        m = ref_model.to(dt)
        m.zero_grad(set_to_none=True)
        s_, n_, r_, _ = reference_field(m, verts, x.reshape(-1, 3), v.reshape(-1, 3), idx, w, with_color=rgb is not None)
        l_ = (s_ * bs.reshape(-1, 1).to(s_)).sum()
        if nabla is not None:
            l_ = l_ + (n_ * bn.reshape(-1, 3).to(n_)).sum()
        if rgb is not None:
            l_ = l_ + (r_ * br.reshape(-1, 3).to(r_)).sum()
        l_.backward()
        o = {"sdf": s_}
        if nabla is not None:
            o["nabla"] = n_
        if rgb is not None:
            o["rgb"] = r_
        o.update({k: p.grad.clone() if p.grad is not None else torch.zeros_like(p) for k, p in m.named_parameters()
                  if k != "ln_s"})
        out[dt] = o
    got = {k: t.reshape(out[torch.float64][k].shape) for k, t in got.items()}
    return got, out[torch.float64], out[torch.float32]


@pytest.mark.parametrize("entry", ENTRIES)
def test_grad_mode_entry_points_sequencing_cpu(entry):
    """forward_density_only / forward_with_nablas in grad mode (the op with with_color False), an empty batch and
    [R, S, 3] inputs, on torch primitives against the float64 reference."""
    cfg, mesh, sd = _case("A")
    ref_model = nb.NeuMesh(helpers.OracleMeshGrid(mesh), **cfg.model_kwargs())
    ref_model.load_state_dict(sd)
    res = _api_patterns(entry, _cpu_model("A", fused=True), ref_model, mesh, "cpu")
    if res is not None:
        _compare(f"cpu entry {entry}", *res, 2e-6, 2e-5, fixed=True)


# ------------------------------------------------------------------------------------------------------------------
# CPU: whole training step, fused sequencing on torch primitives against float64
# ------------------------------------------------------------------------------------------------------------------
STEP_ROWS = ["A", "B", "F", "D_color_8"]
N_STEP_RAYS = 16
# measured on an H100 (CUDA error / fp32 yardstick): loss 4.3e-6 / 9.6e-7 (row A); worst gradient excess over 2 x the
# yardstick 3.6e-5 (row B, density_linear.bias 5.5e-5 / 4.6e-6).  The sharpness s ~ 245 of the alpha amplifies the
# fp32 sdf rounding, and the colour MLP's ReLU kinks are not avoided at 2 000 samples
STEP_FLOOR_FWD, STEP_FLOOR_GRAD = 1e-5, 1e-4


def _step_loss(rgb, depth, ex):
    """helpers.train_loss with the depth term weighted by opacity: depth = sum(w z) / (sum(w) + 1e-10) means nothing on
    a ray whose opacity is ~0, and fp32 / float64 differ there by whole units."""
    nab, acc = ex["implicit_nablas"], ex["mask_volume"]
    return rgb.mean() + 0.5 * acc.mean() + 0.1 * (depth * acc).mean() + 0.1 * ((nab.norm(dim=-1) - 1.0) ** 2).mean()


def _step(model, o, d, z):
    model.zero_grad(set_to_none=True)
    rgb, depth, ex = nb.volume_render(o, d, model, rayschunk=4096, z_samples=z, **helpers.TRAIN_KW)
    loss = _step_loss(rgb, depth, ex)
    loss.backward()
    return {"loss": loss.detach().reshape(1), **{k: p.grad.detach() for k, p in model.named_parameters()
                                                 if p.grad is not None}}


def _step_rays(golden_dir):
    g = dict(np.load(f"{golden_dir}/train_step_small.npz", allow_pickle=False))
    sl = slice(0, N_STEP_RAYS)
    return (torch.from_numpy(g["rays_o"])[sl], torch.from_numpy(g["rays_d"])[sl], torch.from_numpy(g["d_all"])[sl])


def _step_references(row, o, d, z):
    refs = {}
    for dt in (torch.float64, torch.float32):
        refs[dt] = _step(_cpu_model(row, dtype=dt), o.to(dt), d.to(dt), z.to(dt))
    return refs[torch.float64], refs[torch.float32]


@pytest.mark.parametrize("row", STEP_ROWS)
def test_train_step_sequencing_vs_float64_cpu(row, golden_dir):
    """The whole step through ``volume_render`` (torch-primitive sequencing of the fused op, teacher-forced depths of
    the golden file) against the torch-op path in float64; the yardstick is that path in fp32."""
    o, d, z = _step_rays(golden_dir)
    ref, yard = _step_references(row, o, d, z)
    got = _step(_cpu_model(row, fused=True), o, d, z)
    assert set(got) == set(ref)
    _compare(f"cpu step {row}", got, ref, yard, STEP_FLOOR_FWD, STEP_FLOOR_GRAD)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the CUDA kernels
# ------------------------------------------------------------------------------------------------------------------
def _dev():
    return torch.device("cuda:0")


def _sizes():
    """Batch sizes from the kernels' geometry; P = 32 x SMs (the *_out_bwd kernels run min(ceil(M/8), 4 SMs) blocks of 8
    warps, so from P on a warp strides over several points)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    P = 32 * sms
    return {"1": 1, "7": 7, "8": 8, "9": 9, "P-1": P - 1, "P": P, "P+1": P + 1, "3P+5": 3 * P + 5,
            "4095": 4095, "4096": 4096, "4097": 4097, "65539": 65539}


SIZE_IDS = ["1", "7", "8", "9", "P-1", "P", "P+1", "3P+5", "4095", "4096", "4097", "65539"]
MID_SIZE = "3P+5"
# measured on an H100 80GB HBM3 (132 SMs) at a 400 W power limit, outside the high-band rows C / D: worst error 1.3e-5
# (row raw_codes_and_view, geometry_features; 1.0e-5 on the fixed-bar rows), always within 2 x the fp32 yardstick + these
GPU_FLOOR_FWD, GPU_FLOOR_GRAD = 2e-6, 2e-5


@functools.lru_cache(maxsize=None)
def _gpu_model(row):
    cfg, mesh, sd = _case(row)
    return helpers.cuda_model(mesh, cfg, sd, "tcgen05").train()


def _gpu_field_check(row, size_id):
    dev = _dev()
    cfg, mesh, sd = _case(row)
    M = _sizes()[size_id]
    model = _gpu_model(row)
    x, v = _off_relu_kinks(row, model, *_points(M, mesh, seed=15), seed=15)
    up = _upstream(M, seed=16)
    n0 = nb._lib.launch_count()
    got, idx, w = _fused_run(model, x.to(dev), v.to(dev), up)
    torch.cuda.synchronize()
    assert nb._lib.launch_count() - n0 >= 10, "the field op did not run on the library's kernels"
    ref = _reference_run(row, torch.float64, dev, x, v, idx, w, up)
    yard = _reference_run(row, torch.float32, dev, x, v, idx, w, up)
    _compare(f"gpu {row} M={M}", got, ref, yard, GPU_FLOOR_FWD, GPU_FLOOR_GRAD, fixed=row in FIXED_BAR_ROWS,
             bands=cfg.multires_d)


@pytest.mark.gpu
@pytest.mark.parametrize("row", list(MATRIX))
def test_field_op_matrix_vs_float64(row):
    _gpu_field_check(row, MID_SIZE)


@pytest.mark.gpu
@pytest.mark.parametrize("size_id", [s for s in SIZE_IDS if s != MID_SIZE])
@pytest.mark.parametrize("row", ["A", "F"])
def test_field_op_batch_sizes_vs_float64(row, size_id):
    _gpu_field_check(row, size_id)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PATTERNS))
def test_upstream_patterns_vs_float64(name):
    """field_backward on the CUDA kernels with None for each upstream gradient a pattern leaves out."""
    _pattern_check(name, train_ops.CudaPrims(_dev()), _dev(), 3 * 32 * 132 + 5, GPU_FLOOR_FWD, GPU_FLOOR_GRAD)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ENTRIES)
def test_grad_mode_entry_points_vs_float64(entry):
    dev = _dev()
    cfg, mesh, sd = _case("A")
    model = helpers.cuda_model(mesh, cfg, sd, "tcgen05").train()
    ref_model = nb.NeuMesh(helpers.OracleMeshGrid(mesh), **cfg.model_kwargs())
    ref_model.load_state_dict(sd)
    ref_model = ref_model.to(dev)
    res = _api_patterns(entry, model, ref_model, mesh, dev)
    if res is not None:
        _compare(f"gpu entry {entry}", *res, GPU_FLOOR_FWD, GPU_FLOOR_GRAD, fixed=True)


# ---- kernel edges ------------------------------------------------------------------------------------------------
def _f32_neighbours(z, n):
    out = [z]
    a = b = torch.tensor([z], dtype=torch.float32)
    for _ in range(n):
        a = torch.nextafter(a, torch.tensor([math.inf]))
        b = torch.nextafter(b, torch.tensor([-math.inf]))
        out += [a.item(), b.item()]
    return out


@pytest.mark.gpu
def test_softplus_kernels_at_the_threshold_vs_float64():
    """nmb_tr_softplus_fwd / _bwd at z = 0.2f and its neighbours (beta z = 20: the branch follows torch's fp32
    ``z * 100 > 20``), in the band 100 z in (12, 20] where 1 - s1 cancels in fp32, and far below 0."""
    dev = _dev()
    zs = _f32_neighbours(0.2, 3) + list(np.linspace(0.1201, 0.2, 257)) + [-1e-3, -0.05, -0.3, -1.0, -30.0, 0.0, 0.05,
                                                                         0.11, 0.25, 1.0, 7.0]
    z = torch.tensor(zs, dtype=torch.float32)
    n = z.numel()
    g = torch.Generator().manual_seed(21)
    a, bh, bt = (torch.randn(n, generator=g) for _ in range(3))
    P = train_ops.CudaPrims(dev)
    h, t, bz, ba = (torch.empty(n, device=dev) for _ in range(4))
    P.softplus_fwd(z.to(dev), a.to(dev), h, t)
    P.softplus_bwd(z.to(dev), a.to(dev), bh.to(dev), bt.to(dev), bz, ba)
    torch.cuda.synchronize()
    # float64 with the fp32 branch decision
    sat = (z * torch.tensor(100.0)) > 20
    z64, a64, bh64, bt64 = z.double(), a.double(), bh.double(), bt.double()
    s1 = torch.where(sat, torch.ones_like(z64), torch.sigmoid(100 * z64))
    s2 = torch.where(sat, torch.zeros_like(z64), 100 * torch.sigmoid(100 * z64) * torch.sigmoid(-100 * z64))
    h64 = torch.where(sat, z64, F.softplus(z64, beta=100, threshold=1e9))
    # torch's own fp32 softplus, first and second derivative (the yardstick of the cancelling s2 term)
    zt = z.clone().requires_grad_(True)
    ht = F.softplus(zt, beta=100)
    (tt,) = torch.autograd.grad(ht, zt, a, create_graph=True)
    (bzt,) = torch.autograd.grad((ht * bh).sum() + (tt * bt).sum(), zt)
    ref = {"h": h64, "t": s1 * a64, "ba": bt64 * s1}
    worst = 0.0
    for k, got in (("h", h), ("t", t), ("ba", ba)):
        e = ((got.cpu().double() - ref[k]).abs() / ref[k].abs().clamp_min(1e-30)).max().item()
        worst = max(worst, e)
        assert e <= 1e-6, (k, e)   # a few ulps (measured on an H100: 7.3e-7, log1pf in the softplus branch)
    bz64 = bh64 * s1 + bt64 * a64 * s2
    e_bz = (bz.cpu().double() - bz64).abs()
    e_torch = (bzt.detach().double() - bz64).abs()
    assert torch.equal(sat[:7], torch.tensor([False, True, False, True, False, True, False])), sat[:7]
    assert (e_bz <= 2 * e_torch + 4e-7 * bz64.abs() + 1e-12).all(), (e_bz - 2 * e_torch).max()
    print(f"softplus kernels at the threshold: worst relative error {worst:.2e}; bz max error {e_bz.max():.2e} "
          f"(torch fp32 {e_torch.max():.2e})")


def _split_plan(M, N, K, sms):
    """nmb_tr_gemm's split-K choice (csrc/train.cu) -> (splits first chosen, k_chunk, splits launched)."""
    gm, gn = -(-M // 128), -(-N // 128)
    if gm * gn < 2 * sms and K >= 4096:
        s0 = max(1, min(-(-2 * sms // (gm * gn)), -(-K // 1024)))
    else:
        return 1, K, 1
    kc = -(-(-(-K // s0)) // 16) * 16
    return s0, kc, -(-K // kc) if s0 > 1 else 1


@pytest.mark.gpu
def test_gemm_edges_vs_float64():
    """nmb_tr_gemm around the split-K switch (K = 4096), at K where the aligned k_chunk launches fewer splits than first
    chosen, at M = 1 and N = 1, split-K accumulating into C with ldc > N, and K = 0."""
    dev = _dev()
    P = train_ops.CudaPrims(dev)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    # dW products of the training op: A = dZ [K, M] (not K-contiguous), B = X [K, N]
    cases = [(256, 256, K) for K in (4095, 4096, 4097)] + [(256, 17, 4096 + 16 * k + s) for k in (1, 7, 64)
                                                            for s in (-1, 1)]
    # first K = 4096 + 16 k +- 1 per output shape at which ceil(K / k_chunk) < the splits first chosen (K ~ 7e4 - 3e5
    # for 114 - 132 SMs)
    shrink = []
    for M, N in ((256, 256), (256, 17), (1, 300)):
        hit = next(((M, N, K) for k in range(20000) for K in (4096 + 16 * k - 1, 4096 + 16 * k + 1)
                    if _split_plan(M, N, K, sms)[2] < _split_plan(M, N, K, sms)[0]), None)
        if hit:
            shrink.append(hit)
    assert len(shrink) >= 2, "no K where the aligned chunk reduces the split count"
    cases += shrink + [(1, 256, 5000), (256, 1, 5000), (1, 1, 4097), (1, 256, 177), (333, 1, 77)]
    g = torch.Generator().manual_seed(31)
    worst = 0.0
    for (M, N, K) in cases:
        for acc in (False, True):
            A = torch.randn(K, M, generator=g)
            B = torch.randn(K, N + 3, generator=g)
            C0 = torch.randn(M, N + 5, generator=g)
            ref = A.double().t() @ B[:, :N].double()
            if acc:
                ref = ref + C0[:, :N].double()
            C = C0.clone().to(dev)
            P.gemm(A.to(dev), M, False, B.to(dev), N + 3, False, C, N + 5, M, N, K, accumulate=acc)
            C = C.cpu()
            assert torch.equal(C[:, N:], C0[:, N:]), "wrote outside the N columns"
            # fp32 dot products of length K: error ~ sqrt(K) u sum|a b|; bound by the row norms
            bound = (A.double().abs().t() @ B[:, :N].double().abs()) * (K ** 0.5) * 6e-8 * 4 + 1e-6
            err = (C[:, :N].double() - ref).abs()
            worst = max(worst, (err / bound).max().item())
            assert (err <= bound).all(), ((M, N, K), acc, _split_plan(M, N, K, sms), (err / bound).max().item())
    # K = 0: C is the bias (or zero), or unchanged when accumulating
    one = torch.ones(1, device=dev)
    bias = torch.randn(7, generator=g).to(dev)
    C = torch.randn(5, 9, device=dev)
    C0 = C.clone()
    P.gemm(one, 1, True, one, 1, True, C, 9, 5, 7, 0, bias=bias)
    assert torch.equal(C[:, :7], bias.expand(5, 7)) and torch.equal(C[:, 7:], C0[:, 7:])
    C = C0.clone()
    P.gemm(one, 1, True, one, 1, True, C, 9, 5, 7, 0, accumulate=True)
    assert torch.equal(C, C0)
    P.gemm(one, 1, True, one, 1, True, C, 9, 5, 7, 0)
    assert (C[:, :7] == 0).all() and torch.equal(C[:, 7:], C0[:, 7:])
    print(f"nmb_tr_gemm edges: {len(cases)} shapes, worst error / bound {worst:.2e}; shrinking split plans "
          f"{[(c, _split_plan(*c, sms)) for c in shrink]}")


@pytest.mark.gpu
def test_colsum_many_rows_vs_float64():
    """nmb_tr_colsum with more rows than its grid covers in one pass (512 blocks x 8 rows) and N not a multiple of 32."""
    dev = _dev()
    P = train_ops.CudaPrims(dev)
    g = torch.Generator().manual_seed(41)
    for M, N in ((4097, 33), (70001, 77), (512 * 8 * 3 + 5, 1)):
        X = torch.randn(M, N, generator=g) + 0.5
        out = torch.full((N,), 0.25, device=dev)
        P.colsum(X.to(dev), out)
        ref = X.double().sum(0) + 0.25
        # fp32 summation: n_terms u sum|x| (n_terms: the rows one thread adds + the 8-way and atomic levels)
        terms = -(-M // (8 * 512)) + 8 + 512
        bound = terms * 6e-8 * X.double().abs().sum(0)
        err = (out.cpu().double() - ref).abs()
        assert (err <= bound).all(), (M, N, (err / bound).max().item())
        print(f"nmb_tr_colsum M={M} N={N}: max error {err.max():.2e}, {(err / bound).max():.2e} of the bound")


@pytest.mark.gpu
def test_atomic_scatter_cluster_vs_float64():
    """1e5 points that all share the same 8 neighbours: every code / indicator gradient of those rows is 1e5 atomic
    adds.  Bar per element: the fp32 summation-error bound gamma_n sum |terms| of the row, plus the per-point error."""
    dev = _dev()
    row = "A"
    cfg, mesh, sd = _case(row)
    model = _gpu_model(row)
    pv = torch.from_numpy(mesh.vertices).double()
    # the point just off a vertex whose 8th and 9th neighbours are furthest apart; the cluster is a ball well inside
    # that gap
    cand = pv[::10] * 1.02
    d = torch.cdist(cand, pv).sort(-1).values
    j = int((d[:, 8] - d[:, 7]).argmax())
    radius = float(d[j, 8] - d[j, 7]) / 8
    g = torch.Generator().manual_seed(51)
    M = 100_000
    x = (cand[j] + radius * torch.nn.functional.normalize(torch.randn(M, 3, generator=g, dtype=torch.float64), dim=-1)
         * torch.rand(M, 1, generator=g, dtype=torch.float64)).float()
    v = torch.nn.functional.normalize(torch.randn(M, 3, generator=g), dim=-1)
    up = _upstream(M, seed=52)
    got, idx, w = _fused_run(model, x.to(dev), v.to(dev), up)
    rows = idx[0].sort().values
    assert (idx.sort(-1).values == rows).all(), "the cluster's points do not share their neighbours"
    ref = _reference_run(row, torch.float64, dev, x, v, idx, w, up)
    yard = _reference_run(row, torch.float32, dev, x, v, idx, w, up)
    # every point sits in the same spot: ReLU kinks of the colour MLP are not avoided here, the yardstick rule alone
    # applies
    _compare("gpu cluster", got, ref, yard, GPU_FLOOR_FWD, GPU_FLOOR_GRAD)
    # per element of the 8 rows: |error| <= 2 x the fp32 reference's + gamma_M sum_p |term_p| (fp32 summation of M
    # terms in any order) + 1e-5 sum_p |term_p| (the terms' own fp32 error)
    T = _reference_named(row, torch.float64, dev, x, v, idx, w, up, "snr", terms=True)
    fi, w64 = idx.reshape(-1).to(dev), w.to(dev, torch.float64)
    S = {"geometry_features": (w64[..., None] * T["_fg"].abs()[:, None, :]).reshape(-1, cfg.geometry_dim),
         "color_features": (w64[..., None] * T["_fc"].abs()[:, None, :]).reshape(-1, cfg.color_dim),
         "indicator_vector": T["_ind_rows"].abs().reshape(-1, 3)}
    u = 2.0 ** -24
    gamma = M * u / (1 - M * u)
    worst = 0.0
    for k, terms in S.items():
        s = torch.zeros(ref[k].shape, dtype=torch.float64, device=dev).index_add_(0, fi, terms)[rows]
        e = (got[k][rows].double() - ref[k][rows].double()).abs()
        ey = (yard[k][rows].double() - ref[k][rows].double()).abs()
        bound = 2 * ey + (gamma + 1e-5) * s
        worst = max(worst, (e / bound.clamp_min(1e-30)).max().item())
        assert (e <= bound).all(), (k, (e / bound.clamp_min(1e-30)).max().item())
        assert got[k].abs().sum(-1).count_nonzero().item() <= 8, k
    print(f"cluster of {M} points on 8 shared rows: worst error {worst:.2e} of the fp32 summation bound")


# ---- whole step --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("row", STEP_ROWS)
def test_train_step_cuda_vs_float64(row, golden_dir):
    """The training step on the CUDA kernels (fused op in grad mode) at sample depths teacher-forced to the CUDA
    cascade's own ``d_all`` (the golden file's depths where the fused renderer does not take the row), against the
    torch-op path in float64 on CPU at those depths; yardstick: the torch-op path in fp32."""
    dev = _dev()
    cfg, mesh, sd = _case(row)
    model = _gpu_model(row)
    o, d, z = _step_rays(golden_dir)
    if model.fused_supported():
        with torch.no_grad():
            _, _, ex = nb.volume_render(o.to(dev), d.to(dev), model, rayschunk=4096, **helpers.TRAIN_KW)
        z = ex["d_all"].cpu()
    n0 = nb._lib.launch_count()
    got = _step(model, o.to(dev), d.to(dev), z.to(dev))
    torch.cuda.synchronize()
    assert nb._lib.launch_count() - n0 > 20, "the training step did not run on the library's kernels"
    ref, yard = _step_references(row, o, d, z)
    assert set(got) == set(ref)
    _compare(f"gpu step {row}", got, ref, yard, STEP_FLOOR_FWD, STEP_FLOOR_GRAD)


# ---- NeuS teacher ------------------------------------------------------------------------------------------------
NEUS_CASES = {
    "D8_skip4_em6_W256": dict(),
    "D8_noskip_em6_W256": dict(surface=dict(skips=[])),
    "D8_skip2_6_em0_W64": dict(surface=dict(skips=[2, 6], embed_multires=0), W_geo_feat=64),
    "D8_skip4_em10_W64": dict(surface=dict(embed_multires=10), W_geo_feat=64),
    "D2_noskip_em10_W256": dict(surface=dict(D=2, skips=[], embed_multires=10)),
    "D2_noskip_em0_W64_noview": dict(surface=dict(D=2, skips=[], embed_multires=0), W_geo_feat=64,
                                     radiance=dict(use_view_dirs=False)),
    "D8_skip4_em6_W256_noview": dict(radiance=dict(use_view_dirs=False)),
}


def _neus(case):
    c = NEUS_CASES[case]
    kw = dict(helpers.NEUS_KW)
    kw["surface_cfg"] = dict(kw["surface_cfg"], **c.get("surface", {}))
    kw["radiance_cfg"] = dict(kw["radiance_cfg"], **c.get("radiance", {}))
    kw["W_geo_feat"] = c.get("W_geo_feat", kw["W_geo_feat"])
    m = NeuS(**kw)
    m.load_state_dict(helpers.neus_state_dict(m, 60))
    return m.eval()


def _neus_points(M, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(M, 3, generator=g) * 1.6 - 0.8
    v = torch.nn.functional.normalize(torch.randn(M, 3, generator=g), dim=-1)
    return x, v


def _neus_eval(m, x, v):
    s = m.implicit_surface
    sdf, nabla, feat = s.forward_with_nablas(x, has_grad_bypass=False)
    with torch.no_grad():
        rad = m.radiance_net.forward(x, v, nabla, feat)
    return {"sdf": sdf, "nabla": nabla, "feature": feat, "radiance": rad}


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 127, 4099])
@pytest.mark.parametrize("case", list(NEUS_CASES))
def test_neus_teacher_fused_vs_float64(case, M):
    """The fused no-grad teacher (value + 3 tangent row blocks through nmb_tr_gemm / nmb_tr_softplus_fwd, the
    radiance net with the fused ReLU epilogue) against the same module's torch-op path in float64 (autograd nabla)."""
    dev = _dev()
    m = _neus(case)
    x, v = _neus_points(M, seed=61)
    ref = _neus_eval(m.double(), x.double(), v.double())
    yard = _neus_eval(m.float(), x, v)
    md = m.to(dev)
    n0 = nb._lib.launch_count()
    with torch.no_grad():
        got = _neus_eval(md, x.to(dev), v.to(dev))
        sdf2, nabla2 = md.forward_with_nablas(x.to(dev))
    torch.cuda.synchronize()
    D = md.implicit_surface.D
    assert nb._lib.launch_count() - n0 >= (D + 1) + 3 * D + md.radiance_net.D + 1, "the teacher did not run fused"
    assert torch.equal(sdf2, got["sdf"]) and torch.equal(nabla2, got["nabla"])
    got = {k: t.reshape(ref[k].shape) for k, t in got.items()}
    lines, bad = [], []
    for k in ref:
        e, y = _rel(got[k], ref[k], 1e-3), _rel(yard[k], ref[k], 1e-3)
        bar = 2 * y + 1e-5      # measured on an H100: nabla 5.3e-6 with the fp32 path at 1.6e-6
        lines.append(f"{k} {e:.1e}/{y:.1e}")
        if not e <= bar:
            bad.append((k, e, y, bar))
    print(f"[neus {case} M={M}] error / fp32 yardstick: " + ", ".join(lines))
    assert not bad, bad


@pytest.mark.gpu
def test_neus_radiance_with_skips_takes_the_torch_path():
    dev = _dev()
    net = RadianceNet(D=4, skips=[2], W_geo_feat=64, embed_multires=-1, embed_multires_view=4).to(dev).eval()
    x, v = _neus_points(33, seed=71)
    x, v = x.to(dev), v.to(dev)
    feat = torch.randn(33, 64, device=dev)
    n0 = nb._lib.launch_count()
    with torch.no_grad():
        rad = net.forward(x, v, v, feat)
    torch.cuda.synchronize()
    assert nb._lib.launch_count() == n0, "a radiance net with skips ran on the fused kernels"
    assert rad.shape == (33, 3) and torch.isfinite(rad).all()
