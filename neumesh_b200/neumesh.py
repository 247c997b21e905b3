"""``NeuMesh`` field model - drop-in for ``models/frameworks/neumesh/neumesh.py`` (same constructor arguments,
``state_dict`` keys and method protocol), evaluated by the fused CUDA kernels whenever no gradient is required.

* no-grad queries (rendering, mesh extraction): ``forward_density_only`` / ``forward_with_nablas`` / ``forward`` call
  ``nmb_field_sdf`` / ``nmb_field_forward`` - octree KNN, gather + blend + positional encoding, tensor-core MLPs and
  the forward-mode nabla in hand-written kernels;
* grad-enabled queries (training, editing fine-tunes): the neighbour search is still the CUDA octree walk, the
  differentiable remainder is expressed in torch ops so autograd (including the eikonal loss' double backward) works.
"""
from __future__ import annotations

import contextlib
import ctypes as C

import torch
import torch.nn as nn
from torch.nn.utils import weight_norm

from . import _lib


class Embedder(nn.Module):
    """NeRF positional encoding with the reference's ordering (``models/base.py:15-87``):
    ``[x, sin(2^0 x), cos(2^0 x), ..., sin(2^(L-1) x), cos(2^(L-1) x)]``."""

    def __init__(self, input_dim: int, n_freqs: int):
        super().__init__()
        self.input_dim, self.n_freqs = input_dim, n_freqs
        self.out_dim = input_dim * (1 + 2 * n_freqs)
        self.freq_bands = [2.0 ** k for k in range(n_freqs)]

    def forward(self, x):
        out = [x]
        for f in self.freq_bands:
            out += [torch.sin(x * f), torch.cos(x * f)]
        return torch.cat(out, dim=-1)


def get_embedder(multires, input_dim=3):
    if multires < 0:
        return nn.Identity(), input_dim
    e = Embedder(input_dim, multires)
    return e, e.out_dim


def interpolation(features, indices, weights):
    return (features[indices] * weights.unsqueeze(-1)).sum(dim=-2)


def _mlp_stack(make_linear, act, in_dim, width, depth):
    """``Sequential(L0, act, Sequential(L, act), ...)`` - the module nesting fixes the state_dict key names
    (``pts_linears.0``, ``pts_linears.2.0``, ...; reference ``neumesh.py:76-100``)."""
    mods = [make_linear(in_dim, width), act()]
    for _ in range(depth - 1):
        mods.append(nn.Sequential(make_linear(width, width), act()))
    return nn.Sequential(*mods)


# MLP engines of the CUDA library (nmb_field_create's mlp_engine).  "tcgen05_f16" = fp16x3 split operands on fp16 wgmma
# (default: held to the oracle, the float64 truth and the reference's frame goldens by the tests); "tcgen05" = 3xTF32 on
# tf32 wgmma; "fp32" = CUDA-core verification engine.  The names predate the Hopper port and are kept for compatibility.
MLP_ENGINES = {"tcgen05": 0, "fp32": 1, "tcgen05_f16": 2}
DEFAULT_MLP_ENGINE = "tcgen05_f16"


class NeuMesh(nn.Module):
    def __init__(self, mesh_grid, D_density: int, D_color: int, W: int, geometry_dim: int, color_dim: int,
                 multires_view: int, multires_d: int, multires_fg: int, multires_ft: int, enable_nablas_input: bool,
                 input_view_dim=3, input_d_dim=1, ln_s=0.2996, speed_factor=1.0, learn_indicator_weight=True,
                 mlp_engine: str = DEFAULT_MLP_ENGINE):
        super().__init__()
        self.mesh_grid = mesh_grid
        V = mesh_grid.get_number_of_vertices()
        self.ln_s = nn.Parameter(torch.tensor([float(ln_s)]))
        self.speed_factor = speed_factor
        self.geometry_features = nn.Parameter(torch.randn(V, geometry_dim))
        self.color_features = nn.Parameter(torch.randn(V, color_dim))
        self.indicator_vector = nn.Parameter(mesh_grid.get_vertex_normal_torch().float().clone())
        self.learn_indicator_weight = learn_indicator_weight
        if learn_indicator_weight:
            self.indicator_weight_raw = nn.Parameter(torch.tensor([-2.0]))

        self.embed_fn_d, ch_d = get_embedder(multires_d, input_dim=input_d_dim)
        self.embed_fn_view, ch_view = get_embedder(multires_view, input_dim=input_view_dim)
        self.embed_fn_fg, ch_fg = get_embedder(multires_fg, input_dim=geometry_dim)
        self.embed_fn_ft, ch_ft = get_embedder(multires_ft, input_dim=color_dim)

        self.softplus = nn.Softplus(beta=100)
        self.pts_linears = _mlp_stack(lambda i, o: weight_norm(nn.Linear(i, o)), lambda: self.softplus,
                                      ch_d + ch_fg, W, D_density)
        self.enable_nablas_input = enable_nablas_input
        ch_color = ch_view + ch_ft + ch_d + (3 if enable_nablas_input else 0)
        self.views_linears = _mlp_stack(nn.Linear, lambda: nn.ReLU(inplace=True), ch_color, W, D_color)
        self.density_linear = weight_norm(nn.Linear(W, 1))
        self.color_linear = nn.Sequential(nn.Linear(W, 3), nn.Sigmoid())

        self._cfg = dict(D_density=D_density, D_color=D_color, W=W, geometry_dim=geometry_dim, color_dim=color_dim,
                         multires_view=multires_view, multires_d=multires_d, multires_fg=multires_fg,
                         multires_ft=multires_ft, input_view_dim=input_view_dim, input_d_dim=input_d_dim)
        if mlp_engine not in MLP_ENGINES:
            raise ValueError(f"mlp_engine must be one of {sorted(MLP_ENGINES)}")
        self.mlp_engine = mlp_engine
        self._field = None
        self._field_key = None
        self._field_check = {}        # mlp_engine -> None or the library's reason for refusing _cfg on that engine
        # grad-enabled queries on CUDA run the fused training op (train_ops.FusedFieldFn); False = torch-op path
        self.fused_train = True
        self._train_prims = None      # tests inject a torch implementation of the kernel interface here (CPU)

    # ------------------------------------------------------------------------------------------------------
    # packed CUDA field
    # ------------------------------------------------------------------------------------------------------
    def _geo_linears(self):
        return [self.pts_linears[0]] + [self.pts_linears[i][0] for i in range(2, len(self.pts_linears))] + \
            [self.density_linear]

    def _col_linears(self):
        return [self.views_linears[0]] + [self.views_linears[i][0] for i in range(2, len(self.views_linears))] + \
            [self.color_linear[0]]

    def _field_desc(self):
        """``nmb_field_desc`` with the configuration's integer fields set: all ``nmb_field_check`` reads."""
        c = self._cfg
        d = _lib.FieldDesc()
        d.D_density, d.D_color, d.W = c["D_density"], c["D_color"], c["W"]
        d.geometry_dim, d.color_dim = c["geometry_dim"], c["color_dim"]
        d.multires_d, d.multires_fg, d.multires_ft, d.multires_view = (c["multires_d"], c["multires_fg"],
                                                                       c["multires_ft"], c["multires_view"])
        d.enable_nablas_input = 1 if self.enable_nablas_input else 0
        return d

    def _fused_problem(self):
        """None if the fused kernels take this model, otherwise why not.  The input widths and the mesh grid are not in
        the descriptor and are tested here, first (a CPU or oracle grid never loads the library); the library's
        ``nmb_field_check`` owns every other limit."""
        c = self._cfg
        if c["input_view_dim"] != 3 or c["input_d_dim"] != 1:
            return "the fused kernels take input_view_dim = 3 and input_d_dim = 1"
        if not hasattr(getattr(self.mesh_grid, "grid", None), "handle"):
            return "the mesh grid is not a CUDA neumesh_b200.MeshGrid"
        if self.mlp_engine not in self._field_check:
            L = _lib.lib()
            rc = L.nmb_field_check(C.byref(self._field_desc()), MLP_ENGINES[self.mlp_engine])
            self._field_check[self.mlp_engine] = L.nmb_last_error().decode() if rc else None
        return self._field_check[self.mlp_engine]

    def fused_supported(self) -> bool:
        return self._fused_problem() is None

    def indicator_weight_value(self) -> float:
        return float(self.forward_indicator_weight()) if self.learn_indicator_weight else 0.1

    def packed_field(self):
        """``nmb_field`` handle, (re)packed when any parameter, the mesh grid or the engine changed.
        Editors hot-swap ``mesh_grid`` and re-assign ``indicator_vector`` (SURVEY.md section 7.3) - the key below
        covers tensor identity *and* in-place version counters.  A grid deformed in place (``MeshGrid.deform_``) has a
        new generation: the same handle is re-packed (``nmb_field_update``) into the grid's new slot order."""
        problem = self._fused_problem()
        if problem is not None:
            raise RuntimeError("this NeuMesh configuration is outside the fused CUDA kernels' specialisation: " + problem)
        params = list(self.parameters())
        key = (id(self.mesh_grid), id(self.mesh_grid.grid), self.mlp_engine, self.mesh_grid.grid.generation,
               float(self.speed_factor), tuple((p.data_ptr(), p._version) for p in params))
        if self._field is not None and key == self._field_key:
            return self._field
        dev = self.geometry_features.device
        _lib.require_cuda(self.geometry_features, "NeuMesh")
        d = self._field_desc()
        d.indicator_weight = self.indicator_weight_value()
        d.s = float(self.forward_s())
        keep = []

        def dp(t):
            t = t.detach().float().contiguous()
            keep.append(t)
            return t.data_ptr()

        d.geometry_features, d.color_features = dp(self.geometry_features), dp(self.color_features)
        d.indicator_vector = dp(self.indicator_vector)
        for i, lin in enumerate(self._geo_linears()):
            d.geo_v[i], d.geo_g[i], d.geo_b[i] = dp(lin.weight_v), dp(lin.weight_g), dp(lin.bias)
        for i, lin in enumerate(self._col_linears()):
            d.col_w[i], d.col_b[i] = dp(lin.weight), dp(lin.bias)
        engine = MLP_ENGINES[self.mlp_engine]
        with torch.cuda.device(dev):
            if self._field is not None and self._field_key is not None and self._field_key[:3] == key[:3]:
                _lib.check(_lib.lib().nmb_field_update(self._field, C.byref(d), _lib.stream_ptr(dev)))
            else:
                self._release_field()
                h = C.c_void_p()
                _lib.check(_lib.lib().nmb_field_create(self.mesh_grid.grid.handle, C.byref(d), engine,
                                                       _lib.stream_ptr(dev), C.byref(h)))
                self._field = h
        self._field_key = key
        return self._field

    def shell_free_grid(self):
        """(cells [G,G,G] uint8 CUDA tensor indexed [z,y,x], B): cells == 1 where every point of the cell of the grid
        over [-B,B]^3 provably has mesh distance >= 0.1 (the certificate the bounded near/far scan skips by)."""
        field = self.packed_field()
        dev = self.geometry_features.device
        G, B = C.c_int32(0), C.c_float(0.0)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().nmb_field_shell_grid(field, None, C.byref(G), C.byref(B), _lib.stream_ptr(dev)))
            cells = torch.zeros(max(G.value, 1) ** 3, dtype=torch.uint8, device=dev)
            if G.value > 0:
                _lib.check(_lib.lib().nmb_field_shell_grid(field, _lib.ptr(cells), C.byref(G), C.byref(B),
                                                           _lib.stream_ptr(dev)))
        g = max(G.value, 1)
        return cells.reshape(g, g, g), float(B.value)

    def _release_field(self):
        h = self.__dict__.get("_field")
        self.__dict__["_field"] = None   # plain attribute: bypass nn.Module.__setattr__ (safe at interpreter exit)
        if h:
            try:
                _lib.lib().nmb_field_destroy(h)
            except Exception:
                pass

    def __del__(self):
        self._release_field()

    def _fused_ok(self, *tensors) -> bool:
        """Fused kernels serve calls that cannot need a graph: grad mode off, CUDA inputs, supported config."""
        return (not torch.is_grad_enabled()) and all(t.is_cuda for t in tensors) and self.fused_supported() \
            and self.geometry_features.is_cuda

    def _fused_query(self, xyz, view_dirs=None, want_nabla=False, want_neighbours=False):
        """-> (sdf [...,1], nabla [...,3] | None, rgb [...,3] | None, neighbours) where neighbours is () or
        (ds [...,1], indices [...,8] int64, weights [...,8]) as ``forward(..., return_ds=True)`` returns them."""
        lead = xyz.shape[:-1]
        flat = xyz.detach().reshape(-1, 3).float().contiguous()
        M = flat.shape[0]
        dev = flat.device
        field = self.packed_field()
        sdf = torch.empty(M, 1, device=dev)
        nabla = torch.empty(M, 3, device=dev) if want_nabla else None
        rgb = dirs = None
        if view_dirs is not None:
            dirs = view_dirs.detach().reshape(-1, 3).float().contiguous()
            rgb = torch.empty(M, 3, device=dev)
        ds = idx = w = None
        if want_neighbours:
            ds = torch.empty(M, 1, device=dev)
            idx = torch.empty(M, 8, dtype=torch.int64, device=dev)
            w = torch.empty(M, 8, device=dev)
        if M > 0:
            with torch.cuda.device(dev):
                _lib.check(_lib.lib().nmb_field_forward_ex(field, _lib.ptr(flat), _lib.ptr(dirs), M, _lib.ptr(sdf),
                                                           _lib.ptr(rgb), _lib.ptr(nabla), _lib.ptr(ds), _lib.ptr(idx),
                                                           _lib.ptr(w), _lib.stream_ptr(dev)))
        nbr = (ds.reshape(*lead, 1), idx.reshape(*lead, 8), w.reshape(*lead, 8)) if want_neighbours else ()
        return (sdf.reshape(*lead, 1), (nabla.reshape(*lead, 3) if want_nabla else None),
                (rgb.reshape(*lead, 3) if rgb is not None else None), nbr)

    # ------------------------------------------------------------------------------------------------------
    # fused training op (grad-enabled queries): CUDA forward + backward, see train_ops.py
    # ------------------------------------------------------------------------------------------------------
    def _fused_train_ok(self, *tensors) -> bool:
        if not (self.fused_train and torch.is_grad_enabled()):
            return False
        c = self._cfg
        if c["W"] != 256 or min(c["multires_d"], c["multires_fg"], c["multires_ft"], c["multires_view"]) < 0 \
                or c["input_view_dim"] != 3 or c["input_d_dim"] != 1:
            return False
        if self._train_prims is not None:
            return True
        return all(t.is_cuda for t in tensors) and self.geometry_features.is_cuda \
            and hasattr(self.mesh_grid, "grid") and hasattr(self.mesh_grid.grid, "handle")

    def _train_field(self, xyz, view_dirs, with_color):
        """-> (sdf [...,1], nabla [...,3], rgb [...,3] | None, (ds-less) neighbours (idx, w)), differentiable w.r.t. every
        parameter; idx / w come from the CUDA octree (detached, as in mesh_grid.py:121-127)."""
        from . import train_ops
        lead = xyz.shape[:-1]
        flat = xyz.detach().reshape(-1, 3).float().contiguous()
        if flat.shape[0] == 0:   # nothing to evaluate (empty shard): empty outputs, no kernel launch
            z = flat.new_zeros(*lead, 1)
            return z, flat.new_zeros(*lead, 3), (flat.new_zeros(*lead, 3) if with_color else None), \
                (flat.new_zeros(*lead, 8, dtype=torch.int64), flat.new_zeros(*lead, 8))
        dirs = (view_dirs.detach().reshape(-1, 3).float().contiguous() if view_dirs is not None
                else torch.zeros_like(flat))
        w1_t = self.forward_indicator_weight().reshape(()) if self.learn_indicator_weight else \
            torch.tensor(0.1, device=flat.device)
        with torch.no_grad():
            _, idx, w = self.mesh_grid.compute_distance(flat, indicator_vector=self.indicator_vector.detach(),
                                                        indicator_weight=float(w1_t))
        c = self._cfg
        spec = train_ops.FieldSpec(c["geometry_dim"], c["color_dim"], c["multires_d"], c["multires_fg"], c["multires_ft"],
                                   c["multires_view"], self.enable_nablas_input, c["D_density"], c["D_color"])
        prims = self._train_prims if self._train_prims is not None else train_ops.CudaPrims(flat.device)
        params = [self.indicator_vector, w1_t, self.geometry_features, self.color_features]
        geo = self._geo_linears()
        for lin in geo[:-1]:
            params += [torch._weight_norm(lin.weight_v, lin.weight_g, 0), lin.bias]
        params += [torch._weight_norm(geo[-1].weight_v, geo[-1].weight_g, 0), geo[-1].bias]
        for lin in self._col_linears():
            params += [lin.weight, lin.bias]
        sdf, nabla, rgb = train_ops.FusedFieldFn.apply(spec, prims, bool(with_color), flat, dirs, idx, w,
                                                       self.mesh_grid.get_vertices_torch(), *params)
        return (sdf.reshape(*lead, 1), nabla.reshape(*lead, 3), rgb.reshape(*lead, 3) if with_color else None,
                (idx.reshape(*lead, 8), w.reshape(*lead, 8)))

    # ------------------------------------------------------------------------------------------------------
    # reference protocol (neumesh.py:113-174, 262-273)
    # ------------------------------------------------------------------------------------------------------
    def forward(self, xyz, view_dirs, need_nablas=True, nablas_only=False, return_ds=False):
        if need_nablas and not return_ds and self._fused_train_ok(xyz, view_dirs):
            sdf, nabla, rgb, _ = self._train_field(xyz, view_dirs, with_color=not nablas_only)
            return (sdf, nabla) if nablas_only else (sdf, rgb)
        if self._fused_ok(xyz, view_dirs):
            if nablas_only:
                sdf, nabla, _, nbr = self._fused_query(xyz, None, want_nabla=need_nablas,
                                                       want_neighbours=return_ds)
                return (sdf, (nabla if need_nablas else torch.zeros_like(sdf))) + nbr
            if need_nablas or not self.enable_nablas_input:
                sdf, _, rgb, nbr = self._fused_query(xyz, view_dirs, want_nabla=False,
                                                     want_neighbours=return_ds)
                return (sdf, rgb) + nbr
        if need_nablas:
            xyz.requires_grad_(True)
        with (torch.enable_grad() if need_nablas else contextlib.nullcontext()):
            ds, indices, weights = self.compute_distance(xyz)
        density, nablas, d_emb = self._forward_density(xyz, ds, self.geometry_features, indices, weights,
                                                       need_nablas=need_nablas)
        if nablas_only:
            out = (density, nablas)
        else:
            out = (density, self._forward_color(d_emb, view_dirs, self.color_features, indices, weights, nablas))
        if return_ds:
            out = out + (ds, indices, weights)
        return out

    def forward_density_only(self, xyz):
        if self._fused_train_ok(xyz):
            return self._train_field(xyz, None, with_color=False)[0]
        if self._fused_ok(xyz):
            return self._fused_query(xyz)[0]
        ds, indices, weights = self.compute_distance(xyz)
        return self._forward_density(xyz, ds, self.geometry_features, indices, weights, need_nablas=False)[0]

    def forward_with_nablas(self, xyz):
        if self._fused_train_ok(xyz):
            sdf, nabla, _, _ = self._train_field(xyz, None, with_color=False)
            return sdf, nabla
        if self._fused_ok(xyz):
            sdf, nabla, _, _ = self._fused_query(xyz, None, want_nabla=True)
            return sdf, nabla
        xyz.requires_grad_(True)
        with torch.enable_grad():
            ds, indices, weights = self.compute_distance(xyz)
        density, nablas, _ = self._forward_density(xyz, ds, self.geometry_features, indices, weights, need_nablas=True)
        return density, nablas

    def forward_color(self, d, view_dirs, color_features, indices=None, weights=None, nabla=None):
        """Colour network on caller-supplied neighbours (``neumesh.py:156-168``); ``color_features`` may be this
        model's own table or any ``[rows, color_dim]`` table ``indices`` points into (the texture editors pass another
        mesh's codes, ``editing/texture_neumesh/texture_neumesh.py:104-111``)."""
        if (indices is not None and weights is not None and (nabla is not None or not self.enable_nablas_input)
                and self._fused_ok(d, view_dirs, color_features, indices, weights)
                and color_features.dim() == 2 and color_features.shape[1] == self._cfg["color_dim"]):
            return self._fused_color(d, view_dirs, color_features, indices, weights, nabla)
        return self._forward_color(self.embed_fn_d(d), view_dirs, color_features, indices, weights, nabla)

    def _fused_color(self, d, view_dirs, color_features, indices, weights, nabla):
        lead = d.shape[:-1]
        dev = d.device
        ds = d.detach().reshape(-1).float().contiguous()
        M = ds.shape[0]
        rgb = torch.empty(M, 3, device=dev)
        if M == 0:
            return rgb.reshape(*lead, 3)
        dirs = view_dirs.detach().reshape(-1, 3).float().contiguous()
        idx = indices.detach().reshape(-1, 8).to(torch.int64).contiguous()
        w = weights.detach().reshape(-1, 8).float().contiguous()
        nab = nabla.detach().reshape(-1, 3).float().contiguous() if self.enable_nablas_input else None
        own = (color_features.data_ptr() == self.color_features.data_ptr()
               and color_features.shape == self.color_features.shape)
        table = None if own else color_features.detach().float().contiguous()
        field = self.packed_field()
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().nmb_field_color(field, _lib.ptr(table), 0 if own else table.shape[0], _lib.ptr(ds),
                                                  _lib.ptr(idx), _lib.ptr(w), _lib.ptr(nab), _lib.ptr(dirs), M,
                                                  _lib.ptr(rgb), _lib.stream_ptr(dev)))
        return rgb.reshape(*lead, 3)

    def forward_s(self):
        return torch.exp(self.ln_s * self.speed_factor)

    def forward_indicator_weight(self):
        return torch.sigmoid(self.indicator_weight_raw)

    def compute_distance(self, xyz):
        ds, indices, weights = self.mesh_grid.compute_distance(
            xyz.view(-1, 3), indicator_vector=self.indicator_vector,
            indicator_weight=self.forward_indicator_weight() if self.learn_indicator_weight else 0.1)
        lead = xyz.shape[:-1]
        return ds.reshape(*lead, -1), indices.reshape(*lead, -1), weights.reshape(*lead, -1)

    # ---- differentiable torch-op path (training / editing) ---------------------------------------------------
    def _forward_density(self, xyz, d, geometry_features, indices=None, weights=None, need_nablas=False):
        with (torch.enable_grad() if need_nablas else contextlib.nullcontext()):
            d_emb = self.embed_fn_d(d)
            fg_emb = self.embed_fn_fg(interpolation(geometry_features, indices, weights))
            density = self.density_linear(self.pts_linears(torch.cat([d_emb, fg_emb], dim=-1)))
        if not need_nablas:
            return density, torch.zeros_like(density), d_emb
        has_grad = torch.is_grad_enabled()
        nabla = torch.autograd.grad(density, xyz, torch.ones_like(density), create_graph=has_grad,
                                    retain_graph=has_grad, only_inputs=True)[0]
        if not has_grad:
            nabla = nabla.detach()
        return density, nabla, d_emb

    def _forward_color(self, d_emb, view_dirs, color_features, indices=None, weights=None, nabla=None):
        parts = [nabla] if self.enable_nablas_input else []
        parts += [d_emb, self.embed_fn_view(view_dirs),
                  self.embed_fn_ft(interpolation(color_features, indices, weights))]
        return self.color_linear(self.views_linears(torch.cat(parts, dim=-1)))
