"""Training path of the NeuMesh field as ONE differentiable op on hand-written CUDA kernels (BASELINE config 4).

Reference: ``models/frameworks/neumesh/neumesh.py:113-138,204-260`` evaluated under autograd by
``models/trainer.py:75-80``; the nabla comes from ``autograd.grad(sdf, xyz, create_graph=True)`` and the eikonal /
colour losses back-propagate through it (a double backward through the geometry MLP).  Here:

* ``field_forward`` / ``field_backward`` sequence the ``nmb_tr_*`` kernels (``csrc/train.cu``): gather + blend +
  encodings, value AND forward-mode tangent rows through the softplus MLP (the tangent chain makes the nabla an ordinary
  output, so its backward is a first-order reverse pass - derivation and float64 check: ``tools/train_math_proto.py``),
  colour MLP, and the reverse pass with split-K weight-gradient GEMMs and atomic scatter-adds into the vertex tables
  (under ``torch.use_deterministic_algorithms(True)``: a sorted, segmented scatter and fixed reduction orders, so that
  the gradients are bit-reproducible);
* ``FusedFieldFn`` wraps them in a ``torch.autograd.Function``; weight normalisation (``g * v / |v|``) stays in torch
  ops around it (a [256, K] element-wise op per layer), so ``weight_g`` / ``weight_v`` receive their gradients through
  the ordinary graph.

The two functions are written against a small "primitives" interface: ``CudaPrims`` binds the C ABI; the tests inject a
torch implementation of the same interface on CPU to check the SEQUENCING against autograd without a GPU (the kernels
themselves are checked one by one on the GPU).  The product never falls back: ``FusedFieldFn`` requires CUDA tensors.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib

HIDDEN = 256


class TrInputs(C.Structure):
    _fields_ = [
        ("xyz", C.c_void_p), ("dirs", C.c_void_p), ("idx", C.c_void_p), ("w", C.c_void_p), ("vertices", C.c_void_p),
        ("indicator_vector", C.c_void_p), ("geometry_features", C.c_void_p), ("color_features", C.c_void_p),
        ("indicator_weight", C.c_float), ("geometry_dim", C.c_int32), ("color_dim", C.c_int32),
        ("multires_d", C.c_int32), ("multires_fg", C.c_int32), ("multires_ft", C.c_int32), ("multires_view", C.c_int32),
        ("enable_nablas_input", C.c_int32), ("M", C.c_int64), ("ds", C.c_void_p), ("G", C.c_void_p), ("Xg", C.c_void_p),
        ("ldg", C.c_int64), ("T0", C.c_void_p), ("ldt", C.c_int64), ("Xc", C.c_void_p), ("ldc", C.c_int64),
    ]


class FieldSpec:
    """Static description of the field (embedding widths, layer counts)."""

    def __init__(self, geometry_dim, color_dim, multires_d, multires_fg, multires_ft, multires_view, enable_nablas_input,
                 D_density, D_color):
        self.Fg, self.Fc = int(geometry_dim), int(color_dim)
        self.Ld, self.Lfg, self.Lft, self.Lv = int(multires_d), int(multires_fg), int(multires_ft), int(multires_view)
        self.use_nabla = bool(enable_nablas_input)
        self.NLg, self.NLc = int(D_density), int(D_color)
        self.chd = 1 + 2 * self.Ld
        self.chv = 3 * (1 + 2 * self.Lv)
        self.Kg = self.chd + (1 + 2 * self.Lfg) * self.Fg
        self.offd = 3 if self.use_nabla else 0
        self.Kc = self.offd + self.chd + self.chv + (1 + 2 * self.Lft) * self.Fc


class CudaPrims:
    """The ``nmb_tr_*`` kernels on the current CUDA stream of the tensors' device.  The calls that reduce across threads
    first set the library's deterministic mode from ``torch.are_deterministic_algorithms_enabled()``."""

    def __init__(self, device):
        self.dev = torch.device(device)
        self.L = _lib.lib()

    def _s(self):
        return _lib.stream_ptr(self.dev)

    def empty(self, *shape, dtype=torch.float32):
        return torch.empty(*shape, dtype=dtype, device=self.dev)

    def zeros(self, *shape):
        return torch.zeros(*shape, dtype=torch.float32, device=self.dev)

    def gemm(self, A, lda, a_kc, B, ldb, b_kc, Cm, ldc, M, N, K, bias=None, epilogue=0, mask=None, ldmask=0,
             accumulate=False):
        _lib.sync_deterministic()
        with torch.cuda.device(self.dev):
            _lib.check(self.L.nmb_tr_gemm(_lib.ptr(A), lda, int(a_kc), _lib.ptr(B), ldb, int(b_kc), _lib.ptr(Cm), ldc,
                                          M, N, K, _lib.ptr(bias), epilogue, _lib.ptr(mask), ldmask, int(accumulate),
                                          self._s()))

    def _inputs(self, spec, t):
        s = TrInputs()
        for k in ("xyz", "dirs", "idx", "w", "vertices", "indicator_vector", "geometry_features", "color_features", "ds",
                  "G", "Xg", "T0", "Xc"):
            setattr(s, k, t[k].data_ptr())
        s.indicator_weight = float(t["w1"])
        s.geometry_dim, s.color_dim = spec.Fg, spec.Fc
        s.multires_d, s.multires_fg, s.multires_ft, s.multires_view = spec.Ld, spec.Lfg, spec.Lft, spec.Lv
        s.enable_nablas_input = int(spec.use_nabla)
        s.M = t["xyz"].shape[0]
        s.ldg, s.ldt, s.ldc = t["Xg"].shape[1], t["T0"].shape[1], t["Xc"].shape[1]
        return s

    def prep(self, spec, t):
        with torch.cuda.device(self.dev):
            _lib.check(self.L.nmb_tr_prep(C.byref(self._inputs(spec, t)), self._s()))

    def softplus_fwd(self, z, a, h, t):
        with torch.cuda.device(self.dev):
            _lib.check(self.L.nmb_tr_softplus_fwd(_lib.ptr(z), _lib.ptr(a), _lib.ptr(h), _lib.ptr(t), z.numel(), self._s()))

    def softplus_bwd(self, z, a, bh, bt, bz, ba):
        with torch.cuda.device(self.dev):
            _lib.check(self.L.nmb_tr_softplus_bwd(_lib.ptr(z), _lib.ptr(a), _lib.ptr(bh), _lib.ptr(bt), _lib.ptr(bz),
                                                  _lib.ptr(ba), z.numel(), self._s()))

    def geo_out_fwd(self, h, t, w_out, b_out, G, sdf, g, nabla, Xc):
        with torch.cuda.device(self.dev):
            _lib.check(self.L.nmb_tr_geo_out_fwd(_lib.ptr(h), _lib.ptr(t), _lib.ptr(w_out), _lib.ptr(b_out), _lib.ptr(G),
                                                 h.shape[0], h.shape[1], _lib.ptr(sdf), _lib.ptr(g), _lib.ptr(nabla),
                                                 _lib.ptr(Xc), Xc.shape[1] if Xc is not None else 0, self._s()))

    def color_out_fwd(self, c, w_out, b_out, rgb):
        with torch.cuda.device(self.dev):
            _lib.check(self.L.nmb_tr_color_out_fwd(_lib.ptr(c), _lib.ptr(w_out), _lib.ptr(b_out), c.shape[0], c.shape[1],
                                                   _lib.ptr(rgb), self._s()))

    def color_out_bwd(self, b_rgb, rgb, c, w_out, bz, dw_out, db_out):
        _lib.sync_deterministic()
        with torch.cuda.device(self.dev):
            _lib.check(self.L.nmb_tr_color_out_bwd(_lib.ptr(b_rgb), _lib.ptr(rgb), _lib.ptr(c), _lib.ptr(w_out),
                                                   c.shape[0], c.shape[1], _lib.ptr(bz), _lib.ptr(dw_out),
                                                   _lib.ptr(db_out), self._s()))

    def colsum(self, X, out):
        _lib.sync_deterministic()
        with torch.cuda.device(self.dev):
            _lib.check(self.L.nmb_tr_colsum(_lib.ptr(X), X.shape[1], X.shape[0], X.shape[1], _lib.ptr(out), self._s()))

    def geo_out_bwd(self, b_sdf, b_nabla, bXc, G, g, h, t, w_out, bh, bt, b_G, dw_out, db_out):
        _lib.sync_deterministic()
        with torch.cuda.device(self.dev):
            _lib.check(self.L.nmb_tr_geo_out_bwd(_lib.ptr(b_sdf), _lib.ptr(b_nabla), _lib.ptr(bXc),
                                                 bXc.shape[1] if bXc is not None else 0, _lib.ptr(G), _lib.ptr(g),
                                                 _lib.ptr(h), _lib.ptr(t), _lib.ptr(w_out), h.shape[0], h.shape[1],
                                                 _lib.ptr(bh), _lib.ptr(bt), _lib.ptr(b_G), _lib.ptr(dw_out),
                                                 _lib.ptr(db_out), self._s()))

    def input_bwd(self, spec, t, bXg, bT0, bXc, b_G, d_fg, d_fc, d_ind, d_w1):
        _lib.sync_deterministic()
        with torch.cuda.device(self.dev):
            _lib.check(self.L.nmb_tr_input_bwd(C.byref(self._inputs(spec, t)), _lib.ptr(bXg), bXg.shape[1], _lib.ptr(bT0),
                                               bT0.shape[1], _lib.ptr(bXc), bXc.shape[1], _lib.ptr(b_G), _lib.ptr(d_fg),
                                               _lib.ptr(d_fc), _lib.ptr(d_ind), _lib.ptr(d_w1), self._s()))


# ------------------------------------------------------------------------------------------------------------------
# sequencing (shared by the CUDA primitives and the tests' torch primitives)
# ------------------------------------------------------------------------------------------------------------------
def _linear(P, X, K, W, b, out, relu=False):
    """out[M,256] = X[:, :K] . W[:, :K]^T (+ b) (torch.nn.Linear: weight [out, in])."""
    M = X.shape[0]
    P.gemm(X, X.shape[1], True, W, W.shape[1], True, out, out.shape[1], M, W.shape[0], K, bias=b,
           epilogue=1 if relu else 0)


def _bwd_data(P, dZ, W, K, out, mask=None):
    """out[M, :K] = dZ . W[:, :K] (optionally zeroed where mask <= 0)."""
    M = dZ.shape[0]
    P.gemm(dZ, dZ.shape[1], True, W, W.shape[1], False, out, out.shape[1], M, K, W.shape[0],
           epilogue=2 if mask is not None else 0, mask=mask, ldmask=mask.shape[1] if mask is not None else 0)


def _bwd_weight(P, dZ, X, K, dW, accumulate):
    """dW[:, :K] (+)= dZ^T . X[:, :K]."""
    M = dZ.shape[0]
    P.gemm(dZ, dZ.shape[1], False, X, X.shape[1], False, dW, dW.shape[1], dZ.shape[1], K, M, accumulate=accumulate)


def field_forward(P, spec: FieldSpec, t: dict, geo, geo_out, col, col_out, with_color=True):
    """t: xyz, dirs, idx, w, vertices, indicator_vector, geometry_features, color_features (tensors), w1 (float).
    geo / col: lists of (W [256, K], b [256]); geo_out: (w [1,256], b [1]); col_out: (W [3,256], b [3]).
    -> (sdf [M], nabla [M,3], rgb [M,3], saved dict)."""
    M = t["xyz"].shape[0]
    S = dict(t)
    S["ds"], S["G"] = P.empty(M), P.empty(M, 3)
    S["Xg"], S["T0"], S["Xc"] = P.empty(M, spec.Kg), P.empty(M, spec.chd), P.empty(M, spec.Kc)
    P.prep(spec, S)
    hs, ts, zs, as_ = [S["Xg"]], [S["T0"]], [], []
    for l, (W, b) in enumerate(geo):
        K = spec.Kg if l == 0 else HIDDEN
        Kt = spec.chd if l == 0 else HIDDEN       # the tangent seed is non-zero in the PE(ds) columns only
        z, a = P.empty(M, HIDDEN), P.empty(M, HIDDEN)
        _linear(P, hs[-1], K, W, b, z)
        _linear(P, ts[-1], Kt, W, None, a)
        h, tt = P.empty(M, HIDDEN), P.empty(M, HIDDEN)
        P.softplus_fwd(z, a, h, tt)
        zs.append(z); as_.append(a); hs.append(h); ts.append(tt)
    sdf, g, nabla = P.empty(M), P.empty(M), P.empty(M, 3)
    P.geo_out_fwd(hs[-1], ts[-1], geo_out[0], geo_out[1], S["G"], sdf, g, nabla, S["Xc"] if spec.use_nabla else None)
    cs, rgb = [S["Xc"]], None
    if with_color:
        for l, (W, b) in enumerate(col):
            K = spec.Kc if l == 0 else HIDDEN
            c = P.empty(M, HIDDEN)
            _linear(P, cs[-1], K, W, b, c, relu=True)
            cs.append(c)
        rgb = P.empty(M, 3)
        P.color_out_fwd(cs[-1], col_out[0], col_out[1], rgb)
    S.update(hs=hs, ts=ts, zs=zs, as_=as_, cs=cs, g=g, rgb=rgb)
    return sdf, nabla, rgb, S


def field_backward(P, spec: FieldSpec, S: dict, geo, geo_out, col, col_out, b_sdf, b_nabla, b_rgb, want_w1=True):
    """Upstream gradients (any may be None) -> dict: geometry_features, color_features, indicator_vector, w1,
    geo [(dW, db)], geo_out (dw, db), col [(dW, db)], col_out (dW, db)."""
    M = S["xyz"].shape[0]
    out = {}
    # ---- colour MLP ----
    dWo, dbo = P.zeros(3, HIDDEN), P.zeros(3)
    col_grads = [None] * len(col)
    bXc = P.zeros(M, spec.Kc)
    if b_rgb is not None and S["rgb"] is not None:
        bz = P.empty(M, HIDDEN)
        P.color_out_bwd(b_rgb, S["rgb"], S["cs"][-1], col_out[0], bz, dWo, dbo)
        for l in reversed(range(len(col))):
            W, _ = col[l]
            K = spec.Kc if l == 0 else HIDDEN
            dW, db = P.empty(HIDDEN, W.shape[1]), P.zeros(HIDDEN)
            _bwd_weight(P, bz, S["cs"][l], K, dW, accumulate=False)
            P.colsum(bz, db)
            col_grads[l] = (dW, db)
            if l > 0:
                nxt = P.empty(M, HIDDEN)
                _bwd_data(P, bz, W, HIDDEN, nxt, mask=S["cs"][l])   # ReLU of the layer below
                bz = nxt
            else:
                _bwd_data(P, bz, W, spec.Kc, bXc)
    else:
        for l, (W, _) in enumerate(col):
            col_grads[l] = (P.zeros(HIDDEN, W.shape[1]), P.zeros(HIDDEN))
    out["col"], out["col_out"] = col_grads, (dWo, dbo)
    # ---- geometry MLP: value and tangent chains ----
    bh, bt, b_G = P.empty(M, HIDDEN), P.empty(M, HIDDEN), P.empty(M, 3)
    dwo, dbo_g = P.zeros(1, HIDDEN), P.zeros(1)
    P.geo_out_bwd(b_sdf, b_nabla, bXc if (spec.use_nabla and b_rgb is not None and S["rgb"] is not None) else None,
                  S["G"], S["g"], S["hs"][-1],
                  S["ts"][-1], geo_out[0], bh, bt, b_G, dwo, dbo_g)
    geo_grads = [None] * len(geo)
    for l in reversed(range(len(geo))):
        W, _ = geo[l]
        K = spec.Kg if l == 0 else HIDDEN
        Kt = spec.chd if l == 0 else HIDDEN
        bz, ba = P.empty(M, HIDDEN), P.empty(M, HIDDEN)
        P.softplus_bwd(S["zs"][l], S["as_"][l], bh, bt, bz, ba)
        dW, db = P.empty(HIDDEN, W.shape[1]), P.zeros(HIDDEN)
        _bwd_weight(P, bz, S["hs"][l], K, dW, accumulate=False)
        _bwd_weight(P, ba, S["ts"][l], Kt, dW, accumulate=True)
        P.colsum(bz, db)
        geo_grads[l] = (dW, db)
        bh, bt = P.empty(M, K), P.empty(M, Kt)
        _bwd_data(P, bz, W, K, bh)
        _bwd_data(P, ba, W, Kt, bt)
    out["geo"], out["geo_out"] = geo_grads, (dwo, dbo_g)
    # ---- encodings, vertex tables, mesh distance ----
    V = S["geometry_features"].shape[0]
    d_fg, d_fc, d_ind = P.zeros(V, spec.Fg), P.zeros(V, spec.Fc), P.zeros(V, 3)
    d_w1 = P.zeros(1)
    P.input_bwd(spec, S, bh, bt, bXc, b_G, d_fg, d_fc, d_ind, d_w1 if want_w1 else None)
    out.update(geometry_features=d_fg, color_features=d_fc, indicator_vector=d_ind, w1=d_w1)
    return out


class FusedFieldFn(torch.autograd.Function):
    """(sdf [M,1], nabla [M,3], rgb [M,3]) = field(xyz, dirs | neighbours, tables, weights), CUDA forward and backward.

    ``params``: indicator_vector, w1 (0-dim tensor), geometry_features, color_features, then per geometry layer (W, b),
    the geometry output (w [1,256], b [1]), per colour layer (W, b), the colour output (W [3,256], b [3])."""

    @staticmethod
    def forward(ctx, spec, prims, with_color, xyz, dirs, idx, w, vertices, *params):
        params = [p.detach().float().contiguous() for p in params]
        ind, w1, fg, fc = params[:4]
        rest = params[4:]
        geo = [(rest[2 * i], rest[2 * i + 1]) for i in range(spec.NLg)]
        rest = rest[2 * spec.NLg:]
        geo_out, rest = (rest[0], rest[1]), rest[2:]
        col = [(rest[2 * i], rest[2 * i + 1]) for i in range(spec.NLc)]
        col_out = (rest[2 * spec.NLc], rest[2 * spec.NLc + 1])
        t = dict(xyz=xyz.detach().float().contiguous(), dirs=dirs.detach().float().contiguous(),
                 idx=idx.detach().to(torch.int64).contiguous(), w=w.detach().float().contiguous(),
                 vertices=vertices.detach().float().contiguous(), indicator_vector=ind, geometry_features=fg,
                 color_features=fc, w1=float(w1))
        sdf, nabla, rgb, S = field_forward(prims, spec, t, geo, geo_out, col, col_out, with_color=with_color)
        ctx.spec, ctx.prims, ctx.S = spec, prims, S
        ctx.weights = (geo, geo_out, col, col_out)
        if rgb is None:
            rgb = nabla.new_zeros(nabla.shape[0], 3)
            ctx.mark_non_differentiable(rgb)
        return sdf.unsqueeze(-1), nabla, rgb

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, b_sdf, b_nabla, b_rgb):
        geo, geo_out, col, col_out = ctx.weights
        if ctx.S is None:
            raise RuntimeError("FusedFieldFn: backward called twice (the activations are released after the first pass)")
        prep = lambda g: None if g is None else g.detach().float().contiguous()   # noqa: E731
        b_sdf = None if b_sdf is None else b_sdf.detach().float().reshape(-1).contiguous()
        G = field_backward(ctx.prims, ctx.spec, ctx.S, geo, geo_out, col, col_out, b_sdf, prep(b_nabla), prep(b_rgb),
                           want_w1=True)
        ctx.S = None   # release the activations
        grads = [G["indicator_vector"], G["w1"].reshape(()), G["geometry_features"], G["color_features"]]
        for dW, db in G["geo"]:
            grads += [dW, db]
        grads += [G["geo_out"][0], G["geo_out"][1]]
        for dW, db in G["col"]:
            grads += [dW, db]
        grads += [G["col_out"][0], G["col_out"][1]]
        return (None, None, None, None, None, None, None, None, *grads)
