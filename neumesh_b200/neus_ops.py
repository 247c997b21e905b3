"""Training path of the NeuS surface and radiance nets as differentiable ops on the library's kernels.

Reference: ``models/base.py:139-311,363-440`` under autograd; ``ImplicitSurface.forward_with_nablas`` takes the nabla with
``autograd.grad(sdf, x, create_graph=True)``, so the eikonal loss and the radiance net (which reads the nabla) need a
double backward through the 8 x 256 softplus MLP.  Here (derivation: DESIGN.md section 4.6):

* ``surface_forward`` runs the value chain and the reverse-mode adjoint of sdf (one adjoint row block per layer instead
  of three forward-mode tangent blocks: the input is 3-D); the nabla is an ordinary output, so ``surface_backward`` is a
  first-order pass: an upward pass over the adjoint chain, then a downward pass over the value chain;
* ``FusedRadianceFn`` is the colour half of the NeuMesh field op (``train_ops.color_forward`` / ``color_backward``).

Both are written against the primitives interface of ``train_ops.CudaPrims`` (the tests inject torch primitives on CPU)
and take effective weights: weight normalisation and the 1/sqrt(2) of the skip layers stay in torch around the ops.
Nothing falls back: on a device the ops need ``CudaPrims`` and CUDA tensors.
"""
from __future__ import annotations

import torch

from . import train_ops
from .train_ops import _bwd_data, _bwd_weight, _linear


def _at(T, off):
    """T from flat element ``off`` on (a column offset inside a row-major matrix; the row stride is passed beside it)."""
    return T.reshape(-1)[off:]


def _h_width(l, K, C, skips):
    """Columns of layer l's input that come from the layer below (the rest, at layer 0 and skip layers, are PE(x))."""
    return K - C if l == 0 or l in skips else K


def surface_forward(P, x, L, skips, layers, out_layer, with_nabla=True, save=True):
    """x [M,3] fp32; ``layers``: [(W [N_l, K_l], b [N_l])] of the softplus layers (a skip layer's input is
    [h_{l-1}, PE(x)], its W already scaled by 1/sqrt(2)); ``out_layer``: (W_o [1+F, N_{D-1}], b_o [1+F]).
    -> (out [M, 1+F] = (sdf, feature), nabla [M,3] or None, saved dict or None)."""
    M, D = x.shape[0], len(layers)
    C = 3 * (1 + 2 * L)
    X = P.empty(M, C)
    P.pe(x, L, X, C)
    Xs, zs = [X], []
    for l, (W, b) in enumerate(layers):
        N = W.shape[0]
        z = P.empty(M, N)
        _linear(P, X, X.shape[1], W, b, z)
        skip = (l + 1) in skips and l + 1 < D
        X = P.empty(M, N + C if skip else N)
        P.softplus(z, X, X.shape[1])
        if skip:
            P.pe(x, L, _at(X, N), N + C)
        zs.append(z)
        if save:
            Xs.append(X)
    Wo, bo = out_layer
    out = P.empty(M, Wo.shape[0])
    _linear(P, X, X.shape[1], Wo, bo, out)
    if not with_nabla:
        return out, None, (dict(x=x, Xs=Xs, zs=zs, gs=None, us=None) if save else None)
    # adjoint: u_l = g_l * sp'(z_l), g_{l-1} = u_l W_l (h part), e-parts of the input adjoints summed into ebar
    N = zs[-1].shape[1]
    u = P.empty(M, N)
    P.gate(None, Wo[0], zs[-1], u)
    us, gs = [None] * D, [None] * D
    ebar, first = P.empty(M, C), True
    for l in reversed(range(D)):
        W = layers[l][0]
        N, K = W.shape
        Nh = _h_width(l, K, C, skips)
        if l == 0 or l in skips:
            P.gemm(u, N, True, _at(W, Nh), K, False, ebar, C, M, C, N, accumulate=not first)
            first = False
        if save:
            us[l] = u
        if l > 0:
            g = P.empty(M, Nh)
            _bwd_data(P, u, W, Nh, g)
            u = P.empty(M, Nh)
            P.gate(g, None, zs[l - 1], u)
            if save:
                gs[l - 1] = g
    nabla = P.empty(M, 3)
    P.pe_jt(x, L, ebar, nabla)
    return out, nabla, (dict(x=x, Xs=Xs, zs=zs, gs=gs, us=us) if save else None)


def surface_backward(P, S, L, skips, layers, out_layer, b_out, b_nabla):
    """Upstream b_out [M, 1+F], b_nabla [M,3] (either may be None) -> ([(dW_l, db_l)], (dW_o, db_o))."""
    x, Xs, zs, gs, us = S["x"], S["Xs"], S["zs"], S["gs"], S["us"]
    M, D = x.shape[0], len(layers)
    C = 3 * (1 + 2 * L)
    Wo, _ = out_layer
    has_n = b_nabla is not None and us is not None
    grads = [(P.empty(*W.shape), P.zeros(W.shape[0])) for W, _ in layers]
    if b_out is None and not has_n:
        return [(dW.zero_(), db) for dW, db in grads], (P.zeros(*Wo.shape), P.zeros(Wo.shape[0]))
    # ---- upward pass over the adjoint chain: b_u_l = b_gin_l W_l^T, dW_l = u_l^T b_gin_l, b_g_l = b_u_l * sp'(z_l)
    bus = [None] * D
    if has_n:
        be = P.empty(M, C)
        P.pe_j(x, L, b_nabla, be)
        bg = None
        for l in range(D):
            W = layers[l][0]
            N, K = W.shape
            Nh = _h_width(l, K, C, skips)
            dW = grads[l][0]
            bu = P.empty(M, N)
            if l > 0:
                P.gemm(bg, Nh, True, W, K, True, bu, N, M, N, Nh)
                P.gemm(us[l], N, False, bg, Nh, False, dW, K, N, Nh, M)
            if l == 0 or l in skips:
                P.gemm(be, C, True, _at(W, Nh), K, True, bu, N, M, N, C, accumulate=l > 0)
                P.gemm(us[l], N, False, be, C, False, _at(dW, Nh), K, N, C, M)
            bg = P.empty(M, N)
            P.gate(bu, None, zs[l], bg)
            bus[l] = bu
    # ---- output layer: out = X_D W_o^T + b_o; the adjoint's seed row w_o = W_o[0] receives colsum(b_g_{D-1})
    N = zs[-1].shape[1]
    if b_out is not None:
        dWo, dbo = P.empty(*Wo.shape), P.zeros(Wo.shape[0])
        bh = P.empty(M, N)
        _bwd_data(P, b_out, Wo, N, bh)
        _bwd_weight(P, b_out, Xs[-1], N, dWo, accumulate=False)
        P.colsum(b_out, dbo)
    else:
        dWo, dbo = P.zeros(*Wo.shape), P.zeros(Wo.shape[0])
        bh = P.zeros(M, N)
    if has_n:
        P.colsum(bg, dWo[0])
    # ---- downward pass over the value chain: b_z_l = b_h_l * sp'(z_l) + b_u_l * g_l * sp''(z_l)
    scratch = P.empty(M * max(z.shape[1] for z in zs)) if has_n else None
    for l in reversed(range(D)):
        W = layers[l][0]
        N, K = W.shape
        bz = P.empty(M, N)
        if has_n:
            g = gs[l]
            if g is None:          # top layer: g_{D-1} is the broadcast row w_o
                g = P.empty(M, N)
                P.gate(None, Wo[0], None, g)
            P.softplus_bwd(zs[l], g, bh, bus[l], bz, scratch[:M * N].view(M, N))
        else:
            P.gate(bh, None, zs[l], bz)
        dW, db = grads[l]
        _bwd_weight(P, bz, Xs[l], K, dW, accumulate=has_n)
        P.colsum(bz, db)
        if l > 0:
            Nh = layers[l - 1][0].shape[0]    # only the h part of a skip layer's input travels on
            bh = P.empty(M, Nh)
            _bwd_data(P, bz, W, Nh, bh)
    return grads, (dWo, dbo)


def _unpack(params):
    params = [p.detach().float().contiguous() for p in params]
    layers = [(params[2 * i], params[2 * i + 1]) for i in range(len(params) // 2 - 1)]
    return layers, (params[-2], params[-1])


def _flat(layers, out_layer):
    return [t for pair in layers for t in pair] + list(out_layer)


class FusedSurfaceFn(torch.autograd.Function):
    """(out [M, 1+F] = (sdf, feature), nabla [M,3]) = surface(x; weights), or ``out`` alone with ``with_nabla=False``.

    ``params``: per softplus layer (W, b) with effective weights, then the output layer (W_o, b_o).  ``x`` receives no
    gradient: callers route an ``x`` that requires one to the torch-op path."""

    @staticmethod
    def forward(ctx, prims, L, skips, with_nabla, x, *params):
        layers, out_layer = _unpack(params)
        if x.shape[0] == 0:     # nothing to launch (the GEMMs refuse the null pointers of empty tensors)
            out, nabla, S = prims.empty(0, out_layer[0].shape[0]), prims.empty(0, 3), "empty"
        else:
            out, nabla, S = surface_forward(prims, x.detach().float().contiguous(), L, skips, layers, out_layer,
                                            with_nabla=with_nabla)
        ctx.prims, ctx.L, ctx.skips, ctx.S, ctx.weights = prims, L, skips, S, (layers, out_layer)
        ctx.set_materialize_grads(False)
        return (out, nabla) if with_nabla else out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, b_out, b_nabla=None):
        if ctx.S is None:
            raise RuntimeError("FusedSurfaceFn: backward called twice (the activations are released after the first pass)")
        prep = lambda g: None if g is None else g.detach().float().contiguous()   # noqa: E731
        layers, out_layer = ctx.weights
        if isinstance(ctx.S, str):
            ctx.S = None
            return (None, None, None, None, None, *(ctx.prims.zeros(*p.shape) for p in _flat(layers, out_layer)))
        grads, (dWo, dbo) = surface_backward(ctx.prims, ctx.S, ctx.L, ctx.skips, layers, out_layer, prep(b_out),
                                             prep(b_nabla))
        ctx.S = None
        flat = [g for pair in grads for g in pair]
        return (None, None, None, None, None, *flat, dWo, dbo)


class FusedRadianceFn(torch.autograd.Function):
    """rgb [M,3] = radiance net(inp [M,K]; weights): ReLU layers of width 256, then a 3-wide sigmoid.

    ``params``: per ReLU layer (W, b), then the output layer (W [3,256], b [3]), effective weights."""

    @staticmethod
    def forward(ctx, prims, inp, *params):
        layers, out_layer = _unpack(params)
        X = inp.detach().float().contiguous()
        if X.shape[0] == 0:
            rgb, cs = prims.empty(0, 3), [X]
        else:
            rgb, cs = train_ops.color_forward(prims, X, X.shape[1], layers, out_layer)
        ctx.prims, ctx.cs, ctx.rgb, ctx.weights = prims, cs, rgb, (layers, out_layer)
        return rgb

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, b_rgb):
        if ctx.cs is None:
            raise RuntimeError("FusedRadianceFn: backward called twice (the activations are released after the first pass)")
        P = ctx.prims
        layers, out_layer = ctx.weights
        X = ctx.cs[0]
        if X.shape[0] == 0:
            ctx.cs = ctx.rgb = None
            return (None, P.empty(*X.shape), *(P.zeros(*p.shape) for p in _flat(layers, out_layer)))
        bX = P.empty(*X.shape)
        grads, (dWo, dbo) = train_ops.color_backward(P, ctx.cs, ctx.rgb, X.shape[1], layers, out_layer,
                                                     b_rgb.detach().float().contiguous(), bX)
        ctx.cs = ctx.rgb = None
        flat = [g for pair in grads for g in pair]
        return (None, bX, *flat, dWo, dbo)
