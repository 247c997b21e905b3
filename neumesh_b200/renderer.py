"""``volume_render`` / ``SingleRenderer`` - drop-ins for ``models/renderer.py``.

``volume_render(rays_o, rays_d, model, **kwargs) -> (rgb, depth, extras)`` keeps the reference's keyword set
(``renderer.py:105-135``; unknown kwargs are ignored as there).  A ``neumesh_b200.NeuMesh`` on CUDA with grad mode off
is rendered by ``nmb_render`` (``csrc/render.cu``), a texture-edit model (``TextureEditableNeuMesh`` or any object with
its attributes) over such models by ``nmb_render_edit``; every other case - arbitrary models such as the NeuS teacher,
grad-enabled training steps, ``perturb=True``, batched inputs with B > 1 - runs the generic torch-op path below, which
follows the same algorithm through the model's public protocol.
"""
from __future__ import annotations

import ctypes as C
from collections import OrderedDict
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from .neumesh import NeuMesh
from .texture_neumesh import edit_fused_supported, is_edit_model, packed_edit

_WORKSPACES: "dict[tuple, torch.Tensor]" = {}
DEFAULT_FUSED_CHUNK = 1 << 20  # rays per kernel chunk on the fused path (scratch ~19 KB / ray: 12 GB for an 800x800 frame)


def _workspace(device, nbytes):
    # one scratch per (device, stream): renders issued on different streams of one device never share scratch
    key = (device.type, device.index, torch.cuda.current_stream(device).cuda_stream)
    ws = _WORKSPACES.get(key)
    if ws is None or ws.numel() < nbytes:
        _WORKSPACES.pop(key, None)
        ws = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
        _WORKSPACES[key] = ws
    return ws


def release_workspace(device: Optional[torch.device] = None) -> None:
    """Drop the cached ``nmb_render`` scratch of ``device`` (all devices when None).  The fused path keeps one scratch
    tensor per device and stream sized for the largest chunk rendered so far (~21 GB at the default 2^20-ray chunk)."""
    if device is None:
        _WORKSPACES.clear()
    else:
        device = torch.device(device)
        for key in [k for k in _WORKSPACES if k[:2] == (device.type, device.index)]:
            _WORKSPACES.pop(key, None)


def _cascade_eligible(geo, rays_o, *, batched, use_view_dirs, N_samples, N_importance, N_upsample_iters) -> bool:
    """Whether the fused sampling cascade can serve the geometry model ``geo`` with these arguments: every fused route
    of ``volume_render`` needs this."""
    return (isinstance(geo, NeuMesh) and rays_o.is_cuda and geo.geometry_features.is_cuda and geo.fused_supported()
            and use_view_dirs and (not batched or rays_o.shape[0] == 1) and N_samples >= 2 and N_upsample_iters >= 0
            and (N_upsample_iters == 0 or N_importance % N_upsample_iters == 0))


def fused_eligible(model, rays_o, *, batched, random_color_direction, use_view_dirs, N_samples, N_importance,
                   N_upsample_iters) -> bool:
    """Whether ``nmb_render`` renders the whole call: grad mode off, and a ``NeuMesh`` or a texture edit it can render."""
    if torch.is_grad_enabled() or random_color_direction:
        return False
    if isinstance(model, NeuMesh):
        geo = model
    elif is_edit_model(model) and getattr(model, "fused_render", True) and edit_fused_supported(model):
        geo = model.main_model
    else:
        return False
    return _cascade_eligible(geo, rays_o, batched=batched, use_view_dirs=use_view_dirs, N_samples=N_samples,
                             N_importance=N_importance, N_upsample_iters=N_upsample_iters)


def fused_cascade_model(model, rays_o, *, z_samples, random_color_direction, **cascade_kwargs):
    """For a call ``nmb_render`` does not render whole: the geometry model whose fused sampling cascade supplies the
    generic path's sample depths, or None.  Without grad that is the main model of a texture edit (the edit's colour
    blend then runs per chunk on the generic path); in grad mode a ``NeuMesh`` itself (a training step: the
    differentiable evaluation at the final samples follows on the generic path)."""
    if z_samples is not None:
        return None
    if torch.is_grad_enabled():
        geo = model if isinstance(model, NeuMesh) else None
    elif random_color_direction:
        return None
    else:
        geo = getattr(model, "main_model", None)
    return geo if _cascade_eligible(geo, rays_o, **cascade_kwargs) else None


# Outputs of render_fused that nmb_render writes: its rgb, depth, acc and normals arguments, then the fields of
# nmb_render_detail in order ("density" is detail->sdf_mid: [N, P-1] and [N, P-1, 1] share one layout).
_DETAIL_OUTPUTS = ("d_all", "implicit_surface", "implicit_nablas", "radiance", "density", "near_far")
_KERNEL_OUTPUTS = ("rgb", "depth_volume", "mask_volume", "normals_volume") + _DETAIL_OUTPUTS


def _fused_output_shapes(P, *, calc_normal, detailed_output, samples_output, sampling_only):
    """Every output of ``render_fused`` with its per-ray shape, in the order returned (P samples per ray)."""
    if sampling_only:
        return OrderedDict(d_all=(P,), implicit_surface=(P,), near_far=(2,))
    out = OrderedDict(rgb=(3,), depth_volume=(), mask_volume=())
    if calc_normal:
        out["normals_volume"] = (3,)
    if detailed_output:
        if calc_normal:
            out["implicit_nablas"] = (P, 3)
        out.update(implicit_surface=(P,), radiance=(P - 1, 3), alpha=(P - 1,), cdf=(P,), visibility_weights=(P - 1,),
                   d_final=(P - 1,), d_all=(P,), near_far=(2,))
        if samples_output:
            out.update(xyz=(P - 1, 3), dirs=(P - 1, 3), density=(P - 1, 1), colors=(P - 1, 3))
    return out


def render_fused(rays_o, rays_d, model, *, obj_bounding_radius=1.0, calc_normal=False, white_bkgd=False,
                 near_bypass=None, far_bypass=None, N_samples=64, N_importance=64, N_upsample_iters=4,
                 bounded_near_far=True, detailed_output=False, samples_output=False, chunk=None,
                 normalize_dirs=True, skip_dead_samples=True, min_chunk=None, perturb=False, perturb_u=None,
                 sampling_only=False):
    """Flat [N,3] rays -> dict of flat outputs, through ``nmb_render``.

    ``perturb=True`` draws the up-sampling uniforms with ``torch.rand`` (``rend_util.py:292-295``); ``perturb_u``
    [N_upsample_iters, N, N_importance / N_upsample_iters] injects them instead (parity runs).  ``sampling_only=True``
    runs the no-grad sampling cascade only and returns ``{"d_all", "implicit_surface", "near_far"}``.

    ``model`` is a ``NeuMesh`` or a texture-edit model (``texture_neumesh.packed_edit``): its main model drives the
    cascade and ``nmb_render_edit`` blends the reference models' colours into every evaluated mid-point."""
    dev = rays_o.device
    o = rays_o.detach().reshape(-1, 3).float().contiguous()
    d = rays_d.detach().reshape(-1, 3).float().contiguous()
    N = o.shape[0]
    P = N_samples + (N_importance if N_upsample_iters > 0 else 0)
    shapes = _fused_output_shapes(P, calc_normal=calc_normal, detailed_output=detailed_output,
                                  samples_output=samples_output, sampling_only=sampling_only)
    if N == 0:
        # an empty shard (multi-GPU renders of fewer than 128 * world rays leave some ranks without rays): same keys,
        # empty tensors, no library call (empty tensors have null data pointers)
        return OrderedDict((k, o.new_zeros(0, *s)) for k, s in shapes.items())
    u_dev = None
    if (perturb or perturb_u is not None) and N_upsample_iters > 0:
        n_new = N_importance // N_upsample_iters
        u = perturb_u if perturb_u is not None else torch.rand(N_upsample_iters, N, n_new, device=dev)
        u = u.to(dev).float().reshape(N_upsample_iters, N, n_new)
        # the new samples are merged into the sorted ones, so only the SET of draws matters: each ray's ascending
        u_dev = torch.sort(u, dim=-1)[0].permute(0, 2, 1).contiguous()      # [iters, n_new, N]
    cfg = _lib.RenderCfg(float(obj_bounding_radius), int(N_samples), int(N_importance), int(N_upsample_iters),
                         int(bool(bounded_near_far)), int(bool(calc_normal)), int(bool(white_bkgd)),
                         int(near_bypass is not None), float(near_bypass or 0.0), int(far_bypass is not None),
                         float(far_bypass or 0.0), int(bool(normalize_dirs)),
                         int(bool(skip_dead_samples) and not detailed_output), int(bool(sampling_only)),
                         u_dev.data_ptr() if u_dev is not None else None)
    edit = None
    if isinstance(model, NeuMesh):
        geo = model
    else:
        if sampling_only:
            raise ValueError("sampling_only renders the geometry only: pass the edit's main_model")
        geo = model.main_model
        edit = packed_edit(model)
    field = geo.packed_field()
    L = _lib.lib()
    chunk = int(min(chunk or DEFAULT_FUSED_CHUNK, max(N, 1)))
    if min_chunk is not None:
        # the caller's ``rayschunk`` exists to bound memory (render.py passes 4096): never let the scratch of a chunk
        # take more than half of the device memory that is free right now, but never go below the caller's own chunk
        per_ray = L.nmb_render_edit_workspace_bytes(C.byref(cfg), edit, 1 << 16) / float(1 << 16)
        cached = _WORKSPACES.get((dev.type, dev.index, torch.cuda.current_stream(dev).cuda_stream))
        free = torch.cuda.mem_get_info(dev)[0] + (cached.numel() if cached is not None else 0)
        chunk = int(min(chunk, max(int(min_chunk), int(0.5 * free / per_ray))))
    nbytes = L.nmb_render_edit_workspace_bytes(C.byref(cfg), edit, chunk)
    ws = _workspace(dev, nbytes)
    # the outputs the kernels write; the rest are recomputed from them below
    buf = {k: o.new_empty(N, *s) for k, s in shapes.items() if k in _KERNEL_OUTPUTS}
    det = None
    if any(k in buf for k in _DETAIL_OUTPUTS):
        det = _lib.RenderDetail(*[buf[k].data_ptr() if k in buf else None for k in _DETAIL_OUTPUTS])
    args = (C.byref(cfg), _lib.ptr(o), _lib.ptr(d), N, chunk, *[_lib.ptr(buf.get(k)) for k in _KERNEL_OUTPUTS[:4]],
            C.byref(det) if det is not None else None, _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev))
    with torch.cuda.device(dev):
        _lib.check(L.nmb_render(field, *args) if edit is None else L.nmb_render_edit(field, edit, *args))
    if detailed_output and not sampling_only:
        # same quantities the reference returns (renderer.py:335-348), recomputed from the exported samples
        z = buf["d_all"]
        buf["cdf"], buf["alpha"], buf["visibility_weights"] = sdf_to_w(buf["implicit_surface"], geo.forward_s().detach())
        buf["d_final"] = 0.5 * (z[..., 1:] + z[..., :-1])
        if samples_output:
            dn = F.normalize(d, dim=-1) if normalize_dirs else d
            buf["xyz"] = o[:, None, :] + dn[:, None, :] * buf["d_final"][..., None]
            buf["dirs"] = dn[:, None, :].expand_as(buf["xyz"])
            buf["colors"] = buf["radiance"]
    return OrderedDict((k, buf[k]) for k in shapes)


# --------------------------------------------------------------------------------------------------------------
# generic torch-op path (any model with the 4-method protocol; differentiable)
# --------------------------------------------------------------------------------------------------------------
def cdf_Phi_s(x, s):
    return torch.sigmoid(x * s)


def sdf_to_alpha(sdf, s):
    cdf = cdf_Phi_s(sdf, s)
    alpha = ((cdf[..., :-1] - cdf[..., 1:]) / (cdf[..., :-1] + 1e-10)).clamp_min(0)
    return cdf, alpha


def alpha_to_w(alpha):
    ones = torch.ones_like(alpha[..., :1])
    return alpha * torch.cumprod(torch.cat([ones, 1.0 - alpha + 1e-10], dim=-1), dim=-1)[..., :-1]


def sdf_to_w(sdf, s):
    cdf, alpha = sdf_to_alpha(sdf, s)
    return cdf, alpha, alpha_to_w(alpha)


def near_far_from_sphere(rays_o, rays_d, r=1.0, keepdim=True):
    mid = -(rays_o * rays_d).sum(dim=-1, keepdim=keepdim)
    return (mid - r).clamp_min(0.0), (mid + r).clamp_min(r)


def sample_pdf(bins, weights, N_importance, det=False, eps=1e-5, u=None):
    weights = weights + 1e-5
    pdf = weights / weights.sum(dim=-1, keepdim=True)
    cdf = torch.cumsum(pdf, dim=-1)
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], dim=-1)
    shape = list(cdf.shape[:-1]) + [N_importance]
    if u is not None:
        u = u.expand(shape)     # caller-provided uniforms (parity runs of perturb=True)
    elif det:
        u = torch.linspace(0.0, 1.0, steps=N_importance, device=cdf.device).expand(shape)
    else:
        u = torch.rand(shape, device=cdf.device)
    u = u.contiguous()
    inds = torch.searchsorted(cdf.detach(), u, right=False)
    below, above = (inds - 1).clamp_min(0), inds.clamp_max(cdf.shape[-1] - 1)
    c0, c1 = torch.gather(cdf, -1, below), torch.gather(cdf, -1, above)
    b0, b1 = torch.gather(bins, -1, below), torch.gather(bins, -1, above)
    denom = c1 - c0
    denom = torch.where(denom < eps, torch.ones_like(denom), denom)
    return b0 + (u - c0) / denom * (b1 - b0)


def batchify_query(query_fn, *args, chunk, dim_batchify):
    """[(B), N_rays, N_pts, ...] inputs -> flatten rays x pts, call in chunks, restore (utils/train_util.py:25-82)."""
    n_rays, n_pts = args[0].shape[dim_batchify], args[0].shape[dim_batchify + 1]
    flat = [a.flatten(dim_batchify, dim_batchify + 1) for a in args]
    total = flat[0].shape[dim_batchify]
    pieces = []
    for s in range(0, total, chunk):
        r = query_fn(*[a.narrow(dim_batchify, s, min(chunk, total - s)) for a in flat])
        pieces.append(r if isinstance(r, tuple) else (r,))

    def restore(v):
        return v.reshape(*v.shape[:dim_batchify], n_rays, n_pts, *v.shape[dim_batchify + 1:])

    outs = []
    for group in zip(*pieces):
        if isinstance(group[0], dict):
            outs.append({k: restore(torch.cat([g[k] for g in group], dim=dim_batchify)) for k in group[0]})
        else:
            outs.append(restore(torch.cat(group, dim=dim_batchify)))
    return outs[0] if len(outs) == 1 else tuple(outs)


def compute_bounded_near_far(model, rays_o, rays_d, near, far, sample_grid=256, distance_thresh=0.1):
    t = torch.linspace(0, 1, sample_grid, device=rays_o.device)
    depth = (near * (1 - t) + far * t).unsqueeze(-1)
    ds, _, _ = model.compute_distance(rays_o.unsqueeze(-2) + depth * rays_d.unsqueeze(-2))
    inside = ds < distance_thresh
    lo = torch.where(inside, depth, torch.full_like(depth, 1e10)).min(dim=-2)[0]
    hi = torch.where(inside, depth, torch.full_like(depth, -1e10)).max(dim=-2)[0]
    lo = torch.where(lo > 1e5, near, lo)
    hi = torch.where(hi < -1e5, far, hi)
    thin = (hi - lo) < 0.1
    return torch.where(thin, lo - 0.05, lo), torch.where(thin, hi + 0.05, hi)


def _sample_cascade(rays_o, rays_d, model, query, *, obj_bounding_radius, near_bypass, far_bypass, perturb, N_samples,
                    N_importance, N_upsample_iters, bounded_near_far, perturb_u=None):
    """Torch-op sampling cascade (renderer.py:156-259) through the model protocol -> sorted depths z [..., P]."""
    dev = rays_o.device
    near, far = near_far_from_sphere(rays_o, rays_d, r=obj_bounding_radius)
    if bounded_near_far:
        near, far = compute_bounded_near_far(model, rays_o, rays_d, near, far)
    if near_bypass is not None:
        near = torch.full_like(near, near_bypass)
    if far_bypass is not None:
        far = torch.full_like(far, far_bypass)
    pts_at = lambda z: rays_o.unsqueeze(-2) + z.unsqueeze(-1) * rays_d.unsqueeze(-2)  # noqa: E731
    t = torch.linspace(0, 1, N_samples, device=dev)
    with torch.no_grad():
        z = near * (1 - t) + far * t
        sdf = query(model.forward_density_only, pts_at(z)).squeeze(-1)
        for it in range(N_upsample_iters):
            s0, s1, z0, z1 = sdf[..., :-1], sdf[..., 1:], z[..., :-1], z[..., 1:]
            mid = (s0 + s1) * 0.5
            raw = (s1 - s0) / (z1 - z0 + 1e-5)
            slope = torch.minimum(torch.cat([torch.zeros_like(raw[..., :1]), raw[..., :-1]], dim=-1), raw)
            slope = slope.clamp(-10.0, 0.0)
            dist = z1 - z0
            inv_s = 256 * (2 ** it)
            c0 = cdf_Phi_s(mid - slope * dist * 0.5, inv_s)
            c1 = cdf_Phi_s(mid + slope * dist * 0.5, inv_s)
            alpha = (c0 - c1 + 1e-5) / (c0 + 1e-5)
            z_new = sample_pdf(z, alpha_to_w(alpha), N_importance // N_upsample_iters, det=not perturb,
                               u=None if perturb_u is None else perturb_u[it])
            sdf_new = query(model.forward_density_only, pts_at(z_new)).squeeze(-1)
            z, order = torch.sort(torch.cat([z, z_new], dim=-1), dim=-1)
            sdf = torch.gather(torch.cat([sdf, sdf_new], dim=-1), -1, order)
    return z


def _render_from_samples(rays_o, rays_d, model, z_all, query, *, calc_normal, use_view_dirs, white_bkgd, detailed_output,
                         samples_output, random_color_direction):
    """Field evaluation at the final samples + compositing (renderer.py:264-348); differentiable."""
    pts_at = lambda z: rays_o.unsqueeze(-2) + z.unsqueeze(-1) * rays_d.unsqueeze(-2)  # noqa: E731
    z_mid = 0.5 * (z_all[..., 1:] + z_all[..., :-1])
    pts, pts_mid = pts_at(z_all), pts_at(z_mid)
    if calc_normal:
        sdf, nablas = query(model.forward_with_nablas, pts)
    else:
        sdf, nablas = query(model.forward_density_only, pts), None
    sdf = sdf.squeeze(-1)
    cdf, alpha = sdf_to_alpha(sdf, model.forward_s())
    if random_color_direction:
        dirs = torch.rand_like(pts_mid)
        dirs = dirs / torch.linalg.norm(dirs, dim=-1, keepdim=True)
    else:
        view_dirs = rays_d if use_view_dirs else None
        dirs = view_dirs.unsqueeze(-2).expand_as(pts_mid)
    w = alpha_to_w(alpha)
    if not torch.is_grad_enabled() and not detailed_output and pts_mid.dim() == 3:
        # live-sample evaluation (as csrc/render.cu does for a plain NeuMesh): colour is multiplied by the visibility
        # weight below, so mid-points whose weight is exactly 0.0 are not evaluated - adding 0 * c is exact
        live = w != 0
        radiances = torch.zeros_like(pts_mid)
        if bool(live.any()):
            _, c_live = model.forward(pts_mid[live], dirs[live])
            radiances[live] = c_live
        sdf_mid = None
    else:
        sdf_mid, radiances = query(model.forward, pts_mid, dirs)
    rgb = (w[..., None] * radiances).sum(dim=-2)
    depth = (w / (w.sum(dim=-1, keepdim=True) + 1e-10) * z_mid).sum(dim=-1)
    acc = w.sum(dim=-1)
    if white_bkgd:
        rgb = rgb + (1.0 - acc[..., None])
    out = OrderedDict([("rgb", rgb), ("depth_volume", depth), ("mask_volume", acc)])
    if calc_normal:
        nn_ = F.normalize(nablas, dim=-1)
        k = min(w.shape[-1], nn_.shape[-2])
        out["normals_volume"] = (nn_[..., :k, :] * w[..., :k, None]).sum(dim=-2)
    if detailed_output:
        if calc_normal:
            out["implicit_nablas"] = nablas
        out["implicit_surface"] = sdf
        out["radiance"] = radiances
        out["alpha"] = alpha
        out["cdf"] = cdf
        out["visibility_weights"] = w
        out["d_final"] = z_mid
        if samples_output:
            out["xyz"] = pts_mid
            out["dirs"] = rays_d.unsqueeze(-2).expand_as(pts_mid)
            out["density"] = sdf_mid
            out["colors"] = radiances
    return out


def _render_generic(rays_o, rays_d, model, *, dim_batchify, obj_bounding_radius, calc_normal, use_view_dirs, netchunk,
                    white_bkgd, near_bypass, far_bypass, detailed_output, perturb, N_samples, N_importance,
                    N_upsample_iters, samples_output, bounded_near_far, random_color_direction, z_samples=None,
                    perturb_u=None):
    query = lambda fn, *a: batchify_query(fn, *a, chunk=netchunk, dim_batchify=dim_batchify)  # noqa: E731
    if z_samples is None:
        z_samples = _sample_cascade(rays_o, rays_d, model, query, obj_bounding_radius=obj_bounding_radius,
                                    near_bypass=near_bypass, far_bypass=far_bypass, perturb=perturb, N_samples=N_samples,
                                    N_importance=N_importance, N_upsample_iters=N_upsample_iters,
                                    bounded_near_far=bounded_near_far, perturb_u=perturb_u)
    return _render_from_samples(rays_o, rays_d, model, z_samples, query, calc_normal=calc_normal,
                                use_view_dirs=use_view_dirs, white_bkgd=white_bkgd, detailed_output=detailed_output,
                                samples_output=samples_output, random_color_direction=random_color_direction)


def volume_render(rays_o, rays_d, model, obj_bounding_radius=1.0, batched=False, batched_info={}, calc_normal=False,
                  use_view_dirs=True, rayschunk=65536, netchunk=1048576, white_bkgd=False,
                  near_bypass: Optional[float] = None, far_bypass: Optional[float] = None, detailed_output=True,
                  show_progress=False, perturb=False, fixed_s_recp=1 / 64.0, N_samples=64, N_importance=64,
                  N_nograd_samples=2048, N_upsample_iters=4, samples_output=False, bounded_near_far=True,
                  random_color_direction=False, perturb_u=None, z_samples=None, **dummy_kwargs):
    """rays_o, rays_d: [(B,) N_rays, 3] (directions need not be normalised) -> (rgb, depth_volume, extras).

    Beyond the reference's keywords (``renderer.py:105-135``): ``perturb_u`` [N_upsample_iters, N_rays, n] injects the
    uniforms ``perturb=True`` would draw, ``z_samples`` [N_rays, P] skips the sampling cascade (teacher-forced depths);
    both exist for parity runs of the training step."""
    if batched:
        dim_batchify, B = 1, rays_d.shape[0]
        flat_shape = [B, -1, 3]
    else:
        dim_batchify, flat_shape = 0, [-1, 3]
    rays_o = torch.reshape(rays_o, flat_shape).float()
    rays_d = torch.reshape(rays_d, flat_shape).float()

    route = dict(batched=batched, random_color_direction=random_color_direction, use_view_dirs=use_view_dirs,
                 N_samples=N_samples, N_importance=N_importance, N_upsample_iters=N_upsample_iters)
    if fused_eligible(model, rays_o, **route):
        out = render_fused(rays_o, rays_d, model, obj_bounding_radius=obj_bounding_radius, calc_normal=calc_normal,
                           white_bkgd=white_bkgd, near_bypass=near_bypass, far_bypass=far_bypass,
                           N_samples=N_samples, N_importance=N_importance, N_upsample_iters=N_upsample_iters,
                           bounded_near_far=bounded_near_far, detailed_output=detailed_output,
                           samples_output=samples_output, min_chunk=rayschunk, perturb=perturb, perturb_u=perturb_u)
        if batched:  # B == 1
            out = OrderedDict((k, v.unsqueeze(0)) for k, v in out.items())
        return out["rgb"], out["depth_volume"], out

    rays_d = F.normalize(rays_d, dim=-1)
    geo = fused_cascade_model(model, rays_o, z_samples=z_samples, **route)
    if geo is not None:
        # texture edit (editing/texture_neumesh/texture_renderer.py) or training step (config 4): the no-grad sampling
        # cascade runs in the fused CUDA kernels; the evaluation at the final samples goes through the model protocol below
        # (the edit's colour blend per live sample through the fused field kernels, FusedFieldFn in grad mode)
        with torch.no_grad():
            z_samples = render_fused(rays_o.reshape(-1, 3), rays_d.reshape(-1, 3), geo,
                                     obj_bounding_radius=obj_bounding_radius, near_bypass=near_bypass,
                                     far_bypass=far_bypass, N_samples=N_samples, N_importance=N_importance,
                                     N_upsample_iters=N_upsample_iters, bounded_near_far=bounded_near_far,
                                     normalize_dirs=False, min_chunk=rayschunk, perturb=perturb, perturb_u=perturb_u,
                                     sampling_only=True)["d_all"]
        if batched:
            z_samples = z_samples.unsqueeze(0)
    n = rays_o.shape[dim_batchify]
    pieces = []
    it = range(0, n, rayschunk)
    if show_progress:
        try:
            from tqdm import tqdm
            it = tqdm(it)
        except Exception:
            pass
    for s in it:
        sl = (slice(None), slice(s, s + rayschunk)) if batched else (slice(s, s + rayschunk),)
        pieces.append(_render_generic(
            rays_o[sl], rays_d[sl], model, dim_batchify=dim_batchify, obj_bounding_radius=obj_bounding_radius,
            calc_normal=calc_normal, use_view_dirs=use_view_dirs, netchunk=netchunk, white_bkgd=white_bkgd,
            near_bypass=near_bypass, far_bypass=far_bypass, detailed_output=detailed_output, perturb=perturb,
            N_samples=N_samples, N_importance=N_importance, N_upsample_iters=N_upsample_iters,
            samples_output=samples_output, bounded_near_far=bounded_near_far,
            random_color_direction=random_color_direction,
            z_samples=None if z_samples is None else z_samples[sl],
            perturb_u=None if perturb_u is None else (perturb_u[(slice(None),) + sl] if not batched else perturb_u)))
    ret = OrderedDict((k, torch.cat([p[k] for p in pieces], dim=dim_batchify)) for k in pieces[0])
    return ret["rgb"], ret["depth_volume"], ret


class SingleRenderer(nn.Module):
    def __init__(self, model):
        super().__init__()
        self.model = model

    def forward(self, rays_o, rays_d, **kwargs):
        return volume_render(rays_o, rays_d, self.model, **kwargs)


def upsample_step(z, sdf, n_new, inv_s):
    """CUDA ``nmb_upsample_step``: z, sdf [N, n] (sorted depths, their sdf) -> [N, n_new] new depths
    (reference: renderer.py:209-245 + rend_util.sample_pdf(det=True))."""
    _lib.require_cuda(z, "upsample_step")
    zt, st = z.detach().float().t().contiguous(), sdf.detach().float().t().contiguous()
    n, N = zt.shape
    out = torch.empty(n_new, N, device=z.device)
    scratch = torch.empty(n, N, device=z.device)
    with torch.cuda.device(z.device):
        _lib.check(_lib.lib().nmb_upsample_step(_lib.ptr(zt), _lib.ptr(st), N, n, n_new, float(inv_s), _lib.ptr(out),
                                                _lib.ptr(scratch), _lib.stream_ptr(z.device)))
    return out.t().contiguous()


def get_rays(c2w, intrinsics, H, W, device=None):
    """CUDA ray generation for a full H x W image (reference ``utils/rend_util.py:123-176`` with N_rays=-1):
    c2w [4,4]/[3,4], intrinsics [3,3]/[4,4] -> rays_o, rays_d [H*W, 3]."""
    import numpy as np
    device = torch.device(device or "cuda")
    c = np.asarray(torch.as_tensor(c2w).detach().cpu().float().numpy())[:3, :4].astype(np.float32).reshape(-1)
    K = np.asarray(torch.as_tensor(intrinsics).detach().cpu().float().numpy())
    intr = np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2], K[0, 1]], dtype=np.float32)
    o = torch.empty(H * W, 3, device=device)
    d = torch.empty(H * W, 3, device=device)
    with torch.cuda.device(device):
        _lib.check(_lib.lib().nmb_get_rays(c.ctypes.data_as(C.POINTER(C.c_float)),
                                           intr.ctypes.data_as(C.POINTER(C.c_float)), H, W, _lib.ptr(o), _lib.ptr(d),
                                           _lib.stream_ptr(device)))
    return o, d


def pack_bgr8(rgb, H=None, W=None):
    """CUDA ``nmb_pack_bgr8``: rgb [N,3] float -> uint8 BGR (``[H,W,3]`` if H, W given), the conversion ``render.py``
    does on the host before ``cv2.imwrite`` (render.py:219-241)."""
    _lib.require_cuda(rgb, "pack_bgr8")
    flat = rgb.detach().reshape(-1, 3).float().contiguous()
    out = torch.empty(flat.shape[0], 3, dtype=torch.uint8, device=flat.device)
    with torch.cuda.device(flat.device):
        _lib.check(_lib.lib().nmb_pack_bgr8(_lib.ptr(flat), flat.shape[0], _lib.ptr(out), _lib.stream_ptr(flat.device)))
    return out.reshape(H, W, 3) if H and W else out


def vertex_normals(vertices, triangles):
    """CUDA ``nmb_vertex_normals``: area-weighted vertex normals (Open3D ``compute_vertex_normals`` semantics); bit-
    reproducible under ``torch.use_deterministic_algorithms(True)``."""
    _lib.require_cuda(vertices, "vertex_normals")
    v = vertices.detach().float().contiguous()
    t = triangles.detach().to(torch.int32).contiguous()
    out = torch.empty_like(v)
    _lib.sync_deterministic()
    with torch.cuda.device(v.device):
        _lib.check(_lib.lib().nmb_vertex_normals(_lib.ptr(v), v.shape[0], _lib.ptr(t), t.shape[0], _lib.ptr(out),
                                                 _lib.stream_ptr(v.device)))
    return out
