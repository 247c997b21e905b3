"""CPU restatement of the NeuMesh volume renderer - TEST INFRASTRUCTURE (see ``oracle/__init__.py``).

Restates ``models/renderer.py`` (``sdf_to_alpha`` :17-24, ``alpha_to_w`` :49-63, ``compute_bounded_near_far`` :66-102,
``volume_render`` :105-368) and ``utils/rend_util.py`` (``near_far_from_sphere`` :179-199, ``sample_pdf`` :276-319) for
the un-batched, ``perturb=False`` case, as fp32 torch-CPU code over any object with the field protocol
(``compute_distance``, ``forward_density_only``, ``forward_with_nablas``, ``forward``, ``forward_s``).

Pinned against the verbatim-imported reference renderer by ``tests/test_oracle.py::test_oracle_vs_unmodified_reference`` and the committed
``tests/golden/*.npz``.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def sphere_near_far(o, d, r=1.0):
    """rend_util.py:179-199."""
    mid = -(o * d).sum(dim=-1, keepdim=True)
    return (mid - r).clamp_min(0.0), (mid + r).clamp_min(r)


def transmittance_weights(alpha):
    """renderer.py:49-63: w_i = alpha_i * prod_{j<i} (1 - alpha_j + 1e-10)."""
    ones = torch.ones_like(alpha[..., :1])
    trans = torch.cumprod(torch.cat([ones, 1.0 - alpha + 1e-10], dim=-1), dim=-1)[..., :-1]
    return alpha * trans


def inverse_cdf_samples(bins, weights, n, u=None):
    """rend_util.py:276-319 with det=True (u = linspace(0,1,n)) unless ``u`` is given."""
    weights = weights + 1e-5
    pdf = weights / weights.sum(dim=-1, keepdim=True)
    cdf = torch.cumsum(pdf, dim=-1)
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], dim=-1)
    if u is None:
        u = torch.linspace(0.0, 1.0, steps=n).expand(*cdf.shape[:-1], n)
    u = u.contiguous()
    inds = torch.searchsorted(cdf, u, right=False)
    below = (inds - 1).clamp_min(0)
    above = inds.clamp_max(cdf.shape[-1] - 1)
    c0, c1 = torch.gather(cdf, -1, below), torch.gather(cdf, -1, above)
    b0, b1 = torch.gather(bins, -1, below), torch.gather(bins, -1, above)
    denom = c1 - c0
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    return b0 + (u - c0) / denom * (b1 - b0)


def mesh_bounded_near_far(field, o, d, near, far, n_grid=256, thresh=0.1):
    """renderer.py:66-102."""
    t = torch.linspace(0, 1, n_grid).to(near.device)   # the CPU values, also for tensors on a GPU
    depth = (near * (1 - t) + far * t)[..., None]  # [N, G, 1]
    pts = o[:, None, :] + depth * d[:, None, :]
    ds, _, _ = field.compute_distance(pts)
    inside = ds < thresh
    lo = (depth * inside.float() + (~inside).float() * 1e10).min(dim=-2)[0]
    hi = (depth * inside.float() - (~inside).float() * 1e10).max(dim=-2)[0]
    lo = torch.where(lo > 1e5, near, lo)
    hi = torch.where(hi < -1e5, far, hi)
    thin = (hi - lo) < 0.1
    hi = torch.where(thin, hi + 0.05, hi)
    lo = torch.where(thin, lo - 0.05, lo)
    return lo, hi


def _render_chunk(field, o, d, *, radius, calc_normal, white_bkgd, n_samples, n_importance, n_iters, bounded,
                  near_bypass, far_bypass, detailed, perturb_u=None):
    near, far = sphere_near_far(o, d, radius)
    if bounded:
        near, far = mesh_bounded_near_far(field, o, d, near, far)
    if near_bypass is not None:
        near = torch.full_like(near, near_bypass)
    if far_bypass is not None:
        far = torch.full_like(far, far_bypass)

    def pts_at(depths):
        return o[:, None, :] + depths[..., None] * d[:, None, :]

    t = torch.linspace(0, 1, n_samples)
    z = near * (1 - t) + far * t  # [N, S]
    sdf = field.forward_density_only(pts_at(z)).squeeze(-1)
    for it in range(n_iters):  # renderer.py:208-258
        s0, s1, z0, z1 = sdf[..., :-1], sdf[..., 1:], z[..., :-1], z[..., 1:]
        mid = (s0 + s1) * 0.5
        slope = (s1 - s0) / (z1 - z0 + 1e-5)
        prev_slope = torch.cat([torch.zeros_like(slope[..., :1]), slope[..., :-1]], dim=-1)
        slope = torch.minimum(prev_slope, slope).clamp(-10.0, 0.0)
        dist = z1 - z0
        est0 = mid - slope * dist * 0.5
        est1 = mid + slope * dist * 0.5
        inv_s = 256 * (2 ** it)
        c0, c1 = torch.sigmoid(est0 * inv_s), torch.sigmoid(est1 * inv_s)
        alpha = (c0 - c1 + 1e-5) / (c0 + 1e-5)
        # perturb=True (rend_util.py:292-295) draws u = torch.rand; parity runs inject the draws: perturb_u [iters, N, n]
        z_new = inverse_cdf_samples(z, transmittance_weights(alpha), n_importance // n_iters,
                                    u=None if perturb_u is None else perturb_u[it])
        sdf_new = field.forward_density_only(pts_at(z_new)).squeeze(-1)
        z, order = torch.sort(torch.cat([z, z_new], dim=-1), dim=-1)
        sdf = torch.gather(torch.cat([sdf, sdf_new], dim=-1), -1, order)

    z_mid = 0.5 * (z[..., 1:] + z[..., :-1])
    if calc_normal:
        sdf_pts, nablas = field.forward_with_nablas(pts_at(z))
    else:
        sdf_pts, nablas = field.forward_density_only(pts_at(z)), None
    sdf_pts = sdf_pts.squeeze(-1)
    cdf = torch.sigmoid(sdf_pts * field.forward_s())  # renderer.py:13-24
    alpha = ((cdf[..., :-1] - cdf[..., 1:]) / (cdf[..., :-1] + 1e-10)).clamp_min(0)
    pm = pts_at(z_mid)
    sdf_mid, radiance = field.forward(pm, d[:, None, :].expand_as(pm))
    w = transmittance_weights(alpha)
    rgb = (w[..., None] * radiance).sum(dim=-2)
    depth = (w / (w.sum(dim=-1, keepdim=True) + 1e-10) * z_mid).sum(dim=-1)
    acc = w.sum(dim=-1)
    if white_bkgd:
        rgb = rgb + (1.0 - acc[..., None])
    out = {"rgb": rgb, "depth_volume": depth, "mask_volume": acc}
    if calc_normal:
        nn_ = F.normalize(nablas, dim=-1)
        k = min(w.shape[-1], nn_.shape[-2])
        out["normals_volume"] = (nn_[..., :k, :] * w[..., :k, None]).sum(dim=-2)
    if detailed:
        if calc_normal:
            out["implicit_nablas"] = nablas
        out.update({"implicit_surface": sdf_pts, "radiance": radiance, "alpha": alpha, "cdf": cdf,
                    "visibility_weights": w, "d_final": z_mid, "d_all": z, "near": near, "far": far})
    return out


def volume_render(rays_o, rays_d, field, obj_bounding_radius=1.0, calc_normal=False, rayschunk=65536,
                  white_bkgd=False, near_bypass=None, far_bypass=None, detailed_output=False, N_samples=64,
                  N_importance=64, N_upsample_iters=4, bounded_near_far=True, perturb_u=None, **_ignored):
    """renderer.py:105-368, un-batched; perturb=False, or perturb=True with the uniforms given as ``perturb_u``
    [N_upsample_iters, N, N_importance / N_upsample_iters].  Returns (rgb [N,3], depth [N], extras)."""
    o = rays_o.reshape(-1, 3).float()
    d = F.normalize(rays_d.reshape(-1, 3).float(), dim=-1)
    chunks = []
    with torch.no_grad():
        for s in range(0, o.shape[0], rayschunk):
            chunks.append(_render_chunk(field, o[s:s + rayschunk], d[s:s + rayschunk], radius=obj_bounding_radius,
                                        calc_normal=calc_normal, white_bkgd=white_bkgd, n_samples=N_samples,
                                        n_importance=N_importance, n_iters=N_upsample_iters,
                                        bounded=bounded_near_far, near_bypass=near_bypass, far_bypass=far_bypass,
                                        detailed=detailed_output,
                                        perturb_u=None if perturb_u is None else perturb_u[:, s:s + rayschunk]))
    out = {k: torch.cat([c[k] for c in chunks], dim=0) for k in chunks[0]}
    return out["rgb"], out["depth_volume"], out
