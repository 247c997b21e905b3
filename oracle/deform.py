"""CPU restatement of ``deform_model``'s indicator rotation (``editing/render_geometry_editing.py:37-67``) - TEST
INFRASTRUCTURE (see ``oracle/__init__.py``), the specification ``nmb_indicator_rotate`` (``csrc/deform.cu``) computes.

The reference, per vertex, with the old and the new vertex normal:

    axis = torch.cross(n_old, n_new)                                       :46-48
    c    = clamp(sum(n_old * n_new) / (|n_old| |n_new|), -1, 1)            :49-51 (cos_between_vectors)
    aa   = axis * acos(c)                                                  :53-55
    R    = kornia.geometry.conversions.angle_axis_to_rotation_matrix(aa)
    out  = R @ ind;  out[c == -1] *= -1                                    :58-62

``|aa| = theta |axis| = theta |n_old| |n_new| sin(theta)``, not theta: the rotation applied is not the one between the
normals.  That is what the reference computes, so it is what is restated here.

kornia (not a dependency of this project) computes ``angle_axis_to_rotation_matrix`` as (its form, from ceres'
rotation.h)::

    theta2 = aa . aa
    if theta2 > 1e-6:                       # "normal" branch, Rodrigues' formula
        theta = sqrt(theta2);  w = aa / (theta + 1e-6);  c = cos(theta);  s = sin(theta)
        R = [[c + wx wx (1 - c),    wx wy (1 - c) - wz s,  wy s + wx wz (1 - c)],
             [wz s + wx wy (1 - c), c + wy wy (1 - c),     -wx s + wy wz (1 - c)],
             [-wy s + wx wz (1 - c), wx s + wy wz (1 - c), c + wz wz (1 - c)]]
    else:                                   # first-order Taylor branch
        R = [[1, -az, ay], [az, 1, -ax], [-ay, ax, 1]]

Every sum below is written out in the order the CUDA kernel rounds it (``((x0 y0 + x1 y1) + x2 y2)``), so the fp32
form differs from the kernel only through ``acos`` / ``cos`` / ``sin``, which are not correctly rounded on either side.
"""
from __future__ import annotations

import torch

THETA2_EPS = 1e-6   # kornia: mask = theta2 > eps
W_EPS = 1e-6        # kornia: wxyz = angle_axis / (theta + eps)


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return torch.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1],
                        a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                        a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], dim=-1)


def angle_axis_to_rotation_matrix(aa: torch.Tensor) -> torch.Tensor:
    """kornia's ``angle_axis_to_rotation_matrix`` (see the module docstring): [N,3] -> [N,3,3]."""
    theta2 = _dot(aa, aa)
    theta = torch.sqrt(theta2)
    w = aa / (theta + W_EPS)[:, None]
    wx, wy, wz = w.unbind(-1)
    c, s = torch.cos(theta), torch.sin(theta)
    omc = 1.0 - c
    normal = torch.stack([
        c + wx * wx * omc, wx * wy * omc - wz * s, wy * s + wx * wz * omc,
        wz * s + wx * wy * omc, c + wy * wy * omc, -wx * s + wy * wz * omc,
        -wy * s + wx * wz * omc, wx * s + wy * wz * omc, c + wz * wz * omc], dim=-1)
    ax, ay, az = aa.unbind(-1)
    one = torch.ones_like(ax)
    taylor = torch.stack([one, -az, ay, az, one, -ax, -ay, ax, one], dim=-1)
    return torch.where((theta2 > THETA2_EPS)[:, None], normal, taylor).reshape(-1, 3, 3)


def cos_between(n_old: torch.Tensor, n_new: torch.Tensor, dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """``cos_between_vectors`` (``render_geometry_editing.py:20-34``, clamped) in ``dtype``: the rows with exactly -1
    are negated.  That test is a discontinuity of the reference: a pair of normals within rounding of opposite is
    negated in one precision and rotated (by almost nothing: |axis| ~ 0) in another."""
    a, b = n_old.to(dtype), n_new.to(dtype)
    return torch.clamp(_dot(a, b) / (torch.sqrt(_dot(a, a)) * torch.sqrt(_dot(b, b))), -1, 1)


def indicator_rotate(n_old: torch.Tensor, n_new: torch.Tensor, ind: torch.Tensor,
                     dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """The rotated indicator vectors [V,3], computed in ``dtype`` (float32: the kernel's arithmetic; float64: the
    reference formula without fp32 rounding)."""
    a, b, v = n_old.to(dtype), n_new.to(dtype), ind.to(dtype)
    axis = _cross(a, b)
    c = cos_between(a, b, dtype)
    flip = c == -1
    aa = axis * torch.acos(c)[:, None]
    R = angle_axis_to_rotation_matrix(aa)
    out = torch.stack([_dot(R[:, 0], v), _dot(R[:, 1], v), _dot(R[:, 2], v)], dim=-1)
    return torch.where(flip[:, None], -out, out)
