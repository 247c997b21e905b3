"""``TextureEditableNeuMesh`` - drop-in for ``editing/texture_neumesh/texture_neumesh.py`` (SURVEY.md section 8f item 2).

Texture swap / fill: the main model supplies geometry and its own colour everywhere; inside each painted region the
colour comes from a reference model's colour network evaluated on the main mesh's neighbours with the painted
vertices' (transferred) colour codes, blended by how much of a point's interpolation weight sits on painted vertices.

With ``neumesh_b200.NeuMesh`` models and grad mode off every field evaluation below runs in the CUDA library:
``forward(..., nablas_only=True, return_ds=True)`` -> ``nmb_field_forward_ex`` and both ``forward_color`` calls ->
``nmb_field_color`` (the reference model's colour network reading the edited code table through ``color_table``).

Rendering (``volume_render`` / ``render_fused``) runs the whole edit in ``nmb_render_edit``: the main model's fused
cascade, and after the main colour MLP the per-point blend of every reference model (``packed_edit``).  The helpers
below accept this class or any object with its attributes (``main_model``, ``ref_models``, ``main_editing_masks``,
``main_editing_colorfeats``, ``rot_s_m``), such as the reference's own class.
"""
from __future__ import annotations

import ctypes as C
import weakref

import torch
import torch.nn as nn

from . import _lib
from .neumesh import NeuMesh

EDIT_ATTRS = ("main_model", "ref_models", "main_editing_masks", "main_editing_colorfeats", "rot_s_m")
_EDITS: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()


def is_edit_model(model) -> bool:
    return all(hasattr(model, a) for a in EDIT_ATTRS)


def _edit_problem(model):
    """None if ``nmb_render_edit`` can render ``model``, otherwise why not."""
    if not is_edit_model(model):
        return "not a texture-edit model (needs the attributes %s)" % ", ".join(EDIT_ATTRS)
    main, refs = model.main_model, list(model.ref_models)
    masks, codes, rot = model.main_editing_masks, model.main_editing_colorfeats, model.rot_s_m
    if not isinstance(main, NeuMesh) or not refs or not all(isinstance(r, NeuMesh) for r in refs):
        return "the main model and at least one reference model must be neumesh_b200.NeuMesh models"
    V = main.geometry_features.shape[0]
    if masks.dim() != 2 or tuple(masks.shape) != (len(refs), V):
        return "main_editing_masks has shape %s, expected [n_ref, V_main] = [%d, %d]" % (tuple(masks.shape), len(refs), V)
    if codes.dim() != 2 or codes.shape[0] != V:
        return "main_editing_colorfeats has shape %s, expected [V_main = %d, color_dim]" % (tuple(codes.shape), V)
    for i, r in enumerate(refs):
        if r._cfg["color_dim"] != codes.shape[1]:
            return "reference model %d has color_dim %d but main_editing_colorfeats is %d wide" % (
                i, r._cfg["color_dim"], codes.shape[1])
    if rot is not None and tuple(rot.shape) != (len(refs), 3, 3):
        return "rot_s_m has shape %s, expected [n_ref, 3, 3]" % (tuple(rot.shape),)
    if not main.fused_supported() or not all(r.fused_supported() for r in refs):
        return "a model's configuration is outside the fused kernels' specialisation (NeuMesh.fused_supported)"
    tensors = [main.geometry_features, masks, codes] + [r.color_features for r in refs]
    if not all(t.is_cuda for t in tensors):
        return "the models, masks and codes must be on a CUDA device"
    return None


def edit_fused_supported(model) -> bool:
    """True if ``nmb_render_edit`` can render this texture-edit model (the main model and every reference model fused-
    capable, CUDA tensors, colour widths that match the code table, masks of shape [n_ref, V_main])."""
    return _edit_problem(model) is None


class _PackedEdit:
    def __init__(self, handle, key):
        self.handle, self.key = handle, key

    def __del__(self):
        if self.handle:
            try:
                _lib.lib().nmb_edit_destroy(self.handle)
            except Exception:
                pass
            self.handle = None


def _tensor_key(t):
    return None if t is None else (id(t), t.data_ptr(), t._version)


def packed_edit(model):
    """``nmb_edit`` handle of a texture-edit model, cached per model and rebuilt when a field handle, the masks, the
    codes or the rotations changed (tensor identity and in-place version counters, as ``NeuMesh.packed_field``), or the
    main model's grid was deformed in place (its generation: the masks and codes are re-permuted by ``nmb_edit_update``)."""
    problem = _edit_problem(model)
    if problem is not None:
        raise ValueError("neumesh_b200: cannot render this texture edit on the fused path: " + problem)
    main, refs = model.main_model, list(model.ref_models)
    masks, codes, rot = model.main_editing_masks, model.main_editing_colorfeats, model.rot_s_m
    fields = [main.packed_field()] + [r.packed_field() for r in refs]
    # the handle objects themselves (kept alive by the cache entry): a re-created field is a new object
    key_fields = tuple(id(h) for h in fields)
    key_vals = (_tensor_key(masks), _tensor_key(codes), _tensor_key(rot), main.mesh_grid.grid.generation)
    entry = _EDITS.get(model)
    if entry is not None and entry.key == (key_fields, key_vals):
        return entry.handle
    dev = main.geometry_features.device
    m = masks.detach().to(device=dev, dtype=torch.uint8).contiguous()
    c = codes.detach().to(device=dev, dtype=torch.float32).contiguous()
    r = None
    if rot is not None:
        r_host = rot.detach().to("cpu", torch.float32).reshape(-1).contiguous()
        r = (C.c_float * r_host.numel())(*r_host.tolist())
    L = _lib.lib()
    with torch.cuda.device(dev):
        if entry is not None and entry.key[0] == key_fields:
            _lib.check(L.nmb_edit_update(entry.handle, _lib.ptr(m), _lib.ptr(c), r, _lib.stream_ptr(dev)))
            entry.key = (key_fields, key_vals)
            return entry.handle
        arr = (C.c_void_p * len(refs))(*[h.value for h in fields[1:]])
        h = C.c_void_p()
        _lib.check(L.nmb_edit_create(fields[0], len(refs), arr, _lib.ptr(m), _lib.ptr(c), m.shape[1], c.shape[1], r,
                                     _lib.stream_ptr(dev), C.byref(h)))
    entry = _PackedEdit(h, (key_fields, key_vals))
    entry.fields = fields
    _EDITS[model] = entry
    return h


class TextureEditableNeuMesh(nn.Module):
    """Same constructor and model protocol as the reference class (``texture_neumesh.py:8-122``).

    ``fused_render = False`` keeps ``volume_render`` on the generic path (fused cascade, torch-op blend per chunk)."""

    fused_render = True

    def __init__(self, main_model, ref_models, main_editing_masks, main_editing_colorfeats, T_r_m_list=None):
        super().__init__()
        self.main_model = main_model
        self.ref_models = nn.ModuleList(ref_models)
        self.register_buffer("main_editing_masks", main_editing_masks)          # [n_ref, V_main] bool
        self.register_buffer("main_editing_colorfeats", main_editing_colorfeats)  # [V_main, color_dim]
        if T_r_m_list is not None:   # main -> reference frame transforms; only the rotation acts on directions
            self.register_buffer("rot_s_m", torch.stack([T[:3, :3] for T in T_r_m_list], dim=0))
            self.register_buffer("t_s_m", torch.stack([T[:3, 3] for T in T_r_m_list], dim=0))
        else:
            self.rot_s_m = None
            self.t_s_m = None
        self.enable_nablas_input = main_model.enable_nablas_input

    # ---- geometry: the main model's (texture_neumesh.py:40-50) ----
    def compute_distance(self, xyz):
        return self.main_model.compute_distance(xyz)

    def forward_s(self):
        return self.main_model.forward_s()

    def forward_density_only(self, xyz):
        return self.main_model.forward_density_only(xyz)

    def forward_with_nablas(self, xyz):
        return self.main_model.forward_with_nablas(xyz)

    # ---- colour: main colour, over-painted region by region (texture_neumesh.py:52-122) ----
    def forward(self, xyz, view_dirs, need_nablas=True, nablas_only=False):
        main = self.main_model
        sdf, nabla, ds, idx, w = main.forward(xyz, view_dirs, need_nablas=need_nablas, nablas_only=True, return_ds=True)
        out = main.forward_color(ds, view_dirs, main.color_features, indices=idx, weights=w, nabla=nabla).clone()
        for i, ref in enumerate(self.ref_models):
            painted = self.main_editing_masks[i][idx]                 # [..., 8] neighbour is a painted vertex
            w_paint = (w * painted).sum(dim=-1)
            w_rest = (w * (painted == False)).sum(dim=-1)             # noqa: E712  (kept as a separate sum, as there)
            region = w_paint > 0
            total = w_paint + w_rest
            a_paint = (w_paint / total)[region]
            a_rest = (w_rest / total)[region]
            w_ref = w * painted
            w_ref = w_ref / (w_ref.sum(dim=-1, keepdim=True) + 1e-8)   # painted neighbours only, renormalised
            if self.rot_s_m is not None:
                R = self.rot_s_m[i]
                dirs_ref = torch.matmul(R, view_dirs.unsqueeze(-1)).squeeze(-1)
                nabla_ref = torch.matmul(R, nabla.unsqueeze(-1)).squeeze(-1)
            else:
                dirs_ref, nabla_ref = view_dirs, nabla
            if bool(region.any()):
                c_ref = ref.forward_color(ds[region], dirs_ref[region], self.main_editing_colorfeats,
                                          indices=idx[region], weights=w_ref[region], nabla=nabla_ref[region])
                out[region] = out[region] * a_rest.unsqueeze(-1) + c_ref * a_paint.unsqueeze(-1)
        return sdf, out
