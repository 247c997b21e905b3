"""TEST-ONLY pieces shared by ``tests/test_neus_train.py`` and ``tests/golden/make_neus_train_golden.py``:

* ``NeusTorchPrims``: ``train_prims_torch.TorchPrims`` plus the NeuS surface op's primitives (``nmb_ns_*``), in torch ops;
  on CPU it is injected into ``neus_ops`` to check the op's sequencing, on the GPU it is the per-kernel reference;
* ``neus_loss``: the NeuS stage-1 loss as ``models/trainer.py:173-262`` computes it (image L1 over the masked rays, mask
  BCE, eikonal) with the loss weights of ``configs/neus_dtu_scan63.yaml``.
Nothing in the product imports this module."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from train_prims_torch import TorchPrims, pe, softplus_terms


def _pe_d1_cols(x, L):
    """[M, 3(1+2L)] derivative of each PE column with respect to its own coordinate."""
    out = [torch.ones_like(x)]
    for k in range(L):
        f = 2.0 ** k
        out += [f * torch.cos(x * f), -f * torch.sin(x * f)]
    return torch.cat(out, -1)


def _rows(T, ld, rows, cols):
    return T.reshape(-1).as_strided((rows, cols), (ld, 1))


class NeusTorchPrims(TorchPrims):
    def pe(self, x, L, out, ldo):
        _rows(out, ldo, x.shape[0], 3 * (1 + 2 * L)).copy_(pe(x, L))

    def pe_jt(self, x, L, ebar, nabla):
        nabla.copy_((ebar * _pe_d1_cols(x, L)).reshape(x.shape[0], 1 + 2 * L, 3).sum(1))

    def pe_j(self, x, L, b_nabla, b_e):
        b_e.copy_(b_nabla.repeat(1, 1 + 2 * L) * _pe_d1_cols(x, L))

    def softplus(self, z, h, ldh):
        _rows(h, ldh, z.shape[0], z.shape[1]).copy_(softplus_terms(z)[0])

    def gate(self, g, row, z, out):
        v = g if g is not None else row.reshape(1, -1).expand(out.shape)
        out.copy_(v * softplus_terms(z)[1] if z is not None else v)


NEUS_LOSS_WEIGHTS = dict(img=1.0, mask=1.0, eikonal=0.1)


def neus_loss(rgb, target_rgb, target_mask, extras):
    nab = extras["implicit_nablas"].norm(dim=-1)
    acc = extras["mask_volume"].clamp(1e-3, 1 - 1e-3)
    m = target_mask.to(rgb.dtype)
    l_img = (F.l1_loss(rgb, target_rgb, reduction="none") * m[..., None]).sum() / (m.sum() + 1e-10)
    l_mask = F.binary_cross_entropy(acc, m, reduction="mean")
    l_eik = F.mse_loss(nab, nab.new_ones(nab.shape), reduction="mean")
    w = NEUS_LOSS_WEIGHTS
    return w["img"] * l_img + w["mask"] * l_mask + w["eikonal"] * l_eik
