"""CPU emulation of the aero_gan_loss_fwd / _bwd contract (include/aero_b200.h) on aero_b200.gan term tables, and the reference's
loss functions (src/models/discriminators.py:211-244 of the unmodified reference when a checkout is found, else restated)."""
import importlib
import os
import sys

import torch

from aero_b200 import cabi


def owned(m):
    """[n_seg, H, C] view of the owned rows of a Map."""
    return m.t.view(m.n_seg, m.seg, m.C)[:, m.halo:m.halo + m.H]


def _adv(kind, x):
    if kind in (cabi.GAN_LSGAN_REAL, cabi.GAN_LSGAN_GEN):
        return (1 - x) ** 2, -2 * (1 - x)
    if kind == cabi.GAN_LSGAN_FAKE:
        return x * x, 2 * x
    if kind in (cabi.GAN_HINGE_REAL, cabi.GAN_HINGE_GEN):
        return torch.relu(1 - x), -((1 - x) > 0).to(x.dtype)
    if kind == cabi.GAN_HINGE_FAKE:
        return torch.relu(1 + x), ((1 + x) > 0).to(x.dtype)
    return torch.zeros_like(x), torch.zeros_like(x)


def emulate(terms):
    """out [n_terms, 2] fp64 as aero_gan_loss_fwd; writes every term's dx as aero_gan_loss_bwd."""
    out = torch.zeros(len(terms), 2, dtype=torch.float64)
    for k, t in enumerate(terms):
        x = owned(t.x)
        v, d = _adv(t.adv, x)
        g = torch.zeros_like(x)
        if t.adv != cabi.GAN_NONE:
            out[k, 0] = t.adv_scale * v.double().sum()
            g = g + t.adv_scale * d
        if t.ref is not None:
            diff = x - owned(t.ref)
            out[k, 1] = t.l1_scale * diff.abs().double().sum()
            g = g + t.l1_scale * torch.sign(diff)
        if t.dx is not None:
            full = torch.zeros(t.x.n_seg, t.x.seg, t.x.C)
            full[:, t.x.halo:t.x.halo + t.x.H] = g
            t.dx.copy_(full.reshape(-1))
    return out


def reference_losses(ref_root=None):
    """(discriminator_loss, generator_loss, feature_loss) of the unmodified reference at `ref_root` (default $AERO_REFERENCE, else
    ./reference), or restated when there is no checkout.  Second value: whether the reference's own functions were found."""
    from util import ROOT
    root = os.path.abspath(ref_root or os.environ.get("AERO_REFERENCE") or "reference")
    if os.path.isdir(root):
        saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "src" or k.startswith("src.")}
        path_saved = list(sys.path)
        sys.path[:] = [root] + [p for p in sys.path if os.path.abspath(p or ".") != ROOT]
        try:
            mod = importlib.import_module("src.models.discriminators")
        finally:
            sys.path[:] = path_saved
            for k in [k for k in sys.modules if k == "src" or k.startswith("src.")]:
                del sys.modules[k]
            sys.modules.update(saved)
        return (mod.discriminator_loss, mod.generator_loss, mod.feature_loss), True

    def discriminator_loss(real, fake):
        return sum(torch.mean((1 - r) ** 2) + torch.mean(g ** 2) for r, g in zip(real, fake))

    def generator_loss(fake):
        return sum(torch.mean((1 - g) ** 2) for g in fake)

    def feature_loss(f_r, f_g):
        terms = [torch.mean(torch.abs(a - b)) for dr, dg in zip(f_r, f_g) for a, b in zip(dr, dg)]
        return sum(terms) / len(terms)
    return (discriminator_loss, generator_loss, feature_loss), False
