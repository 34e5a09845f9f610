"""The reference's adversarial losses (``src/solver.py:428-520, 580-612``, loss functions of ``src/models/discriminators.py:211-244``)
against the discriminators of ``discriminator_models`` that this package provides: ``msd_melgan``
(``aero_b200.discriminator.Discriminator``) and ``mpd`` (``aero_b200.mpd.MultiPeriodDiscriminator``).

Two routes compute the same losses and gradients:

* ``autograd_losses``: the reference's ``_get_losses`` restated on the discriminators' ``torch.autograd.Function`` s -- every
  discriminator runs on the real clips twice and its backward computes weight gradients the generator step throws away;
* ``MelganAdversary`` / ``MpdAdversary``: the two passes ``aero_b200.trainer.GanTrainer`` drives directly on the engines' tapes
  (DESIGN.md, "The adversarial step"): one joint forward over ``[hr, pr.detach()]`` whose backward computes parameter gradients but
  no input gradient, then one forward of ``pr`` whose backward computes the input gradient only.  The loss terms and their gradients
  are read and written in the engines' own storage by ``aero_gan_loss_fwd`` / ``_bwd`` (``csrc/ganloss.cu``).

A loss term (``Term``) is one feature map in that storage -- ``n_seg`` segments of ``seg`` rows x ``C`` channels whose rows
``[halo, halo + H)`` are owned -- with an optional adversarial component on it and an optional L1 component against the kept
real-clip map of the same geometry.
"""
from __future__ import annotations

import ctypes as C
from collections.abc import Mapping

import torch
import torch.nn.functional as F

from . import cabi
from .cabi import (GAN_HINGE_FAKE, GAN_HINGE_GEN, GAN_HINGE_REAL, GAN_LSGAN_FAKE, GAN_LSGAN_GEN, GAN_LSGAN_REAL, GAN_NONE)
from .discriminator import Discriminator, _DiscEngine
from .mpd import MultiPeriodDiscriminator, _MpdEngine, period_layout
from .train_engine import _ptr

__all__ = ["DISCRIMINATORS", "MelganAdversary", "MpdAdversary", "Map", "Term", "autograd_losses", "build_discriminators",
           "check_discriminators", "gan_loss_bwd", "gan_loss_fwd"]

# discriminator_models name -> (class, short name of its generator losses)
DISCRIMINATORS = {"msd_melgan": (Discriminator, "melgan"), "mpd": (MultiPeriodDiscriminator, "mpd")}
_WHY = ("the HiFi-GAN multi-scale discriminator ('msd_hifi', and 'hifi' which needs it) is not implemented on the kernels "
        "(DESIGN.md section 1)")


def check_discriminators(discs):
    """discs: {discriminator_models name: module}; returns it as an ordered dict after checking names and types."""
    if not isinstance(discs, Mapping) or not discs:
        raise TypeError("expected a non-empty mapping {name: discriminator} keyed like discriminator_models")
    out = {}
    for name, d in discs.items():
        if name not in DISCRIMINATORS:
            raise NotImplementedError(f"discriminator {name!r}: aero_b200 trains against 'msd_melgan' and 'mpd'; {_WHY}")
        cls = DISCRIMINATORS[name][0]
        if not isinstance(d, cls):
            raise TypeError(f"discriminator {name!r} must be {cls.__module__}.{cls.__name__}, got {type(d).__name__}")
        out[name] = d
    return out


def build_discriminators(experiment):
    """{name: module} for an experiment config (aero_b200.load_experiment), as reference ``modelFactory.get_model`` builds them:
    ``Discriminator(**melgan_discriminator)`` then ``MultiPeriodDiscriminator(**mpd)`` (that construction order, so that one seed
    gives the reference's weights), keyed and ordered like ``discriminator_models``.  Empty unless ``adversarial`` is set."""
    if not experiment.get("adversarial", False):
        return {}
    names = list(experiment["discriminator_models"])
    for n in names:
        if n not in DISCRIMINATORS:
            raise NotImplementedError(f"discriminator_models entry {n!r}: {_WHY}")
    built = {}
    if "msd_melgan" in names:
        built["msd_melgan"] = Discriminator(**experiment["melgan_discriminator"])
    if "mpd" in names:
        built["mpd"] = MultiPeriodDiscriminator(**experiment["mpd"])
    return {n: built[n] for n in names}


# ---------------------------------------------------------------------------------------------------------- the autograd route
def _lsgan_d(y_r, y_g):
    return sum(torch.mean((1 - r) ** 2) + torch.mean(g ** 2) for r, g in zip(y_r, y_g))


def _feature_loss(f_r, f_g):
    terms = [torch.mean(torch.abs(a - b)) for dr, dg in zip(f_r, f_g) for a, b in zip(dr, dg)]
    return sum(terms) / len(terms)


def autograd_losses(pr, hr, discs, stft_loss=None, features_loss_lambda=100.0, only_features_loss=False, only_adversarial_loss=False):
    """The reference's ``Solver._get_losses`` for ``losses: [stft]`` (if stft_loss is given) and the discriminators of `discs`, through
    plain autograd: ``{'generator': {...}, 'discriminator': {...}}``.  ``sum(generator).backward()`` gives the generator's gradients
    (and discriminator gradients the reference discards); ``sum(discriminator).backward()`` the discriminators'."""
    discs = check_discriminators(discs)
    gl, dl = {}, {}
    if stft_loss is not None:
        sc, mag = stft_loss(pr.squeeze(1), hr.squeeze(1))
        gl["stft"] = sc + mag
    for name, d in discs.items():
        short = DISCRIMINATORS[name][1]
        if name == "msd_melgan":
            fake_det, real, fake = d(pr.detach()), d(hr), d(pr)
            d_loss = sum(F.relu(1 + s[-1]).mean() for s in fake_det) + sum(F.relu(1 - s[-1]).mean() for s in real)
            w = (1.0 / d.num_D) * (4.0 / (melgan_n_layers(d) + 1))
            feat = 0.0
            for i in range(d.num_D):
                for j in range(len(fake[i]) - 1):
                    feat = feat + w * F.l1_loss(fake[i][j], real[i][j].detach())
            adv = sum(F.relu(1 - s[-1]).mean() for s in fake)
        else:
            y_r, y_g, _, _ = d(hr, pr.detach())
            d_loss = _lsgan_d(y_r, y_g)
            _, y_g, f_r, f_g = d(hr, pr)
            feat = _feature_loss(f_r, f_g)
            adv = sum(torch.mean((1 - g) ** 2) for g in y_g)
        if not only_features_loss:
            gl["adversarial_" + short] = adv
        if not only_adversarial_loss:
            gl["features_" + short] = features_loss_lambda * feat
        dl[name] = d_loss
    return {"generator": gl, "discriminator": dl}


def melgan_n_layers(disc):
    """n_layers of a MelGAN Discriminator (its scales have n_layers + 3 convolutions)."""
    return len(disc.model["disc_0"].specs) - 3


# ---------------------------------------------------------------------------------------------------------- loss terms
class Map:
    """A feature map in engine storage: flat fp32 tensor t holding n_seg segments of seg rows x C channels, rows [halo, halo + H) of
    each segment owned.  A half of a map (see half) remembers the map it was cut from (base) and its element offset there (off)."""
    __slots__ = ("t", "n_seg", "seg", "halo", "H", "C", "base", "off")

    def __init__(self, t, n_seg, seg, halo, H, C_, base=None, off=0):
        self.t, self.n_seg, self.seg, self.halo, self.H, self.C = t, int(n_seg), int(seg), int(halo), int(H), int(C_)
        self.base, self.off = (self if base is None else base), off

    @property
    def count(self):
        return self.n_seg * self.H * self.C

    def half(self, i):
        """The map of segment half i (0: the real clips of a joint [real, generated] batch, 1: the generated ones)."""
        n = self.n_seg // 2
        size = n * self.seg * self.C
        return Map(self.t[i * size:(i + 1) * size], n, self.seg, self.halo, self.H, self.C, self.base, self.off + i * size)


class Term:
    """One loss term: adv_scale * sum adv(x) + l1_scale * sum |x - ref| over the owned elements of map x (see include/aero_b200.h,
    aero_gan_term).  dx: the flat gradient storage the backward writes (every element)."""
    __slots__ = ("x", "ref", "dx", "adv", "adv_scale", "l1_scale")

    def __init__(self, x, adv=GAN_NONE, adv_scale=0.0, ref=None, l1_scale=0.0, dx=None):
        self.x, self.adv, self.adv_scale, self.ref, self.l1_scale, self.dx = x, adv, float(adv_scale), ref, float(l1_scale), dx


def discriminator_terms(maps, kinds):
    """Terms of the discriminator loss on the logits of joint [real, generated] passes: maps = one logits Map per scale / period,
    kinds = (adversarial kind on the real half, on the generated half).  Each mean has weight 1 (the reference sums them)."""
    terms = []
    for m in maps:
        for i, kind in enumerate(kinds):
            h = m.half(i)
            terms.append(Term(h, kind, 1.0 / h.count))
    return terms


def generator_terms(fake, real, adv_kind, feat_weight, adversarial=True, features=True, l1_on_logits=False):
    """Terms of the generator losses: fake / real = per scale or period, the list of layer Maps (last: logits) of the generated clips
    and of the real clips.  The logits carry the adversarial mean (weight 1) when `adversarial`; with `features`, every feature layer
    (and the logits when l1_on_logits, as the MPD's fmap includes them) carries mean |fake - real| with weight feat_weight."""
    terms = []
    for fl, rl in zip(fake, real):
        for j, (fm, rm) in enumerate(zip(fl, rl)):
            logits = j == len(fl) - 1
            adv = adversarial and logits
            l1 = features and (l1_on_logits or not logits)
            if adv or l1:
                terms.append(Term(fm, adv_kind if adv else GAN_NONE, 1.0 / fm.count if adv else 0.0, rm if l1 else None,
                                  feat_weight / fm.count if l1 else 0.0))
    return terms


def _table(terms, dev):
    arr = (cabi.GanTerm * len(terms))()
    for k, t in enumerate(terms):
        x = t.x
        arr[k] = cabi.GanTerm(x.t.data_ptr(), t.ref.t.data_ptr() if t.ref is not None else None,
                              t.dx.data_ptr() if t.dx is not None else None, t.adv_scale, t.l1_scale, x.n_seg, x.seg, x.halo,
                              x.H, x.C, t.adv)
    host = torch.empty(C.sizeof(arr), dtype=torch.uint8, pin_memory=True)
    C.memmove(host.data_ptr(), C.addressof(arr), C.sizeof(arr))
    return host.to(dev, non_blocking=True)          # pinned: no host synchronisation; the caching allocator keeps `host` alive


def gan_loss_fwd(terms, lib=None):
    """[n_terms, 2] fp64 on the device: each term's weighted adversarial and L1 sums (aero_gan_loss_fwd, one call)."""
    lib = lib or cabi.load()
    dev = terms[0].x.t.device
    table = _table(terms, dev)
    out = torch.empty(len(terms), 2, dtype=torch.float64, device=dev)
    work = torch.empty(len(terms) * 2 * cabi.GAN_FWD_BLOCKS, dtype=torch.float64, device=dev)
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    cabi.check(lib.aero_gan_loss_fwd(_ptr(table), len(terms), _ptr(out), _ptr(work), st), lib)
    return out


def gan_loss_bwd(terms, lib=None):
    """Write every term's dx (aero_gan_loss_bwd, one call)."""
    lib = lib or cabi.load()
    dev = terms[0].x.t.device
    table = _table(terms, dev)
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    cabi.check(lib.aero_gan_loss_bwd(_ptr(table), len(terms), st), lib)


def _attach_grads(terms, maps):
    """Give every map a term touches one gradient buffer (terms on its halves get slices of it); returns the buffers aligned with
    `maps` (None: no term reads that map, so it gets no gradient)."""
    grads = [None] * len(maps)
    where = {id(m): k for k, m in enumerate(maps)}
    for t in terms:
        k = where[id(t.x.base)]
        if grads[k] is None:
            grads[k] = torch.empty_like(maps[k].t)
        t.dx = grads[k][t.x.off:t.x.off + t.x.t.numel()]
    return grads


# ---------------------------------------------------------------------------------------------------------- the two passes
class _Adversary:
    """One discriminator's part of GanTrainer.step.  Subclasses provide _forward(x, need_input_grad, param_grads) -> (engines, per
    engine list of layer Maps, autograd inputs), and the loss kinds."""

    def __init__(self, disc, sink, features_loss_lambda, adversarial, features):
        self.disc, self.sink = disc, sink
        self.lmbda, self.adversarial, self.features = float(features_loss_lambda), adversarial, features
        self._real = None

    def d_terms(self, maps):
        """Per engine (scale / period), the discriminator-loss terms on the logits of the joint pass; maps: per engine, its layer Maps."""
        return [discriminator_terms([ms[-1]], self.d_kinds) for ms in maps]

    def g_terms(self, maps, real):
        """Per engine, the generator-loss terms of the generated clips' maps against the real clips' maps of the same geometry."""
        w = self.feat_weight(maps)
        return [generator_terms([ms], [rs], self.g_kind, w, self.adversarial, self.features, self.l1_on_logits)
                for ms, rs in zip(maps, real)]

    def discriminator_pass(self, hr, pr):
        """One joint forward over [hr, pr] (pr detached), the discriminator loss, and a backward that writes parameter gradients
        (into sink(name)) and no input gradient.  Keeps the real clips' feature maps for generator_pass.  Returns the loss (0-dim
        fp32 device tensor)."""
        x = torch.cat([hr, pr.detach()], 0)
        engines, maps, _ = self._forward(x, False, True)
        per = self.d_terms(maps)
        grads = [_attach_grads(p, ms) for p, ms in zip(per, maps)]
        terms = [t for p in per for t in p]
        out = gan_loss_fwd(terms)
        gan_loss_bwd(terms)
        for eng, g in zip(engines, grads):
            eng.backward(g, grad_sink=self._sink_for(eng), owned=True)
        self._real = [[m.half(0) for m in ms] for ms in maps]
        return out[:, 0].sum().float()

    def generator_pass(self, pr):
        """One forward of the generated clips pr (a leaf that requires grad), the generator's adversarial and feature-matching losses
        against the kept real feature maps, and a backward that computes the input gradient only.  Returns ({short loss name: 0-dim
        fp32 device tensor}, autograd roots, their gradients): torch.autograd.backward(roots, grads) adds d loss / d pr to pr.grad."""
        engines, maps, inputs = self._forward(pr, True, False)
        per = self.g_terms(maps, self._real)
        self._real = None
        terms = [t for p in per for t in p]
        if not terms:
            return {}, [], []
        grads = [_attach_grads(p, ms) for p, ms in zip(per, maps)]
        out = gan_loss_fwd(terms)
        gan_loss_bwd(terms)
        sums = out.sum(0).float()
        short = DISCRIMINATORS[self.name][1]
        losses = {}
        if self.adversarial:
            losses["adversarial_" + short] = sums[0]
        if self.features:
            losses["features_" + short] = sums[1]
        roots, gs = [], []
        for eng, g, inp in zip(engines, grads, inputs):
            gx, _ = eng.backward(g, owned=True)
            if gx is None:
                continue
            if roots and roots[-1] is inp:              # the MPD's periods all read pr itself: one sum
                gs[-1].add_(gx.view_as(inp))
            else:
                roots.append(inp)
                gs.append(gx.view_as(inp))
        return losses, roots, gs

    def _sink_for(self, eng):
        return None if self.sink is None else (lambda name, pre=self._prefix(eng): self.sink(pre + name))


class MelganAdversary(_Adversary):
    """MelGAN multi-scale discriminator (hinge loss, feature matching on every layer but the logits with weight
    4 / (n_layers + 1) / num_D, reference solver.py:475-520).  Scale i runs on AvgPool1d^i of the input, reflection-padded by 7."""
    name = "msd_melgan"
    d_kinds = (GAN_HINGE_REAL, GAN_HINGE_FAKE)
    g_kind = GAN_HINGE_GEN
    l1_on_logits = False

    def feat_weight(self, maps):
        d = self.disc
        return self.lmbda * (1.0 / d.num_D) * (4.0 / (melgan_n_layers(d) + 1))

    def _prefix(self, eng):
        return self._prefixes[id(eng)]

    def _forward(self, x, need_input_grad, param_grads):
        d = self.disc
        engines, maps, inputs = [], [], []
        self._prefixes = {}
        ctx = torch.enable_grad() if need_input_grad else torch.no_grad()
        with ctx:
            for i, (key, scale) in enumerate(d.model.items()):
                if i:
                    x = d.downsample(x)
                xp = F.pad(x, (7, 7), mode="reflect")
                eng = _DiscEngine(scale)
                eng.param_grads = param_grads
                outs = eng.forward(xp.detach(), need_input_grad)
                N = xp.shape[0]
                maps.append([Map(y.view(-1), N, y.shape[1], 0, y.shape[1], y.shape[2]) for y in outs])
                engines.append(eng)
                inputs.append(xp)
                self._prefixes[id(eng)] = f"model.{key}."
        return engines, maps, inputs


class MpdAdversary(_Adversary):
    """HiFi-GAN multi-period discriminator (LSGAN loss, feature matching on all six maps of every period including the logits, mean
    over them, reference discriminators.py:211-244 and solver.py:580-598)."""
    name = "mpd"
    d_kinds = (GAN_LSGAN_REAL, GAN_LSGAN_FAKE)
    g_kind = GAN_LSGAN_GEN
    l1_on_logits = True

    def feat_weight(self, maps):
        return self.lmbda / sum(len(ms) for ms in maps)

    def _prefix(self, eng):
        return self._prefixes[id(eng)]

    def _forward(self, x, need_input_grad, param_grads):
        d = self.disc
        N, _, T = x.shape
        xf = x.detach().reshape(N, T).contiguous()
        engines, maps, inputs = [], [], []
        self._prefixes = {}
        for i, dp in enumerate(d.discriminators):
            eng = _MpdEngine(dp)
            eng.param_grads = param_grads
            outs = eng.forward(xf, need_input_grad)
            lay = period_layout(T, dp.period)
            maps.append([Map(o, N * dp.period, seg, halo, H, c) for o, (H, seg, halo), c in zip(outs, lay[1:], dp.channels + [1])])
            engines.append(eng)
            inputs.append(x)
            self._prefixes[id(eng)] = f"discriminators.{i}."
        return engines, maps, inputs


ADVERSARIES = {"msd_melgan": MelganAdversary, "mpd": MpdAdversary}
