"""One optimisation step of the reference's training loop on the CUDA kernels (SURVEY.md section 8e/8f; reference
``src/solver.py:292-342`` ``_run_one_epoch`` body, ``:602-612`` ``_optimize`` / ``_optimize_adversarial``, ``train.py:83``).

``GeneratorTrainer`` owns what the reference spreads over ``Solver`` + ``DistributedDataParallel`` + ``torch.optim.Adam``:

* the generator's gradients live in ONE flat fp32 buffer, laid out in the order the backward pass finishes them (decoder first);
  ``TrainEngine.backward`` writes parameter gradients straight into views of it;
* under ``torch.distributed`` the buffer is summed across ranks with NCCL in a few large pieces, each launched on a side
  stream as soon as the backward pass has finished the layers it covers -- the all-reduce of the decoder's 16 M gradients
  overlaps the encoder's backward (one flat-buffer all-reduce instead of DDP's per-bucket hooks, ``src/ddp/distrib.py:58-69``);
* ``aero_adam_step`` (one launch) applies Adam to every parameter with the 1/world_size averaging folded in.

The plain autograd route (``loss.backward(); optimizer.step()``, DDP-wrapped or not) keeps working -- this class is the fast path
that ``bench.py --config train`` measures.  The generator is ``aero_b200.Aero`` or ``aero_b200.Seanet``.

``GanTrainer(generator, {name: discriminator, ...})`` runs the reference's full adversarial step against ``msd_melgan`` and / or
``mpd`` (DESIGN.md, "The adversarial step"); ``GanTrainer(aero, Discriminator)`` keeps the original single-MelGAN step.
"""
from __future__ import annotations

from collections.abc import Mapping

import torch
import torch.distributed as dist

from .optim import FusedAdam
from .seanet import Seanet, SeanetTrainEngine
from .train_engine import TrainEngine


def _backward_order(model):
    """Parameter names in the order the backward pass completes them: decoder layers (last first), then encoder layers from
    the deepest to the first, then the frequency embedding (shared by the first encoder layer)."""
    names = [n for n, _ in model.named_parameters()]
    depth = model.depth

    def key(n):
        head, idx = n.split(".")[0], n.split(".")[1]
        if head == "decoder":
            return (0, depth - 1 - int(idx))          # decoder.{depth-1} is the last layer of the forward
        if head == "encoder":
            return (1, depth - 1 - int(idx))
        return (2, 0)
    return sorted(names, key=key)


def _seanet_backward_order(model):
    """SEANet's parameter names in the order SeanetTrainEngine.backward completes them: the decoder's top-level modules from the last
    (decoder.{n+1}, the output convolution) to decoder.0, then the encoder's from encoder.{n+1} (the latent projection) to encoder.0."""
    names = [n for n, _ in model.named_parameters()]

    def key(n):
        head, idx = n.split(".")[0], int(n.split(".")[1])
        return (0 if head == "decoder" else 1, -idx)
    return sorted(names, key=key)


class GeneratorTrainer:
    def __init__(self, model, lr=3e-4, betas=(0.9, 0.999), eps=1e-8, pieces=4):
        self.model = model
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.params = dict(model.named_parameters())
        self.order = _seanet_backward_order(model) if isinstance(model, Seanet) else _backward_order(model)
        dev = next(model.parameters()).device
        total = sum(self.params[n].numel() for n in self.order)
        self.flat = torch.zeros(total, device=dev)
        self.views, off = {}, 0
        self.offsets = {}
        for n in self.order:
            p = self.params[n]
            self.views[n] = self.flat[off:off + p.numel()].view(p.shape)
            self.offsets[n] = (off, off + p.numel())
            off += p.numel()
        for n, p in self.params.items():
            p.grad = self.views[n]                      # optimizers / inspection see ordinary .grad tensors
        self.opt = FusedAdam([self.params[n] for n in self.order], lr=lr, betas=betas, eps=eps)
        # all-reduce pieces: boundaries at layer ends, roughly equal bytes
        self.pieces = self._make_pieces(pieces) if self.world > 1 else []
        self.comm_stream = torch.cuda.Stream(device=dev) if self.world > 1 else None
        self.allreduce_bytes = 0

    def _make_pieces(self, n_pieces):
        layer_ends = []
        prev = None
        for n in self.order:
            tag = ".".join(n.split(".")[:2])
            if prev is not None and tag != prev:
                layer_ends.append(self.offsets[n][0])
            prev = tag
        layer_ends.append(self.flat.numel())
        target = self.flat.numel() / n_pieces
        cuts, last = [], 0
        for e in layer_ends:
            if e - last >= target or e == self.flat.numel():
                cuts.append((last, e))
                last = e
        return cuts

    def zero_grad(self):
        self.flat.zero_()

    def _engine(self):
        return SeanetTrainEngine(self.model) if isinstance(self.model, Seanet) else TrainEngine(self.model)

    def _forward(self, eng, lr_batch):
        out = eng.forward(lr_batch)
        return out[0] if isinstance(out, tuple) else out         # Aero's engine also returns the output spectrogram

    def backward(self, engine, d_wave):
        """Run the tape with parameter gradients accumulating into the flat buffer; all-reduce finished pieces while the rest
        of the backward pass runs."""
        done = {"next": 0}
        main = torch.cuda.current_stream()

        def sink(name):
            return self.views[name]

        def progress(ready_upto):
            # ready_upto: flat offset up to which every gradient is final
            while done["next"] < len(self.pieces) and self.pieces[done["next"]][1] <= ready_upto:
                lo, hi = self.pieces[done["next"]]
                self.comm_stream.wait_stream(main)
                with torch.cuda.stream(self.comm_stream):
                    dist.all_reduce(self.flat[lo:hi])
                self.allreduce_bytes += (hi - lo) * 4
                done["next"] += 1
        engine.backward(d_wave, grad_sink=sink, on_layer_done=(self._layer_progress(progress) if self.world > 1 else None))
        if self.world > 1:
            progress(self.flat.numel())
            main.wait_stream(self.comm_stream)

    def _layer_progress(self, progress):
        ends = {}
        for n in self.order:
            ends[".".join(n.split(".")[:2])] = self.offsets[n][1]

        def cb(layer_tag):
            if layer_tag in ends:
                progress(ends[layer_tag])
        return cb

    def step(self, lr_batch, loss_fn):
        """lr_batch [B, C, L]; loss_fn(pr) -> scalar loss of the estimate (built from differentiable ops, e.g.
        aero_b200.losses.MultiResolutionSTFTLoss).  Returns the loss value (0-dim tensor, not synchronised)."""
        model = self.model
        model.train()
        self.zero_grad()
        with torch.cuda.device(lr_batch.device):
            eng = self._engine()
            wave = self._forward(eng, lr_batch)
            pr = wave.detach().requires_grad_(True)
            loss = loss_fn(pr)
            loss.backward()
            self.backward(eng, pr.grad)
            self.opt.step(grad_scale=1.0 / self.world)
        return loss.detach()


class GanTrainer(GeneratorTrainer):
    """The reference's full step with ``adversarial: True`` (``src/solver.py:292-342,428-520,580-612``, ``train.py:83-95``).

    ``GanTrainer(generator, discs, features_loss_lambda=100, only_features_loss=False, only_adversarial_loss=False)``: generator
    ``Aero`` or ``Seanet``; discs ``{name: module}`` keyed and ordered like ``discriminator_models`` -- ``'msd_melgan'``
    (``aero_b200.discriminator.Discriminator``) and / or ``'mpd'`` (``aero_b200.mpd.MultiPeriodDiscriminator``).  ``step`` drives the
    engines directly (``aero_b200.gan``): per discriminator one joint forward over ``[hr, pr.detach()]`` whose backward writes
    parameter gradients only, and one forward of ``pr`` whose backward computes the input gradient only.  One FusedAdam over all
    discriminators' parameters in ``discriminator_models`` order (as ``train.py`` chains them); their gradients live in one flat
    buffer, summed over NCCL once per step under ``torch.distributed``.

    ``GanTrainer(aero, disc)`` with a single MelGAN ``Discriminator`` module is the original step: generator loss = MR-STFT + hinge
    adversarial + 100 x feature matching, then the discriminator's hinge loss on (detached estimate, target), through autograd on the
    discriminator (n_layers: its ``melgan_discriminator.n_layers``)."""

    def __init__(self, model, disc, lr=3e-4, betas=(0.9, 0.999), eps=1e-8, features_loss_lambda=100.0, n_layers=4, pieces=4,
                 only_features_loss=False, only_adversarial_loss=False):
        super().__init__(model, lr=lr, betas=betas, eps=eps, pieces=pieces)
        if isinstance(disc, Mapping):
            self._init_discs(disc, lr, betas, eps, features_loss_lambda, only_features_loss, only_adversarial_loss)
            return
        self.discs = None
        self.disc = disc
        self.lmbda, self.n_layers = features_loss_lambda, n_layers
        dps = list(disc.parameters())
        self.d_flat = torch.zeros(sum(p.numel() for p in dps), device=dps[0].device)
        off = 0
        for p in dps:
            p.grad = self.d_flat[off:off + p.numel()].view(p.shape)
            off += p.numel()
        self.d_opt = FusedAdam(dps, lr=lr, betas=betas, eps=eps)

    def _init_discs(self, discs, lr, betas, eps, lmbda, only_features, only_adversarial):
        from .gan import check_discriminators
        self.discs = check_discriminators(discs)
        self.disc = None
        self.lmbda = float(lmbda)
        self.only_features, self.only_adversarial = bool(only_features), bool(only_adversarial)
        dps = [(name, n, p) for name, d in self.discs.items() for n, p in d.named_parameters()]
        self.d_flat = torch.zeros(sum(p.numel() for _, _, p in dps), device=dps[0][2].device)
        self.d_views, off = {}, 0
        for name, n, p in dps:
            v = self.d_flat[off:off + p.numel()].view(p.shape)
            self.d_views[(name, n)] = v
            p.grad = v
            off += p.numel()
        self.d_opt = FusedAdam([p for _, _, p in dps], lr=lr, betas=betas, eps=eps)

    def generator_losses(self, pr, hr, stft_loss):
        """reference solver.py:430-473,499-520"""
        relu, l1 = torch.nn.functional.relu, torch.nn.functional.l1_loss
        sc, mag = stft_loss(pr.squeeze(1), hr.squeeze(1))
        fake, real = self.disc(pr), self.disc(hr)
        w = (4.0 / (self.n_layers + 1)) / self.disc.num_D
        feat = 0.0
        for i in range(self.disc.num_D):
            for j in range(len(fake[i]) - 1):
                feat = feat + w * l1(fake[i][j], real[i][j].detach())
        adv = sum(relu(1 - s[-1]).mean() for s in fake)
        return {"stft": sc + mag, "adversarial": adv, "features": self.lmbda * feat}

    def discriminator_loss(self, pr, hr):
        """reference solver.py:489-497"""
        relu = torch.nn.functional.relu
        fake, real = self.disc(pr.detach()), self.disc(hr)
        return sum(relu(1 + s[-1]).mean() for s in fake) + sum(relu(1 - s[-1]).mean() for s in real)

    def step(self, lr_batch, hr_batch, stft_loss):
        """One optimisation step of both networks.  With a discriminator mapping: returns the reference's loss mapping
        ``{'generator': {'stft', 'adversarial_melgan', 'features_melgan', 'adversarial_mpd', 'features_mpd'}, 'discriminator':
        {'msd_melgan', 'mpd'}}`` (the keys that apply), values 0-dim device tensors, not synchronised.  stft_loss(pr, hr) -> (sc, mag),
        e.g. aero_b200.losses.MultiResolutionSTFTLoss(); None leaves the MR-STFT term out."""
        if self.discs is not None:
            return self._step_discs(lr_batch, hr_batch, stft_loss)
        model = self.model
        model.train()
        self.zero_grad()
        with torch.cuda.device(lr_batch.device):
            eng = TrainEngine(model)
            wave, _ = eng.forward(lr_batch)
            pr = wave.detach().requires_grad_(True)
            g_losses = self.generator_losses(pr, hr_batch, stft_loss)
            g_total = sum(g_losses.values())
            g_total.backward()
            self.backward(eng, pr.grad)
            self.opt.step(grad_scale=1.0 / self.world)
            # discriminator step (its gradients from the generator's backward above are discarded, as disc_optimizer.zero_grad() does)
            self.d_flat.zero_()
            d_loss = self.discriminator_loss(pr, hr_batch)
            d_loss.backward()
            if self.world > 1:
                dist.all_reduce(self.d_flat)
                self.allreduce_bytes += self.d_flat.numel() * 4
            self.d_opt.step(grad_scale=1.0 / self.world)
        return {k: v.detach() for k, v in g_losses.items()} | {"discriminator": d_loss.detach()}

    def _step_discs(self, lr_batch, hr_batch, stft_loss):
        from .gan import ADVERSARIES
        model = self.model
        model.train()
        self.zero_grad()
        self.d_flat.zero_()
        g_losses, d_losses = {}, {}
        with torch.cuda.device(lr_batch.device):
            eng = self._engine()
            wave = self._forward(eng, lr_batch)
            if wave.shape != hr_batch.shape:
                raise ValueError(f"generator output {tuple(wave.shape)} and target {tuple(hr_batch.shape)} differ in shape")
            pr = wave.detach().requires_grad_(True)
            hr = hr_batch.detach().float().contiguous()
            roots, grads = [], []
            if stft_loss is not None:
                sc, mag = stft_loss(pr.squeeze(1), hr.squeeze(1))
                g_losses["stft"] = sc + mag
                roots.append(g_losses["stft"])
                grads.append(None)
            for name, d in self.discs.items():
                adv = ADVERSARIES[name](d, lambda n, name=name: self.d_views[(name, n)], self.lmbda, not self.only_features,
                                        not self.only_adversarial)
                d_losses[name] = adv.discriminator_pass(hr, pr)
                losses, r, g = adv.generator_pass(pr)
                g_losses.update(losses)
                roots += r
                grads += g
            main = torch.cuda.current_stream()
            if self.world > 1:                 # the discriminators' all-reduce overlaps the generator's backward
                self.comm_stream.wait_stream(main)
                with torch.cuda.stream(self.comm_stream):
                    dist.all_reduce(self.d_flat)
                self.allreduce_bytes += self.d_flat.numel() * 4
            if roots:
                torch.autograd.backward(roots, grads)
            if pr.grad is not None:
                self.backward(eng, pr.grad)
            elif self.world > 1:
                main.wait_stream(self.comm_stream)
            self.opt.step(grad_scale=1.0 / self.world)
            self.d_opt.step(grad_scale=1.0 / self.world)
        return {"generator": {k: v.detach() for k, v in g_losses.items()}, "discriminator": d_losses}
