"""The adversarial training step of aero_b200.trainer.GanTrainer with a discriminator mapping, against the plain autograd route, one
JSON line.

    python bench_gan.py [--batch 8] [--steps 10] [--warmup 2] [--quick]

For aero_4-16_512_64 and seanet_4-16 (4 kHz -> 16 kHz, --batch x 2 s clips), each against [msd_melgan, mpd] and [msd_melgan]
(the configs' discriminators: MelGAN 3 x 16 x 4 x 4, MPD hidden 32 with periods 2, 3, 5, 7, 11), in train_precision 1 and 0:
  * step time (device events, median over --steps after --warmup) of GanTrainer.step and of the autograd route (generator forward,
    aero_b200.gan.autograd_losses with MR-STFT, backward and FusedAdam for the generator, then for the discriminators -- the
    structure of bench_mpd.adversarial_step), the two alternated step by step in the same run;
  * peak memory of one step of each;
  * the discriminators' convolution GEMM FLOP per step on both routes, from shapes (weight and data gradients counted as one forward
    each; the MPD's executed FLOP of aero_b200.mpd.period_flops);
  * the loss kernels (aero_gan_loss_fwd / _bwd) of one GanTrainer step: time from device events around each call, the bytes their
    contract moves, and that rate against the H100 SXM's 3.35 TB/s.
The card name and power limit are read in the same run.  Nothing is written to the tree.  --quick: one configuration, 3 steps.
"""
import argparse
import json
import statistics

import torch

from bench_mpd import SEED, card

LR_SR, HR_SR, HBM_TBS = 4000, 16000, 3.35


def _generator(name):
    from aero_b200 import Aero, Seanet, aero_kwargs, seanet_kwargs
    torch.manual_seed(SEED)
    return Aero(**aero_kwargs(name)) if name.startswith("aero") else Seanet(**seanet_kwargs(name))


def _discs(names):
    from aero_b200 import load_experiment
    from aero_b200.gan import build_discriminators
    torch.manual_seed(SEED + 1)
    return build_discriminators(load_experiment("aero_4-16_512_64_mpd", discriminator_models=list(names)))


def melgan_flops(disc, B, L):
    """Forward FLOP of the MelGAN discriminator's convolutions on B clips of L samples."""
    total, T = 0, L
    for i, (_, scale) in enumerate(disc.model.items()):
        if i:
            T = (T + 2 - 4) // 2 + 1                     # AvgPool1d(4, 2, 1)
        t = T + 14
        for _, cin, cout, k, s, p, g, _ in scale.specs:
            t = (t + 2 * p - k) // s + 1
            total += 2 * B * t * cout * (cin // g) * k
    return total


def disc_flops(discs, B, L):
    """{route: GFLOP per step} of the discriminators' convolution GEMMs.  Autograd: MelGAN D(pr.detach()), D(hr), D(pr) forward, with
    weight and data gradients through all three; MPD two joint passes over 2B clips, each with both gradients.  GanTrainer: one joint
    forward over 2B clips with both gradients, then a forward of the B generated clips with its data gradient."""
    from aero_b200.mpd import period_flops
    auto = new = 0
    for name, d in discs.items():
        if name == "msd_melgan":
            f = melgan_flops(d, B, L)
            auto += 9 * f
            new += 6 * f + 2 * f
        else:
            f = sum(period_flops(B, L, dp.period, dp.channels)[0] for dp in d.discriminators)
            auto += 2 * 3 * 2 * f
            new += 3 * 2 * f + 2 * f
    return {"autograd": round(auto / 1e9, 1), "gan_trainer": round(new / 1e9, 1), "ratio": round(new / auto, 3)}


def autograd_step(gen, discs, lr_b, hr, mrstft):
    from aero_b200.gan import autograd_losses
    from aero_b200.optim import FusedAdam
    opt_g = FusedAdam(gen.parameters(), lr=3e-4, betas=(0.8, 0.99))
    opt_d = FusedAdam([p for d in discs.values() for p in d.parameters()], lr=3e-4, betas=(0.8, 0.99))

    def step():
        pr = gen(lr_b)
        losses = autograd_losses(pr, hr, discs, mrstft)
        opt_g.zero_grad()
        sum(losses["generator"].values()).backward()
        opt_g.step()
        opt_d.zero_grad()
        sum(losses["discriminator"].values()).backward()
        opt_d.step()
        return losses
    return step


def loss_kernel_rate(tr, lr_b, hr, mrstft):
    """Device time and contract bytes of every aero_gan_loss_fwd / _bwd call of one step."""
    from aero_b200 import gan as G
    calls = []
    fwd, bwd = G.gan_loss_fwd, G.gan_loss_bwd

    def nbytes(terms, backward):
        n = 0
        for t in terms:
            n += 4 * t.x.count * (2 if t.ref is not None else 1)
            if backward:
                n += 4 * t.x.t.numel()
        return n

    def timed(fn, backward):
        def call(terms, lib=None):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn(terms, lib)
            e1.record()
            calls.append((e0, e1, nbytes(terms, backward)))
            return r
        return call
    G.gan_loss_fwd, G.gan_loss_bwd = timed(fwd, False), timed(bwd, True)
    try:
        tr.step(lr_b, hr, mrstft)
        torch.cuda.synchronize()
    finally:
        G.gan_loss_fwd, G.gan_loss_bwd = fwd, bwd
    ms = sum(a.elapsed_time(b) for a, b, _ in calls)
    by = sum(n for _, _, n in calls)
    return {"calls": len(calls), "ms": round(ms, 3), "mbytes": round(by / 1e6, 1), "tb_per_s": round(by / ms / 1e9, 3),
            "of_3.35_tb_per_s": round(by / ms / 1e9 / HBM_TBS, 3)}


def run(gname, dnames, precision, B, steps, warmup):
    from aero_b200.losses import MultiResolutionSTFTLoss
    from aero_b200.trainer import GanTrainer
    L = 2 * HR_SR
    g = torch.Generator().manual_seed(SEED + 3)
    lr_b = (torch.randn(B, 1, 2 * LR_SR, generator=g) * 0.1).cuda()
    hr = (torch.randn(B, 1, L, generator=g) * 0.1).cuda()
    mrstft = MultiResolutionSTFTLoss()
    nets = {}
    for route in ("gan_trainer", "autograd"):
        gen, discs = _generator(gname).cuda().train(), {k: v.cuda() for k, v in _discs(dnames).items()}
        for m in [gen, *discs.values()]:
            m.train_precision = precision
        nets[route] = (gen, discs)
    tr = GanTrainer(*nets["gan_trainer"], lr=3e-4, betas=(0.8, 0.99))
    fns = {"gan_trainer": lambda: tr.step(lr_b, hr, mrstft), "autograd": autograd_step(*nets["autograd"], lr_b, hr, mrstft)}
    res = {"generator": gname, "discriminators": list(dnames), "train_precision": precision, "batch": B,
           "disc_gemm_gflop_per_step": disc_flops(nets["autograd"][1], B, L)}
    for name, fn in fns.items():                               # warm-up, then the peak memory of one step
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        out = fn()
        torch.cuda.synchronize()
        res.setdefault(name, {})["peak_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
        res[name]["finite"] = all(bool(torch.isfinite(v)) for side in out.values() for v in side.values())
    times = {k: [] for k in fns}
    for _ in range(steps):                                     # alternated
        for name, fn in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1))
    for name, v in times.items():
        res[name]["ms"] = round(statistics.median(v), 2)
        res[name]["ms_min_max"] = [round(min(v), 2), round(max(v), 2)]
    res["speedup"] = round(res["autograd"]["ms"] / res["gan_trainer"]["ms"], 3)
    res["loss_kernels"] = loss_kernel_rate(tr, lr_b, hr, mrstft)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--quick", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gan.py measures the CUDA path: no GPU")
    configs = [(g, d, p) for p in (1, 0) for g in ("aero_4-16_512_64", "seanet_4-16") for d in (("msd_melgan", "mpd"), ("msd_melgan",))]
    if args.quick:
        configs, args.steps = configs[:1], 3
    out = {"workload": f"adversarial training step, {args.batch} x 2 s at 16 kHz (4 kHz input): GanTrainer.step vs the autograd route",
           "card": card(), "results": []}
    for g, d, p in configs:
        out["results"].append(run(g, d, p, args.batch, args.steps, args.warmup))
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
