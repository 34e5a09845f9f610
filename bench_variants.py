"""The AERO variants of `act_func` and `spec_upsample` next to the default model, and the device resampler, one JSON line.

    python bench_variants.py [--batch 32] [--gan-batch 8] [--rounds 20] [--warmup 3]

All at 4 kHz -> 16 kHz with 2 s clips, every timing the median of --rounds device-event timings, the variants alternated round by
round in the same run so that they see the same clocks and neighbours:
  * inference: the CUDA-graph replay of one forward at precision 2 (the default engine) on --batch clips, for the default model
    (aero_4-16_512_64, Snake), `act_func` relu and gelu, and `spec_upsample=False` (aero_4-16_512_64_sinc: input already at 16 kHz);
  * `aero_b200.resample` of a --batch x 2 s batch from 4 to 16 kHz;
  * one GanTrainer step against [msd_melgan] (MelGAN 3 x 16 x 4 x 4) at train_precision 1 (TF32) on --gan-batch clips, for the
    default model, relu and sinc.
The variants run the same kernels as the default model (a different DConv activation, or the input STFT at hop 64 / window 512),
so their times are expected within noise of it.  The card name and power limit are read in the same run.  Nothing is written to
the tree.
"""
import argparse
import json
import statistics

import torch

from bench_mpd import SEED, card

LR_SR, HR_SR, SECONDS = 4000, 16000, 2
VARIANTS = {"default": ("aero_4-16_512_64", {}), "relu": ("aero_4-16_512_64_relu", {}), "gelu": ("aero_4-16_512_64", {"act_func": "gelu"}),
            "sinc": ("aero_4-16_512_64_sinc", {})}


def _model(name):
    from aero_b200 import Aero, aero_kwargs
    exp, over = VARIANTS[name]
    torch.manual_seed(SEED)
    return Aero(**dict(aero_kwargs(exp), **over)).cuda()


def _input(model, B, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    L = SECONDS * (model.hr_sr if not model.spec_upsample else model.lr_sr)
    return torch.randn(B, 1, L, device="cuda", generator=g)


def _time(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def alternate(fns, rounds, warmup):
    """{name: median ms} of `fns`, called in turn, `warmup` untimed rounds first."""
    for _ in range(warmup):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            ms[k].append(_time(fn))
    return {k: round(statistics.median(v), 3) for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--gan-batch", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_variants.py measures on a CUDA device; none is visible")
    from aero_b200 import resample
    from aero_b200.discriminator import Discriminator
    from aero_b200.losses import MultiResolutionSTFTLoss
    from aero_b200.trainer import GanTrainer
    result = {"card": card(), "batch": args.batch, "gan_batch": args.gan_batch, "clip_s": SECONDS, "rounds": args.rounds}

    # inference on graph replay, precision 2
    fwd = {}
    for name in VARIANTS:
        m = _model(name).eval()
        m.use_cuda_graph(True)
        assert m._engine().precision == 2
        x = _input(m, args.batch, 1)

        def run(m=m, x=x):
            with torch.no_grad():
                m(x)
        fwd[name] = run
    result["forward_ms"] = alternate(fwd, args.rounds, args.warmup)
    fwd.clear()
    torch.cuda.empty_cache()

    # the resampler, 4 -> 16 kHz
    lr = torch.randn(args.batch, 1, SECONDS * LR_SR, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    rs = alternate({"resample": lambda: resample(lr, LR_SR, HR_SR)}, args.rounds * 5, args.warmup)["resample"]
    moved = lr.numel() * 4 * (1 + HR_SR // LR_SR)
    result["resample_ms"] = rs
    result["resample_gbs"] = round(moved / (rs * 1e-3) / 1e9, 1)     # input read once and output written once, over the time

    # one adversarial step against [msd_melgan], train_precision 1
    mrstft = MultiResolutionSTFTLoss()
    steps = {}
    for name in ("default", "relu", "sinc"):
        gen = _model(name)
        gen.train_precision = 1
        torch.manual_seed(SEED + 1)
        disc = Discriminator(3, 16, 4, 4).cuda()
        disc.train_precision = 1
        tr = GanTrainer(gen, {"msd_melgan": disc}, lr=3e-4, betas=(0.8, 0.99))
        x = _input(gen, args.gan_batch, 3)
        hr = 0.1 * torch.randn(args.gan_batch, 1, SECONDS * HR_SR, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
        steps[name] = lambda tr=tr, x=x, hr=hr: tr.step(x, hr, mrstft)
    result["gan_step_ms"] = alternate(steps, max(3, args.rounds // 2), args.warmup)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
