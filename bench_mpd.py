"""HiFi-GAN multi-period discriminator benchmark (aero_b200.mpd, default MultiPeriodDiscriminator), one JSON line.

    python bench_mpd.py [--batch 8] [--steps 20] [--warmup 3] [--no-step]

Times, with device events (median over --steps after --warmup), at --batch x 2 s / 16 kHz:
  * the reference's MPD work per training step (solver.py:580-590): mpd(hr, pr.detach()) and mpd(hr, pr), each with a backward
    (parameter gradients, and the input gradient of pr for the second), for train_precision 0 and 1;
  * the same on the functional oracle (oracle/mpd_oracle.py) on cuDNN in fp32 and TF32 (PyTorch's default for convolutions);
  * a per-layer breakdown of one period in TF32 mode against the oracle on cuDNN TF32 (forward + backward of each convolution);
  * one [msd_melgan, mpd] adversarial step with the AERO generator (aero_4-16_512_64, 4 kHz -> 16 kHz), train_precision 1
    (skipped with --no-step).
Also reported: executed vs algorithmic GFLOP of the forward, and the peak memory of each timed configuration.  The card name and
its power limit are read in the same run.  Nothing is written to the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
SEED = 2036


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit not read"


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    times = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return round(statistics.median(times), 2), round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)


def mpd_work(forward, params, hr, pr):
    """The MPD part of one reference training step: discriminator loss on (hr, pr.detach()), generator losses on (hr, pr)."""
    def step():
        for p in params:
            p.grad = None
        y_r, y_g, _, _ = forward(hr, pr.detach())
        sum(torch.mean((1 - r) ** 2) + torch.mean(g ** 2) for r, g in zip(y_r, y_g)).backward()
        y_r, y_g, f_r, f_g = forward(hr, pr)
        feat = [torch.mean(torch.abs(a - b)) for dr, dg in zip(f_r, f_g) for a, b in zip(dr, dg)]
        (sum(torch.mean((1 - g) ** 2) for g in y_g) + 2 * sum(feat) / len(feat)).backward()
    return step


def per_layer(d, sd, x, steps, warmup):
    """Forward + backward of each convolution of period d.period in TF32 mode (the engine's per-layer events) and on cuDNN TF32."""
    import torch.nn.functional as F
    from oracle import mpd_oracle as O
    rows = {}
    d.train_precision = 1
    per = {}
    try:
        for it in range(warmup + steps):
            d.layer_events = []
            logits, fmap = d(x)
            (logits.square().mean() + sum(f.abs().mean() for f in fmap[:-1])).backward()
            torch.cuda.synchronize()
            if it >= warmup:
                for name, kind, a, b in d.layer_events:
                    per.setdefault((name, kind), []).append(a.elapsed_time(b))
    finally:
        del d.layer_events
    names = [f"convs.{j}" for j in range(5)] + ["conv_post"]
    for (name, kind), v in per.items():
        rows.setdefault(name, {})[f"cuda_tf32_{kind}_ms"] = round(statistics.median(v), 3)
    # cuDNN TF32: each conv2d forward and backward on the oracle's activations
    torch.backends.cudnn.allow_tf32 = True
    p = d.period
    T = x.shape[-1]
    h = F.pad(x, (0, (-T) % p), mode="reflect").reshape(x.shape[0], 1, -1, p) if T % p else x.reshape(x.shape[0], 1, -1, p)
    for j in range(6):
        key = names[j]
        w = torch._weight_norm(sd[key + ".weight_v"], sd[key + ".weight_g"], 0).detach().requires_grad_(True)
        b = sd[key + ".bias"].detach().requires_grad_(True)
        hin = h.detach().requires_grad_(True)
        kw = dict(stride=(3, 1) if j < 4 else 1, padding=(2, 0) if j < 5 else (1, 0))
        out = F.conv2d(hin, w, b, **kw)
        gout = torch.randn_like(out)

        def fwd():
            F.conv2d(hin, w, b, **kw)

        def fb():
            torch.autograd.grad(F.conv2d(hin, w, b, **kw), (hin, w, b), gout)
        tf, _ = timed(fwd, steps, warmup)
        tfb, _ = timed(fb, steps, warmup)
        rows[names[j]].update(cudnn_tf32_fwd_ms=tf, cudnn_tf32_bwd_ms=round(tfb - tf, 3))
        h = F.leaky_relu(out, O.SLOPE).detach()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-step", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mpd.py measures the CUDA path: no GPU")
    from aero_b200.mpd import MultiPeriodDiscriminator, period_flops
    from oracle import mpd_oracle as O
    torch.manual_seed(SEED)
    d = MultiPeriodDiscriminator().cuda()
    B, L = args.batch, 32000
    gen = torch.Generator().manual_seed(SEED + 2)
    hr = torch.randn(B, 1, L, generator=gen).cuda() * 0.1
    pr = (torch.randn(B, 1, L, generator=gen).cuda() * 0.1).requires_grad_(True)
    ex = al = 0
    for dp in d.discriminators:
        e, a = period_flops(B, L, dp.period, dp.channels)
        ex, al = ex + e, al + a
    res = {"workload": f"MultiPeriodDiscriminator(hidden=32, periods=[2,3,5,7,11]), {B} x 2 s at 16 kHz: "
                       "mpd(hr, pr.detach()) + mpd(hr, pr), each with its backward",
           "card": card(),
           "forward_gflop_per_clip": {"algorithmic": round(al / B / 1e9, 2), "executed": round(ex / B / 1e9, 2),
                                      "ratio": round(ex / al, 3)},
           "reference_step_tflop": {"forward": round(4 * al / 1e12, 2), "with_backward_approx": round(12 * al / 1e12, 2)}}
    params = list(d.parameters())
    cuda = {}
    for prec in (0, 1):
        d.train_precision = prec
        ms, gb = timed(mpd_work(d, params, hr, pr), args.steps, args.warmup)
        cuda[prec] = {"ms": ms, "peak_gib": gb}
    res["cuda"] = cuda
    names = [n for n, _ in d.named_parameters()]
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in d.state_dict().items()}
    periods = [dp.period for dp in d.discriminators]
    oracle = {}
    old = torch.backends.cudnn.allow_tf32
    try:
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            ms, gb = timed(mpd_work(lambda a, b: O.mpd_forward(sd, periods, a, b), [sd[n] for n in names], hr, pr), args.steps,
                           args.warmup)
            oracle["tf32" if tf32 else "fp32"] = {"ms": ms, "peak_gib": gb}
    finally:
        torch.backends.cudnn.allow_tf32 = old
    res["oracle_cudnn"] = oracle
    res["tf32_speedup_over_cudnn_tf32"] = round(oracle["tf32"]["ms"] / cuda[1]["ms"], 3)
    x2 = torch.cat([hr, pr.detach()], 0)
    dsd = {k[len("discriminators.4."):]: v for k, v in sd.items() if k.startswith("discriminators.4.")}
    try:
        res["per_layer_period_11"] = per_layer(d.discriminators[4], dsd, x2, max(args.steps // 2, 3), args.warmup)
    finally:
        torch.backends.cudnn.allow_tf32 = old
    if not args.no_step:
        res["adversarial_step"] = adversarial_step(d, B, args)
    print(json.dumps(res))


def adversarial_step(mpd, B, args):
    """One [msd_melgan, mpd] step (solver.py:292-342 with losses [stft], 475-520, 580-598): generator forward, MR-STFT + both
    adversaries' losses, backward and FusedAdam; then both discriminators' losses, backward and FusedAdam.  train_precision 1."""
    from aero_b200 import Aero, aero_kwargs
    from aero_b200.discriminator import Discriminator
    from aero_b200.losses import MultiResolutionSTFTLoss
    from aero_b200.optim import FusedAdam
    torch.manual_seed(SEED)
    gen = Aero(**aero_kwargs("aero_4-16_512_64")).cuda().train()
    msd = Discriminator(3, 16, 4, 4).cuda()
    for m in (gen, msd, mpd):
        m.train_precision = 1
    opt_g = FusedAdam(gen.parameters(), lr=3e-4, betas=(0.8, 0.99))
    opt_d = FusedAdam(list(msd.parameters()) + list(mpd.parameters()), lr=3e-4, betas=(0.8, 0.99))
    mrstft = MultiResolutionSTFTLoss()
    g = torch.Generator().manual_seed(SEED + 3)
    lr, hr = torch.randn(B, 1, 8000, generator=g).cuda() * 0.1, torch.randn(B, 1, 32000, generator=g).cuda() * 0.1
    w = (1.0 / 3) * (4.0 / 5)
    out = {}

    def step():
        pr = gen(lr)
        sc, mag = mrstft(pr.squeeze(1), hr.squeeze(1))
        fake, real = msd(pr), msd(hr)
        loss_g = sc + mag + sum(torch.relu(1 - f[-1]).mean() for f in fake)
        loss_g = loss_g + 100 * w * sum(torch.abs(b - a.detach()).mean() for fr, ff in zip(real, fake) for a, b in zip(fr[:-1], ff[:-1]))
        y_r, y_g, f_r, f_g = mpd(hr, pr)
        feat = [torch.mean(torch.abs(a - b)) for dr, dg in zip(f_r, f_g) for a, b in zip(dr, dg)]
        loss_g = loss_g + sum(torch.mean((1 - y) ** 2) for y in y_g) + 100 * sum(feat) / len(feat)
        opt_g.zero_grad()
        loss_g.backward()
        opt_g.step()
        d_fake, d_real = msd(pr.detach()), msd(hr)
        loss_d = sum(torch.relu(1 + f[-1]).mean() for f in d_fake) + sum(torch.relu(1 - r[-1]).mean() for r in d_real)
        y_r, y_g, _, _ = mpd(hr, pr.detach())
        loss_d = loss_d + sum(torch.mean((1 - r) ** 2) + torch.mean(f ** 2) for r, f in zip(y_r, y_g))
        opt_d.zero_grad()
        loss_d.backward()
        opt_d.step()
        out["finite"] = bool(torch.isfinite(loss_g)) and bool(torch.isfinite(loss_d))
    ms, gb = timed(step, max(args.steps // 2, 3), args.warmup)
    return {"generator": "aero_4-16_512_64", "train_precision": 1, "ms": ms, "peak_gib": gb, "finite": out["finite"]}


if __name__ == "__main__":
    main()
