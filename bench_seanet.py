"""SEANet generator benchmark (conf/experiment/seanet_4-16.yaml, 2-s clips at 4 kHz -> 16 kHz), one JSON line.

    python bench_seanet.py [--batch 32] [--steps 30] [--warmup 5]     # the CUDA path, precision 2 with sub-lines for 1 and 0
    python bench_seanet.py --impl reference --batch 8                   # the functional oracle on the host (torch CPU)
    python bench_seanet.py --train [--batch 8]                          # one adversarial training step, train_precision 0 and 1

The CUDA path is timed on CUDA-graph replay with device events (median over --steps after --warmup), and the timed outputs
of 2 clips are compared with the oracle.  FLOP and HBM byte counts are computed from the shapes of the launches one forward
issues (recorded through a proxy of the kernel library).  Nothing is written to the tree.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
PEAK = {2: 989e12, 1: 495e12, 0: 67e12}          # H100 SXM data sheet, dense FP16 / TF32 / FP32 (700 W)
HBM = 3.35e12
SEED = 2036


def algorithmic_gflop(m, L):
    """Reference-equivalent convolution GFLOP per clip (2 x MACs of every Conv1d / ConvTranspose1d at the shipped geometry),
    and the count the kernels execute (super-frame convolutions: 3 taps of r*C instead of 2r taps of C)."""
    lev = m.level_lengths(L)
    nlev, nres, ngf, lat = len(m.ratios), m.n_residual_layers, m.ngf, m.latent_space_size
    alg = exe = 2.0 * lev[0] * ngf * m.in_channels * 7 + 2.0 * lev[0] * m.out_channels * ngf * 7
    c = ngf
    for i in range(1, nlev + 1):
        T, r = lev[i - 1], m.ratios[nlev - i]
        rb = 2 * nres * 2.0 * T * c * c * (3 + 1 + 1)            # encoder and decoder residual blocks
        alg += rb + 2 * 2.0 * (T // r) * (2 * c) * c * (2 * r)     # down-conv + transposed conv
        exe += rb + 2 * 2.0 * (T // r) * (2 * c) * c * (3 * r)
        c *= 2
    tail = 2 * 2.0 * lev[nlev] * c * lat * 7
    return (alg + tail) / 1e9, (exe + tail) / 1e9


class _Count:
    """Library proxy that adds up the HBM bytes of each launch from its shapes: activations read and written, weights once."""

    def __init__(self, lib):
        self._lib, self.bytes = lib, 0.0

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def aero_tapgemm_fwd(self, *a):
        p = a[10]._obj
        ea = 2 if p.flags & 2 else 4
        eo = 2 if p.flags & 4 else 4
        self.bytes += p.B * p.T_in * (p.C1 + p.C2) * ea + p.B * p.T * p.N * eo * (2 if a[6] else 1) + \
            p.kt * p.N * (p.C1 + p.C2) * ea
        return self._lib.aero_tapgemm_fwd(*a)

    def aero_reflect_act_fwd(self, x, y, B, T, Cc, xs, ys, halo, act, flags, st):
        self.bytes += B * T * Cc * (2 if flags & 2 else 4) + B * (T + 2 * halo) * Cc * (2 if flags & 4 else 4)
        return self._lib.aero_reflect_act_fwd(x, y, B, T, Cc, xs, ys, halo, act, flags, st)

    def aero_seanet_input_fwd(self, x, f, aff, x0, pp, st):
        p = pp._obj
        self.bytes += 2 * p.B * p.C * p.L_in * 4 + p.B * p.C * (p.L_valid + 2 * p.fill) * 4
        return self._lib.aero_seanet_input_fwd(x, f, aff, x0, pp, st)


def build(batch):
    from aero_b200 import Seanet, seanet_kwargs
    from seanet_util import seanet_recipe_state
    torch.manual_seed(SEED)
    m = Seanet(**seanet_kwargs("seanet_4-16"))
    m.load_state_dict(seanet_recipe_state(m.state_dict()))
    x = torch.randn(batch, 1, 8000, generator=torch.Generator().manual_seed(SEED + 1))
    return m, x


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit not read"


def run_cuda(args):
    from oracle import seanet_oracle as O
    from util import rel_l2
    m, x = build(args.batch)
    m = m.cuda().eval()
    xc = x.cuda()
    eng = m._engine()
    alg, exe = algorithmic_gflop(m, x.shape[-1])
    with torch.no_grad():
        ref = O.seanet_forward(m.cpu().state_dict(), m, x[:2])
    m.cuda()
    lines = {}
    for prec in (2, 1, 0):
        eng.precision = prec
        m.use_cuda_graph(False)
        lib = eng.lib
        eng.lib = cnt = _Count(lib)
        m(xc)
        eng.lib = lib
        m.use_cuda_graph(True)
        for _ in range(args.warmup):
            y = m(xc)
        torch.cuda.synchronize()
        times = []
        for _ in range(args.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            y = m(xc)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) / 1e3)
        t = statistics.median(times)
        flop = exe * 1e9 * args.batch
        t_flop, t_mem = flop / PEAK[prec], cnt.bytes / HBM
        lines[prec] = {
            "precision": prec, "step_ms": round(t * 1e3, 3), "audio_s_per_s": round(args.batch * 2.0 / t, 1),
            "spread_ms": [round(min(times) * 1e3, 3), round(max(times) * 1e3, 3)],
            "rel_l2_vs_oracle_2clips": float(f"{rel_l2(y[:2].cpu(), ref):.3e}"),
            "hbm_gb": round(cnt.bytes / 1e9, 3), "tflops_executed": round(flop / t / 1e12, 1),
            "share_of_peak": round(max(t_flop, t_mem) / t, 3), "bound": "compute" if t_flop > t_mem else "memory"}
    res = {"workload": f"seanet_4-16, {args.batch} x 2 s, CUDA graph", "card": card(),
           "gflop_per_clip_algorithmic": round(alg, 2), "gflop_per_clip_executed": round(exe, 2),
           "audio_s_per_s": lines[2]["audio_s_per_s"], "step_ms": lines[2]["step_ms"], "by_precision": lines}
    print(json.dumps(res))


def run_train(args):
    """One adversarial step at `batch` x 2 s through the autograd route (solver.py with `losses: [stft]` and the MelGAN
    discriminator): generator forward / MR-STFT + adversarial + feature losses / backward / Adam, then the discriminator's step."""
    from aero_b200.discriminator import Discriminator
    from aero_b200.losses import MultiResolutionSTFTLoss
    from aero_b200.optim import FusedAdam
    lines = {}
    for prec in (0, 1):
        gen, lr = build(args.batch)
        gen = gen.cuda().train()
        gen.train_precision = prec
        disc = Discriminator(3, 16, 4, 4).cuda().train()
        disc.train_precision = prec
        opt_g, opt_d = FusedAdam(gen.parameters(), lr=3e-4), FusedAdam(disc.parameters(), lr=3e-4)
        mrstft = MultiResolutionSTFTLoss()
        lr = lr.cuda()
        hr = torch.randn(args.batch, 1, 32000, generator=torch.Generator().manual_seed(SEED + 2)).cuda()

        def step():
            pr = gen(lr)
            sc, mag = mrstft(pr.squeeze(1), hr.squeeze(1))
            fake, real = disc(pr), disc(hr)
            adv = sum(torch.relu(1 - f[-1]).mean() for f in fake)
            feat = sum(torch.nn.functional.l1_loss(a.detach(), b) for fr, ff in zip(real, fake) for a, b in zip(fr[:-1], ff[:-1]))
            opt_g.zero_grad()
            (sc + mag + adv + 100 * feat).backward()
            opt_g.step()
            d_fake, d_real = disc(pr.detach()), disc(hr)
            loss_d = sum(torch.relu(1 + f[-1]).mean() for f in d_fake) + sum(torch.relu(1 - r[-1]).mean() for r in d_real)
            opt_d.zero_grad()
            loss_d.backward()
            opt_d.step()
            return loss_d
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        times = []
        for _ in range(args.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ld = step()
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) / 1e3)
        t = statistics.median(times)
        lines[prec] = {"train_precision": prec, "step_ms": round(t * 1e3, 1), "audio_s_per_s": round(args.batch * 2.0 / t, 1),
                       "finite": bool(torch.isfinite(ld))}
    print(json.dumps({"workload": f"seanet_4-16 adversarial training step, {args.batch} x 2 s", "card": card(), "by_precision": lines}))


def run_reference(args):
    from oracle import seanet_oracle as O
    torch.set_num_threads(args.threads or os.cpu_count())
    m, x = build(args.batch)
    sd = m.state_dict()
    times = []
    with torch.no_grad():
        for i in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            O.seanet_forward(sd, m, x)
            if i >= args.warmup:
                times.append(time.perf_counter() - t0)
    t = statistics.median(times)
    print(json.dumps({"workload": f"seanet_4-16, {args.batch} x 2 s, oracle on the host", "threads": torch.get_num_threads(),
                      "step_ms": round(t * 1e3, 1), "audio_s_per_s": round(args.batch * 2.0 / t, 2)}))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", choices=["cuda", "reference"], default="cuda")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--threads", type=int, default=0)
    ap.add_argument("--train", action="store_true", help="one adversarial training step (default batch 8) instead of inference")
    a = ap.parse_args()
    if a.impl == "cuda" and not torch.cuda.is_available():
        sys.exit("bench_seanet.py: no CUDA device (use --impl reference for the host arm)")
    if a.train:
        if a.batch == 32:
            a.batch = 8
        run_train(a)
    else:
        (run_cuda if a.impl == "cuda" else run_reference)(a)
