"""Many clips of different lengths: the per-file loop of reference test.py / evaluate.py against enhance_batch.

Workload: 64 mono clips, lengths drawn uniformly in 1-8 s at 4 kHz (seeded), aero_4-16_512_64 (random trained-like weights),
engine precision 2.  Times (a) the per-file loop `model(clip[None])` as test.py runs it (every file a new shape: eager, no
CUDA graph), (b) `enhance_batch(model, clips)`, (c) the same clips zero-padded into ordinary batches of the same size (a speed
reference only: its results differ).  Each arm starts from an empty engine and allocator cache, so its peak memory is its own.
A separate profiled pass of (b) attributes its device time to kernel families (torch.profiler, CUDA activities) and
compares it with the wall time.  Prints one JSON line with audio-seconds per second, wall time, peak memory and padded-frame
fraction of each arm, the worst per-clip rel-L2 between (a) and (b), the profile, and the card's name and power limit.
Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:                                 # noqa: BLE001
        name, power = torch.cuda.get_device_name(), "unknown"
    return name, power


FAMILIES = (("masked_stats", "masked_stats"), ("gather_rows", "lstm_gathers"), ("frame_mask", "frame_mask"),
            ("lstm", "lstm_recurrence"), ("tapgemm", "tap_gemm"), ("attn", "attention"), ("stft", "stft_istft"),
            ("norm_act", "norm_act"), ("sample_norm", "sample_norm"))


def profile(fn):
    """Device time of one call of `fn` by kernel family (torch.profiler, its own pass), and the wall time of that call."""
    from torch.profiler import ProfilerActivity, profile as tprof
    torch.cuda.synchronize()
    with tprof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    fam = {}
    for ev in prof.key_averages():
        us = getattr(ev, "self_device_time_total", None)     # kernels and copies only: host ops have no self device time
        if us is None:
            us = ev.self_cuda_time_total
        if not us:
            continue
        name = next((f for k, f in FAMILIES if k in ev.key), "copies" if ev.key.startswith(("Memcpy", "Memset")) else "other")
        fam[name] = fam.get(name, 0.0) + us / 1e3
    dev = sum(fam.values())
    return {"wall_ms": round(wall * 1e3, 2), "device_ms": round(dev, 2),
            "device_ms_by_family": {k: round(v, 2) for k, v in sorted(fam.items(), key=lambda kv: -kv[1])}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ragged.py needs a CUDA device")
    from util import SEED, rel_l2, trained_like_
    from aero_b200 import Aero, aero_kwargs
    from aero_b200.enhance import enhance_batch

    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs("aero_4-16_512_64")).eval()
    m.load_state_dict(trained_like_(m.state_dict()))
    m = m.cuda()
    assert m._engine().precision == 2
    gen = torch.Generator().manual_seed(a.seed)
    sr = m.lr_sr
    lengths = [int(sr * (1 + 7 * float(u))) for u in torch.rand(a.clips, generator=gen)]
    clips = [torch.randn(1, n, generator=gen).mul_(0.1).cuda() for n in lengths]
    audio_s = sum(lengths) / sr
    frames = [m.geom.frames(n) for n in lengths]

    eng = m._engine()

    def per_file():
        return [m(c[None])[0] for c in clips]

    def ragged():
        return enhance_batch(m, clips, max_batch=a.max_batch)

    order = sorted(range(len(clips)), key=lambda i: lengths[i])
    padded_batches = []
    for k in range(0, len(order), a.max_batch):
        idx = order[k:k + a.max_batch]
        L = max(lengths[i] for i in idx)
        x = torch.zeros(len(idx), 1, L, device="cuda")
        for j, i in enumerate(idx):
            x[j, :, :lengths[i]] = clips[i]
        padded_batches.append(x)

    def padded():
        return [m(x) for x in padded_batches]

    def pad_fraction(batches):
        tot = sum(len(b) * max(frames[i] for i in b) for b in batches)
        return 1 - sum(frames) / tot

    groups = [order[k:k + a.max_batch] for k in range(0, len(order), a.max_batch)]
    res = {}
    outs = {}
    for name, fn, pf in (("per_file", per_file, 0.0), ("enhance_batch", ragged, pad_fraction(groups)),
                         ("padded_batch", padded, pad_fraction(groups))):
        eng.invalidate()                               # no workspace set of an earlier arm stays allocated
        eng.use_graph = name == "padded_batch"         # per-file: each file is a new shape once (eager); ragged: always eager
        outs[name] = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        outs[name] = fn()                              # warm-up: workspaces, weights, tensor maps
        fn()
        torch.cuda.synchronize()
        times = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        wall = min(times)
        res[name] = {"wall_s": round(wall, 4), "wall_s_all": [round(t, 4) for t in times],
                     "audio_s_per_s": round(audio_s / wall, 1), "peak_mem_mb": round(torch.cuda.max_memory_allocated() / 2 ** 20, 1),
                     "padded_frame_fraction": round(pf, 4)}
    outs.pop("padded_batch")
    worst = max(rel_l2(x.cpu(), y.cpu()) for x, y in zip(outs["per_file"], outs["enhance_batch"]))
    res["enhance_batch_profile"] = profile(ragged)
    name, power = card()
    print(json.dumps({"workload": f"{a.clips} mono clips, 1-8 s at {sr} Hz (seed {a.seed}), aero_4-16_512_64, precision 2, "
                                  f"max_batch {a.max_batch}", "audio_s": round(audio_s, 2), **res,
                      "speedup_enhance_batch_vs_per_file": round(res["per_file"]["wall_s"] / res["enhance_batch"]["wall_s"], 2),
                      "worst_rel_l2_per_file_vs_enhance_batch": worst, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
