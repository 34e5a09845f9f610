"""Scoring a test set: the per-file loop of reference test.py / evaluate.py against evaluate_batch.

Workload (the test set of bench_ragged.py): 64 mono clips, lengths drawn uniformly in 1-8 s at 4 kHz (seeded), targets `hr` of
4x the length, aero_4-16_512_64 (random trained-like weights), engine precision 2.  Two arms, alternated, each starting from an
empty engine and allocator cache:
  (a) reference: per file `model(clip[None])`, `match_signal` to the target length, `get_lsd(hr, pr).item()`;
  (b) `evaluate_batch(model, clips, hrs)`: ragged enhance_batch, match_signal, one fused get_lsd_batch call.
Reports each arm's wall time (whole arm, and the scoring stage alone on precomputed estimates), the device time of the scoring
stage (torch.profiler, CUDA activities, its own pass), the worst relative difference of the per-file LSDs between the arms,
and the card's name and power limit.  Prints one JSON line; writes nothing.
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_ragged import card  # noqa: E402


def device_ms(fn):
    """Device time (kernels and copies) and wall time of one call of `fn` (torch.profiler, its own pass)."""
    from torch.profiler import ProfilerActivity, profile as tprof
    torch.cuda.synchronize()
    with tprof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    dev, kernels = 0.0, {}
    for ev in prof.key_averages():
        us = getattr(ev, "self_device_time_total", None)
        if us is None:
            us = ev.self_cuda_time_total
        if us:
            dev += us / 1e3
            kernels[ev.key[:60]] = round(kernels.get(ev.key[:60], 0.0) + us / 1e3, 3)
    return {"wall_ms": round(wall * 1e3, 2), "device_ms": round(dev, 3),
            "device_ms_by_kernel": dict(sorted(kernels.items(), key=lambda kv: -kv[1])[:8])}


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return min(times), times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py needs a CUDA device")
    from util import SEED, trained_like_
    from aero_b200 import Aero, aero_kwargs
    from aero_b200.enhance import enhance_batch, evaluate_batch, match_signal
    from aero_b200.metrics import get_lsd, get_lsd_batch

    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs("aero_4-16_512_64")).eval()
    m.load_state_dict(trained_like_(m.state_dict()))
    m = m.cuda()
    eng = m._engine()
    assert eng.precision == 2
    gen = torch.Generator().manual_seed(a.seed)
    sr = m.lr_sr
    lengths = [int(sr * (1 + 7 * float(u))) for u in torch.rand(a.clips, generator=gen)]
    clips = [torch.randn(1, n, generator=gen).mul_(0.1).cuda() for n in lengths]
    hrs = [torch.randn(1, 4 * n, generator=gen).mul_(0.1).cuda() for n in lengths]
    audio_s = sum(lengths) / sr

    def reference():
        return [get_lsd(h, match_signal(m(c[None])[0], h.shape[-1])).item() for c, h in zip(clips, hrs)]

    def batched():
        return evaluate_batch(m, clips, hrs, max_batch=a.max_batch)[0].tolist()

    prs = enhance_batch(m, clips, max_batch=a.max_batch)

    def score_reference():
        return [get_lsd(h, match_signal(p, h.shape[-1])).item() for p, h in zip(prs, hrs)]

    def score_batched():
        return get_lsd_batch(hrs, [match_signal(p, h.shape[-1]) for p, h in zip(prs, hrs)]).tolist()

    arms = {"reference_loop": (reference, score_reference), "evaluate_batch": (batched, score_batched)}
    walls = {k: [] for k in arms}
    outs = {}
    for _ in range(a.reps):                               # alternate the arms; each round starts each arm from an empty engine
        for name, (fn, _) in arms.items():
            eng.invalidate()
            eng.use_graph = False
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            outs[name] = fn()                             # warm-up: workspaces, weights, tensor maps
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            walls[name].append(time.perf_counter() - t0)
    res = {}
    for name, (_, score) in arms.items():
        sw, sw_all = timed(score, a.reps)
        res[name] = {"wall_s": round(min(walls[name]), 4), "wall_s_all": [round(t, 4) for t in walls[name]],
                     "score_wall_ms": round(sw * 1e3, 2), "score_wall_ms_all": [round(t * 1e3, 2) for t in sw_all],
                     "score_profile": device_ms(score)}
    worst = max(abs(x - y) / abs(x) for x, y in zip(outs["reference_loop"], outs["evaluate_batch"]))
    name, power = card()
    print(json.dumps({"workload": f"{a.clips} mono clips, 1-8 s at {sr} Hz (seed {a.seed}), hr at 4x, aero_4-16_512_64, "
                                  f"precision 2, max_batch {a.max_batch}", "audio_s": round(audio_s, 2), **res,
                      "speedup_wall": round(res["reference_loop"]["wall_s"] / res["evaluate_batch"]["wall_s"], 2),
                      "speedup_score_wall": round(res["reference_loop"]["score_wall_ms"] / res["evaluate_batch"]["score_wall_ms"], 2),
                      "worst_rel_diff_lsd": worst, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
