"""Many clips of different lengths through SEANet: the per-file loop of reference test.py / evaluate.py against enhance_batch.

Workload: the test set of bench_ragged.py (64 mono clips, lengths drawn uniformly in 1-8 s at 4 kHz, seed 0), seanet_4-16
(recipe weights of tests/seanet_util.py), engine precision 2, max_batch 32.  Times (a) the per-file loop `model(clip[None])`
(every file a new shape: eager, no CUDA graph), (b) `enhance_batch(model, clips)`, (c) the same clips zero-padded into
ordinary batches of the same size on CUDA-graph replay (a speed reference only: its results differ).  Each arm starts from an
empty engine and allocator cache, so its peak memory is its own; wall times are the best of --reps.  A separate profiled pass
of (a) and of (b) attributes their device time to kernel families (torch.profiler, CUDA activities) and compares it with the
wall time.  Prints one JSON line with audio-seconds per second, wall time, peak memory and padded-frame fraction of each arm,
the worst per-clip difference between (a) and (b), the profiles, and the card's name and power limit.  Writes nothing.
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

FAMILIES = (("tapgemm", "tap_gemm"), ("reflect_act", "reflect_act"), ("seanet_std", "input_stage"),
            ("seanet_resample", "input_stage"), ("frame_mask", "frame_mask"))


def profile(fn):
    """Device time of one call of `fn` by kernel family and its kernel count (torch.profiler, its own pass), and the wall time
    of that call."""
    from torch.profiler import ProfilerActivity, profile as tprof
    torch.cuda.synchronize()
    with tprof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    from torch.autograd import DeviceType
    fam, kernels = {}, 0
    for ev in prof.key_averages():
        if ev.device_type != DeviceType.CUDA:
            continue                                         # a host op also carries the device time of the kernels it launched
        us = getattr(ev, "self_device_time_total", None)
        if us is None:
            us = ev.self_cuda_time_total
        if not us:
            continue
        copy = ev.key.startswith(("Memcpy", "Memset"))
        name = next((f for k, f in FAMILIES if k in ev.key), "copies" if copy else "other")
        fam[name] = fam.get(name, 0.0) + us / 1e3
        kernels += 0 if copy else ev.count
    dev = sum(fam.values())
    return {"wall_ms": round(wall * 1e3, 2), "device_ms": round(dev, 2), "kernels": kernels,
            "device_ms_by_family": {k: round(v, 2) for k, v in sorted(fam.items(), key=lambda kv: -kv[1])}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ragged_seanet.py needs a CUDA device")
    from util import SEED, rel_l2
    from seanet_util import seanet_recipe_state
    from aero_b200 import Seanet, seanet_kwargs
    from aero_b200.enhance import enhance_batch

    torch.manual_seed(SEED)
    m = Seanet(**seanet_kwargs("seanet_4-16"))
    m.load_state_dict(seanet_recipe_state(m.state_dict()))
    m = m.cuda().eval()
    eng = m._engine()
    assert eng.precision == 2
    gen = torch.Generator().manual_seed(a.seed)
    sr = m.lr_sr
    lengths = [int(sr * (1 + 7 * float(u))) for u in torch.rand(a.clips, generator=gen)]
    clips = [torch.randn(1, n, generator=gen).mul_(0.1).cuda() for n in lengths]
    audio_s = sum(lengths) / sr
    frames = [m.level_lengths(n)[0] for n in lengths]

    def per_file():
        return [m(c[None])[0] for c in clips]

    def ragged():
        return enhance_batch(m, clips, max_batch=a.max_batch)

    order = sorted(range(len(clips)), key=lambda i: lengths[i])
    groups = [order[k:k + a.max_batch] for k in range(0, len(order), a.max_batch)]
    padded_batches = []
    for idx in groups:
        x = torch.zeros(len(idx), 1, max(lengths[i] for i in idx), device="cuda")
        for j, i in enumerate(idx):
            x[j, :, :lengths[i]] = clips[i]
        padded_batches.append(x)

    def padded():
        return [m(x) for x in padded_batches]

    # frames of the level-0 activations that are padding (each batch is sized by its longest clip)
    pad_fraction = 1 - sum(frames) / sum(len(b) * max(frames[i] for i in b) for b in groups)
    res, outs = {}, {}
    for name, fn, pf in (("per_file", per_file, 0.0), ("enhance_batch", ragged, pad_fraction), ("padded_batch", padded, pad_fraction)):
        eng.invalidate()                               # no workspace set of an earlier arm stays allocated
        eng.use_graph = name == "padded_batch"         # per-file: each file is a new shape once (eager); ragged: always eager
        outs[name] = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        outs[name] = fn()                              # warm-up: workspaces, weights, tensor maps, graph capture
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
    diffs = [rel_l2(x.cpu(), y.cpu()) for x, y in zip(outs["per_file"], outs["enhance_batch"])]
    identical = all(torch.equal(x, y) for x, y in zip(outs["per_file"], outs["enhance_batch"]))
    eng.invalidate()
    eng.use_graph = False
    res["per_file_profile"] = profile(per_file)
    res["enhance_batch_profile"] = profile(ragged)
    name, power = card()
    print(json.dumps({"workload": f"{a.clips} mono clips, 1-8 s at {sr} Hz (seed {a.seed}), seanet_4-16, precision 2, "
                                  f"max_batch {a.max_batch}", "audio_s": round(audio_s, 2), **res,
                      "speedup_enhance_batch_vs_per_file": round(res["per_file"]["wall_s"] / res["enhance_batch"]["wall_s"], 2),
                      "worst_rel_l2_per_file_vs_enhance_batch": max(diffs), "bit_identical_per_file_vs_enhance_batch": identical,
                      "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
