"""bench.py --config train: BASELINE.json configs[3] -- one training step of aero_4-16_512_64 (generator forward in train mode,
multi-resolution STFT loss, backward, Adam) on 8 synthetic paired clips per GPU, data-parallel over the ranks of one box with a
flat-buffer NCCL gradient all-reduce overlapped with the backward pass (reference: src/solver.py:292-342,602-605, train.py:83,
src/ddp/distrib.py:58-69).

A "step" = forward + loss + backward + all-reduce + optimizer update of one batch.  `value` = audio-seconds of training data per
second, whole job (device-timed, max over ranks); `e2e` adds the H2D copy of the (lr, hr) batch from pinned memory and the D2H
read of the loss every step.  The discriminator half of the reference's step (MelGAN MSD, adversarial + feature losses) is part of
the step when `aero_b200.discriminator` is available (`config.adversarial` says which was measured).
"""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
EXP, BATCH, LR_LEN, SECONDS = "aero_4-16_512_64", 8, 8000, 2.0
GFLOP_FWD = 124.16                      # reference-equivalent forward GFLOP per clip (SURVEY.md 8d); fwd + bwd ~ 3x


def cpu_train_step_times(threads, batch, repeats, warmup):
    """The reference's training step on the host: oracle forward with batch-statistics BatchNorm under torch autograd,
    MR-STFT loss, backward, torch.optim.Adam (what solver.py does with `losses: [stft]`)."""
    from bench import build_model, CONFIGS, SEED
    from oracle import aero_oracle as O
    torch.set_num_threads(threads)
    model = build_model(CONFIGS["4-16"])
    sd = {k: (v.clone().requires_grad_(v.dtype.is_floating_point and "running" not in k)) for k, v in model.state_dict().items()}
    params = [v for v in sd.values() if torch.is_tensor(v) and v.requires_grad]
    opt = torch.optim.Adam(params, lr=3e-4, betas=(0.9, 0.999))
    g = torch.Generator().manual_seed(SEED)
    lr_b = torch.randn(batch, 1, LR_LEN, generator=g)
    hr_b = torch.randn(batch, 1, 4 * LR_LEN, generator=g)
    O.BN_TRAIN = True
    times = []
    try:
        for i in range(warmup + repeats):
            t0 = time.perf_counter()
            opt.zero_grad()
            pr = O.aero_forward(sd, model.geom, lr_b)
            sc, mag = O.mrstft_loss(pr.squeeze(1), hr_b.squeeze(1))
            (sc + mag).backward()
            opt.step()
            if i >= warmup:
                times.append(time.perf_counter() - t0)
    finally:
        O.BN_TRAIN = False
    return times


def main(args):
    sys.path.insert(0, ROOT)
    import bench as B
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if args._cpu_probe:
        th, b, rep, wu = (int(v) for v in args._cpu_probe.split(","))
        os.sched_setaffinity(0, range(os.cpu_count() or 1))
        print(json.dumps(cpu_train_step_times(th, b, rep, wu)), flush=True)
        return
    if args.impl == "reference":
        if rank != 0:
            return
        os.sched_setaffinity(0, range(os.cpu_count() or 1))
        threads = int(os.environ.get("AERO_CPU_THREADS", min(B.physical_cores(), 32)))
        times = cpu_train_step_times(threads, BATCH, args.steps, args.warmup)
        dt = sum(times) / len(times)
        val = BATCH * SECONDS / dt
        print(json.dumps({"impl": "reference", "metric": "audio-seconds/sec training step", "value": val, "unit": "audio-s/s", "n_gpus": args.gpus,
                          "steps": args.steps, "warmup": args.warmup, "ms_per_step": dt * 1e3, "higher_is_better": True, "scaling": "weak",
                          "vs_baseline": None, "dtype": "f32", "data": "synthetic",
                          "config": {"workload": f"{EXP} training step (generator fwd + MR-STFT loss + bwd + Adam), batch {BATCH}", "config_key": "train"},
                          "cpu_baseline": {"value": val, "unit": "audio-s/s", "cores": threads, "kind": "port",
                                           "sample": f"{args.steps} steps of batch {BATCH} after {args.warmup} warm-ups; oracle port under torch autograd + torch.optim.Adam"},
                          "e2e": {"value": val, "unit": "audio-s/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}), flush=True)
        return

    import torch.distributed as dist
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    B.pin_to_gpu_numa(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    from aero_b200 import cabi
    from aero_b200.losses import MultiResolutionSTFTLoss
    from aero_b200.trainer import GanTrainer, GeneratorTrainer
    from aero_b200.discriminator import Discriminator
    lib = cabi.load()
    model = B.build_model(B.CONFIGS["4-16"]).to(dev).train()
    adversarial = not os.environ.get("AERO_TRAIN_NO_GAN")
    env_precision = os.environ.get("AERO_TRAIN_PRECISION")
    train_precision = int(env_precision or "0")
    model.train_precision = train_precision
    if adversarial:
        torch.manual_seed(B.SEED + 1)
        disc = Discriminator(3, 16, 4, 4).to(dev)            # reference conf/experiment/aero_*.yaml melgan_discriminator
        disc.train_precision = train_precision
        trainer = GanTrainer(model, disc, lr=3e-4, betas=(0.9, 0.999))
    else:
        trainer = GeneratorTrainer(model, lr=3e-4, betas=(0.9, 0.999))
    mrstft = MultiResolutionSTFTLoss()
    bsz = args.batch or BATCH
    gen = torch.Generator().manual_seed(B.SEED + rank)
    host_lr = torch.randn(bsz, 1, LR_LEN, generator=gen).pin_memory()
    host_hr = torch.randn(bsz, 1, 4 * LR_LEN, generator=gen).pin_memory()
    lr_d, hr_d = host_lr.to(dev), host_hr.to(dev)

    def loss_fn_for(hr):
        def fn(pr):
            sc, mag = mrstft(pr.squeeze(1), hr.squeeze(1))
            return sc + mag
        return fn

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def one_step(a, b):
        if adversarial:
            out = trainer.step(a, b, mrstft)
            return out["stft"]
        return trainer.step(a, loss_fn_for(b))

    warm = max(args.warmup, 3)
    losses = []
    for _ in range(warm):
        losses.append(one_step(lr_d, hr_d))
    barrier()
    sampler = B.ClockSampler(local)
    if rank == 0:
        sampler.start()
    l0 = lib.aero_launch_count()
    ar0 = trainer.allreduce_bytes
    ms_dev = B.timed_steps(lambda: losses.append(one_step(lr_d, hr_d)), args.steps, barrier)
    launches = lib.aero_launch_count() - l0
    if args.dump_outputs:           # what the last timed step produced: its loss and the parameters it left behind
        sfx = "" if world == 1 else f"_rank{rank}"
        B.dump_outputs(args.dump_outputs, {"loss" + sfx: torch.as_tensor(losses[-1]).reshape(1),
                                           "generator_parameters" + sfx: torch.cat([p.detach().reshape(-1).float() for p in model.parameters()])})
    ar_bytes = (trainer.allreduce_bytes - ar0) / args.steps
    sampler.paused = True
    barrier()
    marks = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
    host_loss = torch.empty((), dtype=torch.float32).pin_memory()
    marks[0].record()
    for i in range(args.steps):
        a, b = host_lr.to(dev, non_blocking=True), host_hr.to(dev, non_blocking=True)
        loss = one_step(a, b)
        host_loss.copy_(loss.float(), non_blocking=True)
        marks[i + 1].record()
        torch.cuda.current_stream().synchronize()
    barrier()
    per_step = [marks[i].elapsed_time(marks[i + 1]) for i in range(args.steps)]
    ms_e2e = B.median(per_step)
    # the other arithmetic mode of the same step, device-timed the same way (exact fp32 <-> TF32 tensor-core GEMMs)
    others = [m_ for m_ in (0, 3, 1) if m_ != train_precision] if env_precision is None else []
    ms_others = {}
    for other in others:
        model.train_precision = other
        if adversarial:
            disc.train_precision = other
        for _ in range(3):
            one_step(lr_d, hr_d)
        barrier()
        ms_others[other] = B.timed_steps(lambda: one_step(lr_d, hr_d), args.steps, barrier)
    model.train_precision = train_precision
    if adversarial:
        disc.train_precision = train_precision
    sampler.stop_flag = True
    from aero_b200.parallel import reduce_max
    ms_dev, ms_e2e = reduce_max(ms_dev, dev), reduce_max(ms_e2e, dev)
    ms_others = {k: reduce_max(v, dev) for k, v in ms_others.items()}
    if rank == 0:
        pk = B.peaks()
        total = bsz * world
        value = total * SECONDS / (ms_dev * 1e-3)
        fp32_peak = 132 * 128 * 2 * 1.98e9 / 1e12                            # SIMT fp32 FMA peak of an H100 SXM at 1980 MHz, TFLOP/s
        step_tflops = bsz * 3 * GFLOP_FWD * 1e9 / (ms_dev * 1e-3) / 1e12
        first, last = float(losses[0]), float(losses[-1])
        line = {"metric": "audio-seconds/sec training step", "value": value, "unit": "audio-s/s", "n_gpus": world, "steps": args.steps,
                "warmup": warm, "ms_per_step": ms_dev, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                "dtype": {0: "f32 (exact-fp32 SIMT tap-GEMMs for forward, dgrad and wgrad; fp64 reduction accumulators)",
                          3: "f32-grade: 3xTF32 tensor-core GEMMs (tensor cores, hi/lo operand split, fp32 accumulate) for the convolutions' forward, dgrad, "
                             "wgrad; fp32 SIMT everything else; fp64 reduction accumulators",
                          1: "tf32 tensor-core GEMMs (wgmma: forward, dgrad, wgrad of the convolutions), fp32 everything else, fp64 reduction "
                             "accumulators"}[train_precision],
                "data": "synthetic",
                "config": {"workload": f"{EXP} training step (G + MelGAN-D + MR-STFT, Adam: reference adversarial config), batch {bsz}/GPU "
                                       f"x 2 s paired white-noise clips (BASELINE configs[3])", "config_key": "train", "global_batch": total,
                           "parallelism": f"data-parallel x{world}: flat-buffer NCCL all-reduce of the generator gradients, overlapped with backward",
                           "adversarial": bool(adversarial), "train_precision": train_precision,
                           "step": ("generator forward (train) + MR-STFT + 3 MelGAN-discriminator forwards + G backward + Adam + D backward + Adam"
                                    if adversarial else "generator forward (train) + MR-STFT + backward + Adam"),
                           "l2": "activations saved for backward (~1 GB/step) exceed the 50 MB L2; no explicit flush"},
                "e2e": {"value": total * SECONDS / (ms_e2e * 1e-3), "unit": "audio-s/s", "ms_per_step": ms_e2e,
                        "statistic": "median of per-step device times (H2D of lr+hr, step, D2H of the loss, one stream sync per step)",
                        "h2d_bytes_per_step": (host_lr.numel() + host_hr.numel()) * 4 * world, "d2h_bytes_per_step": 4 * world},
                "gpu_launches": int(launches), "allreduce_bytes_per_step_per_rank": ar_bytes,
                "loss_first_last": [first, last], "clocks": sampler.summary(),
                "roofline": {"bound": "tensor", "kernel": "whole step (forward + dgrad + wgrad tap-GEMMs dominate)", "achieved": step_tflops,
                             "peak": pk["fp16_tflops"], "unit": "TFLOP/s", "frac": step_tflops / pk["fp16_tflops"],
                             "frac_of_fp32_simt_peak": step_tflops / fp32_peak, "fp32_simt_peak": fp32_peak,
                             "note": "convolution GEMMs: see dtype; LSTM recurrence, attention, normalisation and the grouped discriminator convolutions "
                                     "are fp32 SIMT in every mode; `other_modes` times the same step in the other arithmetic modes", "traffic": None}}
        what = {0: "model.train_precision = 0: exact-fp32 SIMT GEMMs",
                3: "model.train_precision = 3 (3xTF32): every convolution GEMM (forward, dgrad, wgrad) as three TF32 tensor-core products on hi / lo "
                   "operand halves, fp32-grade results; meets the exact mode's gradient-parity bars (tests/test_gpu_train_tc.py)",
                1: "model.train_precision = 1: the convolution GEMMs in plain TF32 on wgmma (what cuDNN does for the reference under PyTorch's "
                   "default allow_tf32); all-gradient deviation from the fp64 reference 6.5e-2, the reference algorithm under PyTorch-default TF32 "
                   "on the same GPU 5.3e-2 (tests/test_gpu_train_tc.py)"}
        if ms_others:
            line["other_modes"] = [{"train_precision": k, "ms_per_step": v, "value": total * SECONDS / (v * 1e-3), "unit": "audio-s/s", "what": what[k]}
                                   for k, v in ms_others.items()]
        if not args.no_cpu_baseline and world == 1:
            os.sched_setaffinity(0, range(os.cpu_count() or 1))
            threads = min(B.physical_cores(), 32)
            cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--config", "train", "--_cpu_probe", f"{threads},4,1,1"]
            import subprocess
            try:
                out = subprocess.run(cmd, capture_output=True, text=True, timeout=600).stdout.strip().splitlines()
                ts = json.loads(out[-1])
            except Exception:
                ts = None
            line["cpu_baseline"] = {"value": (4 * SECONDS / B.median(ts)) if ts else None, "unit": "audio-s/s", "cores": threads, "kind": "port",
                                    "sample": "1 training step of 4 clips (of the 8-clip workload) after 1 warm-up: oracle forward (batch-stat BatchNorm) "
                                              "under torch autograd + MR-STFT loss + torch.optim.Adam"}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()
