#!/usr/bin/env python
"""Run one hot-path kernel shape in isolation (for ncu captures and CUDA-event timing).

    python tools/kprof.py dec0_rw [--precision 1] [--iters 5] [--batch 32]

Shapes are the aero_4-16_512_64, T=501 geometry (SURVEY.md appendix A)."""
import argparse
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from aero_b200 import Aero, aero_kwargs, cabi  # noqa: E402
from aero_b200.engine import AeroEngine, pack_taps, tf32_round  # noqa: E402

T = 501
SHAPES = {
    # name: (kwargs of AeroEngine._gemm without B, note)
    "dec0_rw": dict(F_out=4, N=1536, C1=0, C2=384, kf=3, kt=3, pad_f=1, pad_t=1, stats_mode=1, groups=4),
    "dec1_rw": dict(F_out=8, N=768, C1=192, C2=192, kf=3, kt=3, pad_f=1, pad_t=1, stats_mode=1, groups=4),
    "dec2_rw": dict(F_out=16, N=384, C1=96, C2=96, kf=3, kt=3, pad_f=1, pad_t=1, glu=1),
    "dec3_rw": dict(F_out=64, N=192, C1=48, C2=48, kf=3, kt=3, pad_f=1, pad_t=1, glu=1),
    "dec0_ct": dict(F_out=14, F_in=4, N=192, C1=768, mode=cabi.TAPS_CONVT, kf=8, stride_f=2, stats_mode=1, groups=4),
    "enc3_conv": dict(F_out=4, F_in=8, N=384, C1=192, kf=8, stride_f=2, pad_f=3, stats_mode=1, groups=4),
    "enc0_ftb2": dict(F_out=256, N=48, C1=48, C2=48, act=cabi.ACT_RELU),
    "enc0_conv": dict(F_out=64, F_in=256, N=48, C1=48, kf=8, stride_f=4, pad_f=2, act=cabi.ACT_GELU),
    "enc0_dc_c2": dict(F_out=64, N=96, C1=12, stats_mode=2),
    "enc1_ftb2": dict(F_out=64, N=96, C1=96, C2=96, act=cabi.ACT_RELU),
    "enc0_rw": dict(F_out=64, N=96, C1=48, glu=1),
    "dec3_ct_in": dict(F_out=64, N=192, C1=96),
    "enc3_gin2": dict(F_out=1, N=768, C1=192, T=768 * 200 // 32),
    "dec3_ct": dict(F_out=256, F_in=64, N=2, C1=96, mode=cabi.TAPS_CONVT, kf=8, stride_f=4, f_off=2),
}


def run_lstm(args):
    """enc3-like BiLSTM layer-2 recurrence: H=96 (or 48), 768 (1536) windows of 200 steps."""
    from aero_b200.engine import lstm_gate_reorder, lstm_whh_fp16
    H = 96 if args.shape == "lstm96" else 48
    rows = (4 if H == 96 else 8) * args.batch
    T, n_win, steps, stride = 501, 6, 200, 100
    m = Aero(**aero_kwargs("aero_4-16_512_256")).eval().cuda()
    eng = AeroEngine(m)
    eng.precision = args.precision
    tc = args.precision >= 1
    G = 8 * H
    gin = torch.randn(rows * n_win * steps, G, device="cuda")
    if os.environ.get("KPROF_GIN16"):
        gin = gin.half()
    bias = torch.randn(G, device="cuda")
    whh = torch.randn(2, 4 * H, H) / math.sqrt(H)
    if tc:
        src, ok = lstm_gate_reorder(H)
        whh = lstm_whh_fp16(torch.cat([torch.where(ok[:, None], whh[d][src], torch.zeros(())) for d in range(2)], 0))
    whh = whh.cuda()
    hout = torch.zeros(rows * T, 2 * H, device="cuda", dtype=torch.float16 if args.precision == 2 else torch.float32)
    ms = []
    for i in range(args.iters + 2):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng._lstm_rec(gin, bias, whh, hout, rows=rows, T=T, H=H, n_win=n_win, steps=steps, stride=stride, in_windowed=1,
                      out_windowed=0, tc=tc)
        e1.record()
        torch.cuda.synchronize()
        if i >= 2:
            ms.append(e0.elapsed_time(e1))
    print(f"{args.shape}: precision {args.precision} rows {rows} best {min(ms)*1e3:.1f} us -> {min(ms)*1e3/steps:.2f} us/step")


def run_attn(args):
    H = 96 if args.shape == "attn96" else 48
    rows = (4 if H == 96 else 8) * args.batch
    T = 501
    m = Aero(**aero_kwargs("aero_4-16_512_256")).eval().cuda()
    eng = AeroEngine(m)
    eng.precision = args.precision
    ld = 3 * H + 16
    qkvd = torch.randn(rows * T, ld, device="cuda")
    out = torch.empty(rows * T, H, device="cuda")
    ms = []
    for i in range(args.iters + 2):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); eng._attn(qkvd, out, rows=rows, T=T, H=H, heads=4, ndecay=4, ld=ld); e1.record()
        torch.cuda.synchronize()
        if i >= 2:
            ms.append(e0.elapsed_time(e1))
    print(f"{args.shape}: precision {args.precision} rows {rows} best {min(ms)*1e3:.1f} us")


def run_stft(args):
    """The model's analysis / synthesis pair at BASELINE shapes: 32 x 8000 -> [32,256,501,2] -> 32 x 32000."""
    m = Aero(**aero_kwargs("aero_4-16_512_64")).eval().cuda()
    eng = AeroEngine(m)
    B, L, T, Fq = args.batch, 8000, 501, 256
    x = torch.randn(B, L, device="cuda")
    z = torch.empty(B, Fq, T, 2, device="cuda")
    y = torch.empty(B, 32000, device="cuda")
    stats = torch.zeros(B, 2, dtype=torch.float64, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = {}
    for name, fn, nbytes in (
            ("stft", lambda: eng.stft_into(x, z, stats, n_fft=512, hop=16, win=128, channels=1, bins_out=Fq, strides=(Fq * T * 2, 2, T * 2, 2)),
             4 * B * L + 8 * B * Fq * T),
            ("istft", lambda: eng.istft_into(z, y, n_fft=512, hop=64, win=512, channels=1, frames=T, bins_in=Fq, strides=(Fq * T * 2, 2, T * 2, 2)),
             8 * B * Fq * T + 4 * B * 32000)):
        ms = []
        for i in range(args.iters + 2):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record()
            torch.cuda.synchronize()
            if i >= 2:
                ms.append(e0.elapsed_time(e1))
        print(f"{name}: B={B} {nbytes/1e6:.1f} MB  best {min(ms)*1e3:.1f} us -> {nbytes/min(ms)/1e6:.1f} GB/s")


def run_wgrad(args):
    """Weight gradient of one conv shape, as the training engine launches it (fp32 operands, dW in PyTorch's parameter layout)."""
    import ctypes as C
    lib = cabi.load()
    cfg = dict(SHAPES[args.shape])
    B, Tt = args.batch, cfg.pop("T", T)
    F_out, N, C1 = cfg.pop("F_out"), cfg.pop("N"), cfg.pop("C1")
    C2, F_in = cfg.get("C2", 0), cfg.get("F_in", F_out)
    mode, kf, kt = cfg.get("mode", cabi.TAPS_CONV), cfg.get("kf", 1), cfg.get("kt", 1)
    K = C1 + C2
    a1 = torch.randn(B, F_in, Tt, C1, device="cuda") if C1 else None
    a2 = torch.randn(B, F_in, Tt, C2, device="cuda") if C2 else None
    dy = torch.randn(B, F_out, Tt, N, device="cuda")
    conv = mode == cabi.TAPS_CONV
    gw = torch.zeros((N, K, kf, kt) if conv else (K, N, kf, 1), device="cuda")
    sn, sk = (gw.stride(0), gw.stride(1)) if conv else (gw.stride(1), gw.stride(0))

    def cl(F, C_):
        return (F * Tt * C_, Tt * C_, C_)
    p = cabi.TapGemmParams(B, F_out, Tt, N, F_in, Tt, C1, C2, mode, kf, kt, cfg.get("stride_f", 1), cfg.get("pad_f", 0), 1, cfg.get("pad_t", 0),
                           cfg.get("f_off", 0), cabi.ACT_NONE, 0, 0, 1, *(cl(F_in, C1) if C1 else (0, 0, 0)), *(cl(F_in, C2) if C2 else (0, 0, 0)), 0,
                           *cl(F_out, N), 0, 0, 0, 0, 0, args.precision, 0)
    ntaps = kf * kt if conv else kf // cfg["stride_f"]
    flops = 2.0 * B * F_out * Tt * N * K * ntaps
    nbytes = sum(t.numel() * 4 for t in (a1, a2, dy) if t is not None)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    P = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ms = []
    for i in range(args.iters + 2):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        cabi.check(lib.aero_tapgemm_wgrad(P(a1), P(a2), P(dy), P(gw), C.byref(p), sn, sk, 1, st), lib)
        e1.record()
        torch.cuda.synchronize()
        if i >= 2:
            ms.append(e0.elapsed_time(e1))
    best = min(ms)
    print(f"{args.shape} wgrad: precision {args.precision} B={B} {flops/1e9:.1f} GFLOP  best {best*1e3:.1f} us  median {sorted(ms)[len(ms)//2]*1e3:.1f} us"
          f"  -> {flops/best/1e9:.1f} TFLOP/s; operands {nbytes/1e6:.0f} MB once = {nbytes/best/1e6:.0f} GB/s")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("shape", choices=sorted(SHAPES) + ["lstm96", "lstm48", "stft", "attn96", "attn48"])
    ap.add_argument("--precision", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--no-stats", action="store_true")
    ap.add_argument("--out-f32", action="store_true")
    ap.add_argument("--in-f32", action="store_true")
    ap.add_argument("--wgrad", action="store_true", help="time aero_tapgemm_wgrad of the shape (precision 0 = SIMT, 1 = tensor-core TF32)")
    args = ap.parse_args()
    torch.manual_seed(0)
    if args.shape.startswith("lstm"):
        return run_lstm(args)
    if args.shape == "stft":
        return run_stft(args)
    if args.shape.startswith("attn"):
        return run_attn(args)
    if args.wgrad:
        return run_wgrad(args)
    m = Aero(**aero_kwargs("aero_4-16_512_256")).eval().cuda()
    eng = AeroEngine(m)
    eng.precision = args.precision
    cfg = dict(SHAPES[args.shape])
    if args.no_stats:
        cfg.pop("stats_mode", None); cfg.pop("groups", None)
    B = args.batch
    Tt = cfg.pop("T", T)
    F_out, N, C1 = cfg.pop("F_out"), cfg.pop("N"), cfg.pop("C1")
    C2, F_in = cfg.get("C2", 0), cfg.get("F_in", F_out)
    mode = cfg.get("mode", cabi.TAPS_CONV)
    nslab = cfg.get("kf", 1) * cfg.get("kt", 1)
    K = C1 + C2
    from aero_b200.engine import pack_kmajor_fp16
    w = tf32_round(pack_taps(torch.randn(N, K, nslab) / math.sqrt(K * nslab))).cuda()
    eng._wk[w.data_ptr()] = tf32_round(w.permute(0, 2, 1).contiguous())
    eng._wh[w.data_ptr()] = pack_kmajor_fp16(w)
    sm = cfg.get("stats_mode", 0)
    f16 = args.precision == 2 and C1 % 8 == 0 and C2 % 8 == 0 and not args.in_f32
    adt = torch.float16 if f16 else torch.float32
    odt = torch.float16 if (args.precision == 2 and not args.out_f32) else torch.float32      # (pre-norm outputs are FP16 too since round 2)
    a1 = tf32_round(torch.randn(B, F_in, Tt, C1)).cuda().to(adt) if C1 else None
    a2 = tf32_round(torch.randn(B, F_in, Tt, C2)).cuda().to(adt) if C2 else None
    bias = torch.randn(N).cuda()
    n_out = N // 2 if cfg.get("glu") else N
    out = torch.empty(B, F_out, Tt, n_out, device="cuda", dtype=odt)
    nbytes = sum(t.numel() * t.element_size() for t in (a1, a2, out) if t is not None)
    stats = torch.zeros(max(1, {0: 0, 1: B * cfg.get("groups", 1), 2: B * F_out}[sm]), 2, dtype=torch.float64, device="cuda")
    ntaps = nslab if mode == cabi.TAPS_CONV else cfg["kf"] // cfg["stride_f"]
    flops = 2.0 * B * F_out * Tt * N * K * ntaps
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.iters + 1)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ms = []
    for i in range(args.iters + 2):
        flush.zero_()                       # evict L2 between iterations
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng._gemm(out, w, a1=a1, a2=a2, B=B, F_out=F_out, T=Tt, N=N, C1=C1, bias=bias, stats=stats if sm else None, **cfg)
        e1.record()
        torch.cuda.synchronize()
        if i >= 2:
            ms.append(e0.elapsed_time(e1))
    best = min(ms)
    print(f"{args.shape}: precision {args.precision} B={B} {flops/1e9:.1f} GFLOP  best {best*1e3:.1f} us  median {sorted(ms)[len(ms)//2]*1e3:.1f} us"
          f"  -> {flops/best/1e9:.1f} TFLOP/s, {nbytes/best/1e6:.0f} GB/s of {nbytes/1e6:.0f} MB (best)")


if __name__ == "__main__":
    main()
