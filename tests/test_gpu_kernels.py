"""-m gpu: every C-ABI kernel against the CPU statement of its contract (tests/cpu_emu.py, itself
checked against the reference's golden vectors in test_host_logic.py), on seeded random inputs,
covering ragged sizes, two-source K, transposed taps, GLU, statistics and windowed LSTM."""
import math
import os

import numpy as np
import pytest
import torch

from cpu_emu import EmuEngine
from util import SEED, rel_l2, white_noise

from aero_b200 import Aero, aero_kwargs, cabi
from aero_b200.engine import AeroEngine, pack_taps

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs("aero_4-16_512_256")).eval()
    emu = EmuEngine(m)
    mg = Aero(**aero_kwargs("aero_4-16_512_256")).eval().cuda()
    gpu = AeroEngine(mg)
    gpu.precision = 0          # kernel tests pick the path explicitly
    return gpu, emu


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


GEMM_CASES = [
    # name, dict(B,F_out,F_in,T,N,C1,C2, extra)
    ("1x1_flat", dict(B=1, F_out=1, T=1000, N=96, C1=48)),
    ("k2_thin_in", dict(B=1, F_out=1, T=777, N=48, C1=2)),
    ("thin_out_relu", dict(B=2, F_out=8, T=131, N=5, C1=48, act=cabi.ACT_RELU)),
    ("enc_k8s4_gelu", dict(B=2, F_out=4, F_in=16, T=140, N=96, C1=48, kf=8, stride_f=4, pad_f=2, act=cabi.ACT_GELU)),
    ("enc_k8s2_stats", dict(B=2, F_out=4, F_in=8, T=130, N=192, C1=96, kf=8, stride_f=2, pad_f=3, stats_mode=1, groups=4)),
    ("dconv_k3d2_rowstats", dict(B=2, F_out=3, T=257, N=12, C1=48, kt=3, dil_t=2, pad_t=2, stats_mode=2)),
    ("dec_3x3_two_src_glu", dict(B=1, F_out=5, T=133, N=192, C1=48, C2=48, kf=3, kt=3, pad_f=1, pad_t=1, glu=1)),
    ("dec_3x3_zero_half", dict(B=1, F_out=4, T=70, N=128, C1=0, C2=32, kf=3, kt=3, pad_f=1, pad_t=1, stats_mode=1, groups=4)),
    ("convt_s2_full", dict(B=2, F_out=14, F_in=4, T=129, N=48, C1=96, mode=cabi.TAPS_CONVT, kf=8, stride_f=2, stats_mode=1, groups=4)),
    ("convt_s4_crop_affine", dict(B=2, F_out=64, F_in=16, T=65, N=2, C1=24, mode=cabi.TAPS_CONVT, kf=8, stride_f=4, f_off=2, affine=True)),
    ("convt_s4_crop_gelu", dict(B=1, F_out=16, F_in=4, T=200, N=48, C1=96, mode=cabi.TAPS_CONVT, kf=8, stride_f=4, f_off=2, act=cabi.ACT_GELU)),
    ("residual_1x1", dict(B=1, F_out=1, T=500, N=48, C1=96, residual=True)),
    ("glu_addend", dict(B=2, F_out=6, T=90, N=96, C1=48, glu=1, addend=True)),
    ("k9_conv1d", dict(B=2, F_out=1, T=150, N=48, C1=80, kt=9, pad_t=4, act=cabi.ACT_RELU)),
]


@pytest.mark.parametrize("name,cfg", GEMM_CASES, ids=[c[0] for c in GEMM_CASES])
def test_tapgemm_simt(engines, name, cfg):
    gpu, emu = engines
    cfg = dict(cfg)
    B, F_out, T, N, C1 = cfg["B"], cfg["F_out"], cfg["T"], cfg["N"], cfg["C1"]
    C2, F_in = cfg.get("C2", 0), cfg.get("F_in", F_out)
    mode = cfg.get("mode", cabi.TAPS_CONV)
    nslab = cfg.get("kf", 1) * cfg.get("kt", 1)
    K = C1 + C2
    w = pack_taps(rnd(N, K, nslab, seed=1) / math.sqrt(K * (nslab if mode == cabi.TAPS_CONV else 2)))
    a1 = rnd(B, F_in, T, C1, seed=2) if C1 else None
    a2 = rnd(B, F_in, T, C2, seed=3) if C2 else None
    bias = rnd(N, seed=4)
    glu = cfg.get("glu", 0)
    n_out = N // 2 if glu else N
    extra = {}
    if cfg.pop("residual", False):
        extra["residual"] = rnd(B, F_out, T, n_out, seed=5)
    if cfg.pop("addend", False):
        extra["addend"] = rnd(F_out, n_out, seed=6)
    if cfg.pop("affine", False):
        extra["samp_affine"] = rnd(B, 2, seed=7).abs() + 0.5
    sm = cfg.get("stats_mode", 0)
    nslots = {0: 0, 1: B * cfg.get("groups", 1), 2: B * F_out}[sm]
    for k in ("B", "F_out", "T", "N", "C1"):
        cfg.pop(k)
    res = {}
    for tag, eng, dev in (("cpu", emu, "cpu"), ("gpu", gpu, "cuda")):
        def mv(t):
            return None if t is None else t.to(dev)
        out = torch.zeros(B, F_out, T, n_out, device=dev)
        stats = torch.zeros(max(nslots, 1), 2, dtype=torch.float64, device=dev)
        eng._gemm(out, mv(w), a1=mv(a1), a2=mv(a2), B=B, F_out=F_out, T=T, N=N, C1=C1, bias=mv(bias),
                  stats=stats if sm else None, **{k: mv(v) for k, v in extra.items()}, **cfg)
        res[tag] = (out.cpu(), stats.cpu())
    assert rel_l2(res["gpu"][0], res["cpu"][0]) < 2e-6
    if sm:
        assert torch.allclose(res["gpu"][1], res["cpu"][1], rtol=1e-5, atol=1e-3)


def test_freq_mix_gemm_with_activation_weights(engines):
    """FTB frequency mixing: A = Wfc, 'weights' = the activations, batch-strided (include/aero_b200.h w_sb)."""
    gpu, emu = engines
    B, Fq, T, Cc = 2, 16, 37, 24
    x, wfc, gate = rnd(B, Fq, T, Cc, seed=1), rnd(Fq, Fq, seed=2) / 4, rnd(B, T, Cc, seed=3)
    outs = []
    for eng, dev in ((emu, "cpu"), (gpu, "cuda")):
        y = torch.zeros(B, Fq, T, Cc, device=dev)
        eng._gemm(y, x.to(dev), a1=wfc.to(dev), B=B, F_out=1, T=Fq, T_in=Fq, N=T * Cc, C1=Fq, a1_s=(0, 0, Fq),
                  w_sb=Fq * T * Cc, o_s=(Fq * T * Cc, 0, T * Cc), colscale=gate.to(dev), cs_s=(T * Cc, 0))
        outs.append(y.cpu())
    ref = torch.einsum("gf,bftc->bgtc", wfc, x) * gate[:, None]
    assert rel_l2(outs[0], ref) < 1e-6 and rel_l2(outs[1], ref) < 2e-6


@pytest.mark.parametrize("op", [cabi.NA_NONE, cabi.NA_GELU, cabi.NA_GLU, cabi.NA_SNAKE, cabi.NA_GLU_SCALE_RES])
@pytest.mark.parametrize("scope", [1, 2])
def test_norm_act(engines, op, scope):
    gpu, emu = engines
    B, F_in, T, Cc = 2, 6, 77, 48
    groups = 4 if scope == 1 else 1
    f_off, F_out = (1, 4) if (scope == 1 and op in (cabi.NA_NONE, cabi.NA_GELU)) else (0, F_in)
    x = rnd(B, F_in, T, Cc, seed=1) * 1.7 + 0.3
    gamma, beta = 1 + 0.2 * rnd(Cc, seed=2), 0.1 * rnd(Cc, seed=3)
    glu = op in (cabi.NA_GLU, cabi.NA_GLU_SCALE_RES)
    co = Cc // 2 if glu else Cc
    a = rnd(F_in, seed=4).abs() * 8 + 0.2
    scale, resid = rnd(co, seed=5), rnd(B, F_out, T, co, seed=6)
    xd = x.double()
    if scope == 1:
        g = xd.view(B, F_in * T, groups, Cc // groups)
        stats = torch.stack([g.sum((1, 3)).reshape(-1), (g * g).sum((1, 3)).reshape(-1)], 1)
    else:
        g = xd.view(B * F_in, -1)
        stats = torch.stack([g.sum(1), (g * g).sum(1)], 1)
    outs = []
    for eng, dev in ((emu, "cpu"), (gpu, "cuda")):
        y = torch.zeros(B, F_out, T, co, device=dev)
        eng._norm_act(x.to(dev), stats.to(dev), gamma.to(dev), beta.to(dev), y, B=B, F_in=F_in, F_out=F_out, f_off=f_off,
                      T=T, C_=Cc, groups=groups, scope=scope, op=op, snake_a=a.to(dev), scale=scale.to(dev),
                      residual=resid.to(dev))
        outs.append(y.cpu())
    assert rel_l2(outs[1], outs[0]) < 3e-6


@pytest.mark.parametrize("H,T,rows", [(48, 251, 5), (96, 123, 3), (48, 501, 2), (12, 40, 20)])
def test_lstm_layer_pair(engines, H, T, rows):
    """Both recurrent calls of a BLSTM (windowed when T > 200) against the cell recurrence on CPU."""
    gpu, emu = engines
    steps, stride, n_win = (200, 100, math.ceil(T / 100)) if T > 200 else (T, 0, 1)
    n_seq = rows * n_win
    gin1, b1 = rnd(rows * T, 8 * H, seed=1), rnd(8 * H, seed=2) * 0.3
    whh1, whh2 = rnd(2, 4 * H, H, seed=3) / math.sqrt(H), rnd(2, 4 * H, H, seed=4) / math.sqrt(H)
    gin2 = rnd(n_seq * steps, 8 * H, seed=5)
    outs = []
    for eng, dev in ((emu, "cpu"), (gpu, "cuda")):
        h1 = torch.zeros(n_seq * steps, 2 * H, device=dev)
        eng._lstm_rec(gin1.to(dev), b1.to(dev), whh1.to(dev), h1, rows=rows, T=T, H=H, n_win=n_win, steps=steps,
                      stride=stride, in_windowed=0, out_windowed=1)
        h2 = torch.zeros(rows * T, 2 * H, device=dev)
        eng._lstm_rec(gin2.to(dev), b1.to(dev), whh2.to(dev), h2, rows=rows, T=T, H=H, n_win=n_win, steps=steps,
                      stride=stride, in_windowed=1, out_windowed=0)
        outs.append((h1.cpu(), h2.cpu()))
    assert rel_l2(outs[1][0], outs[0][0]) < 1e-5
    assert rel_l2(outs[1][1], outs[0][1]) < 1e-5


@pytest.mark.parametrize("H,T,rows", [(48, 501, 3), (96, 251, 2), (48, 700, 1), (12, 33, 4)])
def test_local_attention(engines, H, T, rows):
    gpu, emu = engines
    ld = 3 * H + 16
    qkvd = rnd(rows * T, ld, seed=1)
    qkvd[:, 3 * H:] = qkvd[:, 3 * H:] * 1.5 - 1.0
    outs = []
    for eng, dev in ((emu, "cpu"), (gpu, "cuda")):
        o = torch.zeros(rows * T, H, device=dev)
        eng._attn(qkvd.to(dev), o, rows=rows, T=T, H=H, heads=4, ndecay=4, ld=ld)
        outs.append(o.cpu())
    assert rel_l2(outs[1], outs[0]) < 1e-5


def test_sample_norm(engines):
    gpu, emu = engines
    B, n = 3, 4 * 257
    x = rnd(B, n, seed=1) * 2.5 + 0.7
    xd = x.double()
    stats = torch.stack([xd.sum(1), (xd * xd).sum(1)], 1)
    outs = []
    for eng, dev in ((emu, "cpu"), (gpu, "cuda")):
        y, aff = torch.zeros(B, n, device=dev), torch.zeros(B, 2, device=dev)
        eng._sample_norm(x.to(dev), stats.to(dev), y, aff, B, n)
        outs.append((y.cpu(), aff.cpu()))
    assert rel_l2(outs[1][0], outs[0][0]) < 1e-6 and rel_l2(outs[1][1], outs[0][1]) < 1e-6
    ref = (x - x.mean(1, keepdim=True)) / (1e-5 + x.std(1, keepdim=True))
    assert rel_l2(outs[1][0], ref) < 1e-5


@pytest.mark.parametrize("J,N,dt", [(2, 48, torch.float16), (2, 48, torch.float32), (4, 64, torch.float16), (2, 24, torch.float16)])
def test_ftb_through_linear_input(engines, J, N, dt):
    """aero_ftb_lin_out_fwd against the fp64 statement of its formula (padded spectrogram rows, ragged T)."""
    gpu, emu = engines
    B, F, T = 2, 9, 77
    zrow = (T * J + 3) & ~3
    z, zm = rnd(B, F, zrow, seed=1), rnd(B, F, zrow, seed=2)
    M, s_, V, d = rnd(B * T, N * (J + 1), seed=3), rnd(F, seed=4), rnd(N, J, seed=5), rnd(N, seed=6)
    ref = torch.zeros(B, F, T, N)
    emu._ftb_lin_out(z, zm, M, s_, V, d, ref, B=B, F=F, T=T, N=N, J=J, zrow=zrow)
    out = torch.full((B, F, T, N), float("nan"), device="cuda", dtype=dt)
    gpu._ftb_lin_out(z.cuda(), zm.cuda(), M.cuda(), s_.cuda(), V.cuda(), d.cuda(), out, B=B, F=F, T=T, N=N, J=J, zrow=zrow)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    assert rel_l2(out.float().cpu(), ref) < (4e-4 if dt == torch.float16 else 2e-6)


@pytest.mark.parametrize("J,dt", [(2, torch.float16), (2, torch.float32), (4, torch.float16)])
def test_ftb_squeeze_through_linear_input(engines, J, dt):
    gpu, emu = engines
    B, F, T, r = 2, 70, 45, 5
    zrow = (T * J + 3) & ~3
    z, W1p, b1p = rnd(B, F, zrow, seed=1), rnd(r, J, seed=2), rnd(r, seed=3)
    ref = torch.zeros(B, T, F * r)
    emu._ftb_lin_squeeze(z, W1p, b1p, ref, B=B, F=F, T=T, J=J, r=r, zrow=zrow)
    R = torch.full((B, T, F * r), float("nan"), device="cuda", dtype=dt)
    gpu._ftb_lin_squeeze(z.cuda(), W1p.cuda(), b1p.cuda(), R, B=B, F=F, T=T, J=J, r=r, zrow=zrow)
    torch.cuda.synchronize()
    assert torch.isfinite(R).all() and rel_l2(R.float().cpu(), ref) < (4e-4 if dt == torch.float16 else 2e-6)


def test_sample_norm_with_row_padding(engines):
    """statistics over `count` values, transform applied to the padded extent (include/aero_b200.h)."""
    gpu, _ = engines
    B, rows, n, pad = 2, 5, 1002, 1004
    x = torch.zeros(B, rows, pad)
    x[:, :, :n] = rnd(B, rows, n, seed=1) * 2.0 + 0.5
    xd = x[:, :, :n].double().reshape(B, -1)
    stats = torch.stack([xd.sum(1), (xd * xd).sum(1)], 1)
    y, aff = torch.zeros(B, rows, pad, device="cuda"), torch.zeros(B, 2, device="cuda")
    gpu._sample_norm(x.cuda(), stats.cuda(), y, aff, B, rows * n, extent=rows * pad)
    ref = (xd - xd.mean(1, keepdim=True)) / (1e-5 + xd.std(1, keepdim=True))
    assert rel_l2(y.cpu()[:, :, :n].reshape(B, -1), ref.float()) < 1e-5


def test_stft_istft_golden_and_roundtrip(golden_dir):
    """spectro / ispectro drop-ins against the reference's own outputs; round trip <= 1e-5 (north_star)."""
    from aero_b200 import ispectro, spectro
    g = np.load(os.path.join(golden_dir, "stft_cases.npz"))
    i = 0
    while f"{i}/params" in g.files:
        n_fft, hop, win, L, *lead = [int(v) for v in g[f"{i}/params"]]
        x = white_noise((*lead, L), seed=SEED + i)
        z = spectro(x.cuda(), n_fft, hop, win_length=win)
        zr = torch.view_as_real(z).cpu().reshape(-1)[torch.from_numpy(g[f"{i}/z_idx"].astype(np.int64))]
        assert rel_l2(zr, g[f"{i}/z_val"]) < 1e-5, (i, "stft")
        y = ispectro(z, hop, win_length=win).cpu()
        assert y.shape == g[f"{i}/y"].shape
        assert rel_l2(y, g[f"{i}/y"]) < 1e-5, (i, "istft")
        n = min(y.shape[-1], L)
        if hop * 2 <= win:      # COLA holds: analysis->synthesis is the identity on the kept span
            assert rel_l2(y[..., :n], x[..., :n]) < 1e-5, (i, "roundtrip")
        i += 1
    assert i >= 6


# ------------------------------------------------------------------------------------------------
# wgmma path: same contract, TF32 operands.  Inputs are pre-rounded to TF32 so every product is exact
# in fp32 and the comparison is tight (it checks descriptors / swizzle / tap geometry, not TF32 noise).
TC_CASES = [c for c in GEMM_CASES if c[0] not in ("k2_thin_in", "thin_out_relu", "convt_s4_crop_affine")] + [
    ("big_n_tiles", dict(B=1, F_out=2, T=300, N=768, C1=96, kf=3, kt=3, pad_f=1, pad_t=1, stats_mode=1, groups=4)),
    ("k_tail_48", dict(B=2, F_out=3, T=129, N=96, C1=48, C2=48, glu=1)),
    ("n_304", dict(B=1, F_out=1, T=1000, N=304, C1=96)),
    ("hidden12", dict(B=2, F_out=4, T=200, N=12, C1=48, kt=3, dil_t=1, pad_t=1, stats_mode=2)),
    ("deep_k", dict(B=1, F_out=1, T=256, N=48, C1=1280, kt=9, pad_t=4, act=cabi.ACT_RELU)),
]


def _run_gemm_case(gpu, emu, cfg, storage, precision):
    """One tap-GEMM case on the GPU with the given activation storage ('tf32': fp32 rounded to TF32, 'f16': FP16 sources,
    FP16 outputs unless the case collects statistics) against the fp64 CPU statement on the same (pre-rounded) numbers."""
    from aero_b200.engine import pack_kmajor_fp16, tf32_round
    cfg = dict(cfg)
    B, F_out, T, N, C1 = cfg["B"], cfg["F_out"], cfg["T"], cfg["N"], cfg["C1"]
    C2, F_in = cfg.get("C2", 0), cfg.get("F_in", F_out)
    mode = cfg.get("mode", cabi.TAPS_CONV)
    nslab = cfg.get("kf", 1) * cfg.get("kt", 1)
    K = C1 + C2
    f16 = storage == "f16"
    a_f16 = f16 and C1 % 4 == 0 and C2 % 4 == 0 and K > 4          # the K=2 layer reads the fp32 spectrogram
    q = (lambda t: t.half().float()) if f16 else tf32_round
    w = q(pack_taps(rnd(N, K, nslab, seed=1) / math.sqrt(K * (nslab if mode == cabi.TAPS_CONV else 2))))
    a1 = (q(rnd(B, F_in, T, C1, seed=2)) if a_f16 or not f16 else rnd(B, F_in, T, C1, seed=2)) if C1 else None
    a2 = q(rnd(B, F_in, T, C2, seed=3)) if C2 else None
    bias = rnd(N, seed=4)
    glu = cfg.get("glu", 0)
    n_out = N // 2 if glu else N
    extra = {}
    if cfg.pop("residual", False):
        extra["residual"] = q(rnd(B, F_out, T, n_out, seed=5))
    if cfg.pop("addend", False):
        extra["addend"] = rnd(F_out, n_out, seed=6)
    if cfg.pop("affine", False):
        extra["samp_affine"] = rnd(B, 2, seed=7).abs() + 0.5
    sm = cfg.get("stats_mode", 0)
    o_f16 = f16 and sm == 0 and "samp_affine" not in extra
    nslots = {0: 0, 1: B * cfg.get("groups", 1), 2: B * F_out}[sm]
    for k in ("B", "F_out", "T", "N", "C1"):
        cfg.pop(k)
    res = {}
    for tag, eng, dev in (("cpu", emu, "cpu"), ("gpu", gpu, "cuda")):
        on_gpu = tag == "gpu"

        def mv(t, half=False):
            if t is None:
                return None
            t = t.to(dev)
            return t.half() if (half and on_gpu) else t
        out = torch.full((B, F_out, T, n_out), float("nan"), device=dev, dtype=torch.float16 if (o_f16 and on_gpu) else torch.float32)
        stats = torch.zeros(max(nslots, 1), 2, dtype=torch.float64, device=dev)
        wd = mv(w)
        kw = {k: mv(v, half=(k == "residual" and o_f16)) for k, v in extra.items()}
        if on_gpu:
            eng.precision = precision
            eng._wk[wd.data_ptr()] = tf32_round(wd.permute(0, 2, 1).contiguous())
            eng._wh[wd.data_ptr()] = pack_kmajor_fp16(wd)
        try:
            eng._gemm(out, wd, a1=mv(a1, a_f16), a2=mv(a2, a_f16), B=B, F_out=F_out, T=T, N=N, C1=C1, bias=mv(bias),
                      stats=stats if sm else None, **kw, **cfg)
            if on_gpu:
                torch.cuda.synchronize()
        finally:
            if on_gpu:
                eng.precision = 0
                eng._wk.clear()
                eng._wh.clear()
        res[tag] = (out.float().cpu(), stats.cpu())
    assert torch.isfinite(res["gpu"][0]).all()
    err = rel_l2(res["gpu"][0], res["cpu"][0])
    if o_f16:
        assert err < 4e-4, err               # one FP16 rounding of the stored value (rms 2^-11/sqrt(3) relative to its binade)
    else:
        # products are exact; what is left is the fp32 accumulation order/rounding, which grows with K
        assert err < (5e-5 if K * nslab > 4096 else 5e-6), err
    if sm:
        assert torch.allclose(res["gpu"][1], res["cpu"][1], rtol=1e-4, atol=1e-2)


@pytest.mark.parametrize("storage", ["tf32", "f16"])
@pytest.mark.parametrize("name,cfg", TC_CASES, ids=[c[0] for c in TC_CASES])
def test_tapgemm_tcgen05(engines, name, cfg, storage):
    gpu, emu = engines
    _run_gemm_case(gpu, emu, cfg, storage, 2 if storage == "f16" else 1)


@pytest.mark.parametrize("name,cfg", GEMM_CASES, ids=[c[0] for c in GEMM_CASES])
def test_tapgemm_simt_fp16_storage(engines, name, cfg):
    """The fp32 SIMT kernels (generic tile and the thin-N / thin-K / thin-transposed ones) reading and writing FP16 tensors."""
    gpu, emu = engines
    _run_gemm_case(gpu, emu, cfg, "f16", 0)


def test_tcgen05_is_selected_for_the_big_convs(engines):
    gpu, _ = engines
    p = cabi.TapGemmParams(32, 4, 501, 1536, 4, 501, 0, 384, 0, 3, 3, 1, 1, 1, 1, 0, 0, 0, 1, 4,
                           0, 0, 0, 4 * 501 * 384, 501 * 384, 384, 0, 4 * 501 * 1536, 501 * 1536, 1536, 0, 0, 0, 0, 0, 0, 0)
    import ctypes
    assert gpu.lib.aero_tapgemm_tc_eligible(ctypes.byref(p)) == 1


@pytest.mark.parametrize("H,T,rows", [(48, 251, 5), (96, 123, 3), (96, 501, 2), (64, 40, 20), (36, 230, 3)])
def test_lstm_layer_pair_tcgen05(engines, H, T, rows):
    """wgmma recurrence (TF32 h*W_hh, fp32 accumulate, fast sigmoid/tanh) against the fp32 cell recurrence."""
    from aero_b200.engine import lstm_gate_reorder, lstm_whh_fp16, tf32_round
    gpu, emu = engines
    steps, stride, n_win = (200, 100, math.ceil(T / 100)) if T > 200 else (T, 0, 1)
    n_seq = rows * n_win
    gin1, b1 = rnd(rows * T, 8 * H, seed=1), rnd(8 * H, seed=2) * 0.3
    whh1, whh2 = rnd(2, 4 * H, H, seed=3) / math.sqrt(H), rnd(2, 4 * H, H, seed=4) / math.sqrt(H)
    gin2 = rnd(n_seq * steps, 8 * H, seed=5)
    h1c = torch.zeros(n_seq * steps, 2 * H)
    emu._lstm_rec(gin1, b1, whh1, h1c, rows=rows, T=T, H=H, n_win=n_win, steps=steps, stride=stride, in_windowed=0, out_windowed=1)
    h2c = torch.zeros(rows * T, 2 * H)
    emu._lstm_rec(gin2, b1, whh2, h2c, rows=rows, T=T, H=H, n_win=n_win, steps=steps, stride=stride, in_windowed=1, out_windowed=0)

    src, ok = lstm_gate_reorder(H)

    def rows_(w):     # [2, 4H, H] -> [2*nM*128, H]
        return lstm_whh_fp16(torch.cat([torch.where(ok[:, None], w[d][src], torch.zeros(())) for d in range(2)], 0))

    gpu.precision = 1
    try:
        h1 = torch.zeros(n_seq * steps, 2 * H, device="cuda")
        gpu._lstm_rec(gin1.cuda(), b1.cuda(), rows_(whh1).cuda(), h1, rows=rows, T=T, H=H, n_win=n_win,
                      steps=steps, stride=stride, in_windowed=0, out_windowed=1, tc=True)
        h2 = torch.zeros(rows * T, 2 * H, device="cuda")
        gpu._lstm_rec(gin2.cuda(), b1.cuda(), rows_(whh2).cuda(), h2, rows=rows, T=T, H=H, n_win=n_win,
                      steps=steps, stride=stride, in_windowed=1, out_windowed=0, tc=True)
        torch.cuda.synchronize()
    finally:
        gpu.precision = 0
    e1, e2 = rel_l2(h1.cpu(), h1c), rel_l2(h2.cpu(), h2c)
    print(f"lstm wgmma H={H} T={T}: rel_l2 {e1:.2e} {e2:.2e}")
    assert e1 < 1e-3 and e2 < 1e-3


@pytest.mark.parametrize("storage", ["tf32", "f16"])
@pytest.mark.parametrize("B,Fq,T,Cc", [(2, 256, 37, 48), (1, 64, 131, 48), (3, 16, 50, 96), (2, 8, 77, 192)])
def test_freq_mix_tcgen05_mn_major(engines, B, Fq, T, Cc, storage):
    """AERO_TAPS_MIX: contraction over the frequency rows with the activations as the MN-major wgmma operand
    (tf32: A fragments loaded into registers from SWIZZLE_128B boxes; f16: transposed-A wgmma on SWIZZLE_128B atoms)."""
    from aero_b200.engine import pack_kmajor_fp16, tf32_round
    gpu, _ = engines
    f16 = storage == "f16"
    q = (lambda t: t.half().float()) if f16 else tf32_round
    x, wfc, gate = q(rnd(B, Fq, T, Cc, seed=1)), q(rnd(Fq, Fq, seed=2) / math.sqrt(Fq)), rnd(B, T, Cc, seed=3)
    y = torch.full((B, Fq, T, Cc), float("nan"), device="cuda", dtype=torch.float16 if f16 else torch.float32)
    wd = pack_kmajor_fp16(wfc.t()[None].contiguous())[0].cuda() if f16 else wfc.cuda()
    gpu._gemm(y, wd, a1=x.half().cuda() if f16 else x.cuda(), mode=cabi.TAPS_MIX, B=B, F_out=1, T=T * Cc, N=Fq, C1=Fq,
              a1_s=(Fq * T * Cc, 0, T * Cc), o_s=(Fq * T * Cc, 0, T * Cc), colscale=gate.cuda(), cs_s=(T * Cc, 0))
    torch.cuda.synchronize()
    ref = torch.einsum("gf,bftc->bgtc", wfc.double(), x.double()) * gate[:, None].double()
    assert torch.isfinite(y).all()
    assert rel_l2(y.float().cpu(), ref) < (4e-4 if f16 else 5e-6)


@pytest.mark.parametrize("F,dt", [(8, torch.float16), (16, torch.float16), (8, torch.float32), (16, torch.float32)])
def test_freq_mix_small(engines, F, dt):
    """aero_freq_mix_small_fwd (deep FTB layers) against the einsum statement; ragged M."""
    gpu, _ = engines
    B, T, Cc = 3, 77, 36
    M = T * Cc
    x = rnd(B, F, T, Cc, seed=1)
    x = x.half().float() if dt == torch.float16 else x
    wfc, gate = rnd(F, F, seed=2) / math.sqrt(F), rnd(B, T, Cc, seed=3)
    ref = torch.einsum("gf,bftc->bgtc", wfc.double(), x.double()) * gate[:, None].double()
    y = torch.full((B, F, T, Cc), float("nan"), device="cuda", dtype=dt)
    gpu._freq_mix_small(x.cuda().to(dt), wfc.cuda(), gate.cuda(), y, B=B, F=F, M=M)
    torch.cuda.synchronize()
    assert torch.isfinite(y).all()
    assert rel_l2(y.float().cpu(), ref) < (4e-4 if dt == torch.float16 else 2e-6)


def test_fp16_outputs_of_the_other_kernels(engines):
    """norm_act / attention writing FP16: the fp32 result of the same call, rounded once (the LSTM recurrence's FP16 output:
    test_gpu_tc_scale.py)."""
    gpu, _ = engines
    B, F_in, T, Cc = 2, 6, 77, 48
    x = (rnd(B, F_in, T, Cc, seed=1) * 1.7 + 0.3).cuda()
    xd = x.double().view(B * F_in, -1)
    stats = torch.stack([xd.sum(1), (xd * xd).sum(1)], 1)
    gamma, beta, scale = (1 + 0.2 * rnd(Cc, seed=2)).cuda(), (0.1 * rnd(Cc, seed=3)).cuda(), rnd(Cc // 2, seed=5).cuda()
    resid = rnd(B, F_in, T, Cc // 2, seed=6).half()
    ys = []
    for dt in (torch.float32, torch.float16):
        y = torch.zeros(B, F_in, T, Cc // 2, device="cuda", dtype=dt)
        gpu._norm_act(x, stats, gamma, beta, y, B=B, F_in=F_in, T=T, C_=Cc, groups=1, scope=2, op=cabi.NA_GLU_SCALE_RES,
                      scale=scale, residual=resid.cuda().to(dt))
        ys.append(y.float().cpu())
    assert rel_l2(ys[1], ys[0]) < 4e-4 and torch.equal(ys[1], ys[0].half().float())
    H, Tt, rows = 48, 130, 2
    ld = 3 * H + 16
    qkvd = rnd(rows * Tt, ld, seed=1).cuda()
    gpu.precision = 1
    try:
        outs_ = []
        for dt in (torch.float32, torch.float16):
            o = torch.zeros(rows * Tt, H, device="cuda", dtype=dt)
            gpu._attn(qkvd, o, rows=rows, T=Tt, H=H, heads=4, ndecay=4, ld=ld)
            outs_.append(o.float().cpu())
    finally:
        gpu.precision = 0
    assert rel_l2(outs_[1], outs_[0]) < 4e-4



@pytest.mark.parametrize("H,T,rows", [(48, 501, 3), (96, 251, 2), (48, 700, 1), (96, 33, 4), (48, 130, 2)])
def test_local_attention_tensor_core(engines, H, T, rows):
    """mma.sync TF32 attention (engine tensor-core mode) against the fp64 statement of modules.py:104-124."""
    gpu, emu = engines
    ld = 3 * H + 16
    qkvd = rnd(rows * T, ld, seed=1)
    qkvd[:, 3 * H:] = qkvd[:, 3 * H:] * 1.5 - 1.0
    ref = torch.zeros(rows * T, H)
    emu._attn(qkvd, ref, rows=rows, T=T, H=H, heads=4, ndecay=4, ld=ld)
    o = torch.full((rows * T, H), float("nan"), device="cuda")
    gpu.precision = 1
    try:
        gpu._attn(qkvd.cuda(), o, rows=rows, T=T, H=H, heads=4, ndecay=4, ld=ld)
        torch.cuda.synchronize()
    finally:
        gpu.precision = 0
    err = rel_l2(o.cpu(), ref)
    print(f"attention mma H={H} T={T}: rel_l2 {err:.2e}")
    assert torch.isfinite(o).all() and err < 1e-3
