"""-m gpu: the three tensor-core kernels at the sizes production launches reach, against fp64 on exactly the operands they read.

The kernel tests in test_gpu_kernels.py launch at most ~128 tiles, so on an H100 (132 SMs) no persistent tap-GEMM CTA reaches a
second tile, the LSTM recurrence only runs its 8-sequence CTAs, and the split-K walker of the TF32 weight gradient never carries
into the next batch item.  Production (32 x 2 s clips, training at batch 8) runs exactly those paths.  Here:

  1. tap-GEMM (csrc/tapgemm_tc_kernel.cuh): every kernel variant pick_kernel builds, at every tile width, in both tile orders,
     on grids of >= 3 tiles per SM with ragged T (some with whole empty row quarters), plus the generic epilogue;
  2. LSTM recurrence (csrc/lstm_tc.cu): the 16-sequence CTAs, FP16 / fp32 outputs and gate inputs;
  3. TF32 weight gradient (csrc/wgrad_tc.cu) at batch 8 / 16, where one split-K stride spans batch items;
  4. every tap-GEMM and LSTM launch of the benchmarked forward (aero_4-16_512_64, 32 x 2 s), each checked right after it ran.

Reference principle: fp64 on the operand values the kernel consumes -- FP16 tensors as stored, fp32 activations truncated to
TF32 (the tensor core ignores the low 13 mantissa bits), weights as packed in their K-major twins.  Every product is then exact in
fp32, and what is left is fp32 accumulation order plus at most one output rounding, so the bars are tight and are applied per
output tile (128 rows x BN columns), where a wrong tile cannot be averaged away by hundreds of good ones:
  - fp32 outputs: per-tile rel-L2 <= 5e-6 (5e-5 when K * taps > 1024).  The wgmma fp32 accumulation error is flat at
    1.2e-7 .. 2.5e-7 of sum |a * w| on every launch of the benchmarked forward; relative to the result it grows with the reduction
    length, reaching 5.2e-6 .. 7.9e-6 per tile on the decoder convolutions (K * taps = 3072 .. 3456; measured on an H100 80GB HBM3,
    700 W), hence the longer-reduction bar from 1024 on;
  - rounded outputs (FP16 storage, or fp32 rounded to TF32 by the epilogue): every element within one ulp of the fp64 value
    rounded the same way, plus 1e-5 * rms(reference) for cancellation;
  - statistics: per slot, within 1e-5 (relative to sum |x| and sum x^2) of fp64 sums of the values as stored."""
import ctypes as C
import math
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as Fn

from cpu_emu import EmuEngine
from util import SEED, rel_l2, trained_like_

from aero_b200 import Aero, aero_kwargs, cabi
from aero_b200.engine import AeroEngine, lstm_gate_reorder, lstm_whh_fp16, pack_kmajor_fp16, pack_taps, tf32_round

pytestmark = pytest.mark.gpu

KMAX_BN = 128           # widest tile the tap-GEMM is built for (tapgemm_tc.cu pick_bn)


def cdiv(a, b):
    return -(-a // b)


def n_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def rnd(*shape, seed=0, dev="cuda"):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(SEED + seed)).to(dev)


def tf32_trunc(t):
    """The value a tensor core reads from an fp32 operand: the low 13 mantissa bits cleared."""
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def pick_bn(N):
    """Tile width of the wgmma tap-GEMM for N output columns (tapgemm_tc.cu pick_bn)."""
    per = cdiv(N, cdiv(N, KMAX_BN))
    return (per + 31) & ~31


class RecordingLib:
    """Forwards to the kernel library and records the parameter block and weight pointer every tap-GEMM / LSTM launch received,
    so a test knows which path (precision 0 = SIMT, 1 = tf32 wgmma, 2 = f16 wgmma) and which flags actually ran."""

    def __init__(self, lib):
        self._lib = lib
        self.calls = []

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def aero_tapgemm_fwd(self, *args):
        p = args[10]._obj
        self.calls.append(("tapgemm", type(p).from_buffer_copy(p), args[2].value))
        return self._lib.aero_tapgemm_fwd(*args)

    def aero_lstm_rec_fwd(self, *args):
        p = args[4]._obj
        self.calls.append(("lstm", type(p).from_buffer_copy(p), args[2].value))
        return self._lib.aero_lstm_rec_fwd(*args)


@pytest.fixture(scope="module")
def engines():
    torch.manual_seed(SEED)
    emu = EmuEngine(Aero(**aero_kwargs("aero_4-16_512_256")).eval())
    gpu = AeroEngine(Aero(**aero_kwargs("aero_4-16_512_256")).eval().cuda())
    gpu.lib = RecordingLib(gpu.lib)
    return gpu, emu


# ------------------------------------------------------------------------------------------------ comparison per output tile
def _ulp(q, f16):
    """One ulp of FP16 / TF32 (10 stored mantissa bits) at the already rounded values q."""
    _, e = torch.frexp(q)
    tiny = 2.0 ** -24 if f16 else 2.0 ** -133
    u = torch.ldexp(torch.ones_like(q), e - 11).clamp_min(tiny)
    return torch.where(q == 0, torch.full_like(q, tiny), u)


def tile_errors(got, ref, bn_out, rounding, bar_rel):
    """Worst error per output tile of [B, F, T, n] tensors (fp64): tiles of 128 rows (t) x bn_out columns.  Returns the per-tile
    error normalised by its bar (<= 1 passes).  rounding None: tile rel-L2 / bar_rel (the tile norm is floored at 1 % of a typical
    tile's, so an all-but-zero tile cannot blow up the ratio); 'f16' / 'tf32': max over the tile of |got - R(ref)| / (ulp + slack)."""
    B, F, T, n = ref.shape
    tt, nt = cdiv(T, 128), cdiv(n, bn_out)

    def tiles(x):
        return Fn.pad(x, (0, nt * bn_out - n, 0, tt * 128 - T)).view(B, F, tt, 128, nt, bn_out)
    rms = float(ref.pow(2).mean().sqrt())
    if rounding is None:
        d2 = tiles((got - ref) ** 2).sum((3, 5))
        r2 = tiles(ref ** 2).sum((3, 5)).clamp_min((1e-2 * rms) ** 2 * 128 * bn_out)
        return (d2 / r2).sqrt() / bar_rel
    q = ref.half().double() if rounding == "f16" else tf32_round(ref.float()).double()
    ratio = (got - q).abs() / (_ulp(q, rounding == "f16") + 1e-5 * rms)
    return tiles(ratio).amax((3, 5))


def check_stats(stats_delta, out, *, B, F_out, T, n_out, stats_mode, groups):
    """Statistics slots against fp64 sums of the output as stored; returns the worst ratio to the 1e-5 bar."""
    v = out[..., :n_out].double()
    if stats_mode == 1:
        g = v.reshape(B, F_out * T, groups, n_out // groups)
        s, q, a = g.sum((1, 3)).reshape(-1), (g * g).sum((1, 3)).reshape(-1), g.abs().sum((1, 3)).reshape(-1)
    else:
        g = v.reshape(B * F_out, -1)
        s, q, a = g.sum(1), (g * g).sum(1), g.abs().sum(1)
    e_s = ((stats_delta[:, 0] - s).abs() / a.clamp_min(1e-30)).max()
    e_q = ((stats_delta[:, 1] - q).abs() / q.clamp_min(1e-30)).max()
    return float(max(e_s, e_q)) / 1e-5


def _twin_to_kn(tw, f16, K):
    """K-major twin as packed ([slab][pad4 N][K] fp32, or [slab][pad4 N][pad8 K] FP16) -> [slab][K][pad4 N] of what it holds."""
    t = tw[..., :K].float() if f16 else tf32_trunc(tw)
    return t.permute(0, 2, 1).contiguous()


def check_launch(emu, eng, rec, kw, out, stats_before, *, label=None):
    """Check one tap-GEMM launch against fp64 on its own (snapshotted) inputs.  `rec` = (params, weight pointer) the C ABI
    received.  Returns a dict: path, BN, worst per-tile ratio to the bar (output), worst statistics ratio."""
    p, wptr = rec
    prec = p.precision
    mode, B, F_out, T, N, C1, C2 = p.mode, p.B, p.F_out, p.T, p.N, p.C1, p.C2
    glu = p.glu
    n_out = N // 2 if glu else N
    K = C1 + C2
    a16 = bool(p.flags & cabi.TG_A_F16)
    o16 = out.dtype == torch.float16

    def operand(t):
        if t is None:
            return None
        return t.double() if (t.dtype == torch.float16 or prec == 0) else tf32_trunc(t.float()).double()
    if mode == cabi.TAPS_MIX:
        w = kw["w"]
        wref = (w.float() if a16 else tf32_trunc(w)).double()
    elif prec == 0:
        wref = kw["w"].double()
    else:
        twins = eng._wh if a16 else eng._wk
        tw = next(t for t in twins.values() if t.data_ptr() == wptr)
        wref = _twin_to_kn(tw, a16, K).double()
    rkw = {k: v for k, v in kw.items() if k not in ("w", "stats", "o_s", "r_s", "tag", "rnd", "stats_mode", "groups")}
    rkw.update(B=B, F_out=F_out, T=T, N=N, C1=C1, a1=operand(kw.get("a1")), a2=operand(kw.get("a2")))
    for k in ("bias", "addend", "colscale", "samp_affine", "residual"):
        if rkw.get(k) is not None:
            rkw[k] = rkw[k].double()
    if mode == cabi.TAPS_MIX:
        ref = torch.zeros(B, N, T, dtype=torch.float64, device=out.device)
        EmuEngine._gemm(emu, ref, wref, **rkw, o_s=(N * T, 0, T))
        ref = ref.permute(0, 2, 1)[:, None]                                        # [B, 1, M, N]: tiles of 128 m x BN n
        got = torch.as_strided(out.reshape(-1), (B, N, T), (kw["o_s"][0], kw["o_s"][2], 1)).double().permute(0, 2, 1)[:, None]
    else:
        ref = torch.zeros(B, F_out, T, n_out, dtype=torch.float64, device=out.device)
        r_s = kw.get("r_s") or kw.get("o_s")                                       # the residual is read with the output's strides
        if rkw.get("residual") is not None and r_s:
            rkw["residual"] = torch.as_strided(rkw["residual"].reshape(-1), (B, F_out, T, n_out), (*r_s, 1)).contiguous()
        EmuEngine._gemm(emu, ref, wref, **rkw)
        o_s = kw.get("o_s") or (F_out * T * n_out, T * n_out, n_out)
        got = torch.as_strided(out.reshape(-1), (B, F_out, T, n_out), (*o_s, 1)).double()
    ntaps = (p.kf * p.kt) if mode == cabi.TAPS_CONV else (p.kf // p.stride_f if mode == cabi.TAPS_CONVT else 1)
    rounding = "f16" if o16 else ("tf32" if p.flags & cabi.TG_ROUND_TF32 else None)
    bn = pick_bn(N) if prec else 64
    bn_out = bn if mode == cabi.TAPS_MIX else (bn // 2 if glu else bn)
    assert torch.isfinite(got).all(), (label, "non-finite output")
    err = float(tile_errors(got, ref, bn_out, rounding, 5e-5 if K * ntaps > 1024 else 5e-6).max())
    serr = 0.0
    if p.stats_mode:
        delta = kw["stats"].double() - stats_before
        serr = check_stats(delta, got.to(out.dtype), B=B, F_out=F_out, T=T, n_out=n_out, stats_mode=p.stats_mode,
                           groups=p.groups)
    path = {0: "simt", 1: "wgmma-tf32", 2: "wgmma-f16"}[prec]
    tiles = B * (F_out if mode != cabi.TAPS_MIX else 1) * cdiv(T, 128) * cdiv(N, bn)
    amode = 3 if glu else p.act
    variant = (path, "mix" if mode == cabi.TAPS_MIX else f"a{amode}" + ("+res" if kw.get("residual") is not None else "") +
               ("+stats" if p.stats_mode else ""), bn if prec else "-", "f16" if o16 else ("f32/tf32" if rounding else "f32"))
    return dict(variant=variant, err=err, serr=serr, tiles=tiles, rounding=rounding, label=f"{label} K*taps={K * ntaps}")


# ------------------------------------------------------------------------------------------------ 1. tap-GEMM at multi-wave sizes
# geometries (K <= 96, <= 3 taps); T ragged: 401 and 270 and 145 leave whole empty 32-row quarters in the last row tile
GEOMS = {
    "1x1": dict(F_in=2, F_out=2, C1=96, T=401),
    "kt3_dil2": dict(F_in=2, F_out=2, C1=48, T=270, kt=3, dil_t=2, pad_t=2),
    "kf3_two_src": dict(F_in=3, F_out=3, C1=48, C2=32, T=333, kf=3, pad_f=1),
    # transposed conv whose output rows 8, 9 lie past the natural extent (F_in - 1) * stride + kf = 8: no valid tap, bias only
    "convt_bias_rows": dict(F_in=3, F_out=10, C1=64, T=145, mode=cabi.TAPS_CONVT, kf=4, stride_f=2),
}
# N per tile width (ragged 16-column chunks at 24, 40 and 200; two n-tiles at 176 and 200) and the GroupNorm groups of the
# statistics (None: per-row statistics); groups of N = 176 / 200 start inside a tile and straddle the n-tile boundary
WIDTHS = {32: dict(N=24, groups=1, groups_glu=None), 64: dict(N=40, groups=1, groups_glu=None),
          96: dict(N=176, groups=2, groups_glu=1), 128: dict(N=200, groups=5, groups_glu=None)}
# (operand kind, output type, amode, residual, statistics): every non-null entry of pick_kernel
VARIANTS = ([("tf32", "f32", a, r, s) for a in range(4) for r in (False, True) for s in (False, True)] +
            [("f16", "f32", a, False, False) for a in range(4)] + [("f16", "f32", 0, False, True)] +
            [(k, "f16", a, False, False) for k in ("f16", "tf32") for a in range(4)] +
            [(k, "f16", 0, r, s) for k in ("f16", "tf32") for r, s in ((True, False), (False, True))])
TC_SCALE = [(bn, v, list(GEOMS)[(i + j) % len(GEOMS)]) for j, bn in enumerate(WIDTHS) for i, v in enumerate(VARIANTS)]
# generic epilogue (lane = row, scattered stores): Nout % 4 != 0, an output row stride that is not a multiple of 4, colscale on a conv
GENERIC = [
    ("nout42_stats_res", 64, dict(N=42), ("tf32", "f32", 0, True, True), "kt3_dil2"),
    ("nout42_f16_stats", 64, dict(N=42), ("f16", "f16", 0, False, True), "1x1"),
    ("odd_row_stride", 128, dict(N=200, o_pad=1), ("tf32", "f32", 2, False, True), "kf3_two_src"),
    ("colscale_conv_gelu", 96, dict(N=176, colscale=True), ("f16", "f32", 1, False, False), "kt3_dil2"),
    ("colscale_convt_glu", 32, dict(N=24, colscale=True), ("tf32", "f32", 3, False, False), "convt_bias_rows"),
]


def _run_scale_case(gpu, emu, bn, variant, geom, N, groups=None, o_pad=0, colscale=False):
    kind, otype, amode, res, st = variant
    g = dict(GEOMS[geom])
    f16a, f16o = kind == "f16", otype == "f16"
    F_in, F_out, T, C1, C2 = g.pop("F_in"), g.pop("F_out"), g.pop("T"), g.pop("C1"), g.pop("C2", 0)
    mode = g.get("mode", cabi.TAPS_CONV)
    nslab = g.get("kf", 1) * (g.get("kt", 1) if mode == cabi.TAPS_CONV else 1)
    assert pick_bn(N) == bn
    glu = amode == 3
    n_out = N // 2 if glu else N
    B = cdiv(3 * n_sms(), F_out * cdiv(T, 128) * cdiv(N, bn)) + 1        # every CTA runs >= 3 tiles
    K = C1 + C2
    q = (lambda t: t.half()) if f16a else tf32_round
    w = pack_taps(rnd(N, K, nslab, seed=1, dev="cpu") / math.sqrt(K * min(nslab, 3))).cuda()
    w = w.half().float() if f16a else tf32_round(w)
    a1 = q(rnd(B, F_in, T, C1, seed=2))
    a2 = q(rnd(B, F_in, T, C2, seed=3)) if C2 else None
    kw = dict(a1=a1, a2=a2, C2=C2, F_in=F_in, bias=rnd(N, seed=4), act=amode if amode < 3 else cabi.ACT_NONE, glu=int(glu), **g)
    if res:
        kw["residual"] = rnd(B, F_out, T, n_out, seed=5).to(torch.float16 if f16o else torch.float32)
        kw["rnd"] = not f16o                                             # production rounds residual-stream outputs to TF32
    if glu and not colscale:
        kw["addend"] = rnd(F_out, n_out, seed=6)
    if colscale:
        kw["colscale"], kw["cs_s"] = rnd(B, T, N, seed=7), (T * N, N)
    if st:
        gr = groups
        kw["stats_mode"], kw["groups"] = (1, gr) if gr else (2, 1)
        nslots = B * gr if gr else B * F_out
        kw["stats"] = torch.zeros(nslots, 2, dtype=torch.float64, device="cuda")
    row = n_out + o_pad
    if o_pad:
        kw["o_s"] = (F_out * T * row, T * row, row)
    gpu._wk[w.data_ptr()] = tf32_round(w.permute(0, 2, 1).contiguous())
    gpu._wh[w.data_ptr()] = pack_kmajor_fp16(w)
    results = []
    try:
        gpu.precision = 2 if f16a else 1
        for reverse in (False, True):
            gpu.snake, gpu._flip = reverse, False                       # TG_REVERSE on the next launch iff snake
            out = torch.full((B, F_out, T, row), float("nan"), device="cuda", dtype=torch.float16 if f16o else torch.float32)
            if st:
                kw["stats"].zero_()
            n0 = len(gpu.lib.calls)
            gpu._gemm(out, w, B=B, F_out=F_out, T=T, N=N, C1=C1, **kw)
            torch.cuda.synchronize()
            (_, p, wptr), = gpu.lib.calls[n0:]
            assert p.precision == (2 if f16a else 1), "the wgmma kernel did not run"
            assert bool(p.flags & cabi.TG_REVERSE) == reverse
            r = check_launch(emu, gpu, (p, wptr), dict(kw, w=w), out, torch.zeros_like(kw["stats"]) if st else None)
            assert r["tiles"] >= 3 * n_sms()
            results.append(r)
    finally:
        gpu.precision, gpu.snake = 0, False
        gpu._wk.clear()
        gpu._wh.clear()
        gpu.lib.calls.clear()
    return results


@pytest.mark.parametrize("bn,variant,geom", TC_SCALE,
                         ids=[f"bn{bn}-{v[0]}-{v[1]}-a{v[2]}{'-res' if v[3] else ''}{'-stats' if v[4] else ''}-{g}" for bn, v, g in TC_SCALE])
def test_tapgemm_wgmma_multi_wave(engines, bn, variant, geom):
    gpu, emu = engines
    wd = WIDTHS[bn]
    res = _run_scale_case(gpu, emu, bn, variant, geom, wd["N"], groups=wd["groups_glu"] if variant[2] == 3 else wd["groups"])
    for r, order in zip(res, ("forward", "reverse")):
        print(f"{order}: {r['variant']} tiles {r['tiles']}: worst tile {r['err']:.3f} of its bar ({r['rounding'] or 'rel-L2'}), "
              f"stats {r['serr']:.3f}")
        assert r["err"] <= 1.0 and r["serr"] <= 1.0, (order, r)


@pytest.mark.parametrize("name,bn,shape,variant,geom", GENERIC, ids=[c[0] for c in GENERIC])
def test_tapgemm_wgmma_generic_epilogue_multi_wave(engines, name, bn, shape, variant, geom):
    gpu, emu = engines
    gr = None if variant[4] and shape["N"] % 8 else WIDTHS[bn]["groups"]
    res = _run_scale_case(gpu, emu, bn, variant, geom, shape["N"], groups=gr, o_pad=shape.get("o_pad", 0),
                          colscale=shape.get("colscale", False))
    for r, order in zip(res, ("forward", "reverse")):
        print(f"{name} {order}: {r['variant']} tiles {r['tiles']}: worst tile {r['err']:.3f} of its bar, stats {r['serr']:.3f}")
        assert r["err"] <= 1.0 and r["serr"] <= 1.0, (order, r)


# ------------------------------------------------------------------------------------------------ 2. LSTM recurrence, 16-sequence CTAs
def lstm_small_ctas(n_seq, H):
    """Whether aero_lstm_rec_fwd launches its 8-sequence CTAs (csrc/lstm_tc.cu, lstm_tc_launch): all of them resident at once."""
    return cdiv(n_seq, 8) * 2 <= n_sms() * (1 if H > 64 else 2)


def lstm_whh_from_rows(whh_rows, H):
    """The wgmma operand [2 * nM * 128, Kp] FP16 (gate rows re-ordered) -> [2, 4H, H] in PyTorch's gate order, as fp64."""
    src, ok = lstm_gate_reorder(H)
    n = src.shape[0]
    out = torch.zeros(2, 4 * H, H, dtype=torch.float64, device=whh_rows.device)
    for d in range(2):
        out[d][src[ok].to(whh_rows.device)] = whh_rows[d * n:(d + 1) * n][ok.to(whh_rows.device), :H].double()
    return out


def lstm_ref(gin, bias_pad, whh, *, rows, T, H, n_win, steps, stride, in_windowed, out_windowed):
    """fp64 BiLSTM recurrence (tests/cpu_emu.py's statement) on the kernel's operands: the gate inputs as stored, W_hh as the FP16
    values it holds and h rounded to FP16 before each recurrent product.  Returns the output in hout's layout, fp64."""
    G = 4 * H
    n_seq = rows * n_win
    gin = gin.double()
    bias_pad = bias_pad.double()
    if in_windowed:
        gi = gin.reshape(n_seq, steps, 2, G)
    else:
        pad_len = (n_win - 1) * stride + steps if n_win > 1 else steps
        padded = bias_pad.view(1, 1, 2 * G).expand(rows, pad_len, 2 * G).clone()
        padded[:, :T] = gin.reshape(rows, T, 2 * G)
        gi = (padded.unfold(1, steps, stride).permute(0, 1, 3, 2) if n_win > 1 else padded).reshape(n_seq, steps, 2, G)
    out = torch.zeros(n_seq, steps, 2, H, dtype=torch.float64, device=gin.device)
    for d in range(2):
        h = torch.zeros(n_seq, H, dtype=torch.float64, device=gin.device)
        c = torch.zeros_like(h)
        wt = whh[d].t()
        for t in (range(steps - 1, -1, -1) if d else range(steps)):
            g = gi[:, t, d] + h.half().double() @ wt
            i, f, gg, o = g.chunk(4, -1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
            h = torch.sigmoid(o) * torch.tanh(c)
            out[:, t, d] = h
    if out_windowed:
        return out.reshape(n_seq * steps, 2 * H)
    dst = torch.zeros(rows, T, 2 * H, dtype=torch.float64, device=gin.device)
    o4 = out.reshape(rows, n_win, steps, 2 * H)
    half = stride // 2
    for k in range(n_win):
        lo, hi = (0 if k == 0 else half), (steps if k == n_win - 1 else steps - half)
        f0, f1 = k * stride + lo, min(k * stride + hi, T)
        if f1 > f0:
            dst[:, f0:f1] = o4[:, k, lo:lo + (f1 - f0)]
    return dst.reshape(rows * T, 2 * H)


def lstm_block_errors(got, ref, seq_rows):
    """(worst, whole) rel-L2 against the fp64 reference rounded as the kernel stores h (to TF32, which it always does, or to
    FP16): worst over blocks of 16 sequences (windowed output, `seq_rows` = steps) or 16 clip rows (`seq_rows` = T) -- one
    16-sequence CTA's share of the output -- and over the whole tensor."""
    q = ref.half().double() if got.dtype == torch.float16 else tf32_round(ref.float()).double()
    d = (got.double() - q).pow(2).sum(1)
    r = ref.pow(2).sum(1)
    nb = cdiv(d.shape[0], 16 * seq_rows)
    d = Fn.pad(d, (0, nb * 16 * seq_rows - d.shape[0])).view(nb, -1).sum(1)
    r = Fn.pad(r, (0, nb * 16 * seq_rows - r.shape[0])).view(nb, -1).sum(1)
    return float((d / r.clamp_min(1e-30)).sqrt().max()), rel_l2(got, q)


# Against the reference rounded as stored, measured on an H100 80GB HBM3 (700 W): worst 16-sequence block 1.9e-4 (H = 96,
# 600 windowed sequences, FP16 gate inputs), <= 7.1e-5 on every recurrence of the benchmarked forward; fp32 and FP16 outputs
# alike.  What remains is fp32 accumulation, ex2 / rcp.approx in the gates, and the h whose FP16 operand rounding flips between
# the fp32 and the fp64 recurrence, carried forward by the cell state.  Bar: about 3x the worst measured block.
LSTM_BAR = 6e-4
# H, T, rows: n_seq = rows * ceil(T / 100) (windowed when T > 200) above the small-CTA threshold, ragged last CTA
LSTM_CASES = [(96, 501, 100), (96, 160, 613), (64, 230, 365), (64, 150, 1101), (48, 350, 270), (48, 120, 1090)]


def _lstm_run(gpu, gin1, gin2, b1, whh1r, whh2r, *, o16, prec, geom):
    H = geom["H"]
    dt = torch.float16 if o16 else torch.float32
    n_seq, steps = geom["rows"] * geom["n_win"], geom["steps"]
    kw = {k: v for k, v in geom.items()}
    gpu.precision = prec
    try:
        h1 = torch.full((n_seq * steps, 2 * H), float("nan"), device="cuda", dtype=dt)
        gpu._lstm_rec(gin1, b1, whh1r, h1, in_windowed=0, out_windowed=1, tc=True, **kw)
        h2 = torch.full((geom["rows"] * geom["T"], 2 * H), float("nan"), device="cuda", dtype=dt)
        gpu._lstm_rec(gin2, b1, whh2r, h2, in_windowed=1, out_windowed=0, tc=True, **kw)
        torch.cuda.synchronize()
    finally:
        gpu.precision = 0
    return h1, h2


@pytest.mark.parametrize("gin16", [False, True], ids=["gin32", "gin16"])
@pytest.mark.parametrize("H,T,rows", LSTM_CASES)
def test_lstm_wgmma_16_sequence_ctas(engines, H, T, rows, gin16):
    """Both recurrent calls of a BLSTM (windowed output, then windowed input) on the 16-sequence CTA variants, writing fp32
    (rounded to TF32) and FP16, reading fp32 or FP16 gate inputs, against the fp64 recurrence on the kernel's operands."""
    gpu, _ = engines
    steps, stride, n_win = (200, 100, cdiv(T, 100)) if T > 200 else (T, 0, 1)
    n_seq = rows * n_win
    assert not lstm_small_ctas(n_seq, H) and n_seq % 16, (n_seq, H)
    gdt = torch.float16 if gin16 else torch.float32
    gin1 = rnd(rows * T, 8 * H, seed=1).to(gdt)
    gin2 = rnd(n_seq * steps, 8 * H, seed=5).to(gdt)
    b1 = rnd(8 * H, seed=2) * 0.3
    src, ok = lstm_gate_reorder(H)

    def rows_(w):
        return lstm_whh_fp16(torch.cat([torch.where(ok[:, None], w[d][src], torch.zeros(())) for d in range(2)], 0)).cuda()
    whh1r = rows_(rnd(2, 4 * H, H, seed=3, dev="cpu") / math.sqrt(H))
    whh2r = rows_(rnd(2, 4 * H, H, seed=4, dev="cpu") / math.sqrt(H))
    geom = dict(rows=rows, T=T, H=H, n_win=n_win, steps=steps, stride=stride)
    n0 = len(gpu.lib.calls)
    h32 = _lstm_run(gpu, gin1, gin2, b1, whh1r, whh2r, o16=False, prec=1, geom=geom)
    h16 = _lstm_run(gpu, gin1, gin2, b1, whh1r, whh2r, o16=True, prec=2, geom=geom)
    calls = gpu.lib.calls[n0:]
    gpu.lib.calls.clear()
    assert [c[1].precision for c in calls] == [1] * 4 and all(c[0] == "lstm" for c in calls)
    ref1 = lstm_ref(gin1, b1, lstm_whh_from_rows(whh1r, H), in_windowed=0, out_windowed=1, **geom)
    ref2 = lstm_ref(gin2, b1, lstm_whh_from_rows(whh2r, H), in_windowed=1, out_windowed=0, **geom)
    for tag, h, ref in (("fp32 layer-1", h32[0], ref1), ("fp32 layer-2", h32[1], ref2),
                        ("fp16 layer-1", h16[0], ref1), ("fp16 layer-2", h16[1], ref2)):
        assert torch.isfinite(h).all(), tag
        worst, whole = lstm_block_errors(h, ref, steps if "1" in tag else T)
        print(f"lstm 16-seq H={H} T={T} n_seq={n_seq} {'gin16' if gin16 else 'gin32'} {tag}: worst block {worst:.2e}, whole {whole:.2e}")
        assert worst < LSTM_BAR, (tag, worst)
    # the FP16 output is the fp32 result of the same recurrence, rounded to nearest once: the two runs share every operand
    for a, b in zip(h16, h32):
        assert torch.equal(a, b.half()), "FP16 hout is not the round-to-nearest of the fp32 result"


# ------------------------------------------------------------------------------------------------ 3. TF32 weight gradient at training batch
def wgrad_split(B, F_out, T, N, C1, C2, nslab):
    """(splits, d_fo, d_b) that aero_tapgemm_wgrad chooses on the tensor cores (csrc/wgrad_tc.cu, wgrad_tc_launch)."""
    tiles_t = cdiv(T, 32)
    nb = cdiv(C1, 32) + cdiv(C2, 32)
    items = cdiv(nb, 4) * cdiv(N, 128) * nslab
    max_splits = max(B * F_out * tiles_t // 8, 1)
    slots = 2 * n_sms()
    lo = max(min(cdiv(2 * slots, items), max_splits), 1)
    hi = max(min(cdiv(6 * slots, items), max_splits, 65535), lo)
    splits, best = lo, 0.0
    for sp in range(lo, hi + 1):
        ctas = items * sp
        eff = ctas / (cdiv(ctas, slots) * slots)
        if eff > best + 0.02:
            best, splits = eff, sp
    d_row = splits // tiles_t
    return splits, d_row % F_out, d_row // F_out


# name, B, geometry, F_in, F_out, T, T_in, C1, C2, N, channel slice of a wider tensor (width, offset)
WGRAD_CASES = [
    ("k3x3_two_src_b8", 8, dict(kf=3, kt=3, pad_f=1, pad_t=1), 3, 3, 150, 150, 48, 112, 200, None),
    ("k3x3_two_src_b16", 16, dict(kf=3, kt=3, pad_f=1, pad_t=1), 3, 3, 150, 150, 48, 112, 200, None),
    ("convt_k8s4_b16", 16, dict(mode=cabi.TAPS_CONVT, kf=8, stride_f=4, f_off=2), 4, 14, 70, 70, 96, 0, 48, None),
    ("convt_k8s2_c160_b8", 8, dict(mode=cabi.TAPS_CONVT, kf=8, stride_f=2), 3, 6, 61, 61, 160, 0, 72, None),
    ("k5_slice_b16", 16, dict(kt=5), 5, 5, 79, 83, 32, 0, 48, (64, 16)),
]


@pytest.mark.parametrize("name,B,geo,F_in,F_out,T,T_in,C1,C2,N,slc", WGRAD_CASES, ids=[c[0] for c in WGRAD_CASES])
def test_wgrad_tc_training_batch(engines, name, B, geo, F_in, F_out, T, T_in, C1, C2, N, slc):
    """aero_tapgemm_wgrad on the tensor cores where one split-K stride spans more than a batch item (the d_b carry of
    WtWalker::next), on TF32-exact operands, against an fp64 einsum: rel-L2 <= 2e-5 per slab."""
    gpu, _ = engines
    lib = gpu.lib
    mode = geo.get("mode", cabi.TAPS_CONV)
    kf, kt, stride_f = geo.get("kf", 1), geo.get("kt", 1), geo.get("stride_f", 1)
    nslab = kf * kt if mode == cabi.TAPS_CONV else kf
    splits, d_fo, d_b = wgrad_split(B, F_out, T, N, C1, C2, nslab)
    assert d_b > 0, (splits, d_fo, d_b)
    if slc:
        width, off = slc
        a1 = tf32_round(rnd(B, F_in, T_in, width, seed=1))[..., off:off + C1]
        a1_s = (F_in * T_in * width, T_in * width, width)
    else:
        a1 = tf32_round(rnd(B, F_in, T_in, C1, seed=1))
        a1_s = (F_in * T_in * C1, T_in * C1, C1)
    a2 = tf32_round(rnd(B, F_in, T_in, C2, seed=2)) if C2 else None
    a2_s = (F_in * T_in * C2, T_in * C2, C2) if C2 else (0, 0, 0)
    dy = tf32_round(rnd(B, F_out, T, N, seed=3))
    p = cabi.TapGemmParams(B, F_out, T, N, F_in, T_in, C1, C2, mode, kf, kt, stride_f, geo.get("pad_f", 0), geo.get("dil_t", 1),
                           geo.get("pad_t", 0), geo.get("f_off", 0), cabi.ACT_NONE, 0, 0, 1, *a1_s, *a2_s, 0,
                           F_out * T * N, T * N, N, 0, 0, 0, 0, 0, 1, 0)
    P = lambda t: None if t is None else C.c_void_p(t.data_ptr())          # noqa: E731
    assert lib.aero_tapgemm_wgrad_tc_eligible(C.byref(p), P(a1), P(a2), P(dy)) == 1
    K = C1 + C2
    dw = torch.zeros(N, K, nslab, device="cuda")                             # PyTorch's [N][K][kf * kt] order
    cabi.check(lib.aero_tapgemm_wgrad(P(a1), P(a2), P(dy), P(dw), C.byref(p), K * nslab, nslab, 1,
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream)), lib)
    torch.cuda.synchronize()
    A = torch.cat([a1] + ([a2] if C2 else []), -1).double()
    Y = dy.double()
    ref = torch.zeros(N, K, nslab, dtype=torch.float64, device="cuda")
    for slab in range(nslab):
        for fo in range(F_out):
            if mode == cabi.TAPS_CONV:
                jf, jt = divmod(slab, kt)
                fi, dt = fo * stride_f + jf - geo.get("pad_f", 0), jt * geo.get("dil_t", 1) - geo.get("pad_t", 0)
            else:
                fof = fo + geo.get("f_off", 0)
                if fof % stride_f != slab % stride_f:
                    continue
                fi, dt = fof // stride_f - slab // stride_f, 0
            lo, hi = max(0, -dt), min(T, T_in - dt)
            if 0 <= fi < F_in and hi > lo:
                ref[:, :, slab] += torch.einsum("btk,btn->nk", A[:, fi, lo + dt:hi + dt], Y[:, fo, lo:hi])
    errs = [rel_l2(dw[:, :, s], ref[:, :, s]) for s in range(nslab)]
    print(f"wgrad tf32 {name}: splits {splits} (d_fo {d_fo}, d_b {d_b}); worst slab rel_l2 {max(errs):.2e}")
    assert max(errs) <= 2e-5, errs


# ------------------------------------------------------------------------------------------------ 4. per-launch replay of the benchmark
@pytest.fixture(scope="module")
def bench_model():
    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs("aero_4-16_512_64")).eval()
    m.load_state_dict(trained_like_(m.state_dict()))
    return m.cuda()


@pytest.mark.parametrize("precision", [2, 1])
def test_benchmark_forward_every_launch(engines, bench_model, precision):
    """AeroEngine.forward on the benchmarked workload (aero_4-16_512_64, trained-like weights, 32 x 2 s), eager: every tap-GEMM
    and every LSTM recurrence is checked right after it runs, against fp64 on that launch's own inputs (snapshotted before the
    call: the BLSTM output projection adds into its own input, and statistics slots accumulate)."""
    _, emu = engines
    eng = AeroEngine(bench_model)
    eng.use_graph = False
    eng.precision = precision
    eng.lib = RecordingLib(eng.lib)
    rows = defaultdict(lambda: [0, 0.0, 0.0, ""])
    checked, lstm_rows = [], []
    gemm0, lstm0 = eng._gemm, eng._lstm_rec

    def gemm(out, w, **kw):
        snap = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in kw.items()}
        stats_before = kw["stats"].double().clone() if kw.get("stats") is not None else None
        n0 = len(eng.lib.calls)
        gemm0(out, w, **kw)
        torch.cuda.synchronize()
        (_, p, wptr), = eng.lib.calls[n0:]
        snap["stats"] = kw.get("stats")
        r = check_launch(emu, eng, (p, wptr), dict(snap, w=w), out, stats_before, label=kw.get("tag") or eng._wname.get(w.data_ptr()))
        row = rows[r["variant"]]
        row[0] += 1
        if r["err"] >= row[1]:
            row[1], row[3] = r["err"], r["label"]
        row[2] = max(row[2], r["serr"])
        checked.append(r)
        return out

    def lstm(gin, bias_pad, whh, hout, **kw):
        g = gin.clone()
        n0 = len(eng.lib.calls)
        lstm0(gin, bias_pad, whh, hout, **kw)
        torch.cuda.synchronize()
        (_, p, _), = eng.lib.calls[n0:]
        assert kw.get("tc"), "the wgmma recurrence did not run"
        H = kw["H"]
        geom = {k: kw[k] for k in ("rows", "T", "H", "n_win", "steps", "stride", "in_windowed", "out_windowed")}
        ref = lstm_ref(g, bias_pad, lstm_whh_from_rows(whh, H), **geom)
        worst, whole = lstm_block_errors(hout, ref, kw["steps"] if kw["out_windowed"] else kw["T"])
        n_seq = kw["rows"] * kw["n_win"]
        lstm_rows.append((H, n_seq, hout.dtype, gin.dtype, lstm_small_ctas(n_seq, H), worst, whole))

    eng._gemm, eng._lstm_rec = gemm, lstm
    mix = torch.randn(32, bench_model.in_channels, 8000, generator=torch.Generator().manual_seed(SEED)).cuda()
    y = eng.forward(mix)
    torch.cuda.synchronize()
    assert torch.isfinite(y).all()
    print(f"\nprecision {precision}: {len(checked)} tap-GEMM launches, {len(lstm_rows)} LSTM recurrences, {n_sms()} SMs")
    print(f"{'path':<11} {'epilogue':<16} {'BN':>4} {'out':<9} {'launches':>8} {'worst tile / bar':>17} {'stats / bar':>12}  worst launch")
    for key in sorted(rows, key=str):
        n, e, s, lab = rows[key]
        print(f"{key[0]:<11} {key[1]:<16} {key[2]!s:>4} {key[3]:<9} {n:>8} {e:>17.3f} {s:>12.3f}  {lab}")
    for H, n_seq, hd, gd, small, worst, whole in lstm_rows:
        print(f"lstm H={H} n_seq={n_seq} {'8' if small else '16'}-sequence CTAs, hout {hd}, gin {gd}: worst block {worst:.2e}, "
              f"whole {whole:.2e}")
    for key, (n, e, s, _) in rows.items():
        assert e <= 1.0 and s <= 1.0, (key, e, s)
    assert all(worst < LSTM_BAR for *_, worst, _ in lstm_rows)
    assert lstm_rows and not any(small for _, _, _, _, small, _, _ in lstm_rows), "production LSTM launches use 16-sequence CTAs"
    assert any(r["tiles"] > n_sms() and r["variant"][0] != "simt" for r in checked)
    if precision == 2:
        assert any(r["variant"][0] == "wgmma-f16" for r in checked)
