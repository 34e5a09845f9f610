"""-m gpu: GroupNorm inputs whose group mean is large next to their spread.

Every GroupNorm of AERO subtracts its group mean, so adding a constant to every output channel of one group of the convolution
that feeds it (to that conv's bias) leaves the model's function unchanged: the unshifted oracle, goldens and fp64 gradients stay
the reference.  `util.shifted` gives each group of each such conv its own constant of size c .. 2.11 c, of alternating sign and
mostly not a multiple of 1/8, so the engine's per-group bias centring (engine.center_groups) must use the right groups and
leaves a residual offset in what the kernels store.  The parity tests run on `trained_like_` weights, whose conv biases keep PyTorch's default init (|b| < 0.1)
on white-noise input, so none of them puts a GroupNorm input where a trained network routinely has it: a group mean larger
than the group's spread.  That is where FP16 storage of the pre-normalisation values (`AeroEngine.raw16`) keeps only the low
bits of the spread, and where statistics of the form E[x^2] - E[x]^2 built from fp32 partial sums cancel.

The layers are found from the model itself: the oracle's forward is traced, and a convolution whose output is the input of a
group_norm call is a pre-normalisation layer (encoder conv -> norm1, rewrite -> norm2, decoder rewrite -> norm1,
conv_tr -> norm2, DConv conv1.0 / conv2.0 -> conv1.1 / conv2.1)."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from util import SEED, pre_norm_convs, rel_l2, shifted, trained_like_, white_noise

from aero_b200 import Aero, aero_kwargs, cabi
from aero_b200.engine import AeroEngine, _ptr, pack_kmajor_fp16, pack_taps, tf32_round

pytestmark = pytest.mark.gpu
TOL = 1e-3                  # the project's end-to-end bar for the tensor-core engines
TOL_FP32 = 1e-5             # precision 0 (exact fp32 kernels)
SHIFTS = [0.0, 0.3, 1.0, 3.0, 10.0]
U = 2.0 ** -24              # fp32 unit roundoff


def build(exp):
    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs(exp)).eval()
    m.load_state_dict(trained_like_(m.state_dict()))
    return m


@pytest.fixture(scope="module")
def shift_case():
    """Per experiment: (model on the GPU, its unshifted state_dict on the CPU, pre-normalisation layers)."""
    cache = {}

    def get(exp):
        if exp not in cache:
            m = build(exp)
            sd0 = {k: v.clone() for k, v in m.state_dict().items()}
            layers = pre_norm_convs(m)
            cache[exp] = (m.cuda(), sd0, layers)
        return cache[exp]
    return get


def test_pre_norm_layers_are_found_from_the_model(shift_case):
    m, sd, layers = shift_case("aero_4-16_512_64")
    keys = [b for _, b, _ in layers]
    ng = m.geom.kw["norm_groups"]
    n_norm = sum(1 for g in m.geom.layers if g.norm)
    n_dconv = sum(abs(m.geom.kw["dconv_depth"]) for g in m.geom.layers if g.dconv)
    # two GroupNorms per encoder and per decoder layer with norm, two per DConv layer
    assert len(keys) == len(set(keys)) == 4 * n_norm + 2 * n_dconv
    assert all(g == 1 for _, b, g in layers if ".dconv." in b) and all(g == ng for _, b, g in layers if ".dconv." not in b)


def _forward(m, sd, mix, precision):
    m.load_state_dict(sd)
    eng = m._engine()
    eng.precision = precision
    eng.use_graph = False
    out = m(mix.cuda())
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("exp,C,L", [("aero_4-16_512_64", 1, 1600), ("aero_11-44_512_64", 2, 2750)])
def test_forward_is_invariant_to_pre_norm_bias_shifts(shift_case, exp, C, L, precision):
    """Engine defaults at each precision, biases shifted per group by util.shifted, against the oracle's forward of the
    UNSHIFTED weights.  Bars: 1e-3 at precisions 1 / 2, 1e-5 at precision 0.  At precisions 0 and 1 (fp32 GroupNorm inputs) a
    shift may also not double the error against the exact (fp64) function of the weights the engine was given: b + c_i rounded
    to fp32 is itself a slightly different model (~1e-6 at c = 10), which is not the engine's error."""
    from oracle import aero_oracle as O
    m, sd0, layers = shift_case(exp)
    mix = white_noise((1, C, L))

    def exact(sd):
        with torch.no_grad():
            return O.aero_forward({k: v.double() for k, v in sd.items()}, m.geom, mix.double())
    with torch.no_grad():
        ref = O.aero_forward({k: v.clone() for k, v in sd0.items()}, m.geom, mix)
    errs, own = {}, {}
    for c in SHIFTS:
        sd = shifted(sd0, layers, c)
        out = _forward(m, sd, mix, precision)
        errs[c] = rel_l2(out, ref)
        if precision in (0, 1):
            own[c] = rel_l2(out, exact(sd))
    m.load_state_dict(sd0)
    print(f"{exp} precision {precision}: rel_l2 vs unshifted oracle by bias shift: " +
          " ".join(f"c={c:g}: {e:.2e}" for c, e in errs.items()) +
          ("; vs fp64 function of the shifted weights: " + " ".join(f"{e:.2e}" for e in own.values()) if own else ""))
    assert max(errs.values()) < (TOL_FP32 if precision == 0 else TOL), errs
    if own:
        assert max(own.values()) < 2 * own[0.0], own


def weight_offset_keys(layers):
    """One pre-normalisation conv per stage whose input comes out of a GELU: the first DConv conv1 of each encoder layer
    (its input is GELU(norm1(conv))) and the rewrite of each decoder layer after the first (its input is GELU of the previous
    decoder layer's output, next to the skip)."""
    keys = [w for w, _, _ in layers if w.endswith(".dconv.layers.0.conv1.0.weight")]
    keys += [w for w, _, _ in layers if w.startswith("decoder.") and ".rewrite." in w and not w.startswith("decoder.0.")]
    return keys


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("exp,C,L", [("aero_4-16_512_64", 1, 1600), ("aero_11-44_512_64", 2, 2750)])
def test_forward_with_a_common_weight_offset(shift_case, exp, C, L, precision):
    """A common positive offset (one weight standard deviation) on every weight of one pre-normalisation conv per stage whose
    input follows a GELU: the group mean now comes from the input (GELU outputs have a positive mean), several times the group's
    spread.  Not shift invariant, so the reference is the oracle's forward of the same modified weights.  Bars as above."""
    from oracle import aero_oracle as O
    m, sd0, layers = shift_case(exp)
    keys = weight_offset_keys(layers)
    assert any(k.startswith("encoder.") for k in keys) and any(k.startswith("decoder.") for k in keys), keys
    sd = {k: (v + v.std() if k in keys else v.clone()) for k, v in sd0.items()}
    mix = white_noise((1, C, L))
    with torch.no_grad():
        ref = O.aero_forward({k: v.clone() for k, v in sd.items()}, m.geom, mix)
        ref0 = O.aero_forward({k: v.clone() for k, v in sd0.items()}, m.geom, mix)
    err = rel_l2(_forward(m, sd, mix, precision), ref)
    err0 = rel_l2(_forward(m, sd0, mix, precision), ref0)
    m.load_state_dict(sd0)
    print(f"{exp} precision {precision}: weight offset rel_l2 vs oracle {err:.2e} (without offset {err0:.2e}); "
          f"output moved by the offset {rel_l2(ref, ref0):.2e}")
    assert rel_l2(ref, ref0) > 1e-2            # the offset changes the function: the comparison is not vacuous
    assert err < (TOL_FP32 if precision == 0 else TOL), err
    if precision in (0, 1):
        assert err < 2 * err0, (err, err0)


@pytest.mark.parametrize("c", [1.0, 10.0])
@pytest.mark.parametrize("precision", [0, 1, 2])
def test_ragged_batch_with_shifted_biases(shift_case, precision, c):
    """enhance.enhance_batch on clips of different lengths, pre-normalisation biases shifted per group (util.shifted): the
    GroupNorm statistics of a ragged batch come from aero_masked_stats_fwd instead of the GEMM epilogue.  Each clip against its own single-clip
    forward, at the tolerances of test_gpu_ragged.test_ragged_equals_single_clip, and against the unshifted oracle."""
    from oracle import aero_oracle as O
    from test_ragged_host import lengths_for_frames
    from aero_b200.enhance import enhance_batch
    m, sd0, layers = shift_case("aero_4-16_512_64")
    m.load_state_dict(shifted(sd0, layers, c))
    eng = m._engine()
    eng.precision = precision
    eng.use_graph = False
    try:
        lengths = lengths_for_frames(m, [101, 201, 300, 700])
        sigs = [white_noise((1, n), seed=20 + i) for i, n in enumerate(lengths)]
        outs = enhance_batch(m, [s.cuda() for s in sigs])
        worst = worst_ref = 0.0
        for s, got in zip(sigs, outs):
            want = m(s[None].cuda())[0]
            worst = max(worst, rel_l2(got.cpu(), want.cpu()))
            with torch.no_grad():
                ref = O.aero_forward({k: v.clone() for k, v in sd0.items()}, m.geom, s[None])[0]
            worst_ref = max(worst_ref, rel_l2(got.cpu(), ref))
    finally:
        m.load_state_dict(sd0)
    print(f"precision {precision}, bias shift {c:g}: worst rel_l2 ragged vs single clip {worst:.2e}, vs unshifted oracle {worst_ref:.2e}")
    assert worst < (1e-5 if precision == 0 else 5e-4)
    assert worst_ref < (TOL_FP32 if precision == 0 else TOL)


# ------------------------------------------------------------------------------------------------ training
# bars of test_gpu_train / test_gpu_train_tc for the non-strict golden t1: (output, all gradients together, worst parameter,
# whether a third of the parameters must be within 1e-3)
TRAIN_BARS = {0: (2e-5, 5e-3, 5e-2, True), 1: (2e-3, 1e-1, 0.5, False), 3: (2e-5, 1e-2, 5e-2, True)}


@pytest.mark.parametrize("c", [1.0, 10.0])
@pytest.mark.parametrize("train_precision", [0, 1, 3])
def test_training_gradients_with_shifted_biases(golden_dir, train_precision, c):
    """The golden case t1_4-16_hop256 with the pre-normalisation biases shifted per group (util.shifted): the function, and so its gradient at the
    shifted point, is the unshifted one, and the fp64 golden gradients of the reference hold unchanged."""
    from test_gpu_train import GRAD_TOL, cotangent, grad_report
    g = np.load(os.path.join(golden_dir, "t1_4-16_hop256.npz"))
    m = build(str(g["exp"]))
    m.load_state_dict(shifted(m.state_dict(), pre_norm_convs(m), c))
    m = m.cuda().train()
    m.train_precision = train_precision
    mix = white_noise((int(g["B"]), m.in_channels, int(g["L"]))).cuda()
    out = m(mix)
    flat = out.detach().reshape(-1).cpu()
    e_out = rel_l2(flat[torch.from_numpy(g["out_idx"].astype(np.int64))], g["out_val"])
    R = cotangent(tuple(out.shape), SEED).cuda()
    ((out * R).sum() / out.numel()).backward()
    torch.cuda.synchronize()
    rows, total = grad_report(m, g)
    ok = sum(1 for r in rows if r[0] < GRAD_TOL)
    print(f"train_precision {train_precision}, bias shift {c:g}: output rel_l2 {e_out:.3e}; all gradients together {total:.3e}; "
          f"{ok}/{len(rows)} within {GRAD_TOL:g}; worst {rows[0][0]:.3e} {rows[0][1]}")
    b_out, b_total, b_worst, third = TRAIN_BARS[train_precision]
    assert e_out < b_out and total < b_total and rows[0][0] < b_worst, (e_out, total, rows[:3])
    if third:
        assert ok >= len(rows) / 3, (ok, len(rows))


# ------------------------------------------------------------------------------------------------ kernel level
# Statistics against fp64 two-pass values of the STORED outputs (include/aero_b200.h: "statistics of the stored value").
# A group of spread sigma carries an offset k * sigma.  The epilogues add fp32 partial sums of x and x^2 and finish in fp64, so
# sum(x^2) carries a relative error of order u (u = 2^-24) of (1 + k^2) * sigma^2 per element, and the variance
# E[x^2] - E[x]^2 an error of order u * (1 + k^2) relative to sigma^2.  Each test below states its bar as a constant times
# u * (1 + k^2).  The constants are the largest ratio measured on an H100 80GB HBM3 (700 W) over every shape, path, op and k
# here (k >= 3, where the offset term dominates any fixed part of the bar), rounded up to the next power of two:
STATS_C = 2        # tap-GEMM epilogues and aero_masked_stats_fwd: 1.1 (variance), 0.5 (mean, against u * (1 + k))
NORM_ACT_C = 0.5   # aero_norm_act_fwd: 0.27
TRAIN_C = 2        # aero_norm_act_train_fwd / _bwd: 1.04
KS = [0, 3, 30, 300]
GEMM_SHAPES = [   # narrow and wide N (the wgmma path's BN follows N), per-group (stats_mode 1) and per-row (stats_mode 2)
    ("narrow_groups", dict(B=2, F_out=4, T=130, N=64, C1=48, kt=3, pad_t=1, stats_mode=1, groups=4)),
    ("wide_groups", dict(B=2, F_out=3, T=101, N=256, C1=48, kf=3, kt=3, pad_f=1, pad_t=1, stats_mode=1, groups=4)),
    ("narrow_rows", dict(B=2, F_out=3, T=257, N=32, C1=48, kt=3, dil_t=2, pad_t=2, stats_mode=2)),
    ("wide_rows", dict(B=1, F_out=3, T=200, N=256, C1=64, stats_mode=2)),
]
PATHS = {"simt": (0, False), "tf32": (1, False), "f16": (2, True)}    # engine precision, FP16 sources and outputs


@pytest.fixture(scope="module")
def gpu_engine():
    torch.manual_seed(SEED)
    eng = AeroEngine(Aero(**aero_kwargs("aero_4-16_512_256")).eval().cuda())
    eng.precision = 0
    return eng


def _slots(x, cfg):
    """fp64 view of x [B, F, T, N] grouped as its statistics slots: [slots, values]."""
    B, Fo, T, N = x.shape
    x = x.double().cpu()
    if cfg["stats_mode"] == 1:
        g = cfg["groups"]
        return x.reshape(B, Fo * T, g, N // g).permute(0, 2, 1, 3).reshape(B * g, -1)
    return x.reshape(B * Fo, -1)


def _offset_gemm(eng, cfg, path, k):
    """One tap-GEMM on `path` whose output groups carry a mean of k times their spread (through the bias, as in the model)."""
    precision, f16 = PATHS[path]
    cfg = dict(cfg)
    B, Fo, T, N, C1 = (cfg.pop(n) for n in ("B", "F_out", "T", "N", "C1"))
    nslab = cfg.get("kf", 1) * cfg.get("kt", 1)
    q = (lambda t: t.half().float()) if f16 else (tf32_round if precision == 1 else (lambda t: t))
    w = q(pack_taps(torch.randn(N, C1, nslab, generator=torch.Generator().manual_seed(1)) / math.sqrt(C1 * nslab))).cuda()
    a = q(torch.randn(B, Fo, T, C1, generator=torch.Generator().manual_seed(2))).cuda()
    gsz = N // cfg["groups"] if cfg["stats_mode"] == 1 else N
    sign = torch.tensor([1.0, -1.0]).repeat_interleave(gsz).repeat(N // (2 * gsz) + 1)[:N]
    bias = (k * sign + 0.1 * torch.randn(N, generator=torch.Generator().manual_seed(4))).cuda()
    out = torch.empty(B, Fo, T, N, device="cuda", dtype=torch.float16 if f16 else torch.float32)
    nslots = B * cfg["groups"] if cfg["stats_mode"] == 1 else B * Fo
    stats = torch.zeros(nslots, 2, dtype=torch.float64, device="cuda")
    eng.precision = precision
    eng._wk[w.data_ptr()] = tf32_round(w.permute(0, 2, 1).contiguous())
    eng._wh[w.data_ptr()] = pack_kmajor_fp16(w)
    try:
        p = cabi.TapGemmParams(B, Fo, T, N, Fo, T, C1, 0, cabi.TAPS_CONV, cfg.get("kf", 1), cfg.get("kt", 1), 1, cfg.get("pad_f", 0),
                               cfg.get("dil_t", 1), cfg.get("pad_t", 0), 0, 0, 0, cfg["stats_mode"], cfg.get("groups", 1),
                               Fo * T * C1, T * C1, C1, 0, 0, 0, 0, Fo * T * N, T * N, N, 0, 0, 0, 0, 0, 0,
                               cabi.TG_A_F16 | cabi.TG_OUT_F16 if f16 else 0)
        if precision:
            assert eng.lib.aero_tapgemm_tc_eligible(C.byref(p)) == 1, "the case must run on the wgmma path"
        eng._gemm(out, w, a1=a.half() if f16 else a, B=B, F_out=Fo, T=T, N=N, C1=C1, bias=bias, stats=stats, **cfg)
        torch.cuda.synchronize()
    finally:
        eng.precision = 0
        eng._wk.clear()
        eng._wh.clear()
    return out, stats


def _check_stats(stats, x_slots, k, what, count=None):
    """Mean / variance from {sum, sumsq} slots (over `count` values each) against fp64 two-pass values of x_slots."""
    n = x_slots.shape[1] if count is None else count
    mean_ref, var_ref = x_slots.mean(1), x_slots.var(1, unbiased=False)
    st = stats.cpu()
    mean, var = st[:, 0] / n, st[:, 1] / n - (st[:, 0] / n) ** 2
    sd = var_ref.sqrt()
    e_mean = float(((mean - mean_ref).abs() / sd).max())
    e_var = float(((var - var_ref).abs() / var_ref).max())
    print(f"{what} k={k}: mean error {e_mean:.2e} sigma ({e_mean / (U * (1 + k)):.1f} u(1+k)), variance error {e_var:.2e} "
          f"({e_var / (U * (1 + k * k)):.1f} u(1+k^2))")
    assert float((mean_ref.abs() / sd).min()) > 0.5 * k          # the offset is there
    assert e_mean < STATS_C * U * (1 + k), (what, e_mean)
    assert e_var < STATS_C * U * (1 + k * k), (what, e_var)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("name,cfg", GEMM_SHAPES, ids=[s[0] for s in GEMM_SHAPES])
def test_tapgemm_statistics_with_group_offsets(gpu_engine, name, cfg, path, k):
    """The statistics slots of a tap-GEMM whose output groups carry an offset of k sigma give the mean and variance of the
    stored outputs.  Bars: |mean - mean_ref| < STATS_C u (1 + k) sigma and |var - var_ref| < STATS_C u (1 + k^2) var_ref,
    against fp64 two-pass values."""
    out, stats = _offset_gemm(gpu_engine, cfg, path, k)
    _check_stats(stats, _slots(out, cfg), k, f"{name} {path}")


def _groupnorm_ref(x, gamma, beta, groups, scope, op, a=None, scale=None, resid=None):
    """fp64 GroupNorm (two-pass statistics) + op of x [B, F, T, C], as include/aero_b200.h states aero_norm_act_fwd."""
    B, Fi, T, Cc = x.shape
    xd = x.double()
    if scope == 1:
        g = xd.view(B, Fi * T, groups, Cc // groups)
        mu, var = g.mean((1, 3), keepdim=True), g.var((1, 3), unbiased=False, keepdim=True)
    else:
        g = xd.view(B * Fi, 1, 1, T * Cc)
        mu, var = g.mean(3, keepdim=True), g.var(3, unbiased=False, keepdim=True)
    y = ((g - mu) / torch.sqrt(var + 1e-5)).reshape(B, Fi, T, Cc) * gamma.double() + beta.double()
    if op == cabi.NA_GELU:
        return F.gelu(y)
    if op == cabi.NA_RELU:
        return y.clamp_min(0)
    if op == cabi.NA_SNAKE:
        ad = a.double().view(1, Fi, 1, 1)
        return y + torch.sin(ad * y) ** 2 / ad
    if op in (cabi.NA_GLU, cabi.NA_GLU_SCALE_RES):
        h = Cc // 2
        y = y[..., :h] * torch.sigmoid(y[..., h:])
        return y if op == cabi.NA_GLU else resid.double() + scale.double() * y
    return y


NA_OPS = {1: [cabi.NA_NONE, cabi.NA_GELU, cabi.NA_GLU], 2: [cabi.NA_RELU, cabi.NA_GELU, cabi.NA_SNAKE, cabi.NA_GLU_SCALE_RES]}


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("storage", ["f32", "f32_to_f16", "f16"])
@pytest.mark.parametrize("scope", [1, 2])
def test_norm_act_on_offset_groups(gpu_engine, scope, storage, k):
    """aero_norm_act_fwd on tap-GEMM outputs with offset groups and the statistics that GEMM produced, against an fp64
    GroupNorm of the stored values, for each op and storage combination the forward uses (fp32 -> fp32, fp32 -> FP16,
    FP16 -> FP16).  Bar: rel-L2 within 4e-6 (fp32 output) or 4e-4 (FP16 output, one rounding) + NORM_ACT_C u (1 + k^2)."""
    cfg = GEMM_SHAPES[0][1] if scope == 1 else GEMM_SHAPES[2][1]
    out, stats = _offset_gemm(gpu_engine, cfg, "f16" if storage == "f16" else "tf32", k)
    B, Fi, T, Cc = out.shape
    groups = cfg["groups"] if scope == 1 else 1
    gen = torch.Generator().manual_seed(5)
    gamma, beta = 1 + 0.2 * torch.randn(Cc, generator=gen), 0.1 * torch.randn(Cc, generator=gen)
    a = torch.rand(Fi, generator=gen) * 8 + 0.2
    scale = torch.randn(Cc // 2, generator=gen)
    o16 = storage != "f32"
    for op in NA_OPS[scope]:
        co = Cc // 2 if op in (cabi.NA_GLU, cabi.NA_GLU_SCALE_RES) else Cc
        resid = torch.randn(B, Fi, T, co, generator=gen)
        resid = resid.half().float() if o16 else resid
        y = torch.empty(B, Fi, T, co, device="cuda", dtype=torch.float16 if o16 else torch.float32)
        res = op == cabi.NA_GLU_SCALE_RES
        gpu_engine._norm_act(out, stats, gamma.cuda(), beta.cuda(), y, B=B, F_in=Fi, T=T, C_=Cc, groups=groups, scope=scope, op=op,
                             snake_a=a.cuda() if op == cabi.NA_SNAKE else None, scale=scale.cuda() if res else None,
                             residual=resid.to(y.dtype).cuda() if res else None)
        torch.cuda.synchronize()
        ref = _groupnorm_ref(out.float().cpu(), gamma, beta, groups, scope, op, a, scale, resid)
        err = rel_l2(y.float().cpu(), ref)
        print(f"norm_act scope {scope} {storage} op {op} k={k}: rel_l2 {err:.2e}")
        assert err < (4e-4 if o16 else 4e-6) + NORM_ACT_C * U * (1 + k * k), (op, err)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("scope", [1, 2])
def test_masked_stats_on_offset_groups(gpu_engine, scope, dtype, k):
    """aero_masked_stats_fwd (the ragged batch's statistics) over each clip's valid frames of offset groups: scaled by
    T / frames[b], mean and variance over T frames are the clip's own fp64 two-pass values.  Bars as for the tap-GEMM
    statistics: STATS_C u (1 + k) sigma on the mean, STATS_C u (1 + k^2) relative on the variance."""
    from aero_b200.engine import _Ragged
    cfg = GEMM_SHAPES[0][1] if scope == 1 else GEMM_SHAPES[2][1]
    out, _ = _offset_gemm(gpu_engine, cfg, "f16" if dtype == torch.float16 else "simt", k)
    B, Fo, T, N = out.shape
    frames = [T, T // 2 + 1][:B]
    groups = cfg["groups"] if scope == 1 else 1
    gpu_engine._vl = _Ragged(frames, "cuda")
    try:
        nslots = B * groups if scope == 1 else B * Fo
        stats = torch.zeros(nslots, 2, dtype=torch.float64, device="cuda")
        gpu_engine._masked_stats(out, stats, groups=groups, scope=scope)
        torch.cuda.synchronize()
    finally:
        gpu_engine._vl = None
    per = nslots // B
    for b, tb in enumerate(frames):
        xb = out[b:b + 1, :, :tb]
        sl = _slots(xb, dict(cfg, stats_mode=1 if scope == 1 else 2))
        _check_stats(stats[b * per:(b + 1) * per], sl, k, f"masked stats scope {scope} {dtype} clip {b}",
                     count=sl.shape[1] * T / tb)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("scope,op", [(1, cabi.NA_GELU), (1, cabi.NA_GLU), (2, cabi.NA_GLU_SCALE_RES), (2, cabi.NA_SNAKE)])
def test_norm_act_train_on_offset_groups(gpu_engine, scope, op, k):
    """aero_norm_act_train_fwd / _bwd (the training step's GroupNorm) on exact-fp32 tap-GEMM outputs with offset groups and the
    epilogue's statistics, against fp64 autograd of the GroupNorm of the same values: output, dx, dgamma, dbeta, and the
    LayerScale / Snake gradients of the ops that have them.  Bar: 1e-5 + TRAIN_C u (1 + k^2) rel-L2 each."""
    cfg = GEMM_SHAPES[0][1] if scope == 1 else GEMM_SHAPES[2][1]
    x, stats = _offset_gemm(gpu_engine, cfg, "simt", k)
    B, Fi, T, Cc = x.shape
    groups = cfg["groups"] if scope == 1 else 1
    gen = torch.Generator().manual_seed(6)
    gamma, beta = 1 + 0.2 * torch.randn(Cc, generator=gen), 0.1 * torch.randn(Cc, generator=gen)
    a = torch.rand(Fi, generator=gen) * 8 + 0.2
    glu = op in (cabi.NA_GLU, cabi.NA_GLU_SCALE_RES)
    co = Cc // 2 if glu else Cc
    scale, resid = torch.randn(co, generator=gen), torch.randn(B, Fi, T, co, generator=gen)
    dy = torch.randn(B, Fi, T, co, generator=gen)
    lib = gpu_engine.lib
    p = cabi.NormActParams(B, Fi, Fi, 0, T, Cc, groups, scope, op, 1e-5, 0)
    dev = {n: t.cuda().contiguous() for n, t in dict(gamma=gamma, beta=beta, a=a, scale=scale, resid=resid, dy=dy).items()}
    y = torch.empty(B, Fi, T, co, device="cuda")
    stream = gpu_engine._stream()
    res = op == cabi.NA_GLU_SCALE_RES
    sa, sc, rs = dev["a"] if op == cabi.NA_SNAKE else None, dev["scale"] if res else None, dev["resid"] if res else None
    cabi.check(lib.aero_norm_act_train_fwd(_ptr(x), _ptr(stats), _ptr(dev["gamma"]), _ptr(dev["beta"]), _ptr(sa), _ptr(sc), _ptr(rs),
                                           _ptr(y), C.byref(p), stream), lib)
    z64 = lambda n: torch.zeros(n, dtype=torch.float64, device="cuda")
    dg, db = z64(Cc), z64(Cc)
    ds, dsn = (z64(co) if res else None), (z64(Fi) if op == cabi.NA_SNAKE else None)
    ws = torch.zeros(stats.shape[0], 2, dtype=torch.float64, device="cuda")
    dx = torch.empty_like(x)
    for pas in (1, 2):
        cabi.check(lib.aero_norm_act_train_bwd(_ptr(x), _ptr(stats), _ptr(dev["gamma"]), _ptr(dev["beta"]), _ptr(sa), _ptr(sc),
                                               _ptr(dev["dy"]), _ptr(dx), _ptr(dg), _ptr(db), _ptr(ds), _ptr(dsn),
                                               _ptr(ws), pas, C.byref(p), stream), lib)
    torch.cuda.synchronize()
    xr = x.cpu().double().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    ar, sr = a.double().requires_grad_(True), scale.double().requires_grad_(True)
    ref = _groupnorm_ref(xr, gr, br, groups, scope, op, ar, sr, resid)
    (ref * dy.double()).sum().backward()
    bar = 1e-5 + TRAIN_C * U * (1 + k * k)
    errs = {"y": rel_l2(y.cpu(), ref.detach()), "dx": rel_l2(dx.cpu(), xr.grad), "dgamma": rel_l2(dg.cpu(), gr.grad),
            "dbeta": rel_l2(db.cpu(), br.grad)}
    if res:
        errs["dscale"] = rel_l2(ds.cpu(), sr.grad)
    if op == cabi.NA_SNAKE:
        errs["dsnake"] = rel_l2(dsn.cpu(), ar.grad)
    print(f"norm_act_train scope {scope} op {op} k={k}: " + " ".join(f"{n} {e:.2e}" for n, e in errs.items()))
    assert all(e < bar for e in errs.values()), errs
