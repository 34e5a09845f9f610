"""-m gpu: the inference forward's attention, FTB-through-linear-input and small frequency-mix kernels on the branches that
only tile edges, production launch shapes and peaked softmaxes reach, against float64 statements of each operation.

test_gpu_kernels.py checks these kernels at one or two small shapes with one global rel-L2 each.  Here:
  1. local attention (csrc/attention.cu, SIMT; csrc/attention_mma.cu, mma.sync TF32) at T on both sides of the 8-key block,
     32-key chunk, 64-key tile, 64 / 128-query CTA and 256-key tile edges, every head dim, heads 1/4/8, ndecay 1/4/16, the
     benchmark forward's own launch shape, four score regimes (flat, peaked, decay slope at its extremes, the maximum in the
     last tile), the mma kernel's fallbacks to the SIMT kernel, FP16 outputs and ragged batches;
  2. aero_ftb_lin_out_fwd at every frequency-row split (fs = 8/4/2/1, even, uneven and odd-row shares), every N, J = 2/4, padded
     spectrogram rows and the production layer-0 shape; aero_ftb_lin_squeeze_fwd at r = 1..8;
  3. aero_freq_mix_small_fwd with and without gate, an M large enough for the grid-stride loop to run three passes, and the
     mixed-storage error path.
Every output goes into a NaN-filled buffer with a NaN guard after it: what the contract says is written must be finite, what it
does not (guard, padded frames of a ragged batch) must still be NaN.  Errors are checked per query / pixel, never only globally,
so one wrong tile, row share or query fails the test."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

from util import SEED

from aero_b200 import Aero, aero_kwargs, cabi
from aero_b200.engine import tf32_round

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

U32 = 2.0 ** -24             # unit roundoff of fp32
U_TF32 = 2.0 ** -11          # unit roundoff of TF32 / FP16 (10-bit mantissa, round to nearest)
LOG2E = 1.4426950408889634
GUARD = 64                   # NaN elements after every output


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(SEED + seed))


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope="module")
def lib():
    return cabi.load()


def nan_out(n, dtype=torch.float32, offset=0):
    """A NaN-filled device buffer of n elements starting `offset` elements in, with GUARD NaN elements after it."""
    buf = torch.full((offset + n + GUARD,), float("nan"), device="cuda", dtype=dtype)
    return buf, buf[offset:offset + n]


def guard_intact(buf, n, offset=0):
    return bool(torch.isnan(buf[offset + n:]).all())


# ------------------------------------------------------------------------------------------------
# production launch shapes: the benchmark forward's own calls, recorded from the engine
@pytest.fixture(scope="module")
def bench_calls():
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from bench import CONFIGS
    cfg = CONFIGS["4-16"]
    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs(cfg["exp"])).eval().cuda()
    eng = m._engine()
    eng.use_graph = False
    calls = {"attn": [], "ftb": []}
    attn0, ftb0 = eng._attn, eng._ftb_lin_out

    def attn(qkvd, out, **kw):
        calls["attn"].append(dict(kw))
        return attn0(qkvd, out, **kw)

    def ftb(*a, **kw):
        calls["ftb"].append(dict(kw))
        return ftb0(*a, **kw)
    eng._attn, eng._ftb_lin_out = attn, ftb
    try:
        x = torch.randn(cfg["batch"], m.in_channels, cfg["length"], generator=torch.Generator().manual_seed(SEED))
        with torch.no_grad():
            m(x.cuda())
        torch.cuda.synchronize()
    finally:
        del eng._attn, eng._ftb_lin_out
    assert calls["attn"] and calls["ftb"], calls
    uniq = lambda lst: [dict(t) for t in sorted({tuple(sorted(c.items())) for c in lst})]   # noqa: E731
    return {k: uniq(v) for k, v in calls.items()}


# ------------------------------------------------------------------------------------------------
# 1. local attention
def attn_inputs(rows, T, H, heads, ndecay, ld, regime="flat", seed=0, tf32=False):
    """qkvd [rows, T, ld]: q | k | v | decay logits | padding (NaN: never read)."""
    d = H // heads
    x = torch.full((rows, T, ld), float("nan"))
    q, k, v = rnd(rows, T, H, seed=seed), rnd(rows, T, H, seed=seed + 1), rnd(rows, T, H, seed=seed + 2)
    dl = rnd(rows, T, heads * ndecay, seed=seed + 3) * 1.5 - 1.0
    if regime == "peaked":
        # |q.k| / sqrt(d) up to ~50: the running maximum moves up chunk after chunk, every rescale carries weight.  Slopes
        # kept small (logits -6..-2) so that the decay does not confine the softmax to the diagonal's neighbours.
        q, k = q * 10.0 ** 0.5, k * 10.0 ** 0.5           # q.k / sqrt(d) ~ N(0, 10^2): max |score| 50-60 at T = 257
        dl = -4.0 + 2.0 * torch.tanh(dl)
    elif regime == "decay8":
        # every (query, head) at the largest or the smallest slope the sigmoid allows
        dl = torch.where(rnd(rows, T, heads, 1, seed=seed + 4) > 0, 8.0, -8.0).expand(rows, T, heads, ndecay).reshape(rows, T, -1)
    elif regime == "far":
        # every query's largest score is the last key (in the last tile), |score| ~ 50, minimum slope
        u = torch.nn.functional.normalize(rnd(heads, d, seed=seed + 5), dim=-1)
        g = (50.0 * math.sqrt(d)) ** 0.5
        q = (q.view(rows, T, heads, d) * 0.3 + g * u).reshape(rows, T, H)
        k = k.clone()
        k.view(rows, T, heads, d)[:, -1] = g * u
        dl = torch.full_like(dl, -8.0)
    x[..., :H], x[..., H:2 * H], x[..., 2 * H:3 * H] = q, k, v
    x[..., 3 * H:3 * H + heads * ndecay] = dl
    if tf32:        # what the producing GEMM stores in tensor-core mode
        x = tf32_round(x)
    return x


def attn_run(lib, qkvd, rows, T, H, heads, ndecay, ld, flags, dtype=torch.float32, offset=0):
    """One aero_local_attn_fwd call; returns (output [rows, T, H] on the host, guard intact)."""
    src = torch.full((offset + qkvd.numel(),), float("nan"), device="cuda")
    src[offset:] = qkvd.reshape(-1).cuda()
    n = rows * T * H
    buf, out = nan_out(n, dtype)
    p = cabi.AttnParams(rows, T, H, heads, ndecay, ld, flags | (cabi.TG_OUT_F16 if dtype == torch.float16 else 0))
    cabi.check(lib.aero_local_attn_fwd(ptr(src[offset:]), ptr(out), C.byref(p), stream()), lib)
    torch.cuda.synchronize()
    return out.view(rows, T, H).cpu(), guard_intact(buf, n)


def attn_ref(qkvd, T, H, heads, ndecay):
    """fp64 statement of reference modules.py:104-124 on the fp32 values the kernel reads, for rows [R] of qkvd [R, T, ld].
    Returns the output [R, T, heads, d], the softmax weights [R, heads, T(query), T(key)], |v| [R, T, heads, d], and per query
    (in [R, T, heads]) the softmax-weighted absolute logit of the q.k term alone (aq) and with the decay term (af), in log2 units."""
    R, d = qkvd.shape[0], H // heads
    m = qkvd.double()
    q, k, v = (m[..., i * H:(i + 1) * H].reshape(R, T, heads, d) for i in range(3))
    dl = m[..., 3 * H:3 * H + heads * ndecay].reshape(R, T, heads, ndecay)
    slope = (torch.sigmoid(dl) / 2 * torch.arange(1, ndecay + 1, dtype=torch.float64)).sum(-1) / math.sqrt(ndecay)
    idx = torch.arange(T, dtype=torch.float64)
    dist = (idx[:, None] - idx[None, :]).abs()
    pen = dist * slope.permute(0, 2, 1)[..., None]                              # [R, h, s, t]
    sc = torch.einsum("rshc,rthc->rhst", q, k) / math.sqrt(d) - pen
    sc.diagonal(dim1=-2, dim2=-1).fill_(-100.0)
    w = torch.softmax(sc, -1)
    o = torch.einsum("rhst,rthc->rshc", w, v)
    A = torch.einsum("rshc,rthc->rhst", q.abs(), k.abs()) / math.sqrt(d)
    aq = (w * A).sum(-1).permute(0, 2, 1) * LOG2E
    af = (w * (A + pen)).sum(-1).permute(0, 2, 1) * LOG2E
    return o, w, v.abs(), aq, af


def tie_dist(x32):
    """Distance of fp32 values to their TF32 rounding tie (the value whose low 13 mantissa bits are 0x1000)."""
    b = x32.contiguous().view(torch.int32)
    return (x32.double() - ((b & ~0x1FFF) | 0x1000).view(torch.float32).double()).abs()


def tf32_ulp(x):
    return torch.ldexp(torch.ones_like(x), torch.frexp(x)[1] - 11)


def attn_mma_emul(qkvd, T, H, heads, ndecay):
    """fp64 emulation of csrc/attention_mma.cu's roundings on TF32 inputs qkvd [R, T, ld] (fixed length):
      q * (log2e / sqrt(d)) in fp32 (the constant folds to fp32(log2e) * fp32(1/sqrt(d))), rounded to TF32 (nearest, ties away);
      k, v as given; scores in the log2 domain; keys in chunks of 32 with the running maximum M after each chunk;
      p = 2^(s - M[chunk]) rounded to TF32 for P.V while the row sum l takes the unrounded p; both rescaled to the final maximum.
    Returns the output before its final TF32 rounding [R, T, heads, d] and an allowance: where an fp32 p sits within
    2^-21 (8 + the magnitudes summed into s - M) of a TF32 tie, fp32 evaluation order decides its rounding, and the allowance
    admits one TF32 ulp of that term."""
    R, d = qkvd.shape[0], H // heads
    qs = np.float32(np.float32(LOG2E) * np.float32(1.0 / math.sqrt(d)))
    qt = tf32_round(qkvd[..., :H].float() * torch.tensor(qs)).double().reshape(R, T, heads, d)
    k = qkvd[..., H:2 * H].double().reshape(R, T, heads, d)
    v = qkvd[..., 2 * H:3 * H].double().reshape(R, T, heads, d)
    dl = qkvd[..., 3 * H:3 * H + heads * ndecay].double().reshape(R, T, heads, ndecay)
    slope = (torch.sigmoid(dl) / 2 * torch.arange(1, ndecay + 1, dtype=torch.float64)).sum(-1) / math.sqrt(ndecay) * LOG2E
    idx = torch.arange(T, dtype=torch.float64)
    dist = (idx[:, None] - idx[None, :]).abs()
    pen = dist * slope.permute(0, 2, 1)[..., None]
    s = torch.einsum("rshc,rthc->rhst", qt, k) - pen
    s.diagonal(dim1=-2, dim2=-1).fill_(float(np.float32(-100.0) * np.float32(LOG2E)))
    nch = (T + 31) // 32
    sp = torch.full((*s.shape[:-1], nch * 32), -math.inf, dtype=torch.float64)
    sp[..., :T] = s
    M = sp.view(*s.shape[:-1], nch, 32).amax(-1).cummax(-1).values             # running maximum after each chunk
    Mk = M.repeat_interleave(32, -1)[..., :T]
    p = torch.exp2(s - Mk)
    p32 = p.float()
    pr = tf32_round(p32).double()
    sc = torch.exp2(Mk - M[..., -1:])
    l = (p * sc).sum(-1).permute(0, 2, 1)[..., None]                            # [R, s, h, 1]
    o = torch.einsum("rhst,rthc->rshc", pr * sc, v) / l
    mag = 8.0 + torch.einsum("rshc,rthc->rhst", qt.abs(), k.abs()) + pen + M[..., -1:].abs()
    amb = tie_dist(p32) <= 2.0 ** -21 * mag * p
    allow = torch.einsum("rhst,rthc->rshc", torch.where(amb, tf32_ulp(p) * sc, 0.0), v.abs()) / l
    return o, allow


def check_attn(out, qkvd, T, H, heads, ndecay, mma, tag):
    """Per-element bounds, scaled per (row, query, head) by max |v| of that (row, head): the output is a convex combination of
    v, so a perturbation delta_s of the logits moves it by at most 2 max|v| sum_s w_s |delta_s| (first order).
      fp32 evaluation (both kernels): |delta_s| <= c u32 (logit magnitude), c from 24 products summed in fp32, the decay fma,
        ex2 / __expf and the running sums; bound 2^-20 (8 + af) with af the softmax-weighted absolute log2 logit.
      mma vs exact: q is rounded to TF32 after scaling, |delta_s| <= 2^-11 sum_c |q_c k_c| / sqrt(d), giving
        2 * 2^-11 * aq(natural units); P rounded to TF32 for P.V adds 2^-11 max|v| and the final TF32 rounding 2^-11 |o| <=
        2^-11 max|v|: total 2^-11 (2 aq ln2 + 2), times 1.1 for the second-order terms (aq <= ~60: 2^-11 aq < 0.03).
      mma vs its emulation (attn_mma_emul): only the fp32 evaluation differs (the same 2^-20 (8 + af) bound), plus one TF32 ulp
        wherever that much error can move a p or the output across a TF32 rounding tie."""
    R, d = qkvd.shape[0], H // heads
    o = out.double().reshape(R, T, heads, d)
    ref, w, va, aq, af = attn_ref(qkvd, T, H, heads, ndecay)
    vmax = va.amax((1, 3))[:, None, :, None]                                     # [R, 1, h, 1]
    base = 2.0 ** -20 * (8.0 + af)[..., None]
    res = {}
    if mma:
        exact = U_TF32 * (2.0 * aq * math.log(2.0) + 2.0)[..., None] * 1.1 + base
        pre, allow = attn_mma_emul(qkvd, T, H, heads, ndecay)
        tol = base * vmax + allow
        # the kernel's output before rounding is within tol of `pre`: where a TF32 tie lies that close, either neighbour is right
        pre32 = pre.float()
        tol = tol + torch.where(tie_dist(pre32) <= tol, tf32_ulp(pre), 0.0)
        checks = (("exact", ref, exact * vmax), ("emulation", tf32_round(pre32).double(), tol))
    else:
        checks = (("exact", ref, base * vmax),)
    for name, r, bound in checks:
        err = (o - r).abs()
        ratio = float((err / bound).max())
        res[name] = ratio
        qbad = (err > bound).any(-1).any(-1)                                      # [R, T]
        assert not bool(qbad.any()), (f"{tag}: {name} bound broken at (row, query) {qbad.nonzero()[:8].tolist()}, "
                                      f"worst err/bound {ratio:.3g}, worst per-query err/max|v| {float((err / vmax).max()):.3g}")
    print(f"{tag}: err/bound " + " ".join(f"{k} {v:.3g}" for k, v in res.items()))
    return ref


T_EDGES = [1, 2, 7, 8, 9, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 513]
HEADS, NDECAY = [1, 4, 8], [1, 4, 16]
EDGE_CASES = [("simt", d, T) for d in (3, 6, 12, 24) for T in T_EDGES] + [("mma", d, T) for d in (12, 24) for T in T_EDGES]


def attn_ld(H, heads, ndecay, mma):
    ld = 3 * H + heads * ndecay
    return (ld + 3) & ~3 if mma else ld + 1          # the mma kernel needs ld % 4 == 0; the SIMT one is fed an odd ld


@pytest.mark.parametrize("kern,d,T", EDGE_CASES, ids=[f"{k}-d{d}-T{T}" for k, d, T in EDGE_CASES])
def test_attention_tile_edges(lib, kern, d, T):
    """Flat scores at every tile-edge T; heads and ndecay cycle through {1, 4, 8} x {1, 4, 16} across the cases."""
    i = T_EDGES.index(T) + 3 * d
    heads, ndecay = HEADS[i % 3], NDECAY[(i // 3) % 3]
    H, rows, mma = heads * d, 2, kern == "mma"
    ld = attn_ld(H, heads, ndecay, mma)
    x = attn_inputs(rows, T, H, heads, ndecay, ld, seed=i, tf32=mma)
    out, guard = attn_run(lib, x, rows, T, H, heads, ndecay, ld, cabi.TG_ROUND_TF32 if mma else 0)
    assert guard and torch.isfinite(out).all()
    if T == 1:      # the diagonal is the only key: p = 1 (TF32-exact), the output is v itself
        assert torch.equal(out, x[..., 2 * H:3 * H])
    check_attn(out, x, T, H, heads, ndecay, mma, f"{kern} d={d} T={T} heads={heads} ndecay={ndecay}")


REGIME_CASES = [(k, r, T) for k in ("simt", "mma") for r in ("flat", "peaked", "decay8", "far") for T in (33, 129, 257, 513)]


@pytest.mark.parametrize("kern,regime,T", REGIME_CASES, ids=[f"{k}-{r}-T{T}" for k, r, T in REGIME_CASES])
def test_attention_score_regimes(lib, kern, regime, T):
    mma = kern == "mma"
    i = REGIME_CASES.index((kern, regime, T))
    ds = (12, 24) if mma else (3, 6, 12, 24)
    d = ds[(i + i // 4) % len(ds)]
    heads, ndecay = HEADS[i % 3], NDECAY[(i // 2) % 3]
    H, rows = heads * d, 2
    ld = attn_ld(H, heads, ndecay, mma)
    x = attn_inputs(rows, T, H, heads, ndecay, ld, regime=regime, seed=100 + i, tf32=mma)
    out, guard = attn_run(lib, x, rows, T, H, heads, ndecay, ld, cabi.TG_ROUND_TF32 if mma else 0)
    assert guard and torch.isfinite(out).all()
    ref = check_attn(out, x, T, H, heads, ndecay, mma, f"{kern} {regime} d={d} T={T} heads={heads} ndecay={ndecay}")
    if regime == "far":      # the regime does what it says: the last key carries most of the weight for the first query
        assert float((ref[:, 0] - x[:, -1, 2 * H:3 * H].double().view(rows, heads, d)).abs().max()) < 0.1


@pytest.mark.parametrize("kern", ["simt", "mma"])
def test_attention_benchmark_launch_shape(lib, bench_calls, kern):
    """Every distinct attention launch of the benchmark forward (rows, T, H, heads, ndecay, ld as the engine passes them),
    all rows computed, four rows checked against fp64 (rows are independent CTAs: first, second, middle, last)."""
    mma = kern == "mma"
    for c in bench_calls["attn"]:
        rows, T, H, heads, ndecay, ld = c["rows"], c["T"], c["H"], c["heads"], c["ndecay"], c["ld"]
        x = attn_inputs(rows, T, H, heads, ndecay, ld, seed=7, tf32=mma)
        out, guard = attn_run(lib, x, rows, T, H, heads, ndecay, ld, cabi.TG_ROUND_TF32 if mma else 0)
        assert guard and torch.isfinite(out).all()
        sel = sorted({0, 1, rows // 2, rows - 1})
        check_attn(out[sel], x[sel], T, H, heads, ndecay, mma, f"{kern} benchmark rows={rows} T={T} H={H}")


def profiled_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "local_attn" in e.name]


@pytest.mark.parametrize("case", ["ld_odd", "misaligned", "d3", "d6"])
def test_attention_mma_fallback_to_simt(lib, case):
    """With ROUND_TF32 the mma kernel runs only for head dim 12 / 24, ld % 4 == 0 and a 16-byte aligned qkvd; otherwise the
    SIMT kernel runs and rounds its output to TF32: bit for bit round_tf32_rna(the SIMT kernel's fp32 output)."""
    heads, ndecay, T, rows = 4, 4, 129, 2
    d = {"d3": 3, "d6": 6}.get(case, 12)
    H = heads * d
    ld = 3 * H + heads * ndecay + (1 if case == "ld_odd" else 0)
    off = 1 if case == "misaligned" else 0
    x = attn_inputs(rows, T, H, heads, ndecay, ld, seed=11, tf32=True)
    names = profiled_kernels(lambda: attn_run(lib, x, rows, T, H, heads, ndecay, ld, cabi.TG_ROUND_TF32, offset=off))
    assert names and all("mma" not in n for n in names), names
    o_tc, g1 = attn_run(lib, x, rows, T, H, heads, ndecay, ld, cabi.TG_ROUND_TF32, offset=off)
    o_32, g2 = attn_run(lib, x, rows, T, H, heads, ndecay, ld, 0, offset=off)
    assert g1 and g2 and torch.isfinite(o_32).all()
    assert torch.equal(o_tc, tf32_round(o_32))


def test_attention_mma_is_taken(lib):
    heads, ndecay, T, rows, d = 4, 4, 65, 1, 24
    H = heads * d
    ld = attn_ld(H, heads, ndecay, True)
    x = attn_inputs(rows, T, H, heads, ndecay, ld, seed=12, tf32=True)
    names = profiled_kernels(lambda: attn_run(lib, x, rows, T, H, heads, ndecay, ld, cabi.TG_ROUND_TF32))
    assert names and all("local_attn_mma_kernel" in n for n in names), names


@pytest.mark.parametrize("kern,d", [("simt", 3), ("simt", 24), ("mma", 12), ("mma", 24)])
def test_attention_fp16_output(lib, kern, d):
    """SIMT: FP16 output = the fp32 output .half(), bit for bit (one template body, one rounding at the store).
    mma: within one FP16 rounding of its fp32 output."""
    mma = kern == "mma"
    heads, ndecay, T, rows = 4, 4, 257, 2
    H = heads * d
    ld = attn_ld(H, heads, ndecay, mma)
    x = attn_inputs(rows, T, H, heads, ndecay, ld, seed=13, tf32=mma)
    fl = cabi.TG_ROUND_TF32 if mma else 0
    o32, g1 = attn_run(lib, x, rows, T, H, heads, ndecay, ld, fl)
    o16, g2 = attn_run(lib, x, rows, T, H, heads, ndecay, ld, fl, dtype=torch.float16)
    assert g1 and g2 and torch.isfinite(o16).all()
    if mma:
        assert bool(((o16.float() - o32).abs() <= U_TF32 * o32.abs() + 2.0 ** -25).all())
    else:
        assert torch.equal(o16, o32.half())


RAGGED_FRAMES = [1, 7, 8, 9, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 513, 200]
RAGGED_CASES = [(k, d, rpc) for k, ds in (("simt", (6, 24)), ("mma", (12, 24))) for d in ds for rpc in (1, 3)]


@pytest.mark.parametrize("kern,d,rpc", RAGGED_CASES, ids=[f"{k}-d{d}-rpc{r}" for k, d, r in RAGGED_CASES])
def test_attention_ragged_equals_fixed_per_clip(lib, kern, d, rpc):
    """aero_local_attn_varlen_fwd: each clip's rows equal, bit for bit, the fixed-length call on that clip alone (same block
    body with Tr = the clip's length); rows past each clip's length are not written."""
    mma = kern == "mma"
    heads, ndecay = 4, 4
    H = heads * d
    ld = attn_ld(H, heads, ndecay, mma)
    fl = cabi.TG_ROUND_TF32 if mma else 0
    n_clip, Tm = len(RAGGED_FRAMES), max(RAGGED_FRAMES)
    rows = n_clip * rpc
    x = attn_inputs(rows, Tm, H, heads, ndecay, ld, seed=20 + d, tf32=mma)
    frames = torch.tensor(RAGGED_FRAMES, dtype=torch.int32, device="cuda")
    n = rows * Tm * H
    buf, out = nan_out(n)
    p = cabi.AttnParams(rows, Tm, H, heads, ndecay, ld, fl)
    cabi.check(lib.aero_local_attn_varlen_fwd(ptr(x.cuda()), ptr(out), ptr(frames), rpc, C.byref(p), stream()), lib)
    torch.cuda.synchronize()
    assert guard_intact(buf, n)
    o = out.view(n_clip, rpc, Tm, H).cpu()
    for c, Tc in enumerate(RAGGED_FRAMES):
        xc = x[c * rpc:(c + 1) * rpc, :Tc].contiguous()
        ref, _ = attn_run(lib, xc, rpc, Tc, H, heads, ndecay, ld, fl)
        assert torch.equal(o[c, :, :Tc], ref), (c, Tc)
        assert bool(torch.isnan(o[c, :, Tc:]).all()), (c, Tc)


# ------------------------------------------------------------------------------------------------
# 2. FTB through linear input
def ftb_out_run(lib, z, zm, M, s, V, d, *, B, F, T, N, J, zrow, flags, dtype=torch.float32):
    n = B * F * T * N
    buf, out = nan_out(n, dtype)
    p = cabi.FtbLinParams(B, F, T, N, J, flags | (cabi.TG_OUT_F16 if dtype == torch.float16 else 0), F * zrow, zrow, F * zrow, zrow)
    cabi.check(lib.aero_ftb_lin_out_fwd(*(ptr(t) for t in (z, zm, M, s, V, d, out)), C.byref(p), stream()), lib)
    torch.cuda.synchronize()
    return out.view(B, F, T, N).cpu(), guard_intact(buf, n)


def check_three_outputs(run, ref, absdot, n_fma, tag):
    """fp32 output within n_fma fp32 roundings of |terms| per element (max over pixels reported); FP16 output = fp32 output .half()
    bit for bit (explicit fmaf chain, one rounding at the store); ROUND_TF32 output = round_tf32_rna(fp32 output) bit for bit."""
    o32, g = run(0, torch.float32)
    assert g and torch.isfinite(o32).all(), tag
    bound = n_fma * U32 * absdot + 1e-30
    ratio = (o32.double() - ref).abs() / bound
    assert float(ratio.max()) <= 1.0, (tag, float(ratio.max()), (ratio > 1).nonzero()[:8].tolist())
    o16, g = run(0, torch.float16)
    assert g and torch.equal(o16, o32.half()), tag
    ot, g = run(cabi.TG_ROUND_TF32, torch.float32)
    assert g and torch.equal(ot, tf32_round(o32)), tag
    print(f"{tag}: fp32 err / ({n_fma} u |terms|) max {float(ratio.max()):.3g}")


def ftb_out_case(lib, B, F, T, N, J, zrow, seed):
    z, zm = rnd(B, F, zrow, seed=seed), rnd(B, F, zrow, seed=seed + 1)
    M, s, V, d = rnd(B * T, N * (J + 1), seed=seed + 2), rnd(F, seed=seed + 3), rnd(N, J, seed=seed + 4), rnd(N, seed=seed + 5)
    zv = z[:, :, :T * J].reshape(B, F, T, J).double()
    zmv = zm[:, :, :T * J].reshape(B, F, T, J).double()
    Mv = M.reshape(B, T, N, J + 1).double()
    terms = [torch.einsum("btn,bft->bftn", Mv[..., j], zmv[..., j]) for j in range(J)]
    terms += [Mv[..., J][:, None] * s.double()[None, :, None, None]]
    terms += [torch.einsum("n,bft->bftn", V.double()[:, j], zv[..., j]) for j in range(J)]
    terms += [d.double().expand(B, F, T, N)]
    pre = sum(terms)
    ref = pre.clamp_min(0)
    absdot = sum(t.abs() for t in terms)
    g = [t.cuda() for t in (z, zm, M, s, V, d)]
    check_three_outputs(lambda fl, dt: ftb_out_run(lib, *g, B=B, F=F, T=T, N=N, J=J, zrow=zrow, flags=fl, dtype=dt),
                        ref, absdot, 2 * J + 2, f"ftb_lin_out B={B} F={F} T={T} N={N} J={J}")


FTB_F = [1, 2, 3, 15, 16, 17, 33, 63, 64, 65, 70, 256]
FTB_T = [1, 31, 32, 33, 501]
FTB_N = [8, 16, 24, 32, 40, 48, 56, 64]
FTB_CASES = [(F, T) for F in FTB_F for T in FTB_T if not (F == 256 and T == 501)]


@pytest.mark.parametrize("F,T", FTB_CASES)
def test_ftb_lin_out_row_shares(lib, F, T):
    """Every frequency split fs (8/4/2/1) with even, uneven and odd-row last shares; padded zrow (!= T*J); N and J cycle."""
    i = FTB_CASES.index((F, T))
    N, J = FTB_N[i % 8], (2, 4)[(i // 8) % 2]
    zrow = T * J + 6
    ftb_out_case(lib, 2, F, T, N, J, zrow, seed=200 + i)


@pytest.mark.parametrize("J", [2, 4])
@pytest.mark.parametrize("N", FTB_N)
def test_ftb_lin_out_every_n(lib, N, J):
    """Block sizes 64..512 threads (32 frames x N/4), uneven share (F = 70: shares of 9, last of 7)."""
    ftb_out_case(lib, 2, 70, 33, N, J, 33 * J + 2, seed=300 + N + J)


def test_ftb_lin_out_benchmark_layer0(lib, bench_calls):
    """The benchmark forward's own launch (F, T, N, J, zrow as the engine passes them), two clips."""
    for c in bench_calls["ftb"]:
        ftb_out_case(lib, 2, c["F"], c["T"], c["N"], c["J"], c["zrow"], seed=400)


def ftb_sq_case(lib, B, F, T, J, r, zrow, seed):
    z, W1p, b1p = rnd(B, F, zrow, seed=seed), rnd(r, J, seed=seed + 1), rnd(r, seed=seed + 2)
    zv = z[:, :, :T * J].reshape(B, F, T, J).double()
    terms = [torch.einsum("n,bft->btfn", W1p.double()[:, j], zv[..., j]) for j in range(J)] + [b1p.double().expand(B, T, F, r)]
    ref = sum(terms).clamp_min(0).reshape(B, T, F * r)
    absdot = sum(t.abs() for t in terms).reshape(B, T, F * r)
    zg, wg, bg = z.cuda(), W1p.cuda(), b1p.cuda()

    def run(fl, dt):
        n = B * T * F * r
        buf, R = nan_out(n, dt)
        p = cabi.FtbLinParams(B, F, T, 0, J, fl | (cabi.TG_OUT_F16 if dt == torch.float16 else 0), F * zrow, zrow, 0, 0)
        cabi.check(lib.aero_ftb_lin_squeeze_fwd(ptr(zg), ptr(wg), ptr(bg), ptr(R), r, C.byref(p), stream()), lib)
        torch.cuda.synchronize()
        return R.view(B, T, F * r).cpu(), guard_intact(buf, n)
    check_three_outputs(run, ref, absdot, J + 1, f"ftb_lin_squeeze B={B} F={F} T={T} J={J} r={r}")


SQ_CASES = [(r, F) for r in range(1, 9) for F in (1, 31, 32, 33, 256)]


@pytest.mark.parametrize("r,F", SQ_CASES)
def test_ftb_lin_squeeze(lib, r, F):
    i = SQ_CASES.index((r, F))
    T, J = FTB_T[i % 5], (2, 4)[(i // 5) % 2]
    ftb_sq_case(lib, 2, F, T, J, r, T * J + 2, seed=500 + i)


# ------------------------------------------------------------------------------------------------
# 3. aero_freq_mix_small_fwd
def freq_mix_case(lib, B, F, M, gate_on, seed, kinds=("f32", "f16", "tf32")):
    x, W = rnd(B, F, M, seed=seed), rnd(F, F, seed=seed + 1) / math.sqrt(F)
    gate = rnd(B, M, seed=seed + 2) if gate_on else None
    gg = gate.cuda() if gate_on else None
    Wg = W.cuda()
    res = {}
    for kind in kinds:
        f16 = kind == "f16"
        xs = x.half() if f16 else x
        xd = xs.double()
        terms = W.double()[None, :, :, None] * xd[:, None]                       # [B, g, f, M]
        if gate_on:
            terms = terms * gate.double()[:, None, None]
        ref, absdot = terms.sum(2), terms.abs().sum(2)
        dt = torch.float16 if f16 else torch.float32
        fl = (cabi.TG_A_F16 | cabi.TG_OUT_F16) if f16 else (cabi.TG_ROUND_TF32 if kind == "tf32" else 0)
        n = B * F * M
        buf, out = nan_out(n, dt)
        cabi.check(lib.aero_freq_mix_small_fwd(ptr(xs.cuda()), ptr(Wg), ptr(gg), ptr(out), B, F, M, fl, stream()), lib)
        torch.cuda.synchronize()
        o = out.view(B, F, M).cpu()
        assert guard_intact(buf, n) and torch.isfinite(o).all(), kind
        bound = (F + 2) * U32 * absdot + (U_TF32 * ref.abs() + 2.0 ** -25 if f16 else 0.0) + 1e-30
        ratio = (o.double() - ref).abs() / bound
        assert float(ratio.max()) <= 1.0 or kind == "tf32", (kind, float(ratio.max()), (ratio > 1).nonzero()[:8].tolist())
        res[kind] = o
        del terms
    if "tf32" in res:
        assert torch.equal(res["tf32"], tf32_round(res["f32"]))
    return res


FM_CASES = [(F, B, g) for F in (8, 16) for B in (1, 2, 3) for g in (False, True)]


@pytest.mark.parametrize("F,B,gate", FM_CASES)
def test_freq_mix_small(lib, F, B, gate):
    freq_mix_case(lib, B, F, 77 * 36 + 4 * B, gate, seed=600 + FM_CASES.index((F, B, gate)))


def test_freq_mix_small_grid_stride_loop(lib):
    """The grid is capped at 132 * 8 blocks of 256 threads x 4 positions = 1081344 positions per pass; M = 2.5e6 takes three
    passes of the grid-stride loop (FP16, F = 8, B = 1: 40 MB each way)."""
    M = 2_500_000
    assert M > 132 * 8 * 1024 * 2
    freq_mix_case(lib, 1, 8, M, True, seed=700, kinds=("f16",))


@pytest.mark.parametrize("flags", [cabi.TG_OUT_F16, cabi.TG_A_F16])
def test_freq_mix_small_mixed_storage_is_refused(lib, flags):
    """fp32 in / FP16 out (and the reverse) is AERO_ERR_UNSUPPORTED, with no launch and the output untouched."""
    B, F, M = 1, 8, 1024
    x = torch.randn(B, F, M, device="cuda", dtype=torch.float16 if flags == cabi.TG_A_F16 else torch.float32)
    W = torch.randn(F, F, device="cuda")
    buf, out = nan_out(B * F * M, torch.float16 if flags == cabi.TG_OUT_F16 else torch.float32)
    n0 = lib.aero_launch_count()
    rc = lib.aero_freq_mix_small_fwd(ptr(x), ptr(W), None, ptr(out), B, F, M, flags, stream())
    torch.cuda.synchronize()
    assert rc == -2, rc                                        # AERO_ERR_UNSUPPORTED
    assert b"storage type" in lib.aero_last_error()
    assert lib.aero_launch_count() == n0
    assert bool(torch.isnan(buf).all())
