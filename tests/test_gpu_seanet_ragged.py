"""Ragged SEANet batches on the H100 (SeanetEngine.forward_varlen, enhance_batch): the two ragged kernels against fp64
restatements of their contracts and against the single-clip kernels, every clip of a ragged batch bit-identical to its own
forward at every precision, the goldens in one ragged batch, padding that never leaks, and evaluate_batch."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from util import SEED, rel_l2, white_noise
from seanet_util import CASES, case_input, seanet_recipe_state

from aero_b200 import Seanet, cabi
from aero_b200.engine import tf32_round
from aero_b200.enhance import enhance_batch, evaluate_batch, match_signal
from aero_b200.metrics import get_lsd
from aero_b200.seanet import sinc_resample_table

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F = torch.nn.functional
CONFIGS = {"shipped": CASES["s1"][0], "s3": CASES["s3"][0], "s5": CASES["s5"][0], "s6": CASES["s6"][0]}


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _model(cfg, precision):
    torch.manual_seed(SEED)
    m = Seanet(**cfg)
    m.load_state_dict(seanet_recipe_state(m.state_dict()))
    m = m.cuda().eval().use_cuda_graph(False)
    m._engine().precision = precision
    return m


def _shortest(m):
    return next(n for n in range(2, 1 << 16) if not _raises(m.check_length, n))


def _raises(fn, *a):
    try:
        fn(*a)
        return False
    except ValueError:
        return True


def _pad(clips, L, fill=0.0):
    x = torch.full((len(clips), clips[0].shape[0], L), fill, device="cuda")
    for b, c in enumerate(clips):
        x[b, :, :c.shape[-1]] = c
    return x


# ------------------------------------------------------------------------------------------------ input stage
def _input_reference(x, n, filt, width, orig, up, hr, Lv, fill, floor):
    """fp64 restatement of one clip: std of the channel mean over its n samples, x / (floor + std), the polyphase filter over
    its own samples (zero outside [0, n)), zero padding to Lv frames, `fill` frames reflected at both ends -> [Lv + 2 fill, C]."""
    xs = x[:, :n].double()
    std = xs.mean(0).std()
    xn = xs / (floor + std)
    if up == 0:
        y = xn
    else:
        f = filt.double()
        t = torch.arange(hr)
        j = (t // up * orig - width)[:, None] + torch.arange(f.shape[1])[None]
        ok = (j >= 0) & (j < n)
        g = xn[:, j.clamp(0, n - 1)] * ok                         # [C, hr, taps]
        y = (g * f[t % up][None]).sum(-1)
    y = F.pad(y, (0, Lv - y.shape[-1]))
    return F.pad(y[None], (fill, fill), mode="reflect")[0].t(), std


@pytest.mark.parametrize("name", ["shipped", "s3", "s5"])
def test_input_stage_contract(name):
    """aero_seanet_input_varlen_fwd with T_b (the valid length) at halo + 1, mid-buffer and at T_max: std, resampling near
    each clip's end, zero pad, reflection at its own end and zeros beyond, against fp64 and bit for bit against the
    single-clip kernel.  Samples past each clip are NaN: never read."""
    m = Seanet(**CONFIGS[name])
    Cin, H, fill, floor = m.in_channels, 9, 3, 1e-3
    if m.upsample:
        filt, width, orig, up = sinc_resample_table(m.lr_sr, m.hr_sr)
        filt, taps = filt.cuda().contiguous(), filt.shape[1]
    else:
        filt, width, orig, up, taps = None, 0, 1, 0, 0
    hr_of = lambda n: math.ceil(up * n / orig) if up else n
    L_max = 1500
    Lv_max = hr_of(L_max) + 7
    n_first = next(n for n in range(2, 100) if hr_of(n + 1) > H + 1)          # hr(n) <= halo + 1 = T_b
    lengths = [n_first, 701, L_max]
    hr = [hr_of(n) for n in lengths]
    valid = [H + 1, hr[1] + 5, Lv_max]
    clips = [white_noise((Cin, n), seed=20 + b) + 0.3 * b for b, n in enumerate(lengths)]
    x = _pad([c.cuda() for c in clips], L_max, float("nan"))
    B = len(lengths)
    tab = torch.tensor(lengths + hr + valid, dtype=torch.int32, device="cuda")
    x0 = torch.full((B, Lv_max + 2 * H, Cin), float("nan"), device="cuda")
    aff = torch.full((B, 2), float("nan"), device="cuda")
    p = cabi.ResampleParams(B, Cin, L_max, orig, up, width, taps, hr_of(L_max), Lv_max, H, fill, 1, floor)
    lib = cabi.load()
    cabi.check(lib.aero_seanet_input_varlen_fwd(_p(x), _p(filt), _p(aff), _p(x0), _p(tab[:B]), _p(tab[B:2 * B]), _p(tab[2 * B:]),
                                                C.byref(p), None), lib)
    torch.cuda.synchronize()
    for b, (n, h, Lv) in enumerate(zip(lengths, hr, valid)):
        ref, std = _input_reference(clips[b], n, None if filt is None else filt.cpu(), width, orig, up, h, Lv, fill, floor)
        got = x0[b, H - fill:H + Lv + fill].cpu()
        assert rel_l2(got, ref) <= 1e-6, (b, rel_l2(got, ref))
        assert abs(float(aff[b, 0]) - float(std)) <= 1e-6 * float(std) and float(aff[b, 1]) == 0.0
        assert (x0[b, H + Lv + fill:] == 0).all()                             # zeros to the buffer's end
        assert torch.isnan(x0[b, :H - fill]).all()                            # nothing before the requested reflection
        # the single-clip kernel on the clip alone writes the same bits
        one = torch.full((1, Lv + 2 * H, Cin), float("nan"), device="cuda")
        aff1 = torch.empty(1, 2, device="cuda")
        xb = clips[b].cuda()[None].contiguous()
        p1 = cabi.ResampleParams(1, Cin, n, orig, up, width, taps, h, Lv, H, fill, 1, floor)
        cabi.check(lib.aero_seanet_input_fwd(_p(xb), _p(filt), _p(aff1), _p(one), C.byref(p1), None), lib)
        torch.cuda.synchronize()
        assert torch.equal(one[0, H - fill:H + Lv + fill], x0[b, H - fill:H + Lv + fill])
        assert torch.equal(aff1[0], aff[b])


# ------------------------------------------------------------------------------------------------ reflection halo
@pytest.mark.parametrize("halo", [0, 1, 3, 9])
@pytest.mark.parametrize("kind", ["f32", "tf32", "f32->f16", "f16"])
def test_reflect_act_contract(halo, kind):
    """aero_reflect_act_varlen_fwd with T_b at halo + 1, mid-buffer and at T_max: act(x) on [0, T_b), reflection at both of the
    clip's own ends, zeros on [T_b + halo, T_max + halo), nothing outside [-halo, T_max + halo); FP16 / TF32-rounded outputs as the
    flags say.  Frames past each clip are NaN: never read."""
    B, T, Cc, H = 3, 57, 12, 9
    frames = [halo + 1, 30, T]
    g = torch.Generator().manual_seed(halo)
    xd = torch.randn(B, T, Cc, generator=g)
    a16 = kind == "f16"
    o16 = kind in ("f16", "f32->f16")
    x = (xd.half() if a16 else xd).cuda()
    for b, tb in enumerate(frames):
        x[b, tb:] = float("nan")
    ydt = torch.float16 if o16 else torch.float32
    y = torch.full((B, T + 2 * H, Cc), float("nan"), dtype=ydt, device="cuda")
    flags = (cabi.TG_A_F16 if a16 else 0) | (cabi.TG_OUT_F16 if o16 else 0) | (cabi.TG_ROUND_TF32 if kind == "tf32" else 0)
    fr = torch.tensor(frames, dtype=torch.int32, device="cuda")
    lib = cabi.load()
    cabi.check(lib.aero_reflect_act_varlen_fwd(_p(x), _p(y[:, H:]), _p(fr), B, T, Cc, T * Cc, (T + 2 * H) * Cc, halo, cabi.ACT_LEAKY,
                                               flags, None), lib)
    torch.cuda.synchronize()
    yc = y.cpu()
    for b, tb in enumerate(frames):
        # the kernel's own arithmetic: one fp32 product with the slope 0.2f (exact in fp64), one rounding to the output type
        src = x[b, :tb].cpu().float().double()
        ref = torch.where(src > 0, src, src * float(np.float32(0.2))).float().double().t()[None]
        if halo:
            ref = F.pad(ref, (halo, halo), mode="reflect")
        ref = ref[0].t().float()
        if kind == "tf32":
            ref = tf32_round(ref)
        ref = ref.to(ydt)
        assert torch.equal(yc[b, H - halo:H + tb + halo], ref), b
        assert (yc[b, H + tb + halo:H + T + halo] == 0).all()
        assert torch.isnan(yc[b, :H - halo].float()).all() and torch.isnan(yc[b, H + T + halo:].float()).all()


# ------------------------------------------------------------------------------------------------ whole forward
def _lengths(m, name):
    """3-8 clips: the longest (L_max), the shortest admissible, and lengths that are not multiples of the ratio product."""
    lo = _shortest(m)
    prod = int(np.prod(m.ratios))
    L_max = {"shipped": 8000, "s3": 12345, "s5": 5513, "s6": 3000}[name]
    mid = [lo + 1, (lo + L_max) // 2 + 3, L_max - prod - 1, 2 * lo + 7]
    return [L_max, lo] + [n for n in mid if lo <= n <= L_max]


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_every_clip_bit_identical_to_its_own_forward(name, precision):
    m = _model(CONFIGS[name], precision)
    lengths = _lengths(m, name)
    assert 3 <= len(lengths) <= 8 and len(set(lengths)) == len(lengths)
    assert any((m.hr_length(n) % int(np.prod(m.ratios))) for n in lengths)
    clips = [white_noise((m.in_channels, n), seed=100 + b).cuda() for b, n in enumerate(lengths)]
    x = _pad(clips, max(lengths))
    y, out_lens = m._engine().forward_varlen(x, lengths)
    assert y.shape == (len(lengths), m.out_channels, max(out_lens))
    for b, c in enumerate(clips):
        want = m(c[None])[0]
        assert out_lens[b] == want.shape[-1]
        assert torch.equal(y[b, :, :out_lens[b]], want), (name, precision, b, lengths[b], rel_l2(y[b, :, :out_lens[b]], want))
        assert (y[b, :, out_lens[b]:] == 0).all()
    # enhance_batch: sorted, at most max_batch per ragged batch, back in input order
    got = enhance_batch(m, clips, max_batch=3)
    for b, c in enumerate(clips):
        assert torch.equal(got[b], y[b, :, :out_lens[b]])


@pytest.mark.parametrize("precision", [0, 1, 2])
def test_one_clip_and_equal_lengths(precision):
    m = _model(CONFIGS["shipped"], precision)
    x = white_noise((3, 1, 7001), seed=5).cuda()
    y, out_lens = m._engine().forward_varlen(x[:1], [7001])
    assert out_lens == [28004] and torch.equal(y, m(x[:1]))
    y, out_lens = m._engine().forward_varlen(x, [7001] * 3)
    assert torch.equal(y, m(x))


@pytest.mark.parametrize("precision", [2, 1, 0])
def test_goldens_in_one_ragged_batch(precision):
    """s1's two clips of 8000 samples and s2's 7001 (the same configuration) in one ragged batch, against the stored reference
    outputs with the bars of tests/test_gpu_seanet.py."""
    m = _model(CASES["s1"][0], precision)
    xs = [case_input("s1")[0], case_input("s1")[1], case_input("s2")[0]]
    gs = [np.load(os.path.join(GOLDEN, f"seanet_{n}.npz")) for n in ("s1", "s2")]
    refs = [(gs[0], 0), (gs[0], 1), (gs[1], 0)]
    out = enhance_batch(m, [x.cuda() for x in xs])
    for x, y, (g, i) in zip(xs, out, refs):
        y = y.cpu()
        assert tuple(y.shape) == g["y"].shape[1:]
        std = x.double().mean(0).std()
        branch = y.double() / std - torch.from_numpy(g["x0"][i, ..., :y.shape[-1]]).double()
        err, err_b = rel_l2(y, g["y"][i]), rel_l2(branch, g["branch"][i, ..., :y.shape[-1]])
        print(f"precision {precision}: out {err:.2e} branch {err_b:.2e}")
        if precision == 0:
            assert err <= 1e-5 and err_b <= 1e-5
        else:
            assert err <= 1e-3 and err_b <= 2e-3


@pytest.mark.parametrize("precision", [0, 2])
def test_padding_never_leaks(precision):
    m = _model(CONFIGS["s6"], precision)
    lengths = [3000, _shortest(m), 2111]
    clips = [white_noise((1, n), seed=30 + b).cuda() for b, n in enumerate(lengths)]
    y0, _ = m._engine().forward_varlen(_pad(clips, 3000), lengths)
    y1, _ = m._engine().forward_varlen(_pad(clips, 3000, float("nan")), lengths)
    assert torch.equal(y0, y1)


def test_forward_varlen_errors():
    m = _model(CONFIGS["shipped"], 2)
    eng = m._engine()
    x = torch.zeros(2, 1, 4000, device="cuda")
    with pytest.raises(ValueError, match="clip 1 of 160 samples"):
        eng.forward_varlen(x, [4000, 160])
    with pytest.raises(ValueError, match="clip 0"):
        eng.forward_varlen(x, [4001, 4000])
    with pytest.raises(ValueError, match="lengths for a batch"):
        eng.forward_varlen(x, [4000])
    y, lens = eng.forward_varlen(x[:0], [])
    assert y.shape[0] == 0 and lens == []
    assert not any(len(k) == 3 for k in eng._bufsets)               # ragged workspaces are released on return


def test_evaluate_batch_seanet_ragged_set():
    m = _model(CASES["s1"][0], 0)
    lens = [8000, 5003, 7001, 4100, 6000]
    lrs = [white_noise((1, n), seed=60 + i).cuda() for i, n in enumerate(lens)]
    hrs = [white_noise((1, 4 * n + d), seed=70 + i).cuda() for i, (n, d) in enumerate(zip(lens, (4, -2, 0, 3, -5)))]
    lsd, mean, count = evaluate_batch(m, lrs, hrs, max_batch=3)
    want = [float(get_lsd(h, match_signal(m(x[None])[0], h.shape[-1]))) for x, h in zip(lrs, hrs)]
    for g, w in zip(lsd.tolist(), want):
        assert abs(g - w) / w < 1e-5, (g, w)
    assert count == len(lens)
