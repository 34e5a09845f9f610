"""-m gpu: ragged batches (AeroEngine.forward_varlen / enhance.enhance_batch).  Each new kernel against the torch statement of
its contract (tests/test_ragged_host.RaggedEmuEngine, fp64 where it sums), golden clips of different lengths batched
together against the reference, and every clip of a ragged batch against its own single-clip forward."""
import os

import numpy as np
import pytest
import torch

from test_ragged_host import RaggedEmuEngine, lengths_for_frames
from util import SEED, rel_l2, trained_like_, white_noise

from aero_b200 import Aero, aero_kwargs
from aero_b200.engine import AeroEngine, _Ragged
from aero_b200.enhance import enhance_batch

pytestmark = pytest.mark.gpu


def build(exp):
    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs(exp)).eval()
    m.load_state_dict(trained_like_(m.state_dict()))
    return m


def engines(frames):
    """The product engine (CUDA) and the contract statement (CPU), both in ragged mode for `frames`."""
    m = build("aero_4-16_512_64")
    emu = RaggedEmuEngine(m)
    emu._vl = _Ragged(frames, "cpu")
    gpu = AeroEngine(build("aero_4-16_512_64").cuda())
    gpu._vl = _Ragged(frames, "cuda")
    return gpu, emu


def test_kernel_contracts():
    torch.manual_seed(1)
    frames = [37, 80, 5]
    gpu, emu = engines(frames)
    B, F_, T, C_ = 3, 4, 80, 24
    for dt in (torch.float32, torch.float16):
        x = torch.randn(B, F_, T, C_).to(dt)
        a, b = x.clone(), x.cuda()
        emu._frame_mask(a)
        gpu._frame_mask(b)
        assert torch.equal(b.cpu(), a)
        for scope, groups in ((1, 4), (2, 1)):
            n = B * groups if scope == 1 else B * F_
            sa, sb = torch.zeros(n, 2, dtype=torch.float64), torch.zeros(n, 2, dtype=torch.float64, device="cuda")
            emu._masked_stats(x, sa, groups=groups, scope=scope)
            gpu._masked_stats(x.cuda(), sb, groups=groups, scope=scope)
            assert rel_l2(sb.cpu(), sa) < 1e-12
        idx = torch.randint(-1, 40, (50, 2), dtype=torch.int32)
        src = torch.randn(40, 16).to(dt)
        fill = torch.randn(16)
        da, db = torch.zeros(50, 16, dtype=dt), torch.zeros(50, 16, dtype=dt, device="cuda")
        emu._gather_rows(src, da, idx, fill, 50)
        gpu._gather_rows(src.cuda(), db, idx.cuda(), fill.cuda(), 50)
        assert torch.equal(db.cpu(), da)
    # STFT / sample norm / iSTFT with per-clip lengths (n_fft 512, hop 16: the 4-16 input analysis)
    g = gpu.geom
    lengths = [1000, 1270, 77 * 16]
    gpu._vl = _Ragged([1 + (n + (-n) % 16) // 16 for n in lengths], "cuda")
    emu._vl = _Ragged(gpu._vl.frames, "cpu")
    T = max(gpu._vl.frames)
    Lp = 16 * (T - 1)
    x = torch.randn(3, Lp)
    kw = dict(n_fft=512, hop=16, win=512, channels=1, bins_out=256, strides=(256 * T * 2, 0, T * 2, 2))
    za, zb = torch.full((3, 256, T, 2), 7.0), torch.full((3, 256, T, 2), 7.0, device="cuda")
    sa, sb = torch.zeros(3, 2, dtype=torch.float64), torch.zeros(3, 2, dtype=torch.float64, device="cuda")
    emu.stft_varlen_into(x, torch.tensor(lengths), za, sa, **kw)
    gpu.stft_varlen_into(x.cuda(), torch.tensor(lengths, dtype=torch.int32, device="cuda"), zb, sb, **kw)
    assert rel_l2(zb.cpu(), za) < 1e-6 and rel_l2(sb.cpu(), sa) < 1e-6
    for b, tb in enumerate(gpu._vl.frames):
        assert (zb[b, :, tb:] == 0).all()
    ya, yb = torch.empty(3, 256 * T * 2), torch.empty(3, 256 * T * 2, device="cuda")
    aa, ab = torch.empty(3, 2), torch.empty(3, 2, device="cuda")
    emu._sample_norm_varlen(za, sa, ya, aa, 3, 256 * 2, 256 * T * 2)
    gpu._sample_norm_varlen(zb, sb, yb, ab, 3, 256 * 2, 256 * T * 2)
    assert rel_l2(yb.cpu(), ya) < 1e-6 and rel_l2(ab.cpu(), aa) < 1e-6
    out_lens = [min(4 * n, 64 * (tb - 1)) for n, tb in zip(lengths, gpu._vl.frames)]
    ikw = dict(n_fft=512, hop=64, win=512, channels=1, frames_max=T, bins_in=256, strides=(256 * T * 2, 0, T * 2, 2))
    wa, wb = torch.empty(3, max(out_lens)), torch.full((3, max(out_lens)), 7.0, device="cuda")
    emu.istft_varlen_into(za, wa, torch.tensor(gpu._vl.frames), torch.tensor(out_lens), **ikw)
    gpu.istft_varlen_into(zb, wb, gpu._vl.frames_d, torch.tensor(out_lens, dtype=torch.int32, device="cuda"), **ikw)
    assert rel_l2(wb.cpu(), wa) < 1e-5
    # attention with per-row length: exact fp32 SIMT kernel and the TF32 mma.sync kernel (head dim 12)
    H, heads, nd = 48, 4, 4
    ld = 3 * H + heads * nd
    frames = [70, 130, 9]
    gpu._vl, emu._vl = _Ragged(frames, "cuda"), _Ragged(frames, "cpu")
    rows, T = 3 * 2, 130
    q = (torch.randn(rows * T, ld) * 0.5)
    for prec, tol in ((0, 1e-5), (1, 3e-3)):
        gpu.precision = prec
        oa = torch.zeros(rows * T, H)
        ob = torch.zeros(rows * T, H, device="cuda")
        emu._attn(q, oa, rows=rows, T=T, H=H, heads=heads, ndecay=nd, ld=ld)
        gpu._attn(q.cuda(), ob, rows=rows, T=T, H=H, heads=heads, ndecay=nd, ld=ld)
        va = oa.view(rows, T, H)
        vb = ob.view(rows, T, H).cpu()
        for r in range(rows):
            tb = frames[r // 2]
            assert rel_l2(vb[r, :tb], va[r, :tb]) < tol, (prec, r)
            assert (vb[r, tb:] == 0).all()            # padded queries are not written


@pytest.mark.parametrize("pair", [("c1_4-16_hop64_b2", "c6_4-16_hop64_short"), ("c3_12-48_hop128", "c7_12-48_hop128_b2_2s"),
                                  ("c4_11-44_stereo", "c8_11-44_stereo_4s")])
@pytest.mark.parametrize("precision", [0, 1, 2])
def test_golden_clips_batched_together(golden_dir, pair, precision):
    """Golden cases that share weights, all their clips in one ragged batch (4-16: T = 501 and 101; 12-48; 11-44 stereo);
    each case's clips against the reference under the bars of its single-clip golden test: precision 0 as
    test_gpu_parity.test_forward_matches_reference_golden (waveform, spectrogram, input spectrogram), 1 / 2 the waveform
    within 1e-3."""
    from test_gpu_parity import wave_error
    gs = [np.load(os.path.join(golden_dir, c + ".npz")) for c in pair]
    assert str(gs[0]["exp"]) == str(gs[1]["exp"])
    m = build(str(gs[0]["exp"])).cuda()
    m._engine().precision = precision
    sigs, owner = [], []
    for i, g in enumerate(gs):
        mix = white_noise((int(g["B"]), m.in_channels, int(g["L"])))
        sigs += [mix[b].cuda() for b in range(mix.shape[0])]
        owner += [i] * mix.shape[0]
    outs = enhance_batch(m, sigs, return_spec=True, return_lr_spec=True)
    for i, (c, g) in enumerate(zip(pair, gs)):
        out, zc, zl = (torch.stack([o[k] for o, w in zip(outs, owner) if w == i]) for k in range(3))
        err = wave_error(out, g)
        zc_r = torch.view_as_real(zc.contiguous()).cpu().reshape(-1)[torch.from_numpy(g["spec_idx"].astype(np.int64))]
        zl_r = torch.view_as_real(zl.contiguous()).cpu().reshape(-1)[torch.from_numpy(g["lrspec_idx"].astype(np.int64))]
        es, el = rel_l2(zc_r, g["spec_val"]), rel_l2(zl_r, g["lrspec_val"])
        print(f"precision {precision} {c} in a ragged batch: rel_l2 wave {err:.2e} spec {es:.2e} lr_spec {el:.2e}")
        if precision == 0:
            assert err < 2e-5 and es < 2e-5 and el < 1e-5
        else:
            assert err < 1e-3


@pytest.mark.parametrize("exp,C", [("aero_4-16_512_64", 1), ("aero_12-48_512_128", 1), ("aero_11-44_512_64", 2)])
@pytest.mark.parametrize("precision", [0, 1, 2])
def test_ragged_equals_single_clip(exp, C, precision):
    m = build(exp).cuda()
    m._engine().precision = precision
    lengths = lengths_for_frames(m, [101, 200, 201, 299, 300, 301, 700]) if exp == "aero_4-16_512_64" else \
        lengths_for_frames(m, [60, 230, 450])
    sigs = [white_noise((C, n), seed=20 + i).cuda() for i, n in enumerate(lengths)]
    outs = enhance_batch(m, sigs, return_spec=True, return_lr_spec=True)
    # The only arithmetic the ragged batch does differently is the GroupNorm statistics: one fp64 pass over the valid frames
    # instead of the tap-GEMM epilogue's fp32 tile partials (test_one_clip_ragged_batch_is_exact_up_to_statistics).  At
    # precision 0 that is ~1e-6 here.  At precisions 1 / 2 every stored activation has a 10-bit mantissa, and a change of the
    # statistics in their last fp32 bit alone moves the forward by more than 1e-4 (test_statistics_sensitivity_at_reduced_
    # precision); measured 2.9-4.1e-4 on an H100 80GB HBM3 (700 W).
    tol = 1e-5 if precision == 0 else 5e-4
    worst = [0.0, 0.0, 0.0]
    for s, got in zip(sigs, outs):
        want = m(s[None], return_spec=True, return_lr_spec=True)
        for k in range(3):
            a, b = got[k], want[k][0]
            assert a.shape == b.shape
            if a.is_complex():
                a, b = torch.view_as_real(a), torch.view_as_real(b)
            worst[k] = max(worst[k], rel_l2(a.cpu(), b.cpu()))
    print(f"{exp} precision {precision}: worst rel_l2 vs single clip: wave {worst[0]:.2e} spec {worst[1]:.2e} "
          f"lr_spec {worst[2]:.2e}")
    assert max(worst) < tol


@pytest.mark.parametrize("precision", [0, 2])
def test_padding_never_leaks(precision):
    """Samples past each clip's length filled with noise of amplitude 1e3: no output moves."""
    m = build("aero_4-16_512_64").cuda()
    m._engine().precision = precision
    eng = m._engine()
    lengths = lengths_for_frames(m, [101, 301, 700])
    L = max(lengths) + 100
    mix = torch.zeros(3, 1, L, device="cuda")
    noisy = 1e3 * white_noise((3, 1, L), seed=9).cuda()
    for b, n in enumerate(lengths):
        s = white_noise((1, n), seed=30 + b).cuda()
        mix[b, :, :n] = s
        noisy[b, :, :n] = s
    y0, l0, zc0, zl0 = eng.forward_varlen(mix, lengths, return_spec=True, return_lr_spec=True)
    y1, l1, zc1, zl1 = eng.forward_varlen(noisy, lengths, return_spec=True, return_lr_spec=True)
    assert l0 == l1
    for b, n in enumerate(lengths):
        tb = m.geom.frames(n)
        assert rel_l2(y1[b, :, :l0[b]].cpu(), y0[b, :, :l0[b]].cpu()) < 1e-6
        assert rel_l2(torch.view_as_real(zc1[b, ..., :tb]).cpu(), torch.view_as_real(zc0[b, ..., :tb]).cpu()) < 1e-6
        assert rel_l2(torch.view_as_real(zl1[b, ..., :tb]).cpu(), torch.view_as_real(zl0[b, ..., :tb]).cpu()) < 1e-6


def test_errors_match_the_single_clip_forward():
    m = build("aero_4-16_512_256").cuda()
    assert enhance_batch(m, []) == []
    with pytest.raises(Exception, match="reflect padding"):
        enhance_batch(m, [white_noise((1, 3000)).cuda(), white_noise((1, 200)).cuda()])
    with pytest.raises(RuntimeError):
        enhance_batch(m, [white_noise((1, 3000))])
    with pytest.raises(ValueError):
        enhance_batch(m, [white_noise((2, 3000)).cuda()])


def _epilogue_statistics(self, raw, w, st, *, scope, groups, **kw):
    return self._gemm(raw, w, stats=st, stats_mode=scope, groups=groups, **kw)


@pytest.mark.parametrize("precision", [0, 1, 2])
def test_one_clip_ragged_batch_is_exact_up_to_statistics(monkeypatch, precision):
    """A ragged batch of one clip has no padded frame, so the tap-GEMM epilogue's statistics are valid for it.  With them the
    ragged path (varlen STFT / iSTFT fast paths, per-clip sample norm, frame masks, BiLSTM gathers around the wgmma or SIMT
    recurrence, per-row attention) must reproduce model(clip[None]) bit for bit: everything but the masked statistics pass
    is exact."""
    m = build("aero_4-16_512_64").cuda()
    eng = m._engine()
    eng.precision = precision
    eng.use_graph = False
    monkeypatch.setattr(AeroEngine, "_gemm_norm", _epilogue_statistics)
    for i, t in enumerate((101, 301, 700)):
        s = white_noise((1, lengths_for_frames(m, [t])[0]), seed=40 + i).cuda()
        y, lens = eng.forward_varlen(s[None], [s.shape[-1]])
        assert torch.equal(y, m(s[None]))


def test_statistics_sensitivity_at_reduced_precision(monkeypatch):
    """Scaling every GroupNorm statistics slot of the ordinary single-clip forward by (1 + 2^-23), one fp32 ulp, moves the
    precision-2 output by more than 1e-4: 1e-4 is below what any change of summation order in the statistics can hold."""
    m = build("aero_4-16_512_64").cuda()
    eng = m._engine()
    eng.use_graph = False
    s = white_noise((1, lengths_for_frames(m, [301])[0]), seed=41).cuda()
    ref = m(s[None])
    orig = AeroEngine._norm_act

    def nudged(self, x, stats, *a, **k):
        stats.mul_(1 + 2.0 ** -23)
        return orig(self, x, stats, *a, **k)
    monkeypatch.setattr(AeroEngine, "_norm_act", nudged)
    err = rel_l2(m(s[None]).cpu(), ref.cpu())
    print(f"precision 2, GroupNorm statistics scaled by 1 + 2^-23: output moves by {err:.2e} rel-L2")
    assert err > 1e-4
