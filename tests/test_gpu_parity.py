"""-m gpu: end-to-end parity of aero_b200.Aero (CUDA kernels through the C ABI) with the reference
forward, via the committed golden vectors, plus size-independent properties at BASELINE.json's full
batch size.  Tolerance: north_star's 1e-3 relative fp32 (the fp32 path lands around 1e-5)."""
import glob
import os

import numpy as np
import pytest
import torch

from util import SEED, rel_l2, trained_like_, weights_digest, white_noise

from aero_b200 import Aero, aero_kwargs

pytestmark = pytest.mark.gpu
TOL = 1e-3
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "c*.npz")))


def build(exp):
    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs(exp)).eval()
    m.load_state_dict(trained_like_(m.state_dict()))
    return m


def wave_error(out, g):
    """rel-L2 of a waveform against a golden file: the whole waveform, or (full-shape cases c7-c9) its committed
    65536-position sample, whose rms must also agree with the rms of the full reference output."""
    if "out" in g.files:
        assert out.shape == g["out"].shape
        return rel_l2(out.cpu(), g["out"])
    assert tuple(out.shape) == tuple(int(v) for v in g["out_shape"])
    flat = out.reshape(-1).cpu()
    assert abs(float(flat.double().pow(2).mean().sqrt()) / float(g["out_rms"]) - 1) < 2e-3
    return rel_l2(flat[torch.from_numpy(g["out_idx"].astype(np.int64))], g["out_val"])


@pytest.mark.parametrize("case", CASES)
def test_forward_matches_reference_golden(golden_dir, case):
    """All-fp32 kernels (engine.precision = 0): agreement with the reference at fp32 round-off level."""
    g = np.load(os.path.join(golden_dir, case + ".npz"))
    m = build(str(g["exp"]))
    assert weights_digest(m.state_dict()) == pytest.approx(float(g["digest"]), rel=1e-12)
    m = m.cuda()
    m._engine().precision = 0
    mix = white_noise((int(g["B"]), m.in_channels, int(g["L"]))).cuda()
    out, zc, zl = m(mix, return_spec=True, return_lr_spec=True)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    err = wave_error(out, g)
    zc_r = torch.view_as_real(zc.contiguous()).cpu().reshape(-1)[torch.from_numpy(g["spec_idx"].astype(np.int64))]
    zl_r = torch.view_as_real(zl.contiguous()).cpu().reshape(-1)[torch.from_numpy(g["lrspec_idx"].astype(np.int64))]
    print(f"{case}: rel_l2 wave {err:.3e} spec {rel_l2(zc_r, g['spec_val']):.3e} lr_spec {rel_l2(zl_r, g['lrspec_val']):.3e}")
    assert err < 2e-5
    assert rel_l2(zc_r, g["spec_val"]) < 2e-5
    assert rel_l2(zl_r, g["lrspec_val"]) < 1e-5
    # plain call returns the same waveform
    assert torch.equal(m(mix), out)


def test_full_batch_properties():
    """BASELINE configs[1]: B=32 x 2 s.  Clips are independent (per-sample norms), so row b of the batch
    must equal the B=1 forward of clip b; and the output must be finite with the reference's length."""
    m = build("aero_4-16_512_64").cuda()
    mix = white_noise((32, 1, 8000)).cuda()
    out = m(mix)
    torch.cuda.synchronize()
    assert out.shape == (32, 1, 32000) and torch.isfinite(out).all()
    for b in (0, 17, 31):
        single = m(mix[b:b + 1])
        # (global fp64 atomics make the GroupNorm sums order-dependent in the last bit; a TF32 rounding flip is ~1e-4 locally)
        assert rel_l2(out[b:b + 1].cpu(), single.cpu()) < 2e-4
    # linearity of the analysis/synthesis pair at full size (STFT of a*x+y)
    x, y = white_noise((32, 1, 8000), seed=3).cuda(), white_noise((32, 1, 8000), seed=4).cuda()
    lhs = m._spec(0.5 * x + y)
    rhs = 0.5 * m._spec(x) + m._spec(y)
    assert rel_l2(torch.view_as_real(lhs).cpu(), torch.view_as_real(rhs).cpu()) < 1e-5


def test_baseline_batch_rows_match_the_oracle():
    """BASELINE configs[1] itself (B=32 x 2 s, default engine): rows {0, 17, 31} of the batch against the ORACLE's forward of
    those clips (not against this repo's own B=1 forward).  north_star bar: 1e-3 relative."""
    from oracle import aero_oracle as O
    m = build("aero_4-16_512_64")
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    mix = white_noise((32, 1, 8000))
    rows = [0, 17, 31]
    with torch.no_grad():
        ref = O.aero_forward(sd, m.geom, mix[rows])
    m = m.cuda()
    assert m._engine().precision == 2
    out = m(mix.cuda())
    torch.cuda.synchronize()
    errs = [rel_l2(out[b].cpu(), ref[i]) for i, b in enumerate(rows)]
    print("B=32 default engine vs oracle, rows 0/17/31:", " ".join(f"{e:.3e}" for e in errs))
    assert max(errs) < TOL


def speech_like(shape, seed):
    """Band-limited, amplitude-modulated noise with a 60 dB level step in the middle: most of its energy below a quarter of
    the band (like speech), a quiet first half (1e-3 of the loud half after the per-sample standardisation of aero.py:462)."""
    x = white_noise(shape, seed=seed)
    n = shape[-1]
    spec = torch.fft.rfft(x)
    f = torch.linspace(0, 1, spec.shape[-1])
    x = torch.fft.irfft(spec * (1.0 / (1.0 + (f / 0.12) ** 4)), n=n)
    env = 0.55 + 0.45 * torch.sin(torch.linspace(0, 37.0, n)) ** 2
    x = x * env
    x[..., : n // 2] *= 1e-3
    return (x / x.abs().max()).contiguous()


def test_hard_input_fp16_range_and_parity():
    """FP16 activation storage under stress: speech-like input with a 60 dB level step and weights re-scaled so that the
    pre-normalisation tensors reach |x| ~ 1e3 (GroupNorm undoes the scale, so the reference output is well defined).
    Checks (1) no FP16 buffer comes near saturation (cvt.rn.satfinite clamps silently at 65504), (2) the default engine agrees
    with the oracle and with the TF32 engine within the 1e-3 bar, (3) the quiet half of the clip is reproduced too."""
    from oracle import aero_oracle as O
    m = build("aero_4-16_512_64")
    sd = m.state_dict()
    big = {}
    for k, v in sd.items():
        pre_norm = (k.startswith(("encoder.2.conv.", "encoder.3.conv.", "encoder.2.rewrite.", "encoder.3.rewrite.",
                                  "decoder.0.rewrite.", "decoder.1.rewrite.", "decoder.0.conv_tr.", "decoder.1.conv_tr."))
                    or ".dconv.layers." in k and (".conv1.0." in k or ".conv2.0." in k))
        big[k] = v * 300.0 if pre_norm else v.clone()
    m.load_state_dict(big)
    mix = speech_like((2, 1, 4000), seed=21)
    with torch.no_grad():
        ref = O.aero_forward({k: v.clone() for k, v in m.state_dict().items()}, m.geom, mix)
    m = m.cuda()
    eng = m._engine()
    eng.use_graph = False
    outs = {}
    for prec in (2, 1):
        eng.precision = prec
        outs[prec] = m(mix.cuda()).cpu()
        if prec == 2:
            torch.cuda.synchronize()
            halves = [(k[0], float(t.float().abs().max())) for k, t in eng._bufs.items() if t.dtype == torch.float16]
            assert halves, "precision 2 must store activations in FP16"
            worst = max(halves, key=lambda kv: kv[1])
            print(f"largest |x| in an FP16 activation buffer: {worst[1]:.1f} ({worst[0]})")
            assert worst[1] < 0.5 * 65504
    e2, e1, e21 = rel_l2(outs[2], ref), rel_l2(outs[1], ref), rel_l2(outs[2], outs[1])
    half = ref.shape[-1] // 2
    q2 = rel_l2(outs[2][..., : half - 600], ref[..., : half - 600])
    print(f"hard input: precision 2 vs oracle {e2:.3e}, precision 1 vs oracle {e1:.3e}, 2 vs 1 {e21:.3e}, quiet half {q2:.3e}")
    assert torch.isfinite(outs[2]).all() and e2 < TOL and e1 < TOL and e21 < TOL
    assert q2 < 5e-3        # the part of the clip 60 dB down: same order as the bar, no blow-up from FP16 subnormals


def test_repeatable_and_buffer_reuse():
    m = build("aero_4-16_512_256").cuda()
    a = white_noise((2, 1, 8000)).cuda()
    b = white_noise((3, 1, 5000), seed=9).cuda()
    o1 = m(a).clone()
    m(b)
    o2 = m(a)
    assert rel_l2(o2.cpu(), o1.cpu()) < 2e-4
    m._engine().precision = 0
    o3 = m(a).clone()
    m(b)
    assert rel_l2(m(a).cpu(), o3.cpu()) < 1e-6


@pytest.mark.parametrize("precision", [2, 1])
@pytest.mark.parametrize("case", CASES)
def test_forward_tensor_core_paths_within_tolerance(golden_dir, case, precision):
    """Tensor-core engines: precision 2 (default; FP16-stored activations, f16 wgmma, fp32 accumulate, fp32
    GroupNorm inputs / gate pre-activations) and precision 1 (fp32 storage rounded to TF32, tf32 wgmma).
    north_star bar: 1e-3 relative."""
    g = np.load(os.path.join(golden_dir, case + ".npz"))
    m = build(str(g["exp"])).cuda()
    assert m._engine().precision == 2
    m._engine().precision = precision
    mix = white_noise((int(g["B"]), m.in_channels, int(g["L"]))).cuda()
    out, zc = m(mix, return_spec=True)
    torch.cuda.synchronize()
    err = wave_error(out, g)
    zc_r = torch.view_as_real(zc.contiguous()).cpu().reshape(-1)[torch.from_numpy(g["spec_idx"].astype(np.int64))]
    print(f"{case} [precision {precision}]: rel_l2 wave {err:.3e} spec {rel_l2(zc_r, g['spec_val']):.3e}")
    assert torch.isfinite(out).all()
    assert err < TOL


def test_lsd_metric_matches_reference_formula():
    """reference src/metrics.py:59-70 (with the torch>=2 `return_complex` shim applied to its STFTMag)."""
    from aero_b200.metrics import get_lsd
    ref_sig, out_sig = white_noise((3, 32000), seed=11), white_noise((3, 32000), seed=12) * 0.7
    out_sig[:, :4000] = 0.0                                        # exercise the 1e-8 clamp
    win = torch.hann_window(2048)

    def mag2(x):
        return torch.stft(x, 2048, 512, window=win, return_complex=True).abs().square().clamp(1e-8)
    want = (torch.log10(mag2(ref_sig)) - torch.log10(mag2(out_sig))).square().mean(dim=1).sqrt().mean()
    got = get_lsd(ref_sig.cuda(), out_sig.cuda())
    assert abs(float(got) - float(want)) / float(want) < 1e-4


def test_enhance_long_on_gpu_equals_serial():
    from aero_b200.enhance import enhance_long
    m = build("aero_4-16_512_256").cuda()
    m._engine().precision = 0
    sig = white_noise((1, 9000))
    got = enhance_long(m, sig.cuda(), sr=4000, segment_sec=0.5, max_batch=3)
    serial = torch.cat([m(sig[None, :, i:i + 2000].cuda())[0] for i in range(0, 9000, 2000)], -1)
    assert got.shape == serial.shape == (1, 36000) and rel_l2(got.cpu(), serial.cpu()) < 1e-6


def test_cuda_graph_replay_matches_eager():
    m = build("aero_4-16_512_256").cuda()
    a, b = white_noise((2, 1, 8000)).cuda(), white_noise((2, 1, 8000), seed=5).cuda()
    ea, eb = m(a).clone(), m(b).clone()
    m.use_cuda_graph(True)
    ga = m(a)
    gb = m(b)
    ga2 = m(a)
    assert rel_l2(ga.cpu(), ea.cpu()) < 2e-4 and rel_l2(gb.cpu(), eb.cpu()) < 2e-4 and rel_l2(ga2.cpu(), ea.cpu()) < 2e-4
    assert not torch.equal(ga, gb)


def test_auto_graph_kicks_in_on_the_third_call_and_matches():
    m = build("aero_4-16_512_256").cuda()
    eng = m._engine()
    assert eng.use_graph == "auto"
    a = white_noise((2, 1, 8000)).cuda()
    outs = [m(a).clone() for _ in range(5)]
    assert len(eng._graphs) == 1
    b = white_noise((1, 1, 6000), seed=3).cuda()          # a new shape goes eager again
    m.use_cuda_graph(False)
    eb = m(b).clone()
    m.use_cuda_graph("auto")
    for _ in range(4):
        gb = m(b)
    assert len(eng._graphs) == 2
    assert rel_l2(gb.cpu(), eb.cpu()) < 2e-4
    for o in outs[1:]:
        assert rel_l2(o.cpu(), outs[0].cpu()) < 2e-4


def test_faster_than_pytorch_eager_on_the_same_gpu():
    """SURVEY.md section 8(d): the existing kernels to beat are PyTorch's own (cuDNN / cuBLAS / cuFFT) running the
    same forward on the same GPU.  The oracle's library-call form makes exactly the reference's torch calls; here it runs
    on the GPU (TF32 allowed, as PyTorch's defaults for convolutions) as a timing reference -- it is not on the product path."""
    from oracle import aero_oracle as O
    m = build("aero_4-16_512_64").cuda()
    sd = {k: v for k, v in m.state_dict().items()}
    x = white_noise((32, 1, 8000)).cuda()

    def timed(fn, n=3):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    try:
        with torch.no_grad():
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = True, True
            ms_eager_tf32 = timed(lambda: O.aero_forward(sd, m.geom, x))
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = False, False
            ms_eager_fp32 = timed(lambda: O.aero_forward(sd, m.geom, x), n=2)
    except (RuntimeError, TypeError) as e:        # the oracle is written for the CPU; an eager-GPU run is a bonus measurement
        pytest.skip(f"oracle does not run on this GPU: {str(e)[:200]}")
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    for _ in range(3):                       # (the third call of a shape captures its CUDA graph: keep that out of the timing)
        m(x)
    ms_ours = timed(lambda: m(x), n=5)
    print(f"B=32 x 2 s forward: PyTorch eager on this GPU {ms_eager_fp32:.1f} ms (fp32) / {ms_eager_tf32:.1f} ms (TF32 allowed); "
          f"aero_b200 {ms_ours:.2f} ms -> {ms_eager_tf32 / ms_ours:.1f}x")
    assert ms_ours < ms_eager_tf32


def test_empty_batch_and_too_short_clip():
    """edge cases of the boundary: an empty batch maps to an empty batch; a clip shorter than the reflect padding raises
    (as torch.stft does in the reference) instead of reading out of bounds."""
    m = build("aero_4-16_512_256").cuda()
    out, zc, zl = m(torch.zeros(0, 1, 8000, device="cuda"), return_spec=True, return_lr_spec=True)
    assert out.shape == (0, 1, 32000) and zc.shape[:3] == (0, 1, 256) and zl.shape[:3] == (0, 1, 256)
    with pytest.raises(Exception, match="reflect padding"):
        m(white_noise((1, 1, 200)).cuda())


def test_mrstft_loss_matches_reference_golden(golden_dir):
    """SURVEY.md section 8f rank 2: aero_b200.losses.MultiResolutionSTFTLoss (aero_stft_fwd + aero_stft_loss_fwd) against
    the values of the reference's module on the same seeded signals."""
    from aero_b200.losses import MultiResolutionSTFTLoss
    from test_oracle import _mrstft_inputs
    g = np.load(os.path.join(golden_dir, "mrstft_cases.npz"))
    loss = MultiResolutionSTFTLoss()
    i = 0
    while f"{i}/params" in g.files:
        x, y = _mrstft_inputs(g, i)
        sc, mag = loss(x.cuda(), y.cuda())
        print(f"mrstft case {i}: sc {float(sc):.6f} (ref {float(g[f'{i}/sc']):.6f}) mag {float(mag):.6f} (ref {float(g[f'{i}/mag']):.6f})")
        assert abs(float(sc) - float(g[f"{i}/sc"])) < 2e-5 * float(g[f"{i}/sc"])
        assert abs(float(mag) - float(g[f"{i}/mag"])) < 1e-4 * float(g[f"{i}/mag"])
        i += 1
    assert i >= 2
