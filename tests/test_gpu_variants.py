"""-m gpu: the AERO variants switched by `act_func` and `spec_upsample` (reference aero.py:306-307) on the kernels -- forward
against the unmodified reference's golden vectors (tests/golden/vf_*.npz), parameter gradients against its fp64 autograd
(tests/golden/vt_*.npz), one adversarial step against the autograd route -- and `aero_b200.resample` against the fp64
resampler of the oracle."""
import json
import math
import os

import numpy as np
import pytest
import torch

from test_gpu_gan import grad_rows
from test_gpu_parity import TOL
from test_gpu_train import GRAD_TOL, cotangent, grad_report
from util import SEED, rel_l2, trained_like_, weights_digest, white_noise

from aero_b200 import Aero, aero_kwargs, resample
from aero_b200 import gan as G
from aero_b200.discriminator import Discriminator
from aero_b200.enhance import enhance_long
from aero_b200.losses import MultiResolutionSTFTLoss
from aero_b200.trainer import GanTrainer
from oracle import seanet_oracle as SO

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FWD = ["vf_gelu_4-16_hop64", "vf_relu_4-16_hop64_ragged_b2", "vf_sinc_4-16_hop64"]
TRAIN = ["vt_relu_4-16_hop64", "vt_sinc_4-16_hop64"]
RATIOS = [(4000, 16000), (8000, 24000), (12000, 48000), (11025, 44100), (16000, 24000), (16000, 4000), (44100, 16000)]


def build(kw):
    torch.manual_seed(SEED)
    m = Aero(**kw)
    m.load_state_dict(trained_like_(m.state_dict()))
    return m


def load_case(case):
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    kw = dict(aero_kwargs(str(g["exp"])), **json.loads(str(g["overrides"]) if "overrides" in g.files else "{}"))
    m = build(kw)
    assert weights_digest(m.state_dict()) == pytest.approx(float(g["digest"]), rel=1e-12)
    if "mix" in g.files:
        mix = torch.from_numpy(g["mix"])
    else:
        mix = white_noise((int(g["B"]), m.in_channels, int(g["L"])))
    return g, m, mix


def sampled(z, idx):
    return torch.view_as_real(z.contiguous()).cpu().reshape(-1)[torch.from_numpy(idx.astype(np.int64))]


# ------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("case", FWD)
def test_forward_matches_reference_golden(case, precision):
    """Waveform and both spectrogram outputs: fp32 round-off at precision 0 (the bars of test_gpu_parity's exact-fp32 test),
    the 1e-3 bar on the tensor-core engines; graph replay equals the eager forward."""
    g, m, mix = load_case(case)
    m = m.cuda().eval()
    eng = m._engine()
    eng.precision = precision
    mix = mix.cuda()
    out, zc, zl = m(mix, return_spec=True, return_lr_spec=True)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and out.shape == g["out"].shape
    e_w, e_s, e_l = rel_l2(out.cpu(), g["out"]), rel_l2(sampled(zc, g["spec_idx"]), g["spec_val"]), \
        rel_l2(sampled(zl, g["lrspec_idx"]), g["lrspec_val"])
    print(f"{case} [precision {precision}]: rel_l2 wave {e_w:.3e} spec {e_s:.3e} lr_spec {e_l:.3e}")
    if precision == 0:
        assert e_w < 2e-5 and e_s < 2e-5 and e_l < 1e-5
    else:
        assert e_w < TOL and e_s < TOL and e_l < TOL
    eager = m(mix)
    eng.use_graph = True
    replay = [m(mix).clone() for _ in range(2)]
    assert len(eng._graphs) == 1
    if precision == 0:
        assert torch.equal(eager, out) and all(torch.equal(r, out) for r in replay)
    else:   # fp64 atomics order the GroupNorm sums differently from launch to launch: a TF32 / FP16 rounding may flip
        assert all(rel_l2(r.cpu(), eager.cpu()) < 1e-5 for r in replay)


def test_sinc_spec_scale_equals_spec():
    """spec_upsample=False: scale is 1, so `_spec(x, scale=True)` analyses on the input grid."""
    m = build(aero_kwargs("aero_4-16_512_64_sinc")).cuda().eval()
    x = white_noise((2, 1, 8001), seed=5).cuda()
    assert torch.equal(m._spec(x, scale=True), m._spec(x))


# ------------------------------------------------------------------------------------------------ training
@pytest.mark.parametrize("case", TRAIN)
def test_parameter_gradients_match_reference_autograd(case):
    """The tiers of test_gpu_train (neither case is free of activations near the FTB ReLU kinks): all gradients together
    <= 5e-3, at least a third of the parameters <= 1e-3, none above 5e-2; loss and train-mode output as there."""
    g, m, mix = load_case(case)
    m = m.cuda().train()
    out = m(mix.cuda())
    assert tuple(out.shape) == tuple(int(v) for v in g["out_shape"])
    e_out = rel_l2(out.detach().reshape(-1).cpu()[torch.from_numpy(g["out_idx"].astype(np.int64))], g["out_val"])
    R = cotangent(tuple(out.shape), SEED).cuda()
    loss = (out * R).sum() / out.numel()
    loss.backward()
    torch.cuda.synchronize()
    assert not any(".act." in n for n, _ in m.named_parameters()) or m.act_func == "snake"
    rows, total = grad_report(m, g)
    ok = sum(1 for r in rows if r[0] < GRAD_TOL)
    print(f"{case}: output {e_out:.3e}, loss {float(loss):.6e} (ref {float(g['loss']):.6e}), all gradients {total:.3e}, "
          f"{ok}/{len(rows)} within {GRAD_TOL:g}, worst {[(f'{a:.1e}', n) for a, n, _ in rows[:3]]}")
    assert e_out < 2e-5
    assert abs(float(loss) - float(g["loss"])) < 1e-4 * max(abs(float(g["loss"])), 1e-6) + 1e-9
    assert total < 5e-3 and ok >= len(rows) / 3 and rows[0][0] < 5e-2


@pytest.mark.parametrize("exp", ["aero_4-16_512_64_relu", "aero_4-16_512_64_sinc"])
def test_gan_step_matches_the_autograd_route(exp):
    """One GanTrainer step with [msd_melgan] at train_precision 0 against the autograd route (the bars of test_gpu_gan)."""
    kw = aero_kwargs(exp)
    L_hr = 8000
    L_in = L_hr if not kw["spec_upsample"] else L_hr * kw["lr_sr"] // kw["hr_sr"]

    def nets():
        torch.manual_seed(SEED + 1)
        return build(kw).cuda(), {"msd_melgan": Discriminator(3, 16, 4, 4).cuda()}
    (gen, discs), (gen_b, discs_b) = nets(), nets()
    lr_b = white_noise((2, 1, L_in), seed=21).cuda()
    hr = white_noise((2, 1, L_hr), seed=22).cuda() * 0.1
    mrstft = MultiResolutionSTFTLoss()
    got = GanTrainer(gen, discs, lr=3e-4).step(lr_b, hr, mrstft)
    gen_b.train()
    want = G.autograd_losses(gen_b(lr_b), hr, discs_b, mrstft)
    sum(want["generator"].values()).backward()
    for d in discs_b.values():
        d.zero_grad(set_to_none=True)
    sum(want["discriminator"].values()).backward()
    torch.cuda.synchronize()
    rows, num, den = [], 0.0, 0.0
    for a, b in [(gen, gen_b), (discs["msd_melgan"], discs_b["msd_melgan"])]:
        pairs = [(n, pa.grad.double(), pb.grad.double()) for (n, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters())]
        rows += grad_rows(pairs)
        num += sum(float((x - y).pow(2).sum()) for _, x, y in pairs)
        den += sum(float(y.pow(2).sum()) for _, _, y in pairs)
    rows.sort(reverse=True)
    total = (num / den) ** 0.5
    loss_err = max(abs(float(got[s][k]) - float(v)) / max(abs(float(v)), 1e-30) for s in want for k, v in want[s].items())
    print(f"{exp}: losses {loss_err:.2e}, all gradients {total:.2e}, worst {[(f'{a:.1e}', n) for a, n in rows[:3]]}")
    assert loss_err < 1e-5 and rows[0][0] < 2e-2 and total < 1e-5


# ------------------------------------------------------------------------------------------------ resampler
def fp64_with_fp32_table(x, orig, new):
    """The oracle's resampler evaluated in fp64 on the filter table torchaudio builds for an fp32 input (the one
    aero_b200.resample uses): what is left is the device's fp32 arithmetic."""
    kern, width = SO.resample_table(orig, new, torch.float32)
    g = math.gcd(orig, new)
    o = orig // g
    w = torch.nn.functional.pad(x.double().reshape(-1, x.shape[-1]), (width, width + o))
    y = torch.nn.functional.conv1d(w[:, None], kern.double(), stride=o).transpose(1, 2).reshape(w.shape[0], -1)
    return y[..., :math.ceil(new // g * x.shape[-1] / o)].reshape(*x.shape[:-1], -1)


@pytest.mark.parametrize("orig,new", RATIOS)
def test_resample_matches_fp64(orig, new):
    """<= 1e-6 against the fp64 evaluation of the same (fp32) filter table; <= 1e-5 against the all-fp64 resampler, whose table
    differs from torchaudio's fp32 one by the rounding of the sinc arguments (~5e-6 on the 475-tap 441:160 filter)."""
    g = math.gcd(orig, new)
    o = orig // g
    for shape in [(1,), (3,), (2, 1, 1001), (1, 2, 5 * o + 1), (4, 8000)]:
        x = white_noise(shape, seed=sum(shape))
        want = SO.resample(x.double(), orig, new)
        got = resample(x.cuda(), orig, new)
        assert got.shape == want.shape == (*shape[:-1], math.ceil(new // g * shape[-1] / o)), (shape, got.shape)
        err, err64 = rel_l2(got.cpu(), fp64_with_fp32_table(x, orig, new)), rel_l2(got.cpu(), want)
        print(f"{orig}->{new} {shape}: rel_l2 {err:.2e} (same table, fp64), {err64:.2e} (fp64 table)")
        assert err < 1e-6 and err64 < 1e-5, (orig, new, shape, err, err64)
    x = white_noise((2, 100)).cuda()
    assert resample(x, orig, orig) is x


def test_enhance_long_upsample_equals_the_reference_loop():
    """reference predict.py:55-86 with `upsample: true`: the whole file resampled to hr_sr, then 10-s chunks of hr_sr samples each
    through the model on their own."""
    m = build(aero_kwargs("aero_4-16_512_64_sinc")).cuda().eval()
    m.use_cuda_graph(False)
    m._engine().precision = 0             # batched chunks against single ones: no TF32 rounding flips between the two
    sig = white_noise((1, 4000 * 23 + 777), seed=31).cuda()
    got = enhance_long(m, sig, 4000, upsample=True)
    up = resample(sig, 4000, 16000)
    seg = 16000 * 10
    want = torch.cat([m(up[None, :, i:i + seg])[0] for i in range(0, up.shape[-1], seg)], dim=-1)
    assert got.shape == want.shape == up.shape
    assert rel_l2(got.cpu(), want.cpu()) < 1e-5
