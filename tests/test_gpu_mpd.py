"""-m gpu: the HiFi-GAN multi-period discriminator (aero_b200.mpd) on the CUDA kernels against the fp64 goldens of the unmodified
reference (tests/golden/mpd_*.npz) in exact and TF32 mode, plus one [msd_melgan, mpd] adversarial step on AERO."""
import os

import numpy as np
import pytest
import torch

from mpd_util import CASES, case_inputs, mpd_loss
from util import SEED, disc_recipe_state, rel_l2, trained_like_, weights_digest, white_noise

from aero_b200 import cabi
from aero_b200.mpd import MultiPeriodDiscriminator

pytestmark = pytest.mark.gpu


def _model(g, kw):
    torch.manual_seed(SEED)
    d = MultiPeriodDiscriminator(**kw)
    d.load_state_dict(disc_recipe_state(d.state_dict()))
    assert weights_digest(d.state_dict()) == pytest.approx(float(g["digest"]), rel=1e-12)
    return d.cuda()


def _grad_rows(named, g):
    """Per-parameter relative error on the committed samples (normalised as test_melgan_discriminator_matches_reference) and the
    deviation of all gradients together (the 256 samples standing for the whole tensor)."""
    gmax = max(float(g[k]) for k in g.files if k.startswith("g_rms/"))
    rows, num, den = [], 0.0, 0.0
    for name, grad in named:
        ref = torch.from_numpy(g["g_val/" + name]).double()
        got = grad.reshape(-1).cpu().double()[torch.from_numpy(g["g_idx/" + name].astype(np.int64))]
        rows.append((float((got - ref).norm()) / max(float(ref.norm()), 1e-4 * gmax * ref.numel() ** 0.5), name))
        scale = grad.numel() / ref.numel()
        num += scale * float((got - ref).pow(2).sum())
        den += scale * float(ref.pow(2).sum())
    return sorted(rows, reverse=True), (num / den) ** 0.5


def _run(d, name):
    y, y_hat = (t.cuda().requires_grad_(True) for t in case_inputs(name))
    outs = d(y, y_hat)
    loss = mpd_loss(outs)
    loss.backward()
    torch.cuda.synchronize()
    return outs, loss, y.grad, y_hat.grad


@pytest.mark.parametrize("name", sorted(CASES))
def test_mpd_matches_reference(golden_dir, name):
    """Exact fp32 mode (train_precision 0) against the fp64 goldens."""
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    kw = CASES[name][0]
    d = _model(g, kw)
    (y_d_rs, y_d_gs, fmap_rs, fmap_gs), loss, dy, dy_hat = _run(d, name)
    worst_f = 0.0
    for i in range(len(kw["periods"])):
        for side, (logits, fmap) in enumerate(((y_d_rs[i], fmap_rs[i]), (y_d_gs[i], fmap_gs[i]))):
            worst_f = max(worst_f, rel_l2(logits.detach().cpu(), g[f"logits/{i}/{side}"]))
            assert len(fmap) == 6
            for j, f in enumerate(fmap):
                assert tuple(f.shape) == tuple(int(v) for v in g[f"f_shape/{i}/{side}/{j}"])
                got = f.detach().reshape(-1).cpu()[torch.from_numpy(g[f"f_idx/{i}/{side}/{j}"].astype(np.int64))]
                worst_f = max(worst_f, rel_l2(got, g[f"f_val/{i}/{side}/{j}"]))
    e_dx = max(rel_l2(dy.cpu(), g["dy"]), rel_l2(dy_hat.cpu(), g["dy_hat"]))
    rows, total = _grad_rows([(n, p.grad) for n, p in d.named_parameters()], g)
    print(f"{name}: features / logits {worst_f:.2e}, loss {float(loss):.6e} (ref {float(g['loss']):.6e}), "
          f"d input {e_dx:.2e}, all gradients {total:.2e}; worst parameters:", [(f"{a:.1e}", b) for a, b in rows[:3]])
    assert worst_f < 2e-5 and e_dx < 1e-4 and rows[0][0] < 1e-3


def test_tf32_mode_is_as_accurate_as_the_reference_under_pytorchs_default_tf32(golden_dir):
    """TF32 mode against the oracle (the reference's algorithm as torch functional code) on cuDNN with allow_tf32 = True, PyTorch's
    default for convolutions: the all-parameter gradient deviation from the fp64 golden is at most 1.5x the oracle's."""
    from oracle import mpd_oracle as O
    name = "mpd_default"
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    kw = CASES[name][0]
    d = _model(g, kw)
    names = [n for n, _ in d.named_parameters()]
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        sd = {k: v.detach().clone().requires_grad_(True) for k, v in d.state_dict().items()}
        y, y_hat = (t.cuda() for t in case_inputs(name))
        mpd_loss(O.mpd_forward(sd, kw["periods"], y, y_hat)).backward()
    finally:
        torch.backends.cudnn.allow_tf32 = old
    _, dev_ref = _grad_rows([(n, sd[n].grad) for n in names], g)
    d.train_precision = 1
    _run(d, name)
    _, dev = _grad_rows([(n, p.grad) for n, p in d.named_parameters()], g)
    print(f"all-parameter gradient deviation from fp64: oracle on cuDNN TF32 {dev_ref:.2e}, TF32 mode {dev:.2e}")
    assert dev <= 1.5 * dev_ref


class _RecordingLib:
    """Forwards to the kernel library and records the parameter block of every tap-GEMM launch, and of every weight-gradient launch
    with whether it ran on the tensor cores."""

    def __init__(self, lib):
        self._lib = lib
        self.calls, self.wgrads = [], []

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def aero_tapgemm_fwd(self, *args):
        p = args[10]._obj
        self.calls.append(type(p).from_buffer_copy(p))
        return self._lib.aero_tapgemm_fwd(*args)

    def aero_tapgemm_wgrad(self, *args):
        p = args[4]._obj
        tc = p.precision == 1 and bool(self._lib.aero_tapgemm_wgrad_tc_eligible(args[4], args[0], args[1], args[2]))
        self.wgrads.append((type(p).from_buffer_copy(p), tc))
        return self._lib.aero_tapgemm_wgrad(*args)


def test_dense_layers_run_on_the_tensor_cores_in_tf32_mode(monkeypatch):
    """train_precision 1: the forward of layers 2-5 on the wgmma tap-GEMM, their weight gradients on the TF32 weight-gradient kernel."""
    rec = _RecordingLib(cabi.load())
    monkeypatch.setattr(cabi, "load", lambda *a, **k: rec)
    torch.manual_seed(SEED)
    h = 32
    d = MultiPeriodDiscriminator(hidden=h, periods=[3]).cuda()
    d.train_precision = 1
    y, y_hat = white_noise((2, 1, 4000)).cuda(), white_noise((2, 1, 4000), seed=5).cuda().requires_grad_(True)
    _, y_d_gs, _, fmap_gs = d(y, y_hat)
    (y_d_gs[0].square().mean() + sum(f.abs().mean() for f in fmap_gs[0])).backward()
    torch.cuda.synchronize()
    # layers 2-5 as (K, N, taps): (3*32, 128, 2), (3*128, 512, 2), (3*512, 1024, 2), (1024, 1024, 5)
    dense = {(3 * h, 4 * h, 2), (12 * h, 16 * h, 2), (48 * h, 32 * h, 2), (32 * h, 32 * h, 5)}
    fwd, wgrad = {}, {}
    for p in rec.calls:
        if (p.C1, p.N, p.kt) in dense:
            fwd.setdefault((p.C1, p.N, p.kt), set()).add(p.precision)
    for p, tc in rec.wgrads:
        if (p.C1, p.N, p.kt) in dense:
            wgrad.setdefault((p.C1, p.N, p.kt), set()).add(tc)
    assert set(fwd) == dense and all(v == {1} for v in fwd.values()), fwd
    assert set(wgrad) == dense and all(v == {True} for v in wgrad.values()), wgrad


def test_adversarial_step_with_melgan_and_mpd():
    """One [msd_melgan, mpd] step of the reference (solver.py:475-520 and 580-598, loss formulas of discriminators.py:211-244 restated)
    on AERO with plain autograd and FusedAdam for both networks: finite losses, all three parameter sets move."""
    from aero_b200 import Aero, aero_kwargs
    from aero_b200.discriminator import Discriminator
    from aero_b200.optim import FusedAdam
    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs("aero_4-16_512_256"))
    m.load_state_dict(trained_like_(m.state_dict()))
    m = m.cuda().train()
    torch.manual_seed(SEED + 1)
    msd = Discriminator(3, 16, 4, 4).cuda()
    mpd = MultiPeriodDiscriminator().cuda()
    opt_g = FusedAdam(m.parameters(), lr=3e-4, betas=(0.8, 0.99))
    opt_d = FusedAdam(list(msd.parameters()) + list(mpd.parameters()), lr=3e-4, betas=(0.8, 0.99))
    lr_b, hr = white_noise((2, 1, 4000)).cuda(), white_noise((2, 1, 16000), seed=5).cuda() * 0.1
    before = [[p.detach().clone() for p in n.parameters()] for n in (m, msd, mpd)]

    def d_loss(real, fake):
        return sum(torch.mean((1 - r) ** 2) + torch.mean(f ** 2) for r, f in zip(real, fake))

    def feat_loss(fr, fg):
        terms = [torch.mean(torch.abs(a - b)) for dr, dg in zip(fr, fg) for a, b in zip(dr, dg)]
        return sum(terms) / len(terms)

    pr = m(lr_b)
    # discriminators (solver.py:475-486, 583-585)
    real, fake = msd(hr), msd(pr.detach())
    loss_d = sum(torch.relu(1 - s[-1]).mean() + torch.relu(1 + f[-1]).mean() for s, f in zip(real, fake))
    y_r, y_g, _, _ = mpd(hr, pr.detach())
    loss_d = loss_d + d_loss(y_r, y_g)
    opt_d.zero_grad()
    loss_d.backward()
    opt_d.step()
    # generator (solver.py:488-520, 587-590)
    real, fake = msd(hr), msd(pr)
    loss_g = sum(torch.relu(1 - f[-1]).mean() for f in fake)
    w = (1.0 / 3) * (4.0 / (4 + 1))                       # 1 / num_D * 4 / (n_layers + 1)
    loss_g = loss_g + 100 * w * sum(torch.abs(b - a.detach()).mean() for s, f in zip(real, fake) for a, b in zip(s[:-1], f[:-1]))
    y_r, y_g, f_r, f_g = mpd(hr, pr)
    loss_g = loss_g + sum(torch.mean((1 - g_) ** 2) for g_ in y_g) + 100 * feat_loss(f_r, f_g)
    opt_g.zero_grad()
    loss_g.backward()
    opt_g.step()
    torch.cuda.synchronize()
    print(f"adversarial step: discriminators {float(loss_d):.5f}, generator {float(loss_g):.5f}")
    assert torch.isfinite(loss_d) and torch.isfinite(loss_g)
    for net, b in zip((m, msd, mpd), before):
        assert any(not torch.equal(a, p) for a, p in zip(b, net.parameters()))
