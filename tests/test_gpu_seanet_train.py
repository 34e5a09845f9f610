"""SEANet training on the H100: the autograd route (SeanetTrainEngine) against the reference's fp64 gradients (t1 golden), in each
train_precision, and one adversarial step as src/solver.py takes it."""
import os

import numpy as np
import pytest
import torch

from util import SEED, rel_l2
from seanet_util import CASES, seanet_recipe_state, train_case

from aero_b200 import Seanet

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _grads(precision):
    torch.manual_seed(SEED)
    m = Seanet(**CASES["s1"][0])
    m.load_state_dict(seanet_recipe_state(m.state_dict()))
    m = m.cuda().train()
    m.train_precision = precision
    x, R = train_case()
    out = m(x.cuda())
    loss = (out.double() * R.cuda().double()).sum()
    loss.backward()
    torch.cuda.synchronize()
    return float(loss), {k: p.grad.detach().cpu().reshape(-1) for k, p in m.named_parameters()}


def _errors(grads, g):
    per = {}
    num = den = 0.0
    for k, gr in grads.items():
        ref = torch.from_numpy(g[f"grad_val/{k}"])
        got = gr[torch.from_numpy(g[f"grad_idx/{k}"]).long()].double()
        per[k] = rel_l2(got, ref)
        num += float((got - ref).pow(2).sum())
        den += float(ref.pow(2).sum())
    return per, (num / den) ** 0.5


def test_exact_mode_gradients_match_reference():
    g = np.load(os.path.join(GOLDEN, "seanet_t1.npz"))
    loss, grads = _grads(0)
    per, together = _errors(grads, g)
    worst = max(per, key=per.get)
    print(f"t1 precision 0: loss {loss:.8e} (ref {float(g['loss']):.8e}), worst gradient {worst} {per[worst]:.2e}, together {together:.2e}")
    assert len(grads) == 252
    # rms of every full gradient, not only the samples
    for k, gr in grads.items():
        assert float(gr.double().pow(2).mean().sqrt()) == pytest.approx(float(g[f"grad_rms/{k}"]), rel=1e-3), k
    # Per-parameter tier 5e-3 instead of 1e-3, traced: the reference's own ops run in fp32 (oracle/seanet_oracle.py under torch autograd
    # on the CPU, fp32) deviate from its fp64 gradients by up to 5.5e-3 on this golden (decoder.1.3.block.2.weight_v; two parameters
    # above 1e-3).  These gradients are sums over 32256 frames with strong cancellation (sum|a*dy| / |sum a*dy| = 86-223 for the
    # layers measured), so fp32 rounding of the activations alone moves single parameters past 1e-3.  Measured here: worst
    # 1.5e-3 (encoder.0.1.weight_v), all gradients together 3.0e-4.
    assert max(per.values()) <= 5e-3
    assert together <= 1e-3
    # the loss is a sum of 32000 products of fp32 outputs (rel-L2 ~1e-7 against fp64) with R: about 2e-5 of it is that rounding
    assert loss == pytest.approx(float(g["loss"]), rel=1e-5)


def test_tensor_core_modes():
    g = np.load(os.path.join(GOLDEN, "seanet_t1.npz"))
    _, grads3 = _grads(3)
    _, together3 = _errors(grads3, g)
    _, grads1 = _grads(1)
    _, together1 = _errors(grads1, g)
    print(f"t1 all gradients together: precision 3 {together3:.2e}, precision 1 {together1:.2e}")
    assert together3 <= 5e-3
    assert together1 <= 5e-2


def test_adversarial_step_end_to_end():
    """What src/solver.py does with `losses: [stft]` and the MelGAN discriminator: generator and discriminator losses, backward,
    Adam; every value finite and the parameters moved."""
    from aero_b200.discriminator import Discriminator
    from aero_b200.losses import MultiResolutionSTFTLoss
    from aero_b200.optim import FusedAdam
    torch.manual_seed(SEED)
    gen = Seanet(**CASES["s1"][0]).cuda().train()
    disc = Discriminator(3, 16, 4, 4).cuda().train()
    opt_g = FusedAdam(gen.parameters(), lr=3e-4, betas=(0.9, 0.999))
    opt_d = FusedAdam(disc.parameters(), lr=3e-4, betas=(0.9, 0.999))
    mrstft = MultiResolutionSTFTLoss()
    lr, hr = train_case()
    lr, hr = lr.cuda(), torch.randn(2, 1, 16000, generator=torch.Generator().manual_seed(SEED + 3)).cuda()
    before = {k: p.detach().clone() for k, p in gen.named_parameters()}
    pr = gen(lr)
    sc, mag = mrstft(pr.squeeze(1), hr.squeeze(1))
    fake = disc(pr)
    real = disc(hr)
    adv = sum(torch.relu(1 - f[-1]).mean() for f in fake)
    feat = sum(torch.nn.functional.l1_loss(fr.detach(), ff) for f_r, f_f in zip(real, fake) for fr, ff in zip(f_r[:-1], f_f[:-1]))
    loss_g = sc + mag + adv + 100 * feat
    opt_g.zero_grad()
    loss_g.backward()
    opt_g.step()
    d_fake = disc(pr.detach())
    d_real = disc(hr)
    loss_d = sum(torch.relu(1 + f[-1]).mean() for f in d_fake) + sum(torch.relu(1 - r[-1]).mean() for r in d_real)
    opt_d.zero_grad()
    loss_d.backward()
    opt_d.step()
    torch.cuda.synchronize()
    assert torch.isfinite(loss_g) and torch.isfinite(loss_d)
    assert all(torch.isfinite(p.grad).all() for p in gen.parameters())
    assert sum(not torch.equal(before[k], p.detach()) for k, p in gen.named_parameters()) == 252
