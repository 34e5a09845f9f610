"""The adversarial step without a GPU: the loss-term tables GanTrainer builds (aero_b200.gan), evaluated by a CPU emulation of the
aero_gan_loss_fwd / _bwd contract, against the reference's loss functions on small random maps in both storage layouts; the
discriminator factory on the shipped configs; SEANet's backward order."""
import pytest
import torch
import torch.nn.functional as F

from gan_util import emulate, reference_losses
from util import SEED

from aero_b200 import Seanet, load_experiment
from aero_b200.discriminator import Discriminator
from aero_b200.gan import MelganAdversary, Map, MpdAdversary, _attach_grads, build_discriminators, check_discriminators
from aero_b200.mpd import MultiPeriodDiscriminator, period_layout, segment_view
from aero_b200.trainer import _seanet_backward_order

FLAGS = [(True, True), (True, False), (False, True)]     # (adversarial, features): both, only_adversarial_loss, only_features_loss


def _rand(*shape, gen):
    return torch.randn(*shape, generator=gen)


def _mpd_maps(B, T, period, channels, tensors, gen):
    """Segment storage of one period holding `tensors` (the six reference-layout maps [B', C, H, period]); rows no output owns hold
    noise, as the logits' storage does."""
    maps = []
    for t, (H, seg, halo), c in zip(tensors, period_layout(T, period)[1:], channels + [1]):
        n = t.shape[0]
        st = _rand(n * period * seg, c, gen=gen)
        segment_view(st, n, period, H, seg, halo, c).copy_(t)
        maps.append(Map(st.view(-1), n * period, seg, halo, H, c))
    return maps


def _mpd_case(B, T, periods, hidden, gen):
    """Reference-layout real / generated maps per period (leaves requiring grad) and the engines' storage of the joint and the
    generated-only passes."""
    mpd = MultiPeriodDiscriminator(hidden=hidden, periods=periods)
    real, fake, joint, gen_only = [], [], [], []
    for dp in mpd.discriminators:
        lay = period_layout(T, dp.period)
        r = [_rand(B, c, H, dp.period, gen=gen) for (H, _, _), c in zip(lay[1:], dp.channels + [1])]
        f = [_rand(B, c, H, dp.period, gen=gen) for (H, _, _), c in zip(lay[1:], dp.channels + [1])]
        joint.append(_mpd_maps(B, T, dp.period, dp.channels, [torch.cat([a, b]) for a, b in zip(r, f)], gen))
        gen_only.append(_mpd_maps(B, T, dp.period, dp.channels, f, gen))
        real.append([t.requires_grad_(True) for t in r])
        fake.append([t.requires_grad_(True) for t in f])
    return mpd, real, fake, joint, gen_only


def _check_grad(dx, m, expect_ref_layout, to_storage_view):
    got = to_storage_view(dx)
    assert torch.allclose(got, expect_ref_layout, rtol=1e-5, atol=1e-9)
    mask = torch.ones(m.n_seg, m.seg, m.C, dtype=torch.bool)
    mask[:, m.halo:m.halo + m.H] = False
    assert torch.count_nonzero(dx.view(m.n_seg, m.seg, m.C)[mask]) == 0


@pytest.mark.parametrize("adversarial,features", FLAGS)
@pytest.mark.parametrize("T,periods", [(1003, [2, 3, 5]), (97, [2, 7, 11])])       # ragged lengths; 97: the deepest layers hold 1-2 frames
def test_mpd_terms_reproduce_the_reference_losses(T, periods, adversarial, features):
    (d_loss_fn, g_loss_fn, feat_fn), live = reference_losses()
    print("reference loss functions:", "live reference" if live else "restated")
    gen = torch.Generator().manual_seed(SEED)
    B, lam = 2, 100.0
    mpd, real, fake, joint, gen_only = _mpd_case(B, T, periods, 4, gen)
    adv = MpdAdversary(mpd, None, lam, adversarial, features)
    flat = lambda t: torch.flatten(t, 1, -1)                          # noqa: E731  (y_d_r / y_d_g of DiscriminatorP.forward)

    # discriminator loss on the joint pass: logits only, real half LSGAN-real, generated half LSGAN-fake
    per = adv.d_terms(joint)
    grads = [_attach_grads(p, ms) for p, ms in zip(per, joint)]
    out = emulate([t for p in per for t in p])
    ref = d_loss_fn([flat(r[-1]) for r in real], [flat(f[-1]) for f in fake])
    assert float(out[:, 0].sum()) == pytest.approx(float(ref), rel=1e-6)
    assert float(out[:, 1].abs().sum()) == 0.0
    gr = torch.autograd.grad(ref, [r[-1] for r in real] + [f[-1] for f in fake])
    for k, (ms, g) in enumerate(zip(joint, grads)):
        assert all(x is None for x in g[:-1])                           # no gradient into the feature maps
        m, P = ms[-1], periods[k]
        H, seg, halo = period_layout(T, P)[6]
        view = lambda d, m=m, P=P, H=H, seg=seg, halo=halo: segment_view(d.view(-1, 1), 2 * B, P, H, seg, halo, 1)  # noqa: E731
        _check_grad(g[-1], m, torch.cat([gr[k], gr[len(periods) + k]]), view)

    # generator losses on the generated-only pass against the joint pass's real half
    per = adv.g_terms(gen_only, [[m.half(0) for m in ms] for ms in joint])
    grads = [_attach_grads(p, ms) for p, ms in zip(per, gen_only)]
    out = emulate([t for p in per for t in p])
    loss = 0.0
    if adversarial:
        ref_adv = g_loss_fn([flat(f[-1]) for f in fake])
        assert float(out[:, 0].sum()) == pytest.approx(float(ref_adv), rel=1e-6)
        loss = loss + ref_adv
    else:
        assert float(out[:, 0].abs().sum()) == 0.0
    if features:
        ref_feat = lam * feat_fn(real, fake)
        assert float(out[:, 1].sum()) == pytest.approx(float(ref_feat), rel=1e-6)
        loss = loss + ref_feat
    else:
        assert float(out[:, 1].abs().sum()) == 0.0
    leaves = [t for f in fake for t in f]
    gf = torch.autograd.grad(loss, leaves, allow_unused=True)
    k = 0
    for ms, g, P in zip(gen_only, grads, periods):
        for j, m in enumerate(ms):
            want = gf[k] if gf[k] is not None else torch.zeros_like(leaves[k])
            k += 1
            if g[j] is None:
                assert not features and j < 5 and float(want.abs().sum()) == 0.0
                continue
            H, seg, halo = period_layout(T, P)[j + 1]
            view = lambda d, m=m, P=P, H=H, seg=seg, halo=halo: segment_view(d.view(-1, m.C), B, P, H, seg, halo, m.C)  # noqa: E731
            _check_grad(g[j], m, want, view)


def _melgan_case(B, disc, gen):
    """Reference-layout [B, C, T] maps per scale and layer (random lengths) and their [B', T, C] storage."""
    real, fake, joint, gen_only = [], [], [], []
    for i in range(disc.num_D):
        specs = disc.model[f"disc_{i}"].specs
        r, f, jm, gm = [], [], [], []
        Tl = 61 - 9 * i
        for j, (_, _, cout, k, s, p, g, _) in enumerate(specs):
            Tl = max((Tl + 2 * p - k) // s + 1, 1) if j else Tl
            a, b = _rand(B, cout, Tl, gen=gen), _rand(B, cout, Tl, gen=gen)
            st = torch.cat([a, b]).permute(0, 2, 1).contiguous()
            jm.append(Map(st.view(-1), 2 * B, Tl, 0, Tl, cout))
            gm.append(Map(b.permute(0, 2, 1).contiguous().view(-1), B, Tl, 0, Tl, cout))
            r.append(a.requires_grad_(True))
            f.append(b.requires_grad_(True))
        real.append(r), fake.append(f), joint.append(jm), gen_only.append(gm)
    return real, fake, joint, gen_only


@pytest.mark.parametrize("adversarial,features", FLAGS)
def test_melgan_terms_reproduce_the_reference_losses(adversarial, features):
    """solver.py:475-520 restated (the losses are Solver methods there): hinge on the logits, feature matching with weight
    4 / (n_layers + 1) / num_D on every other layer."""
    gen = torch.Generator().manual_seed(SEED + 1)
    B, lam = 3, 100.0
    torch.manual_seed(SEED)
    disc = Discriminator(num_D=3, ndf=4, n_layers=2, downsampling_factor=2)
    real, fake, joint, gen_only = _melgan_case(B, disc, gen)
    adv = MelganAdversary(disc, None, lam, adversarial, features)
    per = adv.d_terms(joint)
    grads = [_attach_grads(p, ms) for p, ms in zip(per, joint)]
    out = emulate([t for p in per for t in p])
    ref = sum(F.relu(1 + f[-1]).mean() for f in fake) + sum(F.relu(1 - r[-1]).mean() for r in real)
    assert float(out[:, 0].sum()) == pytest.approx(float(ref), rel=1e-6)
    gr = torch.autograd.grad(ref, [r[-1] for r in real] + [f[-1] for f in fake])
    for i, (ms, g) in enumerate(zip(joint, grads)):
        want = torch.cat([gr[i], gr[disc.num_D + i]]).permute(0, 2, 1)
        assert torch.allclose(g[-1].view_as(want), want, rtol=1e-6, atol=1e-9)

    per = adv.g_terms(gen_only, [[m.half(0) for m in ms] for ms in joint])
    grads = [_attach_grads(p, ms) for p, ms in zip(per, gen_only)]
    out = emulate([t for p in per for t in p])
    w = (1.0 / 3) * (4.0 / (2 + 1))
    loss = 0.0
    if adversarial:
        ref_adv = sum(F.relu(1 - f[-1]).mean() for f in fake)
        assert float(out[:, 0].sum()) == pytest.approx(float(ref_adv), rel=1e-6)
        loss = loss + ref_adv
    if features:
        ref_feat = lam * sum(w * F.l1_loss(f[j], r[j].detach()) for r, f in zip(real, fake) for j in range(len(f) - 1))
        assert float(out[:, 1].sum()) == pytest.approx(float(ref_feat), rel=1e-6)
        loss = loss + ref_feat
    leaves = [t for f in fake for t in f]
    gf = torch.autograd.grad(loss, leaves, allow_unused=True)
    k = 0
    for ms, g in zip(gen_only, grads):
        for j, m in enumerate(ms):
            want = gf[k]
            k += 1
            if g[j] is None:
                assert want is None or float(want.abs().sum()) == 0.0
                continue
            assert torch.allclose(g[j].view(B, m.H, m.C), want.permute(0, 2, 1), rtol=1e-5, atol=1e-9)


def test_build_discriminators_on_the_shipped_configs():
    e = load_experiment("aero_4-16_512_64_mpd")
    torch.manual_seed(SEED)
    d = build_discriminators(e)
    assert list(d) == ["msd_melgan", "mpd"]
    assert d["msd_melgan"]._init_args_kwargs[1] == dict(num_D=3, ndf=16, n_layers=4, downsampling_factor=4)
    assert d["mpd"]._init_args_kwargs[1] == {"hidden": 32, "periods": [2, 3, 5, 7, 11]}
    torch.manual_seed(SEED)                                   # the reference's construction order: MelGAN first, then the MPD
    m, p = Discriminator(**e["melgan_discriminator"]), MultiPeriodDiscriminator(**e["mpd"])
    for a, b in ((d["msd_melgan"], m), (d["mpd"], p)):
        sa, sb = a.state_dict(), b.state_dict()
        assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)
    s = build_discriminators(load_experiment("seanet_4-16"))
    assert list(s) == ["msd_melgan"] and isinstance(s["msd_melgan"], Discriminator)
    assert build_discriminators(load_experiment("seanet_4-16", adversarial=False)) == {}
    for bad in ("msd_hifi", "hifi"):
        with pytest.raises(NotImplementedError):
            build_discriminators(load_experiment("aero_4-16_512_64_mpd", discriminator_models=["msd_melgan", bad]))
        with pytest.raises(NotImplementedError):
            check_discriminators({bad: d["mpd"]})
    with pytest.raises(TypeError):
        check_discriminators({"mpd": d["msd_melgan"]})


def test_seanet_backward_order():
    """Decoder modules from the output convolution back to decoder.0, then the encoder from the latent projection back to encoder.0;
    each top-level module's parameters contiguous, in named_parameters order."""
    torch.manual_seed(SEED)
    m = Seanet(ngf=8, ratios=[4, 2], n_residual_layers=2, latent_space_size=16, lr_sr=4000, hr_sr=16000)
    order = _seanet_backward_order(m)
    names = [n for n, _ in m.named_parameters()]
    assert sorted(order) == sorted(names)
    tags = []
    for n in order:
        t = ".".join(n.split(".")[:2])
        if not tags or tags[-1] != t:
            tags.append(t)
    n = len(m.ratios)
    assert tags == [f"decoder.{j}" for j in range(n + 1, -1, -1)] + [f"encoder.{i}" for i in range(n + 1, -1, -1)]
    for t in tags:
        assert [x for x in order if x.startswith(t + ".")] == [x for x in names if x.startswith(t + ".")]
