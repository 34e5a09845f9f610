"""HiFi-GAN multi-period discriminator, without a GPU: the functional oracle against the fp64 goldens of the unmodified reference
(tests/golden/mpd_*.npz), module parity with the live reference, the segment layout of aero_b200.mpd, and the constructor checks."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from mpd_util import CASES, case_inputs, mpd_loss, reference_mpd_class
from util import SEED, disc_recipe_state, rel_l2, weights_digest

from aero_b200.mpd import DiscriminatorP, MultiPeriodDiscriminator, period_flops, period_layout, segment_view, superframe_weight
from oracle import mpd_oracle as O


def _golden(golden_dir, name):
    return np.load(os.path.join(golden_dir, name + ".npz"))


def _state(kw):
    torch.manual_seed(SEED)
    m = MultiPeriodDiscriminator(**kw)
    return disc_recipe_state(m.state_dict())


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_golden(golden_dir, name):
    g = _golden(golden_dir, name)
    kw, B, L = CASES[name]
    sd = _state(kw)
    assert weights_digest(sd) == pytest.approx(float(g["digest"]), rel=1e-12)
    sd = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    y, y_hat = (t.double().requires_grad_(True) for t in case_inputs(name))
    outs = O.mpd_forward(sd, kw["periods"], y, y_hat)
    y_d_rs, y_d_gs, fmap_rs, fmap_gs = outs
    for i in range(len(kw["periods"])):
        for side, (logits, fmap) in enumerate(((y_d_rs[i], fmap_rs[i]), (y_d_gs[i], fmap_gs[i]))):
            assert rel_l2(logits.detach(), g[f"logits/{i}/{side}"]) < 1e-6
            for j, f in enumerate(fmap):
                assert tuple(f.shape) == tuple(int(v) for v in g[f"f_shape/{i}/{side}/{j}"])
                got = f.detach().reshape(-1)[torch.from_numpy(g[f"f_idx/{i}/{side}/{j}"].astype(np.int64))]
                assert rel_l2(got, g[f"f_val/{i}/{side}/{j}"]) < 1e-6
    loss = mpd_loss(outs)
    assert float(loss) == pytest.approx(float(g["loss"]), rel=1e-9, abs=1e-12)
    loss.backward()
    assert rel_l2(y.grad, g["dy"]) < 1e-6 and rel_l2(y_hat.grad, g["dy_hat"]) < 1e-6
    for k, p in sd.items():
        got = p.grad.reshape(-1)[torch.from_numpy(g["g_idx/" + k].astype(np.int64))]
        assert rel_l2(got, g["g_val/" + k]) < 1e-6, k


def test_module_matches_live_reference():
    Ref = reference_mpd_class()
    if Ref is None:
        pytest.skip("no reference checkout ($AERO_REFERENCE)")
    for kw in (dict(), dict(hidden=8, periods=[1, 4, 6])):
        torch.manual_seed(SEED)
        ref = Ref(**kw)
        rng_ref = torch.get_rng_state()
        torch.manual_seed(SEED)
        m = MultiPeriodDiscriminator(**kw)
        assert torch.equal(torch.get_rng_state(), rng_ref)
        a, b = ref.state_dict(), m.state_dict()
        assert list(a) == list(b)
        assert all(a[k].shape == b[k].shape and torch.equal(a[k], b[k]) for k in a)
        m.load_state_dict(a, strict=True)
        ref.load_state_dict(b, strict=True)
        assert m._init_args_kwargs == ((), kw) and m.discriminators[0]._init_args_kwargs[1] == dict(hidden=kw.get("hidden", 32))


def test_default_model_size():
    m = MultiPeriodDiscriminator()
    sd = m.state_dict()
    assert len(sd) == 90 and sum(p.numel() for p in m.parameters()) == 41105770
    assert list(sd)[:3] == ["discriminators.0.convs.0.bias", "discriminators.0.convs.0.weight_g", "discriminators.0.convs.0.weight_v"]
    assert list(sd)[-1] == "discriminators.4.conv_post.weight_v"
    assert m._init_args_kwargs == ((), {})


def _emulate_period(sd, prefix, period, channels, x):
    """The CUDA path's data movement restated with torch ops (fp64, CPU), following include/aero_b200.h: the fold, each layer as a
    tap-GEMM over the whole segment sequence (out[j] = sum_d W_d a[j + d], zero past the end; stride-3 layers on super-frames),
    the repack, and the returned views."""
    B, _, T = x.shape
    lay = period_layout(T, period)
    S = B * period
    H, seg, halo = lay[0]
    t = torch.arange(H)[:, None] * period + torch.arange(period)[None]
    t = torch.where(t >= T, 2 * (T - 1) - t, t)
    h = torch.zeros(B, period, seg, 1, dtype=x.dtype)
    h[:, :, halo:halo + H, 0] = x[:, 0][:, t].permute(0, 2, 1)
    fmap, cin = [], 1
    for i, cout in enumerate(channels + [1]):
        key = f"{prefix}convs.{i}" if i < 5 else f"{prefix}conv_post"
        w = torch._weight_norm(sd[key + ".weight_v"], sd[key + ".weight_g"], 0).view(cout, cin, -1)
        seg_in = lay[i][1]
        if i < 4:
            rows, a, w = seg_in // 3, h.reshape(S * seg_in // 3, 3 * cin), superframe_weight(w)
        else:
            rows, a = seg_in, h.reshape(S * seg_in, cin)
        y = F.conv1d(F.pad(a.t()[None], (0, w.shape[2] - 1)), w, sd[key + ".bias"])[0].t()      # [S * rows, cout]
        Ho, seg_o, halo_o = lay[i + 1]
        if i < 5:
            h = torch.zeros(S, seg_o, cout, dtype=x.dtype)
            h[:, halo_o:halo_o + Ho] = F.leaky_relu(y.reshape(S, rows, cout)[:, :Ho], O.SLOPE)
        else:
            h = y
        fmap.append(segment_view(h.reshape(-1), B, period, Ho, seg_o, halo_o, cout))
        cin = cout
    return torch.flatten(fmap[-1], 1, -1), fmap


@pytest.mark.parametrize("name", sorted(CASES))
def test_segment_layout_gives_the_reference_tensors(name):
    kw, B, L = CASES[name]
    sd = {k: v.double() for k, v in _state(kw).items()}
    y, _ = case_inputs(name)
    channels = DiscriminatorP(1, hidden=kw["hidden"]).channels
    for i, p in enumerate(kw["periods"]):
        for T in (L, L - 1, 3 * p + 1):
            x = y[..., :T].double()
            want_l, want_f = O.period_forward(sd, f"discriminators.{i}.", p, x)
            got_l, got_f = _emulate_period(sd, f"discriminators.{i}.", p, channels, x)
            assert got_l.shape == want_l.shape and rel_l2(got_l, want_l) < 1e-12
            for a, b in zip(got_f, want_f):
                assert a.shape == b.shape and rel_l2(a, b) < 1e-12


def test_executed_over_algorithmic_flop():
    """At 8 x 2 s / 16 kHz the tap-GEMMs execute 1.12x the reference's FLOP: the zero sixth super-frame tap of the stride-3 layers
    (1.2x on 42 % of the work), one row per segment that no output owns, and the halos.  The default model's forward is
    35.9 GFLOP per clip (DESIGN.md)."""
    m = MultiPeriodDiscriminator()
    ex = al = 0
    for d in m.discriminators:
        e, a = period_flops(8, 32000, d.period, d.channels)
        assert e / a < 1.2, (d.period, e / a)
        ex, al = ex + e, al + a
    assert ex / al < 1.13, ex / al
    assert al / 8 / 1e9 == pytest.approx(35.9, abs=0.05)


def test_constructor_checks():
    with pytest.raises(NotImplementedError):
        DiscriminatorP(2, use_spectral_norm=True)
    with pytest.raises(NotImplementedError):
        DiscriminatorP(2, kernel_size=3)
    with pytest.raises(NotImplementedError):
        DiscriminatorP(2, stride=2)
    for hidden in (0, 6, 30):
        with pytest.raises(NotImplementedError):
            MultiPeriodDiscriminator(hidden=hidden)
    with pytest.raises(ValueError):
        DiscriminatorP(0)
    m = MultiPeriodDiscriminator(hidden=4, periods=[2])
    for v in (0, 1):
        m.train_precision = v
        assert m.discriminators[0].train_precision == v
    with pytest.raises(NotImplementedError):
        m.train_precision = 3
    assert m.train_precision == 1
    with pytest.raises(ValueError):
        m.train_precision = 2


def test_cpu_input_is_refused():
    m = MultiPeriodDiscriminator(hidden=4, periods=[2])
    x = torch.zeros(1, 1, 64)
    with pytest.raises(RuntimeError, match="CUDA only"):
        m(x, x)


def test_experiment_file_builds_both_adversaries():
    """conf/experiment/aero_4-16_512_64_mpd.yaml: the generator of aero_4-16_512_64, [msd_melgan, mpd], and the `mpd:` block the
    reference's factory passes to MultiPeriodDiscriminator (modelFactory.py:21-23)."""
    from aero_b200.config import aero_kwargs, load_experiment
    exp = load_experiment("aero_4-16_512_64_mpd")
    assert exp["discriminator_models"] == ["msd_melgan", "mpd"]
    assert aero_kwargs("aero_4-16_512_64_mpd") == aero_kwargs("aero_4-16_512_64")
    m = MultiPeriodDiscriminator(**exp["mpd"])
    assert [d.period for d in m.discriminators] == [2, 3, 5, 7, 11] and m.discriminators[0].channels[0] == 32
