"""-m gpu: the adversarial step of GanTrainer with a discriminator mapping (aero_b200.gan): the loss kernels against fp64, one step
against the plain autograd route, which kernels each pass launches, and the two-rank NCCL step."""
import os

import pytest
import torch

from gan_util import owned
from util import SEED, rel_l2, trained_like_, white_noise

from aero_b200 import Aero, Seanet, aero_kwargs, cabi
from aero_b200 import gan as G
from aero_b200.discriminator import Discriminator, _DiscEngine
from aero_b200.losses import MultiResolutionSTFTLoss
from aero_b200.mpd import MultiPeriodDiscriminator, period_layout
from aero_b200.trainer import GanTrainer

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ loss kernels against fp64
def _maps(gen):
    """MPD segment maps (hidden 32, periods 2 and 11 on 97 and 4000 samples: the deepest layers hold 1-2 frames) and MelGAN
    [B, T, C] maps, each with a same-geometry reference map; storage filled with noise everywhere."""
    out = []
    for T, P in ((97, 11), (97, 2), (4000, 2), (4000, 11)):
        for (H, seg, halo), c in zip(period_layout(T, P)[1:], [32, 128, 512, 1024, 1024, 1]):
            n = 2 * P
            out.append([G.Map(torch.randn(n * seg * c, generator=gen).cuda(), n, seg, halo, H, c) for _ in range(2)])
    for T, c in ((32014, 16), (501, 1024), (7, 1)):
        out.append([G.Map(torch.randn(2 * T * c, generator=gen).cuda(), 2, T, 0, T, c) for _ in range(2)])
    return out


def _expect(t, dtype):
    """Value (adv, l1) and gradient of the owned rows of a term, element-wise in `dtype`, summed in fp64."""
    x = owned(t.x).to(dtype)
    v, d = torch.zeros((), dtype=torch.float64, device=x.device), torch.zeros_like(x)
    a = torch.zeros_like(v)
    if t.adv != cabi.GAN_NONE:
        k = t.adv
        if k in (cabi.GAN_LSGAN_REAL, cabi.GAN_LSGAN_GEN):
            a, d = ((1 - x) ** 2).double().sum(), -2 * (1 - x)
        elif k == cabi.GAN_LSGAN_FAKE:
            a, d = (x * x).double().sum(), 2 * x
        elif k in (cabi.GAN_HINGE_REAL, cabi.GAN_HINGE_GEN):
            a, d = torch.relu(1 - x).double().sum(), -((1 - x) > 0).to(dtype)
        else:
            a, d = torch.relu(1 + x).double().sum(), ((1 + x) > 0).to(dtype)
        a, d = t.adv_scale * a, t.adv_scale * d.double()
    if t.ref is not None:
        diff = x - owned(t.ref).to(dtype)
        v = t.l1_scale * diff.abs().double().sum()
        d = d.double() + t.l1_scale * torch.sign(diff).double()
    return a, v, d


def test_loss_kernels_match_fp64():
    """Every adversarial kind, L1 alone and combined with an adversarial component (the MPD logits), in both layouts.  Sums: within
    1e-12 of the same fp32 element values summed in fp64 (the contract), and within 1e-7 of fp64 throughout.  Gradients within fp32
    rounding of fp64.  Every unowned row of the NaN-filled gradient comes back exactly 0; two runs bit-identical."""
    gen = torch.Generator().manual_seed(SEED)
    maps = _maps(gen)
    kinds = [cabi.GAN_LSGAN_REAL, cabi.GAN_LSGAN_FAKE, cabi.GAN_LSGAN_GEN, cabi.GAN_HINGE_REAL, cabi.GAN_HINGE_FAKE, cabi.GAN_HINGE_GEN]
    terms = []
    for i, (x, r) in enumerate(maps):
        kind = kinds[i % len(kinds)] if (i % 3) else cabi.GAN_NONE
        with_l1 = i % 2 == 0 or kind == cabi.GAN_NONE
        terms.append(G.Term(x, kind, 1.0 / x.count if kind else 0.0, r if with_l1 else None, 3.7 / x.count if with_l1 else 0.0,
                            dx=torch.full_like(x.t, float("nan"))))
    outs, grads = [], []
    for _ in range(2):
        for t in terms:
            t.dx.fill_(float("nan"))
        outs.append(G.gan_loss_fwd(terms).cpu())
        G.gan_loss_bwd(terms)
        torch.cuda.synchronize()
        grads.append([t.dx.clone() for t in terms])
    assert torch.equal(outs[0], outs[1]) and all(torch.equal(a, b) for a, b in zip(*grads))
    worst_v, worst_64, worst_g = 0.0, 0.0, 0.0
    for k, t in enumerate(terms):
        a32, v32, _ = _expect(t, torch.float32)
        a, v, d = _expect(t, torch.float64)
        for got, w32, w64 in ((outs[0][k, 0], a32, a), (outs[0][k, 1], v32, v)):
            worst_v = max(worst_v, abs(float(got) - float(w32)) / max(abs(float(w32)), 1e-30))
            worst_64 = max(worst_64, abs(float(got) - float(w64)) / max(abs(float(w64)), 1e-30))
        m = t.x
        g = t.dx.view(m.n_seg, m.seg, m.C)
        mask = torch.ones(m.n_seg, m.seg, dtype=torch.bool, device=g.device)
        mask[:, m.halo:m.halo + m.H] = False
        assert not torch.isnan(g).any()
        assert torch.count_nonzero(g[mask]) == 0, (k, m.n_seg, m.seg, m.halo, m.H)
        err = (g[:, m.halo:m.halo + m.H].double() - d).abs().max() / d.abs().max().clamp_min(1e-30)
        worst_g = max(worst_g, float(err))
    print(f"loss kernels: sums {worst_v:.2e} from fp32 elements summed in fp64, {worst_64:.2e} from fp64; gradients {worst_g:.2e} "
          f"from fp64 ({len(terms)} terms)")
    assert worst_v < 1e-12 and worst_64 < 1e-7 and worst_g < 2e-7


# ------------------------------------------------------------------------------------------------ one step against autograd
def _gen(kind):
    torch.manual_seed(SEED)
    if kind == "aero":
        m = Aero(**aero_kwargs("aero_4-16_512_256"))
        m.load_state_dict(trained_like_(m.state_dict()))
        return m, 4000
    return Seanet(ngf=16, ratios=[4, 4, 2], n_residual_layers=2, latent_space_size=64, lr_sr=4000, hr_sr=16000), 4000


def _discs(names):
    torch.manual_seed(SEED + 1)
    made = {"msd_melgan": lambda: Discriminator(3, 16, 4, 4), "mpd": lambda: MultiPeriodDiscriminator(hidden=16)}
    return {n: made[n]() for n in names}


def _both_routes(kind, names, precision, B=2, **flags):
    (gen, L), (gen_b, _) = _gen(kind), _gen(kind)            # two identical copies (weight-normalised modules do not deepcopy)
    discs, discs_b = _discs(names), _discs(names)
    for m in [gen, gen_b, *discs.values(), *discs_b.values()]:
        m.cuda()
        m.train_precision = precision
    lr_b = white_noise((B, 1, L), seed=21).cuda()
    hr = white_noise((B, 1, 4 * L), seed=22).cuda() * 0.1
    mrstft = MultiResolutionSTFTLoss()
    tr = GanTrainer(gen, discs, lr=3e-4, **flags)
    got = tr.step(lr_b, hr, mrstft)
    # the autograd route: generator loss backward, the discriminators' gradients it leaves dropped, discriminator loss backward
    gen_b.train()
    pr = gen_b(lr_b)
    want = G.autograd_losses(pr, hr, discs_b, mrstft, **flags)
    sum(want["generator"].values()).backward()
    for d in discs_b.values():
        d.zero_grad(set_to_none=True)
    sum(want["discriminator"].values()).backward()
    torch.cuda.synchronize()
    rows, num, den = [], 0.0, 0.0
    for net_a, net_b in [(gen, gen_b)] + [(discs[n], discs_b[n]) for n in names]:
        pairs = [(n, pa.grad.double(), pb.grad.double()) for (n, pa), (_, pb) in zip(net_a.named_parameters(), net_b.named_parameters())]
        rows += grad_rows(pairs)
        num += sum(float((a - b).pow(2).sum()) for _, a, b in pairs)
        den += sum(float(b.pow(2).sum()) for _, _, b in pairs)
    loss_err = {f"{side}/{k}": abs(float(got[side][k]) - float(v)) / max(abs(float(v)), 1e-30)
                for side in ("generator", "discriminator") for k, v in want[side].items()}
    assert {s: list(got[s]) for s in got} == {s: list(want[s]) for s in want}
    return loss_err, sorted(rows, reverse=True), (num / den) ** 0.5


def grad_rows(pairs):
    """(relative L2 error, name) per parameter of one network, the norm floored at 1e-4 x the network's largest per-parameter RMS
    gradient x sqrt(numel) (as tests/test_gpu_mpd.py normalises): a bias ahead of a BatchNorm has an exactly-zero gradient of
    which both routes compute rounding noise, and the hinge / LSGAN gradients of the real and generated halves cancel on the
    discriminators' weight_g, so those entries are compared at the scale of the network's gradients."""
    gmax = max(float(b.pow(2).mean().sqrt()) for _, _, b in pairs)
    return [(float((a - b).norm()) / max(float(b.norm()), 1e-4 * gmax * b.numel() ** 0.5), n) for n, a, b in pairs]


@pytest.mark.parametrize("kind,names", [("aero", ["msd_melgan", "mpd"]), ("seanet", ["msd_melgan", "mpd"]), ("aero", ["mpd"])])
def test_step_matches_the_autograd_route(kind, names):
    """train_precision 0, same seeds and inputs: every loss within 1e-5 and all gradients together within 1e-5 rel-L2.  Per parameter
    (grad_rows) within 2e-2: the worst are the MelGAN logits layer's weight_g, where the real and generated halves' hinge gradients
    cancel on these noise inputs (measured up to 1.3e-2 on an H100 80GB HBM3), and biases ahead of a BatchNorm (2e-3), whose exact
    gradient is zero; every other parameter sits near 1e-4 or below."""
    loss_err, rows, total = _both_routes(kind, names, 0)
    print(f"{kind} + {names}: losses {max(loss_err.values()):.2e}, all gradients {total:.2e}, worst", [(f"{a:.1e}", b) for a, b in rows[:3]])
    assert max(loss_err.values()) < 1e-5, loss_err
    assert rows[0][0] < 2e-2 and total < 1e-5, rows[:3]


@pytest.mark.parametrize("flags", [dict(only_features_loss=True), dict(only_adversarial_loss=True, features_loss_lambda=10.0)])
def test_step_flags_match_the_autograd_route(flags):
    loss_err, rows, total = _both_routes("seanet", ["mpd", "msd_melgan"], 0, **flags)
    print(f"{flags}: losses {max(loss_err.values()):.2e}, all gradients {total:.2e}, worst", [(f"{a:.1e}", b) for a, b in rows[:3]])
    assert max(loss_err.values()) < 1e-5 and rows[0][0] < 2e-2 and total < 1e-5


def test_step_in_tf32_mode_against_the_autograd_route():
    """train_precision 1.  Both routes run the same kernels, but the loss gradients reaching the discriminators differ in the last fp32
    bit (this route's loss kernels against torch's ops), and rounding the operands to TF32 turns some of those one-ulp differences into
    TF32-ulp (2^-11) ones: the losses meet the exact mode's bar, all gradients together stay within 1e-4 (measured 2.6e-5 on an
    H100 80GB HBM3, where exact mode gives 1e-7)."""
    loss_err, rows, total = _both_routes("aero", ["msd_melgan", "mpd"], 1)
    print(f"TF32: losses {max(loss_err.values()):.2e}, all gradients {total:.2e}, worst", [(f"{a:.1e}", b) for a, b in rows[:3]])
    assert max(loss_err.values()) < 1e-5 and total < 1e-4


# ------------------------------------------------------------------------------------------------ what each pass launches
class _RecordingLib:
    """Forwards to the kernel library and logs (phase, symbol, arguments) of every call."""

    def __init__(self, lib):
        self._lib = lib
        self.log, self.phase = [], None

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("aero_"):
            return fn

        def call(*args):
            self.log.append((self.phase, name, args))
            return fn(*args)
        return call


def test_each_pass_launches_only_what_its_optimiser_uses(monkeypatch):
    rec = _RecordingLib(cabi.load())
    monkeypatch.setattr(cabi, "load", lambda *a, **k: rec)
    batches = []
    fwd = _DiscEngine.forward
    monkeypatch.setattr(_DiscEngine, "forward", lambda self, xp, need: (batches.append((rec.phase, xp.shape[0])), fwd(self, xp, need))[1])
    for meth in ("discriminator_pass", "generator_pass"):
        orig = getattr(G._Adversary, meth)

        def wrapped(self, *a, orig=orig, meth=meth):
            rec.phase = (self.name, meth)
            try:
                return orig(self, *a)
            finally:
                rec.phase = None
        monkeypatch.setattr(G._Adversary, meth, wrapped)
    gen, L = _gen("aero")
    discs = {k: v.cuda() for k, v in _discs(["msd_melgan", "mpd"]).items()}
    B = 2
    tr = GanTrainer(gen.cuda(), discs)
    tr.step(white_noise((B, 1, L), seed=21).cuda(), white_noise((B, 1, 4 * L), seed=22).cuda() * 0.1, MultiResolutionSTFTLoss())
    torch.cuda.synchronize()
    n_periods = len(discs["mpd"].discriminators)
    wgrad = {"aero_tapgemm_wgrad", "aero_gconv1d_wgrad", "aero_weight_norm_bwd"}
    gen_calls = [n for ph, n, _ in rec.log if ph and ph[1] == "generator_pass"]
    disc_calls = [n for ph, n, _ in rec.log if ph and ph[1] == "discriminator_pass"]
    assert gen_calls and disc_calls
    assert not wgrad & set(gen_calls), wgrad & set(gen_calls)
    assert "aero_mpd_fold_bwd" not in disc_calls and "aero_mpd_fold_bwd" in gen_calls
    assert {"aero_tapgemm_wgrad", "aero_gconv1d_wgrad", "aero_weight_norm_bwd"} <= set(disc_calls)
    # one forward over the real clips per discriminator: the joint pass (batch 2B); the generator pass sees the B generated clips
    folds = [(ph, a[2]) for ph, n, a in rec.log if n == "aero_mpd_fold_fwd"]
    assert sorted(folds) == sorted([(("mpd", "discriminator_pass"), 2 * B)] * n_periods + [(("mpd", "generator_pass"), B)] * n_periods)
    num_d = discs["msd_melgan"].num_D
    assert sorted(batches) == sorted([(("msd_melgan", "discriminator_pass"), 2 * B)] * num_d + [(("msd_melgan", "generator_pass"), B)] * num_d)


# ------------------------------------------------------------------------------------------------ two ranks over NCCL
def _rank(rank, world, port, q):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    gen, L = _gen("seanet")
    discs = _discs(["msd_melgan", "mpd"])
    gen1, discs1 = _gen("seanet")[0].cuda(), {k: v.cuda() for k, v in _discs(["msd_melgan", "mpd"]).items()}
    lr_b = white_noise((2, 1, L), seed=30 + rank).cuda()
    hr = white_noise((2, 1, 4 * L), seed=40 + rank).cuda() * 0.1
    single = GanTrainer(gen1, discs1)                                 # before init_process_group: one rank's own gradients
    single.step(lr_b, hr, MultiResolutionSTFTLoss())
    own = (single.flat.clone(), single.d_flat.clone())
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        tr = GanTrainer(gen.cuda(), {k: v.cuda() for k, v in discs.items()})
        tr.step(lr_b, hr, MultiResolutionSTFTLoss())
        mean = []
        for t in own:
            dist.all_reduce(t)
            mean.append(t / world)
        params = torch.cat([p.detach().reshape(-1) for m in [gen, *discs.values()] for p in m.parameters()])
        gathered = [torch.empty_like(params) for _ in range(world)]
        dist.all_gather(gathered, params)
        torch.cuda.synchronize()
        q.put((rank, bool(all(torch.equal(gathered[0], g) for g in gathered)),
               rel_l2(tr.flat.cpu() / world, mean[0].cpu()), rel_l2(tr.d_flat.cpu() / world, mean[1].cpu())))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_rank_nccl_step():
    """After one step both ranks hold identical parameters, and the flat buffers hold the mean of the single-rank gradients."""
    import socket
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=120)
    print("two ranks:", res)
    for _, same, eg, ed in res:
        assert same and eg < 1e-6 and ed < 1e-6
