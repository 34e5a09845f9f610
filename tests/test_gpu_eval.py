"""-m gpu: test-set scoring.  get_lsd_batch (the fused aero_lsd_varlen_fwd) against the reference LSD formula in fp64 on the
CPU and against get_lsd file by file; its independence from padding, call order and file order; its errors; evaluate_batch
against the reference's per-file loop (model, match_signal, get_lsd) for AERO and SEANet."""
import pytest
import torch

from util import SEED, trained_like_, white_noise
from seanet_util import CASES, seanet_recipe_state

from aero_b200 import Aero, Seanet, aero_kwargs
from aero_b200.enhance import evaluate_batch, match_signal, nonzero_mean
from aero_b200.metrics import get_lsd, get_lsd_batch, lsd_varlen

pytestmark = pytest.mark.gpu


def oracle_lsd(ref, est):
    """reference src/metrics.py:59-70 with the torch>=2 `return_complex` shim, in fp64 on the CPU; [C, L] files are scored
    over the frames of all their channels."""
    win = torch.hann_window(2048, dtype=torch.float64)

    def lg(x):
        return torch.log10(torch.stft(x.cpu().double(), 2048, 512, window=win, return_complex=True).abs().square().clamp(1e-8))
    return float((lg(ref) - lg(est)).square().mean(dim=-2).sqrt().mean())


def cases():
    """(reference, estimate) CPU pairs: noise, a zeroed stretch (the 1e-8 clamp), the shortest lengths reflect padding takes
    and those around a hop, 8 s at 16 kHz, a stereo file, a pure tone on an exact bin."""
    out = [(white_noise((1, 8000), seed=1), 0.7 * white_noise((1, 8000), seed=2))]
    r, e = white_noise((1, 32000), seed=3), 0.7 * white_noise((1, 32000), seed=4)
    e[:, 4000:12000] = 0.0
    out.append((r, e))
    for k, n in enumerate((1025, 1536, 2049)):
        out.append((white_noise((n,), seed=10 + k), white_noise((n,), seed=20 + k)))
    out.append((white_noise((1, 128000), seed=5), white_noise((1, 128000), seed=5) + 0.1 * white_noise((1, 128000), seed=6)))
    out.append((white_noise((2, 20000), seed=7), 0.5 * white_noise((2, 20000), seed=8)))
    t = torch.sin(2 * torch.pi * 64 * torch.arange(40000, dtype=torch.float64) / 2048).float()[None]
    out.append((t, 0.5 * t))
    return out


def test_batch_matches_the_fp64_reference_formula_and_get_lsd():
    pairs = cases()
    got = get_lsd_batch([r.cuda() for r, _ in pairs], [e.cuda() for _, e in pairs])
    assert got.dtype == torch.float32 and got.is_cuda and got.shape == (len(pairs),)
    for i, (r, e) in enumerate(pairs):
        want = oracle_lsd(r, e)
        assert abs(float(got[i]) - want) / want < 1e-4, (i, float(got[i]), want)
        one = float(get_lsd(r.reshape(-1, r.shape[-1]).cuda(), e.reshape(-1, e.shape[-1]).cuda()))
        assert abs(float(got[i]) - one) / one < 1e-5, (i, float(got[i]), one)


def test_samples_past_each_length_are_never_read():
    pairs = cases()
    rows_r = [r.reshape(-1, r.shape[-1]) for r, _ in pairs]
    rows_e = [e.reshape(-1, e.shape[-1]) for _, e in pairs]
    lengths = [x.shape[-1] for rows in rows_r for x in rows]
    row_file = [i for i, rows in enumerate(rows_r) for _ in rows]
    L = max(lengths) + 700

    def padded(rows, fill):
        x = (1e3 * white_noise((len(lengths), L), seed=99)) if fill else torch.zeros(len(lengths), L)
        for j, row in enumerate(x for file_rows in rows for x in file_rows):
            x[j, :row.shape[-1]] = row
        return x.cuda()
    clean = lsd_varlen(padded(rows_r, False), padded(rows_e, False), lengths, row_file, len(pairs))
    noisy = lsd_varlen(padded(rows_r, True), padded(rows_e, True), lengths, row_file, len(pairs))
    assert torch.equal(clean, noisy)
    assert torch.equal(clean, get_lsd_batch([r.cuda() for r, _ in pairs], [e.cuda() for _, e in pairs]))


def test_repeatable_and_independent_of_file_order():
    pairs = cases()
    refs, ests = [r.cuda() for r, _ in pairs], [e.cuda() for _, e in pairs]
    a, b = get_lsd_batch(refs, ests), get_lsd_batch(refs, ests)
    assert torch.equal(a, b)
    perm = torch.randperm(len(pairs), generator=torch.Generator().manual_seed(SEED)).tolist()
    c = get_lsd_batch([refs[i] for i in perm], [ests[i] for i in perm])
    assert torch.equal(c, a[perm])
    d = get_lsd_batch(refs[2:4], ests[2:4])                        # a file's value does not depend on the others in the call
    assert torch.equal(d, a[2:4])


def test_errors():
    x, y = white_noise((1, 4000)).cuda(), white_noise((1, 1024)).cuda()
    with pytest.raises(ValueError, match=r"file 1 \(row 1\): length 1024"):
        get_lsd_batch([x, y], [x, y])
    with pytest.raises(ValueError, match="file 0"):
        get_lsd_batch([x], [x[:, :3000]])
    with pytest.raises(ValueError, match="file 0"):
        get_lsd_batch([white_noise((2, 4000)).cuda()], [white_noise((1, 4000)).cuda()])
    with pytest.raises(RuntimeError, match="CUDA"):
        get_lsd_batch([x, x.cpu()], [x, x.cpu()])
    with pytest.raises(ValueError, match="row 1"):
        lsd_varlen(torch.zeros(2, 4000).cuda(), torch.zeros(2, 4000).cuda(), [4000, 1000], [0, 1], 2)


def _reference_loop(model, lrs, hrs):
    """What reference evaluate.py does to each file: the model at batch 1, match_signal, get_lsd."""
    return [float(get_lsd(h, match_signal(model(x[None])[0], h.shape[-1]))) for x, h in zip(lrs, hrs)]


def _check_evaluate(model, lrs, hrs):
    lsd, mean, count = evaluate_batch(model, lrs, hrs, max_batch=3)
    want = _reference_loop(model, lrs, hrs)
    assert lsd.shape == (len(lrs),) and lsd.is_cuda
    for g, w in zip(lsd.tolist(), want):
        assert abs(g - w) / w < 1e-5, (g, w)
    assert count == len(lrs) and mean == pytest.approx(nonzero_mean(lsd.tolist())[0])


def test_evaluate_batch_aero_matches_the_per_file_loop():
    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs("aero_4-16_512_64")).eval()
    m.load_state_dict(trained_like_(m.state_dict()))
    m = m.cuda()
    m._engine().precision = 0
    lens = [4000, 2600, 7001, 3333, 5120]
    lrs = [white_noise((1, n), seed=40 + i).cuda() for i, n in enumerate(lens)]
    hrs = [white_noise((1, 4 * n + d), seed=50 + i).cuda() for i, (n, d) in enumerate(zip(lens, (-3, 5, 0, -7, 2)))]
    _check_evaluate(m, lrs, hrs)


def test_evaluate_batch_seanet_matches_the_per_file_loop():
    torch.manual_seed(SEED)
    m = Seanet(**CASES["s1"][0])
    m.load_state_dict(seanet_recipe_state(m.state_dict()))
    m = m.cuda().eval()
    m._engine().precision = 0
    lens = [8000, 7001, 4000]
    lrs = [white_noise((1, n), seed=60 + i).cuda() for i, n in enumerate(lens)]
    hrs = [white_noise((1, 4 * n + d), seed=70 + i).cuda() for i, (n, d) in enumerate(zip(lens, (4, -2, 0)))]
    _check_evaluate(m, lrs, hrs)
