"""SEANet on the CPU: the oracle against the stored reference outputs and, where the reference checkout can be imported, against
the live reference; constructor parity; the factory on the authored experiment file; length and ratio checks."""
import os
import warnings

import numpy as np
import pytest
import torch

from util import SEED, import_reference, rel_l2, weights_digest
from seanet_util import CASES, case_input, seanet_recipe_state

from aero_b200 import Seanet, seanet_kwargs
from aero_b200.seanet import sinc_resample_table, superframe_conv_weight, superframe_convt_weight
from oracle import seanet_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _model(name):
    torch.manual_seed(SEED)
    m = Seanet(**CASES[name][0])
    m.load_state_dict(seanet_recipe_state(m.state_dict()))
    return m


def _reference_seanet():
    root = os.path.abspath(os.environ.get("AERO_REFERENCE") or "reference")
    if import_reference(root) is None:
        return None
    import importlib
    import sys
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "src" or k.startswith("src.")}
    path_saved = list(sys.path)
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:] = [root] + [p for p in sys.path if os.path.abspath(p or ".") != repo]
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return importlib.import_module("src.models.seanet").Seanet
    finally:
        sys.path[:] = path_saved
        for k in [k for k in sys.modules if k == "src" or k.startswith("src.")]:
            del sys.modules[k]
        sys.modules.update(saved)


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_golden_fp32(name):
    g = np.load(os.path.join(GOLDEN, f"seanet_{name}.npz"))
    m = _model(name)
    assert weights_digest(m.state_dict()) == pytest.approx(float(g["digest"]), rel=1e-12)
    stages = {}
    with torch.no_grad():
        y = O.seanet_forward(m.state_dict(), m, case_input(name), stages)
    assert tuple(y.shape) == g["y"].shape
    assert rel_l2(y, g["y"]) <= 2e-5
    assert rel_l2(stages["branch"], g["branch"]) <= 2e-5
    assert rel_l2(stages["x0"], g["x0"]) <= 2e-5
    for k in [k for k in g.files if k.startswith("stage_val/")]:
        st = k.split("/", 1)[1]
        got = stages[st].reshape(-1)[torch.from_numpy(g["stage_idx/" + st]).long()]
        assert rel_l2(got, g[k]) <= 2e-5, st


def test_constructor_and_oracle_match_live_reference():
    Ref = _reference_seanet()
    if Ref is None:
        pytest.skip("reference checkout not importable")
    for name in ("s1", "s5", "s6"):
        kw = CASES[name][0]
        torch.manual_seed(SEED)
        ours = Seanet(**kw)
        after_ours = torch.rand(8)
        torch.manual_seed(SEED)
        ref = Ref(**kw)
        after_ref = torch.rand(8)
        a, b = ours.state_dict(), ref.state_dict()
        assert list(a) == list(b) and len(a) == (252 if name == "s1" else len(b))
        assert all(torch.equal(a[k], b[k]) for k in a)
        assert torch.equal(after_ours, after_ref)
        ours.load_state_dict(ref.state_dict(), strict=True)          # reference checkpoints load unchanged
        ref.load_state_dict(seanet_recipe_state(ref.state_dict()))
        ref = ref.double().eval()
        sd = {k: v.double() for k, v in ref.state_dict().items()}
        x = case_input(name).double()
        with torch.no_grad():
            assert rel_l2(O.seanet_forward(sd, ours, x), ref(x)) <= 1e-10


def test_filter_table_matches_torchaudio():
    ta = pytest.importorskip("torchaudio.functional.functional")
    for lr, hr in ((4000, 16000), (8000, 24000), (11025, 44100), (16000, 48000)):
        g = np.gcd(lr, hr)
        for dt in (torch.float32, torch.float64):
            k, w = ta._get_sinc_resample_kernel(lr, hr, int(g), 6, 0.99, "sinc_interp_hann", None, torch.device("cpu"), dt)
            t, w2, orig, new = sinc_resample_table(lr, hr, dt)
            ko, w3 = O.resample_table(lr, hr, dt)
            assert w == w2 == w3 and torch.equal(k.view(new, -1), t) and torch.equal(k, ko)
    x = torch.randn(2, 1, 777, dtype=torch.float64)
    import torchaudio.functional as F_
    assert torch.equal(O.resample(x, 4000, 16000), F_.resample(x, 4000, 16000))


@pytest.mark.parametrize("r", [2, 3, 4, 8])
def test_superframe_mappings(r):
    """The strided conv and the transposed conv as 3-tap convs over super-frames of r frames (fp64, on the host)."""
    F = torch.nn.functional
    g = torch.Generator().manual_seed(r)
    B, C, N, T = 2, 3, 5, 6 * r
    x = torch.randn(B, C, T, generator=g, dtype=torch.float64)
    w = torch.randn(N, C, 2 * r, generator=g, dtype=torch.float64)
    p = r // 2 + r % 2
    ref = F.conv1d(x, w, stride=r, padding=p)
    xs = x.permute(0, 2, 1).reshape(B, T // r, r * C).permute(0, 2, 1)           # super-frames
    got = F.conv1d(xs, superframe_conv_weight(w, r), padding=1)
    assert ref.shape == got.shape and torch.allclose(ref, got, rtol=0, atol=1e-12)
    wt = torch.randn(C, N, 2 * r, generator=g, dtype=torch.float64)
    ref = F.conv_transpose1d(x, wt, stride=r, padding=p, output_padding=r % 2)
    got = F.conv1d(x, superframe_convt_weight(wt, r), padding=1)                  # [B, r*N, T] = [B, T*r, N]
    got = got.permute(0, 2, 1).reshape(B, T * r, N).permute(0, 2, 1)
    assert ref.shape == got.shape and torch.allclose(ref, got, rtol=0, atol=1e-12)


def test_get_model_on_the_experiment_file():
    from aero_b200.config import load_experiment
    from src.models.modelFactory import get_model
    exp = load_experiment("seanet_4-16")
    assert exp["model"] == "seanet"
    m = get_model({"experiment": exp})["generator"]
    assert isinstance(m, Seanet) and len(m.state_dict()) == 252
    assert sum(p.numel() for p in m.parameters()) == 8875938
    kw = seanet_kwargs("seanet_4-16")
    assert (kw["lr_sr"], kw["hr_sr"], kw["ratios"], kw["floor"]) == (4000, 16000, [8, 8, 2, 2], 1e-3)
    from src.models.seanet import Seanet as Shim
    assert Shim is Seanet


def test_valid_length_and_checks():
    m = Seanet(**CASES["s1"][0])
    for L in list(range(1, 3000, 37)) + [39999]:
        assert m.estimate_output_length(L) == 256 * -(-L // 256)
    x, pad = m.pad_to_valid_length(torch.zeros(1, 1, 1000))
    assert x.shape[-1] == 1024 and pad == 24
    with pytest.raises(ValueError):
        m.check_length(160)
    m.check_length(200)
    with pytest.raises(NotImplementedError):
        Seanet(lr_sr=16000, hr_sr=22050)
    with pytest.raises(RuntimeError):
        m.eval()(torch.zeros(1, 1, 4000))                # a CPU tensor: no fallback
