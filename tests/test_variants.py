"""The AERO variants switched by `act_func` and `spec_upsample` (reference aero.py:306-307), and the resampler the
`spec_upsample=False` route feeds them with, checked on the CPU: constructor parity with the live reference, both oracle
forms and the engine's host logic (through the CPU emulation of the kernel contracts) against the golden vectors of the
unmodified reference (tests/golden/vf_*.npz), and the resampler's host filter table and output lengths against torchaudio."""
import glob
import json
import os

import numpy as np
import pytest
import torch

from cpu_emu import EmuEngine
from util import SEED, import_reference, rel_l2, trained_like_, weights_digest, white_noise

from aero_b200 import Aero, aero_kwargs, load_experiment
from aero_b200 import cabi
from aero_b200.engine import dconv_norm_act_op
from aero_b200.resampler import resampled_length
from aero_b200.seanet import sinc_resample_table
from oracle import aero_variants_oracle as O

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "vf_*.npz")))
# orig, new: the ratios the shipped experiments use (4->16, 8->24, 12->48, 11.025->44.1 kHz) and a 2:3 one
RATIOS = [(4000, 16000), (8000, 24000), (12000, 48000), (11025, 44100), (16000, 24000), (16000, 4000), (44100, 16000)]


def golden_kwargs(g):
    return dict(aero_kwargs(str(g["exp"])), **json.loads(str(g["overrides"])))


def build_case(case):
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    torch.manual_seed(SEED)
    model = Aero(**golden_kwargs(g)).eval()
    model.load_state_dict(trained_like_(model.state_dict()))
    assert weights_digest(model.state_dict()) == pytest.approx(float(g["digest"]), rel=1e-12)
    return g, model, torch.from_numpy(g["mix"])


def check_against_golden(g, out, zc, zlr, tol):
    assert out.shape == g["out"].shape
    assert rel_l2(out, g["out"]) < tol
    zc_r = torch.view_as_real(zc.contiguous()).reshape(-1)[torch.from_numpy(g["spec_idx"].astype(np.int64))]
    assert rel_l2(zc_r, g["spec_val"]) < tol
    zl_r = torch.view_as_real(zlr.contiguous()).reshape(-1)[torch.from_numpy(g["lrspec_idx"].astype(np.int64))]
    assert rel_l2(zl_r, g["lrspec_val"]) < tol


# ------------------------------------------------------------------ constructor
@pytest.mark.parametrize("overrides", [{"act_func": "relu"}, {"act_func": "gelu"}, {"act_func": "tanh"}, {"spec_upsample": False},
                                       {"act_func": "relu", "spec_upsample": False}])
def test_constructor_matches_live_reference(overrides):
    ref = import_reference()
    if ref is None:
        pytest.skip("no reference checkout ($AERO_REFERENCE)")
    kw = dict(aero_kwargs("aero_4-16_512_64"), **overrides)
    torch.manual_seed(SEED)
    r = ref["aero"].Aero(**kw)
    rng_ref = torch.get_rng_state()
    torch.manual_seed(SEED)
    m = Aero(**kw)
    assert torch.equal(torch.get_rng_state(), rng_ref)
    a, b = r.state_dict(), m.state_dict()
    assert list(a) == list(b)
    assert all(torch.equal(a[k], b[k]) for k in a)
    assert (m.scale, m.hop_length, m.win_length) == (r.scale, r.hop_length, r.win_length)


def test_activation_mapping_and_snake_parameters():
    kw = aero_kwargs("aero_4-16_512_64")
    torch.manual_seed(SEED)
    snake = Aero(**kw)
    for act, op in (("snake", cabi.NA_SNAKE), ("gelu", cabi.NA_GELU), ("relu", cabi.NA_RELU), ("anything", cabi.NA_RELU)):
        assert dconv_norm_act_op(act) == op
        torch.manual_seed(SEED)
        m = Aero(**dict(kw, act_func=act))
        keys = set(m.state_dict())
        if act == "snake":
            assert any(k.endswith(".act.a") for k in keys)
        else:
            # reference default model: 8 Snake tensors (4 encoder layers x depth 2) and 184 parameters fewer
            assert not any(".act." in k for k in keys) and len(keys) == len(snake.state_dict()) - 8
            assert sum(p.numel() for p in snake.parameters()) - sum(p.numel() for p in m.parameters()) == 184
            assert isinstance(m.encoder[0].dconv.layers[0]["act"], torch.nn.GELU if act == "gelu" else torch.nn.ReLU)


def test_sinc_geometry_is_scale_one():
    m = Aero(**aero_kwargs("aero_4-16_512_64_sinc"))
    g = m.geom
    assert m.scale == 1 and (g.hop_in, g.win_in, g.hop_out, g.win_out) == (64, 512, 64, 512)
    assert (m.hop_length, m.win_length) == (64, 512)
    for L in (1, 63, 64, 8000, 8001):
        assert g.frames(L) == g.frames(L, scale=True) == 1 + (L + (-L) % 64) // 64


@pytest.mark.parametrize("overrides", [{"cac": False}, {"rewrite": False}, {"dconv_mode": 3}, {"context": 2},
                                       {"context_enc": 1}, {"nfft": 500}])
def test_other_options_still_refused(overrides):
    kw = dict(aero_kwargs("aero_4-16_512_64"), **overrides)
    with pytest.raises(NotImplementedError):
        Aero(**kw)


def test_experiment_files():
    e = load_experiment("aero_4-16_512_64_sinc")
    assert e["upsample"] is True and e["aero"]["spec_upsample"] is False and e["aero"]["act_func"] == "snake"
    e = load_experiment("aero_4-16_512_64_relu")
    assert e["upsample"] is False and e["aero"]["spec_upsample"] is True and e["aero"]["act_func"] == "relu"
    base = aero_kwargs("aero_4-16_512_64")
    assert dict(aero_kwargs("aero_4-16_512_64_sinc"), spec_upsample=True) == base
    assert dict(aero_kwargs("aero_4-16_512_64_relu"), act_func="snake") == base


# ------------------------------------------------------------------ oracle and engine host logic
@pytest.mark.parametrize("case", CASES)
def test_oracle_library_form_matches_reference_golden(case):
    g, model, mix = build_case(case)
    snake = O.O.snake
    with torch.no_grad():
        out, zc, zlr = O.aero_forward(model.state_dict(), model.geom, mix, True, True)
    check_against_golden(g, out, zc, zlr, 2e-5)
    assert O.O.snake is snake                 # the Snake of the restated network is back in place


@pytest.mark.parametrize("case", CASES)
def test_oracle_explicit_form_matches_reference_golden(case):
    g, model, mix = build_case(case)
    with torch.no_grad():
        out, zc, zlr = O.aero_forward(model.state_dict(), model.geom, mix, True, True, explicit=True)
    check_against_golden(g, out, zc, zlr, 1e-4)


class _ReluEmuEngine(EmuEngine):
    """The emulation of norm_act with the DConv ReLU added (the emulated contract in tests/cpu_emu.py predates the op)."""

    def _norm_act(self, x, stats, gamma, beta, y, *, op, **kw):
        super()._norm_act(x, stats, gamma, beta, y, op=cabi.NA_NONE if op == cabi.NA_RELU else op, **kw)
        if op == cabi.NA_RELU:
            y.clamp_(min=0)
            self.calls[-1] = ("norm_act", op)
        return y


@pytest.mark.parametrize("case", CASES)
def test_engine_sequence_matches_reference_golden(case):
    """The product's host logic (weight packing without Snake parameters, the DConv op, the scale-1 geometry) on the
    emulated kernel contracts."""
    g, model, mix = build_case(case)
    object.__setattr__(model, "_engine_obj", _ReluEmuEngine(model))
    out, zc, zl = model(mix, return_spec=True, return_lr_spec=True)
    check_against_golden(g, out, zc, zl, 2e-5)
    ops = {c[1] for c in model._engine_obj.calls if c[0] == "norm_act"}
    assert dconv_norm_act_op(model.act_func) in ops
    assert (cabi.NA_SNAKE in ops) == (model.act_func == "snake")


# ------------------------------------------------------------------ resampler (host side)
@pytest.mark.parametrize("orig,new", RATIOS)
def test_resample_table_and_lengths_match_torchaudio(orig, new):
    taf = pytest.importorskip("torchaudio.functional.functional")
    import math
    gcd = math.gcd(orig, new)
    kern, width = taf._get_sinc_resample_kernel(orig, new, gcd, 6, 0.99, "sinc_interp_hann", None, torch.device("cpu"), torch.float32)
    table, w, o, up = sinc_resample_table(orig, new, torch.float32)
    assert (w, o, up) == (width, orig // gcd, new // gcd)
    assert torch.equal(table, kern.view(up, -1))
    for L in (1, 2, 3, 7, 1001, orig // gcd * 5 + 1, 8000, 44101):
        assert resampled_length(L, orig, new) == taf.resample(torch.zeros(1, L), orig, new).shape[-1], L


def test_resample_refuses_bad_rates():
    from aero_b200 import resample
    x = torch.zeros(1, 10)
    for o, n in ((0, 16000), (4000, -1), (4000.5, 16000)):
        with pytest.raises(ValueError):
            resample(x, o, n)
    with pytest.raises(RuntimeError):
        resample(x, 4000, 16000)                # CPU tensor: no fallback
