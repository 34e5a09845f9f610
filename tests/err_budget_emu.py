"""Error budget of FP16 storage choices, measured WITHOUT a GPU (test infrastructure: it uses the oracle and the CPU emulation).

The emulation (tests/cpu_emu.py) runs the product's host logic with exact arithmetic but stores through the real buffer
dtypes, so the only error is the storage rounding.  This script forces additional fp32 workspaces to FP16 and reports the
end-to-end rel-L2 against the oracle: what a candidate storage change would cost before any kernel is written.

    python tests/err_budget_emu.py

Round-1 result (three configs): LSTM gate inputs and attention q/k/v in FP16: no measurable change (5.43e-4 -> 5.42e-4);
DConv pre-norm tensors in FP16: +2.6 %; every pre-norm GEMM output in FP16: +6 %.
The "pre-norm biases + 10..21" line shifts each GroupNorm group of every conv that feeds one by its own constant of size 10 to 21
(tests/util.py `shifted`: the same function, so the reference is the oracle of the unshifted weights).
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from cpu_emu import EmuEngine
from util import SEED, pre_norm_convs, shifted, trained_like_, white_noise, rel_l2
from aero_b200 import Aero, aero_kwargs
from oracle import aero_oracle as O

def run(exp, B, L, C=1, f16_names=(), bias_shift=0.0):
    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs(exp)).eval()
    m.load_state_dict(trained_like_(m.state_dict()))
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    if bias_shift:
        m.load_state_dict(shifted(sd0, pre_norm_convs(m), bias_shift))
    e = EmuEngine(m); e.precision = 2
    orig = e._buf
    def buf(name, *shape, dtype=torch.float32, zero=False):
        if dtype == torch.float32 and any(name.endswith(sfx) for sfx in f16_names):
            dtype = torch.float16
        return orig(name, *shape, dtype=dtype, zero=zero)
    e._buf = buf
    object.__setattr__(m, "_engine_obj", e)
    x = white_noise((B, C, L))
    with torch.no_grad():
        ref = O.aero_forward(sd0, m.geom, x)
    return rel_l2(m(x), ref)

cases = [("aero_4-16_512_256", 1, 7777, 1), ("aero_4-16_512_64", 1, 1600, 1), ("aero_11-44_512_64", 1, 2750, 2)]
variants = {"baseline (as shipped)": (),
            "+ DConv pre-norm u, h32 in f16": (".u", ".h32"),
            "+ all pre-norm GEMM outputs in f16": (".u", ".h32", ".rw", ".ct", ".conv32"),
            "+ LSTM gate inputs in f16": (".gin1", ".gin2"),
            "+ attention qkvd in f16": (".qkvd",),
            "pre-norm biases + 10..21 (as shipped)": ((), 10.0)}
for exp, B, L, C in cases:
    for name, v in variants.items():
        sfx, shift = v if name.startswith("pre-norm") else (v, 0.0)
        t0 = time.time()
        err = run(exp, B, L, C, sfx, shift)
        print(f"{exp:22s} L={L:5d} {name:40s} rel_l2 {err:.3e}  ({time.time()-t0:.0f}s)", flush=True)
