"""SEANet test helpers shared by the golden generator, the CPU and GPU tests and bench_seanet.py (CPU-only code; no kernels)."""
import torch

from util import SEED

# case name -> (constructor kwargs, input shape [B, C, L], whether the model runs it)
_SHIPPED = dict(latent_space_size=128, ngf=32, n_residual_layers=3, resample=1, normalize=True, floor=1e-3,
                ratios=[8, 8, 2, 2], lr_sr=4000, hr_sr=16000)
CASES = {
    "s1": (dict(_SHIPPED), (2, 1, 8000)),
    "s2": (dict(_SHIPPED), (1, 1, 7001)),
    "s3": (dict(_SHIPPED, upsample=False), (1, 1, 12345)),
    "s4": (dict(_SHIPPED, lr_sr=8000, hr_sr=24000), (1, 1, 4000)),
    "s5": (dict(_SHIPPED, in_channels=2, out_channels=2, lr_sr=11025, hr_sr=44100), (1, 2, 5513)),
    "s6": (dict(_SHIPPED, ngf=16, ratios=[4, 4, 2], n_residual_layers=2, latent_space_size=64), (2, 1, 3000)),
}


def seanet_recipe_state(state, seed=SEED):
    """Deterministic weights for SEANet (the reference and aero_b200 share the 252 state_dict keys): weight_g moved off ||v||
    by up to +-30 %, biases N(0, 0.05^2), weight_v left at its seeded init.  Pure function of (key order, shapes, seed)."""
    g = torch.Generator().manual_seed(seed + 11)
    out = {}
    for k, v in state.items():
        r = torch.randn(v.shape, generator=g)
        if k.endswith("weight_g"):
            out[k] = v * (1.0 + 0.3 * torch.tanh(r))
        elif k.endswith("bias"):
            out[k] = 0.05 * r
        else:
            out[k] = v.clone()
    return {k: out[k].to(state[k].dtype) for k in state}


def case_input(name):
    shape = CASES[name][1]
    return torch.randn(*shape, generator=torch.Generator().manual_seed(SEED + 100 + int(name[1:])))


def train_case():
    """t1 (shipped config, training): B=2 x 1 s of low-rate noise and the cotangent R of loss = sum(out * R)."""
    g = torch.Generator().manual_seed(SEED + 200)
    return torch.randn(2, 1, 4000, generator=g), torch.randn(2, 1, 16000, generator=g)
