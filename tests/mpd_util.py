"""Cases, inputs and cotangents shared by the multi-period discriminator goldens and tests (CPU-only code; no kernels)."""
from util import SEED, white_noise

# name -> (MultiPeriodDiscriminator kwargs, B, L)
CASES = {
    "mpd_default": (dict(hidden=32, periods=[2, 3, 5, 7, 11]), 2, 8192),      # ragged for p = 3, 5, 7, 11
    "mpd_short": (dict(hidden=32, periods=[2, 3, 5, 7, 11]), 2, 1200),        # 1-2 frames in the deepest layers of p = 7, 11
    "mpd_small": (dict(hidden=8, periods=[1, 4, 6]), 2, 3001),                # p = 1, and a non-default hidden
}


def case_inputs(name):
    _, B, L = CASES[name]
    return white_noise((B, 1, L), seed=SEED + 3), 0.5 * white_noise((B, 1, L), seed=SEED + 4)


def cotangent(shape, i, side, j):
    """Seeded cotangent of output j (0-4 feature maps, 5 conv_post, 9 logits) of period i, side 0 (real) / 1 (generated)."""
    return white_noise(tuple(shape), seed=SEED + 2000 + 100 * i + 10 * side + j)


def mpd_loss(outs):
    """sum over every returned tensor of mean(tensor * cotangent): reaches every output of every period on both sides."""
    y_d_rs, y_d_gs, fmap_rs, fmap_gs = outs
    loss = 0.0
    for i in range(len(y_d_rs)):
        for side, (logits, fmap) in enumerate(((y_d_rs[i], fmap_rs[i]), (y_d_gs[i], fmap_gs[i]))):
            loss = loss + (logits * cotangent(logits.shape, i, side, 9).to(logits)).mean()
            for j, f in enumerate(fmap):
                loss = loss + (f * cotangent(f.shape, i, side, j).to(f)).mean()
    return loss


def reference_mpd_class(ref_root=None):
    """MultiPeriodDiscriminator of the unmodified reference package at `ref_root` (default $AERO_REFERENCE, else ./reference);
    None when there is none."""
    import importlib
    import os
    import sys
    from util import ROOT
    root = os.path.abspath(ref_root or os.environ.get("AERO_REFERENCE") or "reference")
    if not os.path.isdir(root):
        return None
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "src" or k.startswith("src.")}
    path_saved = list(sys.path)
    sys.path[:] = [root] + [p for p in sys.path if os.path.abspath(p or ".") != ROOT]
    try:
        mod = importlib.import_module("src.models.discriminators")
    finally:
        sys.path[:] = path_saved
        for k in [k for k in sys.modules if k == "src" or k.startswith("src.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    return mod.MultiPeriodDiscriminator
