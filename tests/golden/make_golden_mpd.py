"""Golden vectors for the HiFi-GAN multi-period discriminator from the UNMODIFIED reference (`src/models/discriminators.py:89-147`)
in fp64:

    AERO_REFERENCE=/path/to/aero python tests/golden/make_golden_mpd.py

Weights are a recipe (tests/util.disc_recipe_state on a model seeded with SEED: 41 M parameters would be 160 MB) plus a digest;
inputs and cotangents are seeded (tests/mpd_util).  Stored per case (tests/mpd_util.CASES): 512 samples of every feature map, the
logits, the gradients of both inputs, and 256 samples + the rms of every parameter gradient of  loss = sum over every returned
tensor of mean(tensor * R)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from util import SEED, disc_recipe_state, sample_indices, weights_digest  # noqa: E402
from mpd_util import CASES, case_inputs, mpd_loss, reference_mpd_class  # noqa: E402


def main():
    torch.set_num_threads(os.cpu_count())
    Ref = reference_mpd_class()
    for name, (kw, B, L) in CASES.items():
        torch.manual_seed(SEED)
        ref = Ref(**kw)
        ref.load_state_dict(disc_recipe_state(ref.state_dict()))
        digest = weights_digest(ref.state_dict())
        ref = ref.double()
        y, y_hat = (t.double().requires_grad_(True) for t in case_inputs(name))
        outs = ref(y, y_hat)
        loss = mpd_loss(outs)
        loss.backward()
        blob = {"digest": np.float64(digest), "B": B, "L": L, "hidden": kw["hidden"], "periods": np.array(kw["periods"]),
                "torch": torch.__version__, "loss": np.float64(float(loss)), "dy": y.grad.float().numpy(),
                "dy_hat": y_hat.grad.float().numpy()}
        y_d_rs, y_d_gs, fmap_rs, fmap_gs = outs
        for i in range(len(y_d_rs)):
            for side, (logits, fmap) in enumerate(((y_d_rs[i], fmap_rs[i]), (y_d_gs[i], fmap_gs[i]))):
                blob[f"logits/{i}/{side}"] = logits.detach().float().numpy()
                for j, f in enumerate(fmap):
                    flat = f.detach().reshape(-1)
                    idx = sample_indices(flat.numel(), 512, seed=17 + j)
                    blob[f"f_shape/{i}/{side}/{j}"] = np.array(f.shape)
                    blob[f"f_idx/{i}/{side}/{j}"] = idx.numpy().astype(np.int32)
                    blob[f"f_val/{i}/{side}/{j}"] = flat[idx].float().numpy()
        for k, p in ref.named_parameters():
            gflat = p.grad.reshape(-1)
            idx = sample_indices(gflat.numel(), 256, seed=13)
            blob["g_idx/" + k] = idx.numpy().astype(np.int32)
            blob["g_val/" + k] = gflat[idx].float().numpy()
            blob["g_rms/" + k] = np.float64(gflat.pow(2).mean().sqrt())
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **blob)
        print(name, "loss", float(loss), "logit shapes", [tuple(t.shape) for t in y_d_rs], os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
