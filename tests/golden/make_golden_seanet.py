"""Golden vectors for the SEANet generator from the UNMODIFIED reference (`src/models/seanet.py`) in fp64:

    AERO_REFERENCE=/path/to/aero python tests/golden/make_golden_seanet.py

Weights are a recipe (tests/seanet_util.seanet_recipe_state on a model seeded with SEED) plus a digest; inputs are seeded
(tests/seanet_util.case_input).  Stored per case: the output, the generated branch (the last decoder layer's tanh output,
before the input skip is added), the padded input x0, and 2048 samples of the input of every encoder level and the output of
every decoder level (so that a failure points at a stage)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from util import SEED, sample_indices, weights_digest  # noqa: E402
from seanet_util import CASES, case_input, seanet_recipe_state, train_case  # noqa: E402


def reference_seanet_class():
    import importlib
    root = os.path.abspath(os.environ.get("AERO_REFERENCE", "reference"))
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "src" or k.startswith("src.")}
    path_saved = list(sys.path)
    repo = os.path.dirname(os.path.dirname(HERE))
    sys.path[:] = [root] + [p for p in sys.path if os.path.abspath(p or ".") != repo]
    try:
        mod = importlib.import_module("src.models.seanet")
    finally:
        sys.path[:] = path_saved
        for k in [k for k in sys.modules if k == "src" or k.startswith("src.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    return mod.Seanet


def main():
    torch.set_num_threads(os.cpu_count())
    Ref = reference_seanet_class()
    for name, (kw, _) in CASES.items():
        torch.manual_seed(SEED)
        ref = Ref(**kw)
        ref.load_state_dict(seanet_recipe_state(ref.state_dict()))
        digest = weights_digest(ref.state_dict())
        ref = ref.double().eval()
        x = case_input(name).double()
        cap = {}
        hooks = [ref.decoder[-1].register_forward_hook(lambda m, i, o: cap.__setitem__("branch", o))]
        for i, enc in enumerate(ref.encoder):
            hooks.append(enc.register_forward_pre_hook(lambda m, inp, i=i: cap.__setitem__(f"enc{i}_in", inp[0])))
        for j, dec in enumerate(ref.decoder[:-1]):
            hooks.append(dec.register_forward_hook(lambda m, i, o, j=j: cap.__setitem__(f"dec{j}_raw", o)))
        with torch.no_grad():
            y = ref(x)
        for h in hooks:
            h.remove()
        blob = {"digest": np.float64(digest), "torch": torch.__version__, "y": y.float().numpy(),
                "branch": cap["branch"].float().numpy(), "x0": cap["enc0_in"].float().numpy()}
        for k, v in cap.items():
            if k in ("branch", "enc0_in") or k.endswith("_raw"):
                continue
            flat = v.reshape(-1)
            idx = sample_indices(flat.numel(), 2048, seed=17)
            blob[f"stage_idx/{k}"] = idx.numpy().astype(np.int32)
            blob[f"stage_val/{k}"] = flat[idx].float().numpy()
        path = os.path.join(HERE, f"seanet_{name}.npz")
        np.savez_compressed(path, **blob)
        print(name, tuple(y.shape), os.path.getsize(path), "bytes")



def main_train():
    """t1: the shipped config in training, B=2 x 1 s, loss = sum(out * R) with a seeded R: the loss and, per parameter, the rms and
    256 samples of its gradient."""
    Ref = reference_seanet_class()
    kw = CASES["s1"][0]
    torch.manual_seed(SEED)
    ref = Ref(**kw)
    ref.load_state_dict(seanet_recipe_state(ref.state_dict()))
    digest = weights_digest(ref.state_dict())
    ref = ref.double().train()
    x, R = train_case()
    loss = (ref(x.double()) * R.double()).sum()
    loss.backward()
    blob = {"digest": np.float64(digest), "torch": torch.__version__, "loss": np.float64(float(loss))}
    for k, p in ref.named_parameters():
        gr = p.grad.reshape(-1)
        idx = sample_indices(gr.numel(), 256, seed=19)
        blob[f"grad_rms/{k}"] = np.float64(float(gr.pow(2).mean().sqrt()))
        blob[f"grad_idx/{k}"] = idx.numpy().astype(np.int32)
        blob[f"grad_val/{k}"] = gr[idx].numpy()
    path = os.path.join(HERE, "seanet_t1.npz")
    np.savez_compressed(path, **blob)
    print("t1 loss", float(loss), os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
    main_train()
