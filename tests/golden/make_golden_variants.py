"""Golden vectors of the AERO variants the reference switches with `act_func` and `spec_upsample` (aero.py:306-307), made by
running the UNMODIFIED reference:

    python tests/golden/make_golden_variants.py [case ...]

Forward cases (vf_*.npz) follow tests/golden/make_golden.py: the reference ``Aero`` built from the experiment kwargs plus the
case's overrides, ``trained_like_`` weights, ``forward(mix, return_spec=True, return_lr_spec=True)`` under ``no_grad`` in fp32
on CPU, with block outputs captured by forward hooks.  Training cases (vt_*.npz) follow tests/golden/make_golden_train.py: the
reference promoted to fp64 in train mode, ``loss = sum(out * R) / out.numel()`` back-propagated, per-parameter gradient samples.
The files are named vf_* / vt_* so that the c* / t* parametrisations (whose input recipe is plain noise) do not pick them up.

Input: seeded white noise at lr_sr; for an experiment with ``upsample: true`` (the sinc cases) it is first resampled to hr_sr
with ``torchaudio.functional.resample`` as the reference's dataset does (datasets.py:143-145), and stored in the file as ``mix``.
The GPU box has no /root/reference; tests there read only the committed .npz files.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from util import ROOT, SEED, import_reference, sample_indices, trained_like_, weights_digest, white_noise  # noqa: E402

sys.path.insert(0, ROOT)
from aero_b200.config import aero_kwargs, load_experiment  # noqa: E402

FORWARD = [  # name, experiment, aero kwarg overrides, batch, low-rate length
    ("vf_relu_4-16_hop64_ragged_b2", "aero_4-16_512_64_relu", {}, 2, 3001),
    ("vf_gelu_4-16_hop64", "aero_4-16_512_64", {"act_func": "gelu"}, 1, 4000),
    ("vf_sinc_4-16_hop64", "aero_4-16_512_64_sinc", {}, 1, 2000),
]
TRAIN = [  # name, experiment, batch, low-rate length
    ("vt_relu_4-16_hop64", "aero_4-16_512_64_relu", 2, 2000),
    ("vt_sinc_4-16_hop64", "aero_4-16_512_64_sinc", 1, 1500),
]


def variant_input(exp, B, L):
    """Seeded white noise at lr_sr, resampled to hr_sr when the experiment sets `upsample`."""
    e = load_experiment(exp)
    mix = white_noise((B, e["aero"]["in_channels"], L))
    if e["upsample"]:
        import torchaudio
        mix = torchaudio.functional.resample(mix, e["lr_sr"], e["hr_sr"])
    return mix


def reference_model(ref, kw):
    torch.manual_seed(SEED)
    model = ref["aero"].Aero(**kw)
    model.load_state_dict(trained_like_(model.state_dict()))
    return model, weights_digest(model.state_dict())


def forward_case(ref, name, exp, overrides, B, L):
    kw = dict(aero_kwargs(exp), **overrides)
    model, digest = reference_model(ref, kw)
    model.eval()
    mix = variant_input(exp, B, L)
    acts = {}

    def hook(tag):
        def fn(mod, inp, out):
            acts[tag] = out.detach()
        return fn
    handles = []
    for i, enc in enumerate(model.encoder):
        handles.append(enc.register_forward_hook(hook(f"encoder.{i}")))
        handles.append(enc.dconv.register_forward_hook(hook(f"encoder.{i}.dconv")))
        handles.append(enc.freq_attn_block.register_forward_hook(hook(f"encoder.{i}.ftb")))
    for j, dec in enumerate(model.decoder):
        handles.append(dec.register_forward_hook(hook(f"decoder.{j}")))
    with torch.no_grad():
        out, zc, zlr = model(mix, return_spec=True, return_lr_spec=True)
    for h in handles:
        h.remove()
    blob = {"digest": np.float64(digest), "B": B, "L": L, "exp": exp, "torch": torch.__version__,
            "overrides": json.dumps(overrides), "mix": mix.numpy(), "out": out.numpy()}
    zc_r, zlr_r = torch.view_as_real(zc).reshape(-1), torch.view_as_real(zlr).reshape(-1)
    blob["spec_idx"] = sample_indices(zc_r.numel(), 8192).numpy().astype(np.int32)
    blob["spec_val"] = zc_r[blob["spec_idx"].astype(np.int64)].numpy()
    blob["lrspec_idx"] = sample_indices(zlr_r.numel(), 8192).numpy().astype(np.int32)
    blob["lrspec_val"] = zlr_r[blob["lrspec_idx"].astype(np.int64)].numpy()
    for tag, a in acts.items():
        flat = a.reshape(-1)
        idx = sample_indices(flat.numel(), 2048)
        blob["act_idx/" + tag] = idx.numpy().astype(np.int32)
        blob["act_val/" + tag] = flat[idx].numpy()
        blob["act_rms/" + tag] = np.float64(flat.double().pow(2).mean().sqrt())
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **blob)
    print(name, "out", tuple(out.shape), "rms", float(out.pow(2).mean().sqrt()), "digest", digest)


def train_case(ref, name, exp, B, L):
    model, digest = reference_model(ref, aero_kwargs(exp))
    # fp64 reference: see make_golden_train.py (gradients that are small differences of large terms)
    model = model.double().train()
    mix = variant_input(exp, B, L).double()
    out = model(mix)
    R = white_noise(tuple(out.shape), seed=SEED + 77).double()        # make_golden_train.cotangent
    loss = (out * R).sum() / out.numel()
    loss.backward()
    blob = {"digest": np.float64(digest), "B": B, "L": L, "exp": exp, "torch": torch.__version__, "loss": np.float64(float(loss.detach())),
            "out_shape": np.array(out.shape), "mix": mix.float().numpy()}
    flat = out.detach().reshape(-1)
    oi = sample_indices(flat.numel(), 16384, seed=11)
    blob["out_idx"], blob["out_val"] = oi.numpy().astype(np.int32), flat[oi].float().numpy()
    for k, p in model.named_parameters():
        gflat = p.grad.reshape(-1)
        idx = sample_indices(gflat.numel(), 256, seed=13)
        blob["g_idx/" + k] = idx.numpy().astype(np.int32)
        blob["g_val/" + k] = gflat[idx].float().numpy()
        blob["g_rms/" + k] = np.float64(gflat.double().pow(2).mean().sqrt())
    for k, b in model.named_buffers():
        if k.endswith(("running_mean", "running_var")):
            blob["buf/" + k] = b.detach().float().numpy()
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **blob)
    print(name, "out", tuple(out.shape), "loss", float(loss.detach()), "params", sum(1 for _ in model.named_parameters()))


def main():
    ref = import_reference()
    assert ref is not None, "needs /root/reference"
    torch.set_num_threads(os.cpu_count())
    only = set(sys.argv[1:])
    for name, *rest in FORWARD:
        if not only or name in only:
            forward_case(ref, name, *rest)
    for name, *rest in TRAIN:
        if not only or name in only:
            train_case(ref, name, *rest)


if __name__ == "__main__":
    main()
