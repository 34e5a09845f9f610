"""Inference drivers with the reference's call shapes (SURVEY.md section 8a16, 8f rank 4).

* ``get_estimate(model, lr_sig)``            -- reference ``src/enhance.py:11-15`` (no_grad forward).
* ``enhance_long(model, lr_sig, sr, ...)``   -- what reference ``predict.py:55-86`` does to a whole file: cut it into
  non-overlapping 10-second chunks, run the generator on each chunk on its own (each chunk is normalised by its own
  statistics, ``aero.py:462-464``) and concatenate.  The reference runs the chunks one by one at batch 1 with a
  host round trip per chunk; here equal-length chunks go through the kernels as one batch and stay on the device.
  Results are identical to the serial loop because samples of a batch never interact.
"""
from __future__ import annotations

import math

import torch

SEGMENT_DURATION_SEC = 10          # reference predict.py:22


def get_estimate(model, lr_sig):
    with torch.no_grad():
        return model(lr_sig)


@torch.no_grad()
def enhance_long(model, lr_sig, sr, segment_sec=SEGMENT_DURATION_SEC, max_batch=8, upsample=False):
    """lr_sig: [C, L] on the model's device, sampled at ``sr`` (= model.lr_sr).  Returns [C_out, ~L * scale].
    ``upsample`` (the experiment's ``upsample: true``, reference predict.py:55-57): the whole signal is first resampled to
    ``model.hr_sr`` on the device (``aero_b200.resample``) and then cut into chunks of ``hr_sr * segment_sec`` samples."""
    if lr_sig.dim() != 2:
        raise ValueError(f"expected [channels, samples], got {tuple(lr_sig.shape)}")
    if upsample:
        from .resampler import resample
        lr_sig = resample(lr_sig, sr, model.hr_sr)
        sr = model.hr_sr
    seg = int(sr * segment_sec)
    total = lr_sig.shape[-1]
    if total == 0 or seg <= 0:
        raise ValueError(f"enhance_long: empty signal or segment (samples {total}, segment {seg})")
    n_chunks = max(1, math.ceil(total / seg))
    n_full = total // seg if total % seg else n_chunks
    outs = []
    if n_full:
        full = lr_sig[:, :n_full * seg].reshape(lr_sig.shape[0], n_full, seg).permute(1, 0, 2).contiguous()   # [n_full, C, seg]
        for i in range(0, n_full, max_batch):
            pr = model(full[i:i + max_batch])                   # [b, C_out, seg*scale]
            outs.extend(pr[j] for j in range(pr.shape[0]))
    if n_full < n_chunks:
        tail = lr_sig[:, n_full * seg:]
        outs.append(model(tail.unsqueeze(0))[0])
    return torch.cat(outs, dim=-1)
