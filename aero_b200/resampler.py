"""``aero_b200.resample``: ``torchaudio.functional.resample`` with its defaults on the sm_90a kernels.

The reference resamples low-rate audio to the high rate before a time-domain model, or before AERO built with
``spec_upsample=False`` (reference ``src/data/datasets.py:143-145``, ``predict.py:55-57``, ``src/evaluate.py:22-25``).
The polyphase filter table is computed on the host exactly as torchaudio computes it for an fp32 input
(``seanet.sinc_resample_table``); ``aero_resample_fwd`` applies it on the device.  Data preparation: no gradient.
"""
from __future__ import annotations

import ctypes as C
import math

import torch

from . import cabi
from .seanet import sinc_resample_table

__all__ = ["resample", "resampled_length"]

_tables = {}


def _reduced(orig_freq, new_freq):
    if orig_freq <= 0 or new_freq <= 0:
        raise ValueError(f"resample: frequencies must be positive (got {orig_freq}, {new_freq})")
    if int(orig_freq) != orig_freq or int(new_freq) != new_freq:
        raise ValueError(f"resample: frequencies must be integers (got {orig_freq}, {new_freq})")
    g = math.gcd(int(orig_freq), int(new_freq))
    return int(orig_freq) // g, int(new_freq) // g


def resampled_length(length, orig_freq, new_freq):
    """Output length of ``torchaudio.functional.resample`` for `length` input samples: ceil(new * length / orig) of the
    reduced ratio, evaluated the way torchaudio evaluates it (a Python float made a default-dtype tensor)."""
    orig, new = _reduced(orig_freq, new_freq)
    if orig == new:
        return length
    return int(torch.ceil(torch.as_tensor(new * length / orig)).long())


def _table(orig_freq, new_freq, device):
    key = (orig_freq, new_freq, device)
    t = _tables.get(key)
    if t is None:
        filt, width, orig, up = sinc_resample_table(orig_freq, new_freq, torch.float32)
        t = _tables[key] = (filt.contiguous().to(device), width, orig, up)
    return t


@torch.no_grad()
def resample(x, orig_freq, new_freq):
    """``torchaudio.functional.resample(x, orig_freq, new_freq)`` (``sinc_interp_hann``, ``lowpass_filter_width=6``,
    ``rolloff=0.99``) on the device.  x: fp32 CUDA tensor ``[..., L]``; returns ``[..., ceil(new * L / orig)]`` for the
    gcd-reduced ratio orig:new, and `x` itself when the rates are equal (as torchaudio does)."""
    orig, new = _reduced(orig_freq, new_freq)
    if not x.is_cuda:
        raise RuntimeError("aero_b200.resample runs on CUDA only (sm_90a kernels in libaero_b200.so); there is no CPU path")
    if x.dtype != torch.float32:
        raise TypeError(f"aero_b200.resample computes in fp32; got {x.dtype}")
    if x.dim() == 0:
        raise ValueError("aero_b200.resample: expected [..., L], got a scalar")
    if orig == new:
        return x
    *lead, length = x.shape
    out_len = resampled_length(length, orig, new)
    y = torch.empty(*lead, out_len, dtype=torch.float32, device=x.device)
    if y.numel() == 0:
        return y
    lib = cabi.load()
    with torch.cuda.device(x.device):
        filt, width, orig, up = _table(int(orig_freq), int(new_freq), x.device)
        x2 = x.contiguous()
        stream = C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)
        cabi.check(lib.aero_resample_fwd(C.c_void_p(x2.data_ptr()), C.c_void_p(filt.data_ptr()), C.c_void_p(y.data_ptr()),
                                         x2.numel() // length, length, out_len, orig, up, width, filt.shape[1], stream), lib)
    return y
