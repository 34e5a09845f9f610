"""Functional torch-CPU restatement of the reference SEANet forward (reference ``src/models/seanet.py``), in any dtype.

Used by the tests and ``bench_seanet.py`` as the comparison point of the CUDA path.  It reads a ``state_dict`` with the
reference's keys (weight_norm ``weight_g`` / ``weight_v``) and a ``Seanet``-like config object (``ratios``, ``ngf``,
``n_residual_layers``, ``normalize``, ``floor``, ``lr_sr``, ``hr_sr``, ``upsample``, ``scale_factor``,
``estimate_output_length``).  The resampler of ``torchaudio.functional.resample`` is written out (``resample_table``,
``resample``) so that the oracle does not depend on torchaudio.
"""
import math

import torch
import torch.nn.functional as F


def resample_table(orig_freq, new_freq, dtype, lowpass_filter_width=6, rolloff=0.99):
    """torchaudio ``_get_sinc_resample_kernel`` (sinc_interp_hann) for an input of `dtype`: [new, 1, 2*width + orig], width."""
    g = math.gcd(int(orig_freq), int(new_freq))
    orig, new = int(orig_freq) // g, int(new_freq) // g
    base = min(orig, new) * rolloff
    width = math.ceil(lowpass_filter_width * orig / base)
    idx = torch.arange(-width, width + orig, dtype=dtype)[None, None] / orig
    t = torch.arange(0, -new, -1, dtype=dtype)[:, None, None] / new + idx
    t *= base
    t = t.clamp_(-lowpass_filter_width, lowpass_filter_width)
    window = torch.cos(t * math.pi / lowpass_filter_width / 2) ** 2
    t *= math.pi
    kern = torch.where(t == 0, torch.tensor(1.0).to(t), t.sin() / t)
    kern *= window * (base / orig)
    return kern, width


def resample(x, orig_freq, new_freq):
    """torchaudio ``_apply_sinc_resample_kernel``: x [..., L] -> [..., ceil(new * L / orig)] (reduced ratio)."""
    g = math.gcd(int(orig_freq), int(new_freq))
    orig, new = int(orig_freq) // g, int(new_freq) // g
    kern, width = resample_table(orig_freq, new_freq, x.dtype)
    shape = x.shape
    w = x.reshape(-1, shape[-1])
    n, length = w.shape
    w = F.pad(w, (width, width + orig))
    y = F.conv1d(w[:, None], kern, stride=orig).transpose(1, 2).reshape(n, -1)
    y = y[..., :math.ceil(new * length / orig)]
    return y.view(*shape[:-1], y.shape[-1])


def _w(sd, key):
    # torch.nn.utils.weight_norm, dim 0: w = g * v / ||v|| over every dimension but the first
    return torch._weight_norm(sd[key + ".weight_v"], sd[key + ".weight_g"], 0)


def _conv(sd, key, x, **kw):
    return F.conv1d(x, _w(sd, key), sd[key + ".bias"], **kw)


def _lrelu(x):
    return F.leaky_relu(x, 0.2)


def _resblock(sd, key, x, dil):
    # seanet.py:10-23
    h = _conv(sd, key + ".block.2", F.pad(_lrelu(x), (dil, dil), mode="reflect"), dilation=dil)
    h = _conv(sd, key + ".block.4", _lrelu(h))
    return _conv(sd, key + ".shortcut", x) + h


def seanet_forward(sd, cfg, signal, stages=None):
    """reference seanet.py:153-179.  `stages` (a dict) receives the input of every encoder level and the output of every
    decoder level: x0, enc{i}_in, dec{j}_out."""
    nres, ratios = cfg.n_residual_layers, list(cfg.ratios)
    nlev = len(ratios)
    target = signal.shape[-1] * (cfg.scale_factor if cfg.upsample else 1)
    if cfg.normalize:                                               # :158-161
        mono = signal.mean(dim=1, keepdim=True)
        std = mono.std(dim=-1, keepdim=True)
        signal = signal / (cfg.floor + std)
    else:
        std = 1
    x = signal
    if cfg.upsample:                                                # :165-166
        x = resample(x, cfg.lr_sr, cfg.hr_sr)
    x = F.pad(x, (0, cfg.estimate_output_length(x.shape[-1]) - x.shape[-1]))     # :168, :147-151
    skips = [x]
    if stages is not None:
        stages["x0"] = x
    # encoder 0 (:106-111): ReflectionPad1d(3), WNConv1d(k7), Tanh
    x = torch.tanh(_conv(sd, "encoder.0.1", F.pad(x, (3, 3), mode="reflect")))
    for i in range(1, nlev + 1):                                    # :72-104 (encoder side)
        skips.append(x)
        if stages is not None:
            stages[f"enc{i}_in"] = x
        r = ratios[nlev - i]
        for k in range(nres):
            x = _resblock(sd, f"encoder.{i}.{k}", x, 3 ** k)
        x = _conv(sd, f"encoder.{i}.{nres + 1}", _lrelu(x), stride=r, padding=r // 2 + r % 2)
    skips.append(x)
    if stages is not None:
        stages[f"enc{nlev + 1}_in"] = x
    x = _conv(sd, f"encoder.{nlev + 1}.2", F.pad(_lrelu(x), (3, 3), mode="reflect"))        # :63-67
    x = _conv(sd, "decoder.0.2", F.pad(_lrelu(x), (3, 3), mode="reflect")) + skips.pop()    # :57-61, :173-176
    if stages is not None:
        stages["dec0_out"] = x
    for j in range(1, nlev + 1):                                    # :83-99 (decoder side)
        r = ratios[j - 1]
        key = f"decoder.{j}.1"
        x = F.conv_transpose1d(_lrelu(x), _w(sd, key), sd[key + ".bias"], stride=r, padding=r // 2 + r % 2, output_padding=r % 2)
        for k in range(nres):
            x = _resblock(sd, f"decoder.{j}.{2 + k}", x, 3 ** k)
        x = x + skips.pop()
        if stages is not None:
            stages[f"dec{j}_out"] = x
    x = torch.tanh(_conv(sd, f"decoder.{nlev + 1}.2", F.pad(_lrelu(x), (3, 3), mode="reflect")))   # :113-118
    if stages is not None:
        stages["branch"] = x
    x = x + skips.pop()
    if target < x.shape[-1]:                                        # :177-179
        x = x[..., :target]
    return std * x
