"""Inference drivers with the reference's call shapes (SURVEY.md section 8a16, 8f rank 4).

* ``get_estimate(model, lr_sig)``            -- reference ``src/enhance.py:11-15`` (no_grad forward).
* ``enhance_long(model, lr_sig, sr, ...)``   -- what reference ``predict.py:55-86`` does to a whole file: cut it into
  non-overlapping 10-second chunks, run the generator on each chunk on its own (each chunk is normalised by its own
  statistics, ``aero.py:462-464``) and concatenate.  The reference runs the chunks one by one at batch 1 with a
  host round trip per chunk; here equal-length chunks go through the kernels as one batch and stay on the device.
  Results are identical to the serial loop because samples of a batch never interact.
* ``enhance_batch(model, signals)``          -- many clips of different lengths (reference ``test.py`` / ``evaluate.py``,
  many-file ``predict.py``): sorted by length and run in ragged batches (``AeroEngine.forward_varlen`` for AERO,
  ``SeanetEngine.forward_varlen`` for SEANet), each clip with the result it gets on its own.
* ``evaluate_batch(model, lr, hr)``           -- reference ``src/evaluate.py:143-185`` ``evaluate()`` without ViSQOL, wandb and
  file writing: every file's estimate, ``match_signal`` to its ``hr`` length, the per-file LSDs of one fused call
  (``metrics.get_lsd_batch``) and their mean over files with a non-zero LSD, averaged over ranks.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

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


def _ragged_batches(signals, cin, max_batch):
    """Sort clips by length and pad them into batches of at most ``max_batch``: yields (input indices, lengths, [b, cin, L_max])."""
    order = sorted(range(len(signals)), key=lambda i: signals[i].shape[-1])
    for k in range(0, len(order), max_batch):
        idx = order[k:k + max_batch]
        lens = [signals[i].shape[-1] for i in idx]
        mix = signals[idx[0]].new_zeros(len(idx), cin, max(lens))
        for j, i in enumerate(idx):
            mix[j, :, :lens[j]] = signals[i]
        yield idx, lens, mix


@torch.no_grad()
def enhance_batch(model, signals, max_batch=32, return_spec=False, return_lr_spec=False):
    """signals: list of [C, L_i] tensors on the model's (CUDA) device at ``model.lr_sr``.  Returns a list, in input order,
    of what ``model(signals[i][None])`` returns with the batch axis dropped: the waveform [C_out, out_len(L_i)], and with
    ``return_spec`` / ``return_lr_spec`` (AERO only) the spectrograms cropped to the clip's own frames.  Clips are sorted by
    length and run in ragged batches of at most ``max_batch``, so that each batch carries as little padding as possible.
    ``model`` is an ``Aero`` or a ``Seanet`` in ``eval()`` mode (``AeroEngine.forward_varlen``, ``SeanetEngine.forward_varlen``)."""
    from .model import Aero
    from .seanet import Seanet
    if isinstance(model, Seanet):
        return _enhance_batch_seanet(model, signals, max_batch, return_spec or return_lr_spec)
    if not isinstance(model, Aero):
        raise NotImplementedError(f"enhance_batch runs the AERO or SEANet generator, got {type(model).__name__}")
    eng = model._engine()
    if model.training:
        eng._check_mode()
    if max_batch < 1:
        raise ValueError(f"max_batch must be >= 1, got {max_batch}")
    signals = list(signals)
    if not signals:
        return []
    cin = model.geom.kw["in_channels"]
    for i, s in enumerate(signals):
        eng._require(s)
        if s.dim() != 2 or s.shape[0] != cin:
            raise ValueError(f"signal {i}: expected [{cin}, L], got {tuple(s.shape)}")
    results = [None] * len(signals)
    for idx, lens, mix in _ragged_batches(signals, cin, max_batch):
        out = eng.forward_varlen(mix, lens, return_spec=return_spec, return_lr_spec=return_lr_spec)
        y, out_lens = out[0], out[1]
        frames = [model.geom.frames(n) for n in lens]
        for j, i in enumerate(idx):
            r = y[j, :, :out_lens[j]].clone()
            if return_spec:
                specs = tuple(sp[j, ..., :frames[j]].clone() for sp in out[2:])
                results[i] = (r, *specs)
            else:
                results[i] = r
    return results


def _enhance_batch_seanet(model, signals, max_batch, specs):
    # everything a SEANet call can be refused for is checked on the host, in this order, before the engine is built or the
    # library is loaded: the mode, the arguments, then each clip's shape and length (the error names the clip)
    if model.training:
        raise NotImplementedError("enhance_batch runs the SEANet inference forward; call model.eval()")
    if specs:
        raise ValueError("return_spec / return_lr_spec: SEANet is a time-domain generator and has no spectrogram output")
    if max_batch < 1:
        raise ValueError(f"max_batch must be >= 1, got {max_batch}")
    signals = list(signals)
    if not signals:
        return []
    cin = model.in_channels
    for i, s in enumerate(signals):
        if s.dim() != 2 or s.shape[0] != cin:
            raise ValueError(f"signal {i}: expected [{cin}, L], got {tuple(s.shape)}")
        try:
            model.check_length(s.shape[-1])
        except ValueError as e:
            raise ValueError(f"signal {i}: {e}") from None
    eng = model._engine()
    for s in signals:
        eng._require(s)
    results = [None] * len(signals)
    for idx, lens, mix in _ragged_batches(signals, cin, max_batch):
        y, out_lens = eng.forward_varlen(mix, lens)
        for j, i in enumerate(idx):
            results[i] = y[j, :, :out_lens[j]].clone()
    return results


def match_signal(signal, ref_len):
    """reference src/utils.py:211-217: crop or zero-pad the last axis of `signal` to `ref_len` samples."""
    n = signal.shape[-1]
    if n < ref_len:
        return F.pad(signal, (0, ref_len - n))
    return signal[..., :ref_len]


def nonzero_mean(values):
    """reference evaluate.py:160-177: the sum of the per-file values over the number of files whose value is not 0 (a file
    scored 0 does not count); (0.0, 0) when there is none.  Returns (mean, count)."""
    values = [float(v) for v in values]
    count = sum(1 for v in values if v != 0)
    return (sum(values) / count if count else 0.0), count


@torch.no_grad()
def evaluate_batch(model, lr_signals, hr_signals, max_batch=32):
    """lr_signals, hr_signals: lists of [C, L_i] CUDA tensors (the model's input and the high-rate target of each file).
    Both generators run the files through ``enhance_batch`` (ragged batches of at most ``max_batch``).  Each
    estimate is cropped or zero-padded to its target's length and all files are scored in one ``get_lsd_batch`` call.
    Returns (per-file LSDs as an fp32 CUDA tensor [N], the mean over files with a non-zero LSD, that count); under
    ``torch.distributed`` the mean is averaged over ranks weighted by each rank's count.  Like the reference, the model
    runs in eval mode and is put back in the mode it came in."""
    from .metrics import get_lsd_batch
    from .model import Aero
    from .parallel import average_over_ranks
    from .seanet import Seanet
    lr_signals, hr_signals = list(lr_signals), list(hr_signals)
    if len(lr_signals) != len(hr_signals):
        raise ValueError(f"{len(lr_signals)} inputs for {len(hr_signals)} targets")
    if not isinstance(model, (Aero, Seanet)):
        raise NotImplementedError(f"evaluate_batch runs AERO or SEANet, got {type(model).__name__}")
    was_training = model.training
    model.eval()
    try:
        prs = enhance_batch(model, lr_signals, max_batch=max_batch)
    finally:
        model.train(was_training)
    prs = [match_signal(p, h.shape[-1]) for p, h in zip(prs, hr_signals)]
    lsd = get_lsd_batch(hr_signals, prs)
    mean, count = nonzero_mean(lsd.tolist())
    return lsd, average_over_ranks(mean, count), count
