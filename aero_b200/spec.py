"""CUDA drop-ins for the reference's ``src/models/spec.py``: ``spectro`` (9-22) and ``ispectro`` (25-38), and the one
place that calls the STFT entry points.

Same signatures and shapes: ``spectro(x[..., L]) -> complex [..., n_fft/2+1, 1+L//hop]`` (normalized, centred
reflect, periodic Hann of ``win_length`` zero-padded to ``n_fft``), ``ispectro`` its inverse.  Inputs must be
CUDA fp32 / complex64 tensors; the work is done by ``aero_stft_fwd`` / ``aero_istft_fwd`` (include/aero_b200.h).

``stft_into`` / ``istft_into`` launch those entry points (or their ragged-batch twins) on a stream the caller names, for
every module that runs an STFT; ``stft_adjoint_into`` / ``istft_adjoint_into`` are their gradients."""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn.functional as F

from . import cabi

_windows = {}
_envelopes = {}


def window(win, device):
    """Periodic Hann of length win on `device`, computed on the host in fp32 as reference spec.py:15 does, then moved."""
    w = _windows.get((win, device))
    if w is None:
        w = _windows[(win, device)] = torch.hann_window(win).to(device)
    return w


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def stft_into(x, z, stats, *, n_fft, hop, win, channels, bins_out, strides, stream, lengths=None, flags=0):
    """STFT of the rows of x [n_signals, length] into z (strides: batch, channel, bin, frame, in floats), adding each
    sample's {sum, sumsq} to stats [B, 2] fp64 when it is given.  With per-clip `lengths` (int32 on the device) row b holds
    lengths[b] samples of a ragged batch (aero_stft_varlen_fwd)."""
    lib = cabi.load()
    n_sig, length = x.shape
    p = cabi.StftParams(n_fft, hop, win, n_sig, channels, length, 1 + length // hop, bins_out, *strides, flags, 0)
    w = window(win, x.device)
    if lengths is None:
        rc = lib.aero_stft_fwd(_ptr(x), _ptr(w), _ptr(z), _ptr(stats), C.byref(p), stream)
    else:
        rc = lib.aero_stft_varlen_fwd(_ptr(x), _ptr(w), _ptr(z), _ptr(stats), _ptr(lengths), C.byref(p), stream)
    cabi.check(rc, lib)


def istft_into(z, y, *, n_fft, hop, win, channels, frames, bins_in, strides, stream, clip_frames=None, out_lens=None,
               flags=0):
    """iSTFT of `frames` frames of z (strides as for stft_into) into y [n_signals, out_len].  With per-clip `clip_frames`
    and `out_lens` (int32 on the device) clip b uses its own frames and writes its own samples of a ragged batch, the rest
    of its rows zeros (aero_istft_varlen_fwd)."""
    lib = cabi.load()
    n_sig, out_len = y.shape
    p = cabi.IstftParams(n_fft, hop, win, n_sig, channels, frames, bins_in, out_len, *strides, flags, 0)
    w = window(win, z.device)
    if clip_frames is None:
        rc = lib.aero_istft_fwd(_ptr(z), _ptr(w), _ptr(y), C.byref(p), stream)
    else:
        rc = lib.aero_istft_varlen_fwd(_ptr(z), _ptr(w), _ptr(y), _ptr(clip_frames), _ptr(out_lens), C.byref(p), stream)
    cabi.check(rc, lib)


def stft_adjoint_into(gz, dx, *, n_fft, hop, win, stream):
    """dx [B, L] += the gradient of x through z = stft(x) (normalised, centred, reflect padded), from gz [B, bins, frames, 2]
    = d/dz with its interior bins already halved (the C2R transform counts them twice): a RAW iSTFT, then the reflect
    padding folded back.  The centre, left and right parts are added in that order."""
    B, bins, frames = gz.shape[:3]
    L = dx.shape[-1]
    span = hop * (frames - 1) + n_fft                    # padded positions covered by a frame (<= L + n_fft)
    gp = torch.empty(B, span, device=gz.device)
    istft_into(gz, gp, n_fft=n_fft, hop=hop, win=win, channels=1, frames=frames, bins_in=bins,
               strides=(bins * frames * 2, 0, frames * 2, 2), stream=stream, flags=cabi.ISTFT_RAW)
    gp = F.pad(gp, (0, L + n_fft - span))
    h = n_fft // 2
    dx += gp[:, h:h + L]
    dx[:, 1:h + 1] += gp[:, :h].flip(1)                  # left reflection: padded pos p < h came from x[h - p]
    dx[:, L - 1 - h:L - 1] += gp[:, h + L:].flip(1)      # right reflection: padded pos h + L + j came from x[L - 2 - j]


def _envelope(n_fft, hop, win, frames, device):
    """sum_t w^2[pos - t*hop] of the synthesis window over the padded axis (what the iSTFT divides by)."""
    key = (n_fft, hop, win, frames, device)
    e = _envelopes.get(key)
    if e is None:
        w = torch.zeros(n_fft, device=device)
        wl = (n_fft - win) // 2
        w[wl:wl + win] = window(win, device)
        w2 = (w * w).view(1, n_fft, 1).expand(1, n_fft, frames)
        e = _envelopes[key] = F.fold(w2, (1, hop * (frames - 1) + n_fft), (1, n_fft), stride=(1, hop)).reshape(-1)
    return e


def istft_adjoint_into(gy, gz, *, n_fft, hop, win, channels, frames, bins, strides, stream):
    """gz (laid out as istft_into reads it) = the gradient of z through y = istft(z), from gy [n_signals, out_len] = d/dy:
    zero-extend, divide by the window envelope, then the STFT with AERO_STFT_ZERO_PAD | AERO_STFT_ADJ_SCALE."""
    full = hop * (frames - 1)
    u = torch.zeros(gy.shape[0], full, device=gy.device)
    u[:, :min(gy.shape[1], full)] = gy[:, :full]
    u.div_(_envelope(n_fft, hop, win, frames, gy.device)[n_fft // 2:n_fft // 2 + full])
    stft_into(u, gz, None, n_fft=n_fft, hop=hop, win=win, channels=channels, bins_out=bins, strides=strides, stream=stream,
              flags=cabi.STFT_ZERO_PAD | cabi.STFT_ADJ_SCALE)


def current_stream():
    """The current device's current stream, as the C entry points take it."""
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _need_cuda(t, what):
    if not t.is_cuda:
        raise RuntimeError(f"aero_b200.{what}: CUDA tensors only (no CPU fallback); got {t.device}")


@torch.no_grad()
def spectro(x, n_fft=512, hop_length=None, pad=0, win_length=None):
    _need_cuda(x, "spectro")
    *other, length = x.shape
    n = n_fft * (1 + pad)
    hop = hop_length or n_fft // 4
    win = win_length or n_fft
    x2 = x.reshape(-1, length).to(torch.float32).contiguous()
    bins, frames = n // 2 + 1, 1 + length // hop
    z = torch.empty(x2.shape[0], bins, frames, 2, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        stft_into(x2, z, None, n_fft=n, hop=hop, win=win, channels=1, bins_out=bins,
                  strides=(bins * frames * 2, 0, frames * 2, 2), stream=current_stream())
    return torch.view_as_complex(z).view(*other, bins, frames)


@torch.no_grad()
def ispectro(z, hop_length=None, length=None, pad=0, win_length=None):
    _need_cuda(z, "ispectro")
    *other, bins, frames = z.shape
    n_fft = 2 * bins - 2
    hop = hop_length or n_fft // 2
    win = win_length or n_fft // (1 + pad)
    zr = torch.view_as_real(z.reshape(-1, bins, frames).to(torch.complex64).contiguous())
    full = hop * (frames - 1)
    out_len = full if length is None else min(length, full)
    y = torch.empty(zr.shape[0], out_len, dtype=torch.float32, device=z.device)
    with torch.cuda.device(z.device):
        istft_into(zr, y, n_fft=n_fft, hop=hop, win=win, channels=1, frames=frames, bins_in=bins,
                   strides=(bins * frames * 2, 0, frames * 2, 2), stream=current_stream())
    if length is not None and length > full:
        y = torch.nn.functional.pad(y, (0, length - full))
    return y.view(*other, y.shape[-1])
