"""``torch.library`` custom ops over the C ABI (SURVEY.md section 8b: "torch.library.custom_op + ctypes shim ...
register_fake for shape inference").

Importing this module registers, for the CUDA dispatch key only (there is no CPU kernel: a CPU tensor fails in the
dispatcher), the ops

  * ``aero_b200::stft(x, n_fft, hop, win) -> float32 [..., n_fft/2+1, 1+L//hop, 2]``   (``aero_stft_fwd``; reference spec.py:9-22)
  * ``aero_b200::istft(z, hop, win, length) -> float32 [..., length]``                  (``aero_istft_fwd``; spec.py:25-38)
  * ``aero_b200::generator_forward(mix, handle) -> float32 [B, C_out, L*scale]``        (the whole launch sequence of
    ``Aero.forward`` for the model registered under ``handle``; aero.py:446-523)

each with a fake (meta) implementation, so the path can sit inside ``torch.compile`` / ``torch.export`` graphs as opaque
nodes with known output shapes.  ``Aero.forward`` itself keeps calling the engine directly; these ops are the registration
a framework integrator asks for.

Autograd: ``stft`` and ``istft`` carry backward formulas that run on the same kernels -- the adjoint of the STFT is
``aero_istft_fwd`` in ``AERO_ISTFT_RAW`` mode plus the fold of the reflect padding, the adjoint of the iSTFT is ``aero_stft_fwd``
with ``AERO_STFT_ZERO_PAD | AERO_STFT_ADJ_SCALE`` on the envelope-divided cotangent (include/aero_b200.h).  The generator trains
through ``Aero.forward`` in ``train()`` mode (one autograd node over aero_b200/train_engine.py); ``generator_forward`` is the
inference op.
"""
from __future__ import annotations

import weakref

import torch

from . import spec

_models = weakref.WeakValueDictionary()


def register_model(model):
    """Handle under which ``generator_forward`` finds ``model`` (an ``aero_b200.Aero``)."""
    h = id(model)
    _models[h] = model
    return h


@torch.library.custom_op("aero_b200::stft", mutates_args=(), device_types="cuda")
def stft(x: torch.Tensor, n_fft: int, hop: int, win: int) -> torch.Tensor:
    return torch.view_as_real(spec.spectro(x, n_fft, hop, win_length=win)).contiguous()


@stft.register_fake
def _(x, n_fft, hop, win):
    return x.new_empty((*x.shape[:-1], n_fft // 2 + 1, 1 + x.shape[-1] // hop, 2), dtype=torch.float32)


@torch.library.custom_op("aero_b200::istft", mutates_args=(), device_types="cuda")
def istft(z: torch.Tensor, hop: int, win: int, length: int) -> torch.Tensor:
    return spec.ispectro(torch.view_as_complex(z.contiguous()), hop, length=length, win_length=win)


@istft.register_fake
def _(z, hop, win, length):
    return z.new_empty((*z.shape[:-3], length), dtype=torch.float32)


def _stft_adjoint(g, n_fft, hop, win, length):
    """d loss / d x [..., length] from g = d loss / d z [..., bins, frames, 2] of z = stft(x) (normalised, centred, reflect)."""
    lead = g.shape[:-3]
    bins, frames = g.shape[-3], g.shape[-2]
    gz = g.reshape(-1, bins, frames, 2).float().clone()
    gz[:, 1:bins - 1] *= 0.5                                   # interior bins count twice in the C2R transform
    dx = torch.zeros(gz.shape[0], length, device=g.device)
    with torch.cuda.device(g.device):
        spec.stft_adjoint_into(gz, dx, n_fft=n_fft, hop=hop, win=win, stream=spec.current_stream())
    return dx.view(*lead, length)


def _istft_adjoint(gy, hop, win, bins, frames):
    """d loss / d z [..., bins, frames, 2] from gy = d loss / d y [..., length] of y = istft(z)."""
    lead, length = gy.shape[:-1], gy.shape[-1]
    gy = gy.reshape(-1, length)
    gz = torch.empty(gy.shape[0], bins, frames, 2, device=gy.device)
    with torch.cuda.device(gy.device):
        spec.istft_adjoint_into(gy, gz, n_fft=2 * (bins - 1), hop=hop, win=win, channels=1, frames=frames, bins=bins,
                                strides=(bins * frames * 2, 0, frames * 2, 2), stream=spec.current_stream())
    return gz.view(*lead, bins, frames, 2)


def _stft_setup(ctx, inputs, output):
    x, n_fft, hop, win = inputs
    ctx.args = (n_fft, hop, win, x.shape[-1])


def _stft_backward(ctx, g):
    n_fft, hop, win, length = ctx.args
    return _stft_adjoint(g.contiguous(), n_fft, hop, win, length), None, None, None


def _istft_setup(ctx, inputs, output):
    z, hop, win, length = inputs
    ctx.args = (hop, win, z.shape[-3], z.shape[-2])


def _istft_backward(ctx, g):
    hop, win, bins, frames = ctx.args
    return _istft_adjoint(g.contiguous(), hop, win, bins, frames), None, None, None


torch.library.register_autograd("aero_b200::stft", _stft_backward, setup_context=_stft_setup)
torch.library.register_autograd("aero_b200::istft", _istft_backward, setup_context=_istft_setup)


@torch.library.custom_op("aero_b200::generator_forward", mutates_args=(), device_types="cuda")
def generator_forward(mix: torch.Tensor, handle: int) -> torch.Tensor:
    model = _models.get(handle)
    if model is None:
        raise RuntimeError("aero_b200::generator_forward: unknown model handle (aero_b200.ops.register_model)")
    return model(mix)


@generator_forward.register_fake
def _(mix, handle):
    model = _models.get(handle)
    if model is None:
        raise RuntimeError("aero_b200::generator_forward: unknown model handle (aero_b200.ops.register_model)")
    g = model.geom
    length = mix.shape[-1]
    padded = length + (-length) % g.hop_in
    frames = 1 + padded // g.hop_in
    out_len = min(int(length * g.scale), g.hop_out * (frames - 1))
    return mix.new_empty((mix.shape[0], g.kw["out_channels"], out_len), dtype=torch.float32)
