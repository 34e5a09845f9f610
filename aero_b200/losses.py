"""Multi-resolution STFT loss on the GPU, with its gradient (SURVEY.md section 8f rank 2).

``MultiResolutionSTFTLoss`` has the constructor and call shape of reference ``src/models/stft_loss.py:96-138`` (three
resolutions 1024/120/600, 2048/240/1200, 512/50/240; spectral convergence ``:30-45`` + log-magnitude L1 ``:48-63``, each
averaged over the resolutions and scaled by ``factor_sc`` / ``factor_mag``).  The six STFTs run on ``aero_stft_fwd``, the
reductions on ``aero_stft_loss_fwd``.  It is differentiable with respect to the estimate ``x`` (the reference calls it with
gradients at ``solver.py:470-473``): one ``torch.autograd.Function`` whose backward is ``aero_stft_loss_bwd`` (gradient of the
normalised spectrogram) followed by the adjoint of the STFT = ``aero_istft_fwd`` in ``AERO_ISTFT_RAW`` mode and the fold of
the reflect padding.  The target ``y`` gets no gradient (the reference never needs one).
The reference's own ``stft()`` calls ``torch.stft`` without ``return_complex`` and raises on torch >= 2 (SURVEY.md appendix
C); the semantics here are the intended ones (tests/golden/make_golden.py applies the one-line shim to the reference to
produce the fixture).
"""
from __future__ import annotations

import ctypes as C

import torch

from . import cabi
from .spec import spectro, stft_adjoint_into


def _spectra(x, y, resolutions):
    lib = cabi.load()
    sums = torch.zeros(len(resolutions), 3, dtype=torch.float64, device=x.device)
    counts, saved = [], []
    with torch.cuda.device(x.device):
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        for i, (n_fft, hop, win) in enumerate(resolutions):
            zx = torch.view_as_real(spectro(x, n_fft, hop, win_length=win)).contiguous()   # [B, bins, frames, 2], x n_fft^-1/2
            zy = torch.view_as_real(spectro(y, n_fft, hop, win_length=win)).contiguous()
            B, bins, frames = zx.shape[:3]
            counts.append(B * bins * frames)
            cabi.check(lib.aero_stft_loss_fwd(C.c_void_p(zx.data_ptr()), C.c_void_p(zy.data_ptr()),
                                              C.c_void_p(sums[i].data_ptr()), B, bins, frames, n_fft, stream), lib)
            saved.append((zx, zy))
    return sums, counts, saved


class _MRSTFTFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, y, resolutions, factor_sc, factor_mag):
        xc, yc = x.detach().float().contiguous(), y.detach().float().contiguous()
        sums, counts, saved = _spectra(xc, yc, resolutions)
        n = torch.tensor(counts, dtype=torch.float64, device=x.device)
        sc = torch.sqrt(sums[:, 0] / sums[:, 1]).mean()
        mag = (sums[:, 2] / n).mean()
        ctx.saved, ctx.sums, ctx.res, ctx.f = saved, sums, resolutions, (factor_sc, factor_mag)
        ctx.shape, ctx.dtype = x.shape, x.dtype
        ctx.set_materialize_grads(False)
        return (factor_sc * sc).float(), (factor_mag * mag).float()

    @staticmethod
    def backward(ctx, g_sc, g_mag):
        lib = cabi.load()
        B, L = ctx.shape
        dev = ctx.sums.device
        R = len(ctx.res)
        k_sc = (float(g_sc) if g_sc is not None else 0.0) * ctx.f[0] / R
        k_mag = (float(g_mag) if g_mag is not None else 0.0) * ctx.f[1] / R
        dx = torch.zeros(B, L, device=dev)
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            for i, (n_fft, hop, win) in enumerate(ctx.res):
                zx, zy = ctx.saved[i]
                _, bins, frames = zx.shape[:3]
                gz = torch.empty_like(zx)
                cabi.check(lib.aero_stft_loss_bwd(C.c_void_p(zx.data_ptr()), C.c_void_p(zy.data_ptr()), C.c_void_p(ctx.sums[i].data_ptr()),
                                                  C.c_void_p(gz.data_ptr()), B, bins, frames, n_fft, k_sc, k_mag, stream), lib)
                stft_adjoint_into(gz, dx, n_fft=n_fft, hop=hop, win=win, stream=stream)
        return dx.to(ctx.dtype), None, None, None, None


class MultiResolutionSTFTLoss(torch.nn.Module):
    def __init__(self, fft_sizes=(1024, 2048, 512), hop_sizes=(120, 240, 50), win_lengths=(600, 1200, 240),
                 window="hann_window", factor_sc=0.1, factor_mag=0.1):
        super().__init__()
        if not (len(fft_sizes) == len(hop_sizes) == len(win_lengths)):
            raise ValueError("fft_sizes, hop_sizes and win_lengths must have the same length")
        if window != "hann_window":
            raise NotImplementedError("aero_b200: only the Hann window of the shipped configs is implemented")
        self.resolutions = list(zip(fft_sizes, hop_sizes, win_lengths))
        self.factor_sc, self.factor_mag = factor_sc, factor_mag

    def forward(self, x, y):
        """x (estimate), y (target): CUDA tensors [B, T].  Returns (factor_sc * sc_loss, factor_mag * mag_loss), 0-dim fp32;
        differentiable with respect to x."""
        if not (x.is_cuda and y.is_cuda):
            raise RuntimeError("aero_b200.losses: CUDA tensors only (no CPU fallback)")
        if x.shape != y.shape or x.dim() != 2:
            raise ValueError(f"expected two [B, T] signals, got {tuple(x.shape)} and {tuple(y.shape)}")
        return _MRSTFTFn.apply(x, y, tuple(self.resolutions), self.factor_sc, self.factor_mag)
