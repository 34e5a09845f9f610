"""GPU metrics next to the hot path (SURVEY.md section 8f rank 4).

``get_lsd(ref_sig, out_sig)`` has the call shape of reference ``src/metrics.py:59-70`` (log-spectral distance with
``STFTMag(2048, 512)``: centred reflect STFT, periodic Hann 2048, magnitude) but runs the two STFTs with
``aero_stft_fwd`` and the distance with ``aero_lsd_fwd`` on the device: no D2H copy of the waveforms and no CPU STFT
per file as in reference ``src/evaluate.py:54-97``.  (The reference's own ``STFTMag`` calls ``torch.stft`` without
``return_complex`` and raises on torch >= 2, SURVEY.md appendix C; the semantics implemented here are the intended ones.)

``get_lsd_batch(refs, ests)`` scores a whole list of files of different lengths in one fused call
(``aero_lsd_varlen_fwd``, DESIGN.md section 13): one LSD per file, each the value ``get_lsd`` gives that file on its own.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import cabi
from .spec import spectro

LSD_NFFT, LSD_HOP = 2048, 512


@torch.no_grad()
def get_lsd(ref_sig, out_sig, n_fft=LSD_NFFT, hop=LSD_HOP):
    """ref_sig, out_sig: CUDA tensors [B, T] or [T].  Returns a 0-dim CUDA tensor (fp32)."""
    if not (ref_sig.is_cuda and out_sig.is_cuda):
        raise RuntimeError("aero_b200.metrics.get_lsd: CUDA tensors only (no CPU fallback)")
    if ref_sig.shape != out_sig.shape:
        raise ValueError(f"shape mismatch {tuple(ref_sig.shape)} vs {tuple(out_sig.shape)}")
    lib = cabi.load()
    r2 = ref_sig.reshape(-1, ref_sig.shape[-1]).float()
    o2 = out_sig.reshape(-1, out_sig.shape[-1]).float()
    zr = torch.view_as_real(spectro(r2, n_fft, hop, win_length=n_fft)).contiguous()      # [B, bins, frames, 2], x n_fft^-1/2
    ze = torch.view_as_real(spectro(o2, n_fft, hop, win_length=n_fft)).contiguous()
    B, bins, frames = zr.shape[:3]
    acc = torch.zeros(1, dtype=torch.float64, device=zr.device)
    with torch.cuda.device(zr.device):
        cabi.check(lib.aero_lsd_fwd(C.c_void_p(zr.data_ptr()), C.c_void_p(ze.data_ptr()), C.c_void_p(acc.data_ptr()),
                                    B, bins, frames, n_fft, C.c_void_p(torch.cuda.current_stream().cuda_stream)), lib)
    return (acc[0] / (B * frames)).float()


def lsd_tables(lengths, row_file):
    """Host tables of aero_lsd_varlen_fwd as one int32 array [lengths | row_file | row_frame_off (rows + 1)], and the largest
    per-row frame count.  A row of L samples has 1 + L // 512 frames; the frames of row r start at row_frame_off[r]."""
    frames = [1 + int(n) // LSD_HOP for n in lengths]
    off = np.concatenate([[0], np.cumsum(frames)])
    return np.concatenate([np.asarray(lengths), np.asarray(row_file), off]).astype(np.int32), max(frames)


@torch.no_grad()
def lsd_varlen(ref, est, lengths, row_file, n_files):
    """ref, est: CUDA tensors [R, L_max]; row r holds lengths[r] valid samples (samples past it are never read) and belongs
    to file row_file[r].  Returns an fp32 CUDA tensor [n_files]: each file's LSD, the mean over all frames of all its rows.
    No host synchronisation: the tables go up in one asynchronous copy from pinned memory."""
    if not (ref.is_cuda and est.is_cuda):
        raise RuntimeError("aero_b200.metrics.lsd_varlen: CUDA tensors only (no CPU fallback)")
    if ref.dim() != 2 or ref.shape != est.shape or ref.device != est.device:
        raise ValueError(f"expected two [rows, samples] tensors on one device, got {tuple(ref.shape)} and {tuple(est.shape)}")
    R, L_max = ref.shape
    lengths, row_file = [int(n) for n in lengths], [int(f) for f in row_file]
    if len(lengths) != R or len(row_file) != R:
        raise ValueError(f"{len(lengths)} lengths and {len(row_file)} file indices for {R} rows")
    for r, n in enumerate(lengths):
        if not LSD_NFFT // 2 < n <= L_max:
            raise ValueError(f"row {r}: length {n} must exceed n_fft/2 ({LSD_NFFT // 2}) for reflect padding and be at most "
                             f"{L_max}")
    if sorted(set(row_file)) != list(range(n_files)):
        raise ValueError(f"every file in [0, {n_files}) needs at least one row and no row may name another: {row_file}")
    lib = cabi.load()
    host, max_frames = lsd_tables(lengths, row_file)
    tab = torch.from_numpy(host).pin_memory().to(ref.device, non_blocking=True)
    frame_lsd = torch.empty(int(host[-1]), dtype=torch.float32, device=ref.device)
    out = torch.empty(n_files, dtype=torch.float32, device=ref.device)
    r32, e32 = ref.float().contiguous(), est.float().contiguous()
    with torch.cuda.device(ref.device):
        cabi.check(lib.aero_lsd_varlen_fwd(C.c_void_p(r32.data_ptr()), C.c_void_p(e32.data_ptr()), R, L_max,
                                           C.c_void_p(tab.data_ptr()), C.c_void_p(tab[R:].data_ptr()),
                                           C.c_void_p(tab[2 * R:].data_ptr()), max_frames, n_files,
                                           C.c_void_p(frame_lsd.data_ptr()), C.c_void_p(out.data_ptr()),
                                           C.c_void_p(torch.cuda.current_stream().cuda_stream)), lib)
    return out


@torch.no_grad()
def get_lsd_batch(refs, ests):
    """refs, ests: lists of CUDA tensors [C, L_i] or [L_i]; reference and estimate of a file have the same shape.  Returns an
    fp32 CUDA tensor [N] whose entry i is the LSD of file i over all its channels, as ``get_lsd(refs[i], ests[i])`` (rows of
    a stereo file are scored together: the mean over the frames of both).  Files must be longer than 1024 samples."""
    refs, ests = list(refs), list(ests)
    if len(refs) != len(ests):
        raise ValueError(f"{len(refs)} references for {len(ests)} estimates")
    if not refs:
        return torch.empty(0, dtype=torch.float32, device="cuda")
    rows_r, rows_e, row_file = [], [], []
    for i, (r, e) in enumerate(zip(refs, ests)):
        if not (r.is_cuda and e.is_cuda):
            raise RuntimeError(f"aero_b200.metrics.get_lsd_batch: file {i}: CUDA tensors only (no CPU fallback)")
        if r.shape != e.shape or r.dim() not in (1, 2):
            raise ValueError(f"file {i}: expected equal shapes [C, L] or [L], got {tuple(r.shape)} vs {tuple(e.shape)}")
        if r.shape[-1] <= LSD_NFFT // 2:
            raise ValueError(f"file {i} (row {len(rows_r)}): length {r.shape[-1]} must exceed n_fft/2 ({LSD_NFFT // 2}) for "
                             "reflect padding")
        rows_r += r.reshape(-1, r.shape[-1]).unbind(0)
        rows_e += e.reshape(-1, e.shape[-1]).unbind(0)
        row_file += [i] * (r.numel() // r.shape[-1])
    pad = torch.nn.utils.rnn.pad_sequence
    ref = pad([x.float() for x in rows_r], batch_first=True)
    est = pad([x.float() for x in rows_e], batch_first=True)
    return lsd_varlen(ref, est, [x.shape[0] for x in rows_r], row_file, len(refs))
