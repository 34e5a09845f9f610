"""SEANet generator (time-domain baseline of AERO): ``aero_b200.Seanet``, a drop-in for reference ``src/models/seanet.py``.

The module tree holds the parameters only, built in the reference's order (``seanet.py:29-121``) so that for a given
``torch.manual_seed`` the 252 ``state_dict`` entries are bit-identical to the reference's and the RNG is left in the same
state (the discriminator that ``get_model`` builds next depends on it).  The forward runs on the sm_90a kernels through
``SeanetEngine``; nothing falls back to PyTorch's convolutions.

Layout: channels-last ``[B, frames, C]``.  Every activation that feeds a reflection-padded convolution is written with a halo of
``max dilation`` frames per clip by ``aero_reflect_act_fwd`` (LeakyReLU + reflection in one pass), so the convolution reads it
with no padding.  Strided convolutions and transposed convolutions run on the tap-GEMM over "super-frames": ``[B, T, C]`` viewed
as ``[B, T/r, r*C]`` (see ``superframe_conv_weight`` / ``superframe_convt_weight`` and DESIGN.md, "SEANet").
``SeanetEngine.forward_varlen`` runs clips of different lengths in one forward, each bit-identical to its own (DESIGN.md section 14).
"""
from __future__ import annotations

import ctypes as C
import math
import warnings

import torch
from torch import nn

from . import cabi
from .cabi import ACT_LEAKY, ACT_NONE, ACT_TANH
from .engine import AeroEngine, _ptr, pack_taps
from .discriminator import _DiscEngine
from .model import _record_ctor_args
from .train_engine import TrainEngine, _Conv

__all__ = ["Seanet", "SeanetEngine", "SeanetTrainEngine", "seanet_ragged_tables", "sinc_resample_table", "superframe_conv_weight",
           "superframe_convt_weight"]

_SLOPE = 0.2          # nn.LeakyReLU(0.2), seanet.py:14,58


def _wn(conv):
    # torch.nn.utils.weight_norm(dim=0), as reference modules.py:10-15 (WNConv1d / WNConvTranspose1d)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return nn.utils.weight_norm(conv)


class _ResnetBlock(nn.Module):
    # reference seanet.py:10-23 (parameter holder: block.2 = dilated k3 conv, block.4 = 1x1 conv, shortcut = 1x1 conv)
    def __init__(self, dim, dilation):
        super().__init__()
        self.block = nn.Sequential(nn.LeakyReLU(_SLOPE), nn.ReflectionPad1d(dilation),
                                   _wn(nn.Conv1d(dim, dim, kernel_size=3, dilation=dilation)),
                                   nn.LeakyReLU(_SLOPE), _wn(nn.Conv1d(dim, dim, kernel_size=1)))
        self.shortcut = _wn(nn.Conv1d(dim, dim, kernel_size=1))

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("parameter holder: compute happens in aero_b200.seanet.SeanetEngine")


def _init_conv_draw(m):
    # reference utils.py:38-44 `weights_init`: normal_ on each conv's computed `weight`.  weight_norm recomputes that tensor from
    # (g, v) on every forward, so the parameters keep their default init -- but the draws advance the RNG, in apply() post-order.
    if "Conv" in type(m).__name__:
        m.weight.data.normal_(0.0, 0.02)


def sinc_resample_table(orig_freq, new_freq, dtype=torch.float32, lowpass_filter_width=6, rolloff=0.99):
    """Polyphase filter of ``torchaudio.functional.resample`` (``sinc_interp_hann``) for the reduced ratio orig:new, computed the
    way torchaudio computes it for an input of ``dtype``.  Returns (table [new, 2*width + orig], width, orig, new)."""
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
    return kern.view(new, -1), width, orig, new


def seanet_ragged_tables(model, lengths):
    """Per-clip length tables of a ragged SEANet batch, in integer arithmetic on the host (numpy, no device): for clip b of
    lengths[b] low-rate samples, ``hr[b]`` = its high-rate length (``model.hr_length``), ``frames[i][b]`` = its frames at U-Net
    level i (``model.level_lengths``; level 0 is its valid length, ``estimate_output_length(hr[b])``) and ``out_lens[b]`` =
    min(target, valid length), the samples ``model(clip[None])`` returns.  Returns int32 arrays (hr [B], frames
    [levels + 1, B], out_lens [B])."""
    import numpy as np
    n = np.asarray([int(v) for v in lengths], np.int64)
    g = math.gcd(int(model.lr_sr), int(model.hr_sr))
    up, orig = int(model.hr_sr) // g, int(model.lr_sr) // g
    hr = (up * n + orig - 1) // orig if model.upsample else n.copy()
    t = hr.copy()
    for s in model.ratios[::-1]:                                  # encoder: strided conv, k = 2s, pad p = s//2 + s%2
        p = s // 2 + s % 2
        t = np.maximum(-((2 * s - 2 * p - t) // s) + 1, 1)        # max(ceil((t - 2s + 2p) / s) + 1, 1)
    for s in model.ratios:                                        # decoder: transposed conv, output_padding s%2
        p = s // 2 + s % 2
        t = (t - 1) * s + 2 * s - 2 * p + s % 2
    frames = [t]
    for r in model.ratios[::-1]:
        frames.append(frames[-1] // r)
    target = n * model.scale_factor if model.upsample else n
    out_lens = np.minimum(target, t)
    return hr.astype(np.int32), np.stack(frames).astype(np.int32), out_lens.astype(np.int32)


class _SeanetRagged:
    """Per-call state of a ragged SEANet batch (SeanetEngine.forward_varlen): the clips' sample lengths, high-rate lengths,
    output lengths and frames at every level as int32 device tables, uploaded from pinned memory in ONE asynchronous copy
    (no host synchronisation in the launch sequence).  ``frames_d`` maps a level's buffer frame count (the longest clip's)
    to that level's table."""

    def __init__(self, model, lengths, L_max, device):
        import numpy as np
        hr, frames, out_lens = seanet_ragged_tables(model, lengths)
        self.out_lens = [int(v) for v in out_lens]
        parts = [np.asarray(lengths, np.int32), hr, out_lens, frames.reshape(-1)]
        flat = torch.from_numpy(np.concatenate(parts))
        if torch.device(device).type == "cuda":
            flat = flat.pin_memory().to(device, non_blocking=True)
        B = len(lengths)
        self.lengths_d, self.hr_d, self.out_lens_d = flat[:B], flat[B:2 * B], flat[2 * B:3 * B]
        self.frames_d = {T: flat[(3 + i) * B:(4 + i) * B] for i, T in enumerate(model.level_lengths(L_max))}


def superframe_conv_weight(w, r):
    """Conv1d(k=2r, stride r, pad r//2 + r%2) weight [N, C, 2r] -> the 3-tap stride-1 conv (pad 1) over super-frames of r frames:
    [N, r*C, 3] with W'[n][j*C + c][d] = w[n][c][r(d-1) + j + p] (zero where that index leaves [0, 2r))."""
    n, c, k = w.shape
    p = r // 2 + r % 2
    out = w.new_zeros(n, r * c, 3)
    for d in range(3):
        for j in range(r):
            kk = r * (d - 1) + j + p
            if 0 <= kk < k:
                out[:, j * c:(j + 1) * c, d] = w[:, :, kk]
    return out


def superframe_convt_weight(w, r):
    """ConvTranspose1d(k=2r, stride r, pad r//2 + r%2, output_pad r%2) weight [Cin, Cout, 2r] -> a 3-tap stride-1 conv (pad 1)
    whose r*Cout output columns are r consecutive output frames: [r*Cout, Cin, 3] with W'[j*Cout + n][c][d] = w[c][n][r(1-d) + j + p]."""
    cin, cout, k = w.shape
    p = r // 2 + r % 2
    out = w.new_zeros(r * cout, cin, 3)
    for d in range(3):
        for j in range(r):
            kk = r * (1 - d) + j + p
            if 0 <= kk < k:
                out[j * cout:(j + 1) * cout, :, d] = w[:, :, kk].t()
    return out


def superframe_conv_weight_adjoint(g, r, k):
    """Adjoint of superframe_conv_weight: [N, r*C, 3] -> [N, C, k].  Every original weight appears once: a gather."""
    n, rc, _ = g.shape
    c, p = rc // r, r // 2 + r % 2
    out = g.new_zeros(n, c, k)
    for d in range(3):
        for j in range(r):
            kk = r * (d - 1) + j + p
            if 0 <= kk < k:
                out[:, :, kk] = g[:, j * c:(j + 1) * c, d]
    return out


def superframe_convt_weight_adjoint(g, r, k):
    """Adjoint of superframe_convt_weight: [r*Cout, Cin, 3] -> [Cin, Cout, k] (a gather)."""
    rco, cin, _ = g.shape
    cout, p = rco // r, r // 2 + r % 2
    out = g.new_zeros(cin, cout, k)
    for d in range(3):
        for j in range(r):
            kk = r * (1 - d) + j + p
            if 0 <= kk < k:
                out[:, :, kk] = g[j * cout:(j + 1) * cout, :, d].t()
    return out


class Seanet(nn.Module):
    """SEANet generator on the sm_90a kernels.  Constructor arguments and defaults follow reference ``seanet.py:29-40``
    (``resample`` is accepted and unused there too)."""

    @_record_ctor_args
    def __init__(self, latent_space_size=128, ngf=32, n_residual_layers=3, resample=1, normalize=True, floor=1e-3,
                 ratios=[8, 8, 2, 2], in_channels=1, out_channels=1, lr_sr=16000, hr_sr=16000, upsample=True):
        super().__init__()
        if int(hr_sr) % int(lr_sr) or hr_sr < lr_sr:
            raise NotImplementedError(f"aero_b200.Seanet: rate ratio {lr_sr} -> {hr_sr} is not an integer up-sampling")
        if any(int(r) < 2 for r in ratios) or n_residual_layers < 1:
            raise NotImplementedError("aero_b200.Seanet: ratios must be >= 2 and n_residual_layers >= 1")
        if ngf % 4 or latent_space_size % 4:
            # channels-last passes (reflection halo, activations) move 4 channels at a time
            raise NotImplementedError("aero_b200.Seanet: ngf and latent_space_size must be multiples of 4")
        if in_channels != out_channels or not 1 <= out_channels <= 8:
            # the output adds the input signal (seanet.py:173-176): the reference needs equal channel counts too
            raise NotImplementedError("aero_b200.Seanet: in_channels == out_channels <= 8")
        self.resample, self.normalize, self.floor = resample, normalize, floor
        self.lr_sr, self.hr_sr = lr_sr, hr_sr
        self.scale_factor = int(hr_sr / lr_sr)
        self.upsample = upsample
        self.ratios = list(ratios)
        self.ngf, self.latent_space_size, self.n_residual_layers = ngf, latent_space_size, n_residual_layers
        self.in_channels, self.out_channels = in_channels, out_channels

        self.encoder = nn.ModuleList()
        self.decoder = nn.ModuleList()
        mult = 2 ** len(ratios)
        # construction order = RNG order of the reference (seanet.py:57-119)
        dec_in = nn.Sequential(nn.LeakyReLU(_SLOPE), nn.ReflectionPad1d(3),
                               _wn(nn.Conv1d(latent_space_size, mult * ngf, kernel_size=7, padding=0)))
        enc_out = nn.Sequential(nn.LeakyReLU(_SLOPE), nn.ReflectionPad1d(3),
                                _wn(nn.Conv1d(mult * ngf, latent_space_size, kernel_size=7, padding=0)))
        self.encoder.insert(0, enc_out)
        self.decoder.append(dec_in)
        for r in ratios:
            c = mult * ngf // 2
            enc = [nn.LeakyReLU(_SLOPE), _wn(nn.Conv1d(c, 2 * c, kernel_size=2 * r, stride=r, padding=r // 2 + r % 2))]
            dec = [nn.LeakyReLU(_SLOPE), _wn(nn.ConvTranspose1d(2 * c, c, kernel_size=2 * r, stride=r, padding=r // 2 + r % 2,
                                                                output_padding=r % 2))]
            for j in range(n_residual_layers - 1, -1, -1):
                enc = [_ResnetBlock(c, 3 ** j)] + enc
            for j in range(n_residual_layers):
                dec = dec + [_ResnetBlock(c, 3 ** j)]
            mult //= 2
            self.encoder.insert(0, nn.Sequential(*enc))
            self.decoder.append(nn.Sequential(*dec))
        self.encoder.insert(0, nn.Sequential(nn.ReflectionPad1d(3), _wn(nn.Conv1d(in_channels, ngf, kernel_size=7, padding=0)),
                                             nn.Tanh()))
        self.decoder.append(nn.Sequential(nn.LeakyReLU(_SLOPE), nn.ReflectionPad1d(3),
                                          _wn(nn.Conv1d(ngf, out_channels, kernel_size=7, padding=0)), nn.Tanh()))
        self.apply(_init_conv_draw)
        self._engine_obj = None
        # training arithmetic of the convolution GEMMs, as aero_b200.Aero: 0 exact fp32, 1 TF32, 3 "3xTF32" on the tensor cores
        self.train_precision = 0

    # ------------------------------------------------------------------ geometry (reference seanet.py:123-151)
    def estimate_output_length(self, length):
        depth = len(self.ratios)
        for idx in range(depth - 1, -1, -1):
            s = self.ratios[idx]
            length = max(math.ceil((length - 2 * s + 2 * (s // 2 + s % 2)) / s) + 1, 1)
        for idx in range(depth):
            s = self.ratios[idx]
            length = (length - 1) * s + 2 * s - 2 * (s // 2 + s % 2) + s % 2
        return int(length)

    def pad_to_valid_length(self, signal):
        valid = self.estimate_output_length(signal.shape[-1])
        pad = valid - signal.shape[-1]
        return torch.nn.functional.pad(signal, (0, pad)), pad

    def hr_length(self, length):
        """High-rate length of a low-rate input of `length` samples (torchaudio's ceil(new * L / orig); L without upsample)."""
        if not self.upsample:
            return length
        g = math.gcd(int(self.lr_sr), int(self.hr_sr))
        return math.ceil((int(self.hr_sr) // g) * length / (int(self.lr_sr) // g))

    def level_lengths(self, length):
        """Frames at every U-Net level for a low-rate input of `length` samples: [L_valid, L_valid/r_1, ...]
        (encoder level i down-samples by ratios[-i])."""
        t = [self.estimate_output_length(self.hr_length(length))]
        for r in self.ratios[::-1]:
            t.append(t[-1] // r)
        return t

    def check_length(self, length):
        """ValueError where the reference's reflection pads would fail (a pad must be shorter than the frames it mirrors)."""
        t = self.level_lengths(length)
        dil = 3 ** (self.n_residual_layers - 1)
        if min(t[:-1]) <= dil or t[-1] <= 3:
            raise ValueError(f"aero_b200.Seanet: input of {length} samples is too short: level lengths {t} do not admit "
                             f"reflection pads of {dil} (residual blocks) and 3 (bottleneck)")

    # ------------------------------------------------------------------ engine plumbing (as aero_b200.Aero)
    def _engine(self):
        if self._engine_obj is None:
            object.__setattr__(self, "_engine_obj", SeanetEngine(self))
        return self._engine_obj

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        if self._engine_obj is not None:
            self._engine_obj.invalidate()
        return out

    def load_state_dict(self, *a, **k):
        out = super().load_state_dict(*a, **k)
        if self._engine_obj is not None:
            self._engine_obj.invalidate()
        return out

    def use_cuda_graph(self, enabled=True):
        """Replay each forward from a CUDA graph captured per input shape (inference; same kernels, same results).
        ``"auto"`` (the default) captures a shape the third time it is seen, ``True`` on first sight, ``False`` never."""
        self._engine().use_graph = "auto" if enabled == "auto" else bool(enabled)
        return self

    def forward(self, signal):
        """signal [B, in_channels, L] (low rate when ``upsample``) -> [B, out_channels, L * scale_factor] (reference seanet.py:153-179).
        In training mode the forward and its backward run on the CUDA kernels behind one autograd node (SeanetTrainEngine); the
        input is data (the reference never differentiates it), so it receives no gradient."""
        if self.training:
            names = [n for n, p in self.named_parameters() if p.requires_grad]
            return _SeanetTrainFn.apply(signal, self, names, *[p for _, p in self.named_parameters() if p.requires_grad])
        return self._engine().forward(signal)


class SeanetEngine(AeroEngine):
    """Launch sequence of the SEANet forward.  Shares AeroEngine's plumbing: workspace shape sets, CUDA-graph replay, device
    handling, weight-version tracking, precision modes (2: FP16 storage / f16 wgmma, 1: TF32, 0: exact fp32 SIMT)."""

    def __init__(self, model):
        self._init_state(model, cabi.load())
        self._filters = {}

    def _check_mode(self):
        if self.model.training:
            raise NotImplementedError("aero_b200.Seanet: the CUDA path implements the inference forward; call model.eval()")

    @property
    def halo(self):
        return max(3 ** (self.model.n_residual_layers - 1), 3)

    # ------------------------------------------------------------------ weights
    @torch.no_grad()
    def _pack(self):
        m = self.model
        dev = self._device()
        W = {}

        def wn(conv):
            return torch._weight_norm(conv.weight_v.detach(), conv.weight_g.detach(), 0)

        def plain(key, conv):
            W[key + ".w"], W[key + ".b"] = pack_taps(wn(conv)), conv.bias.detach().clone()

        def resblock(key, blk):
            plain(key + ".c3", blk.block[2])
            w1, ws = wn(blk.block[4]), wn(blk.shortcut)          # [C, C, 1] each: one GEMM over [h | x]
            W[key + ".c1.w"] = pack_taps(torch.cat([w1, ws], 1))
            W[key + ".c1.b"] = (blk.block[4].bias + blk.shortcut.bias).detach().clone()

        nlev = len(m.ratios)
        plain("enc0", m.encoder[0][1])
        for i in range(1, nlev + 1):
            seq = m.encoder[i]
            r = m.ratios[nlev - i]
            for k in range(m.n_residual_layers):
                resblock(f"enc{i}.rb{k}", seq[k])
            conv = seq[m.n_residual_layers + 1]
            W[f"enc{i}.down.w"] = pack_taps(superframe_conv_weight(wn(conv), r))
            W[f"enc{i}.down.b"] = conv.bias.detach().clone()
        plain(f"enc{nlev + 1}", m.encoder[nlev + 1][2])
        plain("dec0", m.decoder[0][2])
        for j in range(1, nlev + 1):
            seq = m.decoder[j]
            r = m.ratios[j - 1]
            ct = seq[1]
            W[f"dec{j}.up.w"] = pack_taps(superframe_convt_weight(wn(ct), r))
            W[f"dec{j}.up.b"] = ct.bias.detach().repeat(r)
            for k in range(m.n_residual_layers):
                resblock(f"dec{j}.rb{k}", seq[2 + k])
        plain(f"dec{nlev + 1}", m.decoder[nlev + 1][2])
        out = {k: v.to(device=dev, dtype=torch.float32).contiguous() for k, v in W.items()}
        self._wk, self._wh, self._wname = {}, {}, {}
        return self._add_tc_twins(out)

    def _filter(self):
        m = self.model
        key = self._device()
        f = self._filters.get(key)
        if f is None:
            table, width, orig, up = sinc_resample_table(m.lr_sr, m.hr_sr, torch.float32)
            f = self._filters[key] = (table.contiguous().to(key), width, orig, up)
        return f

    # ------------------------------------------------------------------ kernel wrappers
    def _reflect_act(self, x, y, *, B, T, C, x_sb, y_sb, halo, act=ACT_LEAKY):
        """y (pointing at frame 0 of a halo'd buffer) = act(x) with `halo` reflected frames on both sides.  In a ragged batch
        each clip is reflected at its own end and followed by zeros (aero_reflect_act_varlen_fwd with the level's frame table)."""
        flags = (cabi.TG_A_F16 if x.dtype == torch.float16 else 0) | (cabi.TG_OUT_F16 if y.dtype == torch.float16 else 0) | \
                (cabi.TG_ROUND_TF32 if self.precision >= 1 else 0)
        if self._vl is not None:
            rc = self.lib.aero_reflect_act_varlen_fwd(_ptr(x), _ptr(y), _ptr(self._vl.frames_d[T]), B, T, C, x_sb, y_sb, halo, act,
                                                      flags, self._stream())
        else:
            rc = self.lib.aero_reflect_act_fwd(_ptr(x), _ptr(y), B, T, C, x_sb, y_sb, halo, act, flags, self._stream())
        cabi.check(rc, self.lib)

    def _halo_buf(self, name, B, T, C):
        """[B, T + 2*halo, C] activation buffer (zero-filled once: halo frames a pass does not write stay finite)."""
        return self._buf(name, B, T + 2 * self.halo, C, dtype=self._adt(C), zero=True)

    def _resblock(self, x, out, W, key, B, T, C, dil, residual=None):
        """reference seanet.py:22-23: out = shortcut(x) + conv1x1(lrelu(conv_k3,d(reflpad_d(lrelu(x))))) (+ residual)."""
        H = self.halo
        h0 = self._halo_buf(f"h0.{T}.{C}", B, T, C)
        row = (T + 2 * H) * C
        self._reflect_act(x, h0[:, H:], B=B, T=T, C=C, x_sb=T * C, y_sb=row, halo=dil)
        h1 = self._buf(f"h1.{T}.{C}", B, T, C, dtype=self._adt(C))
        self._gemm(h1, W[key + ".c3.w"], a1=h0[:, H - dil:], B=B, F_out=1, T=T, T_in=T + 2 * dil, N=C, C1=C, kt=3, dil_t=dil,
                   a1_s=(row, 0, C), bias=W[key + ".c3.b"], act=ACT_LEAKY, rnd=True)
        self._gemm(out, W[key + ".c1.w"], a1=h1, a2=x, B=B, F_out=1, T=T, N=C, C1=C, C2=C, bias=W[key + ".c1.b"],
                   residual=residual, rnd=True)
        return out

    def _k7(self, x, out, W, key, B, T, C, N, act, residual=None, r_s=None, samp_affine=None, rnd=True):
        """LeakyReLU, ReflectionPad1d(3), WNConv1d(k=7) (+ act, + residual, x samp_affine)."""
        H = self.halo
        h0 = self._halo_buf(f"h0.{T}.{C}", B, T, C)
        row = (T + 2 * H) * C
        self._reflect_act(x, h0[:, H:], B=B, T=T, C=C, x_sb=T * C, y_sb=row, halo=3)
        return self._gemm(out, W[key + ".w"], a1=h0[:, H - 3:], B=B, F_out=1, T=T, T_in=T + 6, N=N, C1=C, kt=7,
                          a1_s=(row, 0, C), bias=W[key + ".b"], act=act, residual=residual, r_s=r_s,
                          samp_affine=samp_affine, rnd=rnd)

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward_varlen(self, signal, lengths):
        """Ragged batch: clip b is signal[b, :, :lengths[b]] (samples past it are never read) and comes out as
        forward(signal[b:b+1, :, :lengths[b]]) gives it.  Returns the padded waveform [B, C_out, max out_len], zero past each
        clip's own output length, and the list of those lengths.  Runs eagerly (no CUDA graph); its workspaces are released
        when it returns."""
        self._require(signal)
        self._check_mode()
        m = self.model
        if signal.dim() != 3 or signal.shape[1] != m.in_channels:
            raise ValueError(f"expected input [B, {m.in_channels}, L], got {tuple(signal.shape)}")
        lengths = [int(n) for n in lengths]
        if len(lengths) != signal.shape[0]:
            raise ValueError(f"{len(lengths)} lengths for a batch of {signal.shape[0]}")
        if not lengths:
            return self._forward(signal), []
        L = signal.shape[2]
        for b, n in enumerate(lengths):
            if not 1 <= n <= L:
                raise ValueError(f"clip {b}: length {n} outside [1, {L}]")
            try:
                m.check_length(n)
            except ValueError as e:
                raise ValueError(f"clip {b} of {n} samples: {e}") from None
        with self._on_device():
            self._vl = _SeanetRagged(m, lengths, L, signal.device)
            try:
                y = self._forward(signal)
                out_lens = self._vl.out_lens
            finally:
                self._vl = None
                # keyed on the batch's exact longest clip, which rarely repeats in an evaluation loop: release, as AERO does
                self._bufsets.pop((tuple(signal.shape), self.precision, "varlen"), None)
                self._bufs = {}
        return y[:, :, :max(out_lens)], out_lens

    @torch.no_grad()
    def _forward(self, signal, return_spec=False, return_lr_spec=False):
        self._require(signal)
        self._check_mode()
        m = self.model
        if signal.dim() != 3 or signal.shape[1] != m.in_channels:
            raise ValueError(f"expected input [B, {m.in_channels}, L], got {tuple(signal.shape)}")
        B, Cin, L = signal.shape
        target = L * m.scale_factor if m.upsample else L
        if B == 0:
            # clips are independent: an empty batch maps to an empty batch, nothing to launch
            return signal.new_zeros(0, m.out_channels, target)
        m.check_length(L)
        W = self._weights()
        vl = self._vl                   # _SeanetRagged while forward_varlen runs
        self._select_shape_set((tuple(signal.shape), self.precision) + (() if vl is None else ("varlen",)))
        H = self.halo
        lev = m.level_lengths(L)
        Lv, L_hr = lev[0], m.hr_length(L)
        nlev = len(m.ratios)

        # input stage: std, normalise, resample, zero pad, reflection halo (x0 stays fp32: enc0 and the output skip read it)
        x0 = self._buf("x0", B, Lv + 2 * H, Cin, zero=True)
        affine = self._buf("affine", B, 2)
        if m.upsample:
            filt, width, orig, up = self._filter()
            taps = filt.shape[1]
        else:
            filt, width, orig, up, taps = None, 0, 1, 0, 0
        p = cabi.ResampleParams(B, Cin, L, orig, up, width, taps, L_hr, Lv, H, 3, 1 if m.normalize else 0, float(m.floor))
        if vl is None:
            rc = self.lib.aero_seanet_input_fwd(_ptr(signal.contiguous()), _ptr(filt), _ptr(affine), _ptr(x0), C.byref(p),
                                                self._stream())
        else:
            rc = self.lib.aero_seanet_input_varlen_fwd(_ptr(signal.contiguous()), _ptr(filt), _ptr(affine), _ptr(x0),
                                                       _ptr(vl.lengths_d), _ptr(vl.hr_d), _ptr(vl.frames_d[Lv]), C.byref(p),
                                                       self._stream())
        cabi.check(rc, self.lib)
        row0 = (Lv + 2 * H) * Cin

        # enc0: ReflectionPad1d(3), WNConv1d(k7, Cin -> ngf), Tanh   (the halo of x0 is the reflection)
        c = m.ngf
        skips = [self._buf("s0", B, Lv, c, dtype=self._adt(c))]
        self._gemm(skips[0], W["enc0.w"], a1=x0[:, H - 3:], B=B, F_out=1, T=Lv, T_in=Lv + 6, N=c, C1=Cin, kt=7,
                   a1_s=(row0, 0, Cin), bias=W["enc0.b"], act=ACT_TANH, rnd=True)
        # encoder levels: residual blocks at T, LeakyReLU, strided conv as a 3-tap conv over super-frames of r frames
        for i in range(1, nlev + 1):
            T, r = lev[i - 1], m.ratios[nlev - i]
            x = skips[-1]
            for k in range(m.n_residual_layers):
                x = self._resblock(x, self._buf(f"rb{k % 2}.{T}.{c}", B, T, c, dtype=self._adt(c)), W, f"enc{i}.rb{k}", B, T, c,
                                   3 ** k)
            h0 = self._halo_buf(f"h0.{T}.{c}", B, T, c)
            row = (T + 2 * H) * c
            self._reflect_act(x, h0[:, H:], B=B, T=T, C=c, x_sb=T * c, y_sb=row, halo=0)
            y = self._buf(f"s{i}", B, T // r, 2 * c, dtype=self._adt(2 * c))
            self._gemm(y, W[f"enc{i}.down.w"], a1=h0[:, H:], B=B, F_out=1, T=T // r, N=2 * c, C1=r * c, kt=3, pad_t=1,
                       a1_s=(row, 0, r * c), bias=W[f"enc{i}.down.b"], rnd=True)
            skips.append(y)
            c *= 2
        T = lev[nlev]
        lat = m.latent_space_size
        z = self._buf("z", B, T, lat, dtype=self._adt(lat))
        self._k7(skips[-1], z, W, f"enc{nlev + 1}", B, T, c, lat, ACT_NONE)
        d = self._buf("d0", B, T, c, dtype=self._adt(c))
        self._k7(z, d, W, "dec0", B, T, lat, c, ACT_NONE, residual=skips[-1])
        # decoder levels: LeakyReLU, transposed conv as a 3-tap conv with r*C/2 output columns (= r frames), residual blocks,
        # + the skip (the input of the mirrored encoder level) in the last block's epilogue
        for j in range(1, nlev + 1):
            r = m.ratios[j - 1]
            co = c // 2
            h0 = self._halo_buf(f"h0.{T}.{c}", B, T, c)
            row = (T + 2 * H) * c
            self._reflect_act(d, h0[:, H:], B=B, T=T, C=c, x_sb=T * c, y_sb=row, halo=0)
            To = T * r
            x = self._buf(f"up.{To}.{co}", B, To, co, dtype=self._adt(co))
            self._gemm(x, W[f"dec{j}.up.w"], a1=h0[:, H:], B=B, F_out=1, T=T, N=r * co, C1=c, kt=3, pad_t=1,
                       a1_s=(row, 0, c), o_s=(To * co, 0, r * co), bias=W[f"dec{j}.up.b"], rnd=True)
            skip = skips[nlev - j]
            for k in range(m.n_residual_layers):
                last = k == m.n_residual_layers - 1
                out = self._buf(f"d{j}" if last else f"rb{k % 2}.{To}.{co}", B, To, co, dtype=self._adt(co))
                x = self._resblock(x, out, W, f"dec{j}.rb{k}", B, To, co, 3 ** k, residual=skip if last else None)
            d, T, c = x, To, co
        # dec5: LeakyReLU, ReflectionPad1d(3), WNConv1d(k7, ngf -> Cout), Tanh, + x0, x std (fp32, exact thin kernel)
        Cout = m.out_channels
        y = self._buf("y", B, Lv, Cout)
        self._k7(d, y, W, f"dec{nlev + 1}", B, Lv, c, Cout, ACT_TANH, residual=x0[:, H:],
                 r_s=(row0, 0, Cin), samp_affine=affine, rnd=False)
        if vl is not None:
            # each clip's samples past its own output length (computed from the zero padding) read as zeros
            cabi.check(self.lib.aero_frame_mask_fwd(_ptr(y), _ptr(vl.out_lens_d), B, 1, Lv, Cout, 0, self._stream()), self.lib)
        return y[:, :min(target, Lv)].permute(0, 2, 1).contiguous()


class SeanetTrainEngine(TrainEngine):
    """Training forward / backward of SEANet on the tape machinery of aero_b200.train_engine (fp32 activations; the convolution GEMMs in
    ``train_precision`` 0, 1 or 3).  Weight norm runs on aero_weight_norm_fwd / _bwd and the super-frame repack is a derived weight
    (``w_override``) whose backward gathers the gradient back onto the original taps.  Reflection padding writes an explicit padded
    tensor (aero_reflect_act_fwd) whose adjoint folds the halo's gradient back (aero_reflect_act_bwd)."""

    wn_weight = _DiscEngine.wn_weight

    def __init__(self, model):
        self.model = model
        self.geom = None
        self.lib = cabi.load()
        self.precision = int(getattr(model, "train_precision", 0))
        self._reset()

    def _wn(self, prefix):
        v = self.params[prefix + ".weight_v"]
        return self.wn_weight(prefix, v.shape[0], v[0].numel())

    def reflect_act(self, x, B, T, C_, halo, act=ACT_LEAKY):
        """y = act(x) reflection-padded by `halo` frames: a contiguous [B, T + 2 halo, C] tensor."""
        Tp = T + 2 * halo
        y = self._new(B * Tp * C_)
        yv = y.view(B, Tp, C_)[:, halo:]
        self._check(self.lib.aero_reflect_act_fwd(_ptr(x), _ptr(yv), B, T, C_, T * C_, Tp * C_, halo, act, 0, self._stream()))

        def bwd():
            dy = self.grad(y)
            if dy is None:
                return
            dx = self._new(B * T * C_)
            self._check(self.lib.aero_reflect_act_bwd(_ptr(x), _ptr(dy.view(B, Tp, C_)[:, halo:]), _ptr(dx), B, T, C_, T * C_, Tp * C_,
                                                      halo, act, self._stream()))
            self.acc(x, dx)
        self.tape.append(bwd)
        self.keep.append((x, y))
        return y

    def resblock(self, x, key, B, T, C_, dil, residual=None):
        """reference seanet.py:22-23; the shortcut and the 1x1 conv are one two-source GEMM over [h | x] (+ the decoder skip)."""
        xp = self.reflect_act(x, B, T, C_, dil)
        h = self.conv(xp, None, C_, 0, None, key + ".block.2.bias", _Conv(kt=3, dil_t=dil), B, 1, 1, T, C_,
                      w_override=self._wn(key + ".block.2"), T_in=T + 2 * dil)
        h = self.norm_act(h, cabi.NA_LEAKY, B=B, F_in=1, T=T, C_=C_, scope=1, no_norm=True)
        (w1, back1), (ws, backs) = self._wn(key + ".block.4"), self._wn(key + ".shortcut")
        b1n, bsn = key + ".block.4.bias", key + ".shortcut.bias"

        def w_back(gw):
            gw = gw.reshape(C_, 2 * C_, 1)
            back1(gw[:, :C_].contiguous())
            backs(gw[:, C_:].contiguous())

        def b_back(gb):
            self.pgrad(b1n).add_(gb)
            self.pgrad(bsn).add_(gb)
        return self.conv(h, x, C_, C_, None, None, _Conv(), B, 1, 1, T, C_, residual=residual,
                         w_override=(torch.cat([w1, ws], 1), w_back), b_override=(self.params[b1n] + self.params[bsn], b_back))

    def k7(self, x, key, B, T, C_, N, residual=None):
        """LeakyReLU, ReflectionPad1d(3), WNConv1d(k=7)."""
        xp = self.reflect_act(x, B, T, C_, 3)
        return self.conv(xp, None, C_, 0, None, key + ".bias", _Conv(kt=7), B, 1, 1, T, N, w_override=self._wn(key), T_in=T + 6,
                         residual=residual)

    def _input(self, signal, halo):
        """aero_seanet_input_fwd into [B, L_valid + 2 halo, C]: the normalised, resampled, zero-padded input with `halo` reflected frames."""
        m = self.model
        B, Cin, L = signal.shape
        Lv = m.level_lengths(L)[0]
        out = self._new(B, Lv + 2 * halo, Cin)
        if m.upsample:
            filt, width, orig, up = sinc_resample_table(m.lr_sr, m.hr_sr, torch.float32)
            filt, taps = filt.contiguous().to(self._device()), filt.shape[1]
        else:
            filt, width, orig, up, taps = None, 0, 1, 0, 0
        p = cabi.ResampleParams(B, Cin, L, orig, up, width, taps, m.hr_length(L), Lv, halo, halo, 1 if m.normalize else 0, float(m.floor))
        self._check(self.lib.aero_seanet_input_fwd(_ptr(signal), _ptr(filt), _ptr(self._affine), _ptr(out), C.byref(p), self._stream()))
        self.keep.append(filt)
        return out.view(-1)

    @torch.no_grad()
    def forward(self, signal):
        """signal [B, C, L] fp32 -> [B, C, L * scale_factor]; records the tape."""
        self._reset()
        self._sync_stream()
        m = self.model
        if signal.dim() != 3 or signal.shape[1] != m.in_channels or signal.dtype != torch.float32:
            raise ValueError(f"expected fp32 input [B, {m.in_channels}, L], got {tuple(signal.shape)} {signal.dtype}")
        B, Cin, L = signal.shape
        m.check_length(L)
        self.params = {k: v.detach() for k, v in m.named_parameters()}
        signal = signal.contiguous()
        lev = m.level_lengths(L)
        Lv, nlev, nres = lev[0], len(m.ratios), m.n_residual_layers
        self._affine = self._new(B, 2)
        xp = self._input(signal, 3)                     # reflect-padded x0 for encoder 0
        x0 = self._input(signal, 0)                     # x0 itself for the output skip
        self.no_grad.update((id(xp), id(x0)))
        c = m.ngf
        h = self.conv(xp, None, Cin, 0, None, "encoder.0.1.bias", _Conv(kt=7), B, 1, 1, Lv, c, w_override=self._wn("encoder.0.1"),
                      T_in=Lv + 6)
        h = self.norm_act(h, cabi.NA_TANH, B=B, F_in=1, T=Lv, C_=c, scope=1, no_norm=True)
        self.marks.append((len(self.tape), "encoder.0"))
        skips = [h]
        for i in range(1, nlev + 1):
            T, r = lev[i - 1], m.ratios[nlev - i]
            x = skips[-1]
            for k in range(nres):
                x = self.resblock(x, f"encoder.{i}.{k}", B, T, c, 3 ** k)
            key = f"encoder.{i}.{nres + 1}"
            hx = self.reflect_act(x, B, T, c, 0)
            w, back = self._wn(key)
            wp = superframe_conv_weight(w, r)
            y = self.conv(hx, None, r * c, 0, None, key + ".bias", _Conv(kt=3, pad_t=1), B, 1, 1, T // r, 2 * c,
                          w_override=(wp, lambda g, back=back, r=r, k=w.shape[2], shp=wp.shape: back(superframe_conv_weight_adjoint(
                              g.reshape(shp), r, k).contiguous())))
            skips.append(y)
            self.marks.append((len(self.tape), f"encoder.{i}"))
            c *= 2
        T = lev[nlev]
        z = self.k7(skips[-1], f"encoder.{nlev + 1}.2", B, T, c, m.latent_space_size)
        self.marks.append((len(self.tape), f"encoder.{nlev + 1}"))
        d = self.k7(z, "decoder.0.2", B, T, m.latent_space_size, c, residual=skips[-1])
        self.marks.append((len(self.tape), "decoder.0"))
        for j in range(1, nlev + 1):
            r, co = m.ratios[j - 1], c // 2
            key = f"decoder.{j}.1"
            hx = self.reflect_act(d, B, T, c, 0)
            w, back = self._wn(key)
            wp = superframe_convt_weight(w, r)
            bn = key + ".bias"
            x = self.conv(hx, None, c, 0, None, None, _Conv(kt=3, pad_t=1), B, 1, 1, T, r * co,
                          w_override=(wp, lambda g, back=back, r=r, k=w.shape[2], shp=wp.shape: back(superframe_convt_weight_adjoint(
                              g.reshape(shp), r, k).contiguous())),
                          b_override=(self.params[bn].repeat(r), lambda gb, bn=bn, r=r, co=co: self.pgrad(bn).add_(gb.view(r, co).sum(0))))
            T, c = T * r, co
            skip = skips[nlev - j]
            for k in range(nres):
                x = self.resblock(x, f"decoder.{j}.{2 + k}", B, T, c, 3 ** k, residual=skip if k == nres - 1 else None)
            d = x
            self.marks.append((len(self.tape), f"decoder.{j}"))
        v = self.k7(d, f"decoder.{nlev + 1}.2", B, Lv, c, m.out_channels)
        self.marks.append((len(self.tape), f"decoder.{nlev + 1}"))
        out = self._new(B * Lv * m.out_channels)
        n = Lv * m.out_channels
        self._check(self.lib.aero_seanet_output_fwd(_ptr(v), _ptr(x0), _ptr(self._affine), _ptr(out), B, n, self._stream()))

        def out_bwd():
            dy = self.grad(out)
            if dy is None:
                return
            dv = self._new(B * n)
            self._check(self.lib.aero_seanet_output_bwd(_ptr(v), _ptr(self._affine), _ptr(dy), _ptr(dv), B, n, self._stream()))
            self.acc(v, dv)
        self.tape.append(out_bwd)
        self.keep.append((v, out))
        self._out, self._shape = out, (B, Lv, m.out_channels)
        target = min(L * m.scale_factor if m.upsample else L, Lv)
        self._target = target
        return out.view(B, Lv, m.out_channels)[:, :target].permute(0, 2, 1).contiguous()

    @torch.no_grad()
    def backward(self, d_out, grad_sink=None, on_layer_done=None):
        """d_out [B, C, target] -> {parameter name: gradient}.  grad_sink(name) -> zeroed tensor to accumulate that parameter's gradient
        into (else fresh tensors); on_layer_done(tag) is called when every gradient of top-level module `tag` ("decoder.5", ...,
        "decoder.0", "encoder.5", ..., "encoder.0") is final (as TrainEngine.backward)."""
        self._sync_stream()
        self._sink = grad_sink
        B, Lv, Co = self._shape
        g = torch.zeros(B, Lv, Co, dtype=torch.float32, device=d_out.device)
        g[:, :self._target] = d_out.permute(0, 2, 1)
        self.acc(self._out, g.view(-1))
        starts, prev = {}, 0
        for end, tag in self.marks:                       # module `tag` owns tape[prev:end]; it is done once tape[prev] has run
            starts[prev] = tag
            prev = end
        for i in range(len(self.tape) - 1, -1, -1):
            self.tape[i]()
            if on_layer_done is not None and i in starts:
                on_layer_done(starts[i])
        pg = self.pg
        self._reset()
        return pg


class _SeanetTrainFn(torch.autograd.Function):
    """forward = SeanetTrainEngine.forward (records a tape), backward = SeanetTrainEngine.backward (parameter gradients; the input is
    data and gets None)."""

    @staticmethod
    def forward(ctx, signal, model, names, *params):
        if not signal.is_cuda or next(model.parameters()).device != signal.device:
            raise RuntimeError("aero_b200.Seanet trains on CUDA only (sm_90a kernels in libaero_b200.so); there is no CPU path")
        with torch.cuda.device(signal.device):
            eng = SeanetTrainEngine(model)
            out = eng.forward(signal.detach())
        ctx.eng, ctx.names, ctx.dev = eng, names, signal.device
        ctx.set_materialize_grads(False)
        return out

    @staticmethod
    def backward(ctx, d_out):
        if d_out is None:
            return (None, None, None, *[None] * len(ctx.names))
        with torch.cuda.device(ctx.dev):
            grads = ctx.eng.backward(d_out.contiguous())
        ctx.eng = None
        return (None, None, None, *[grads.get(n) for n in ctx.names])
