"""HiFi-GAN multi-period discriminator on the CUDA kernels: drop-ins for reference ``src/models/discriminators.py:89-147``
(``DiscriminatorP``, ``MultiPeriodDiscriminator``, the ``mpd`` adversary of ``discriminator_models``).

Same constructor arguments, the same ``state_dict`` keys in the same order (``discriminators.i.convs.j.{bias, weight_g, weight_v}``,
then ``conv_post``: weight-normalised ``Conv2d`` with PyTorch's default initialisation, constructed in the reference's order so that
one seed gives bit-identical parameters), and the same return value ``(y_d_rs, y_d_gs, fmap_rs, fmap_gs)``.

Each period is one ``torch.autograd.Function`` whose forward and backward run on libaero_b200.so through the tape machinery of
``aero_b200.train_engine`` (weight norm on ``aero_weight_norm_*``, convolutions on the tap-GEMM in ``train_precision`` 0 or 1).
Layout (DESIGN.md, "Multi-period discriminator"): the ``[B, 1, H, p]`` view of a period turns into ``B*p`` independent sequences of
H frames.  They are stored back to back as one long channels-last sequence of segments ``[zero halo | H frames | zero tail]``
(``period_layout``), so every tap-GEMM runs over all of them at once with full 128-row tiles.  The four stride-3 layers are 2-tap
convolutions over super-frames of 3 frames (``superframe_weight``).  ``aero_mpd_fold_*`` (reflect pad + fold) and
``aero_mpd_repack_*`` (LeakyReLU(0.1) + the next layer's segment layout) move data between them.  Feature maps are returned as
``[B, C, H, p]`` views of that storage.
"""
from __future__ import annotations

import torch
from torch import nn

from .discriminator import _DiscEngine
from .model import _record_ctor_args
from .seanet import _wn
from .train_engine import _Conv, _ptr

__all__ = ["DiscriminatorP", "MultiPeriodDiscriminator", "period_flops", "period_layout", "segment_view", "superframe_weight",
           "superframe_weight_adjoint"]

_SLOPE = 0.1          # LRELU_SLOPE, discriminators.py:82
_K = 5                # kernel (5, 1) of the five convolutions
_HALO = 2             # their padding (2, 0)


def period_layout(T, period):
    """Segment geometry of one DiscriminatorP on a T-sample input, as (H, seg, halo) per stored tensor: the folded input, the five
    feature maps and the logits.  Segment s = b*period + w of a tensor holds frame h at row s*seg + halo + h; every other row is zero
    (the logits' other rows hold values no output owns).  A stride-3 layer's input has seg = 3*(H_out + 1) rows: H_out + 1 super-frames,
    of which output row o reads o and o + 1."""
    hs = [-(-T // period)]
    for _ in range(4):
        hs.append(-(-hs[-1] // 3))
    lay = [(hs[i], 3 * (hs[i + 1] + 1), _HALO) for i in range(4)]
    lay.append((hs[4], hs[4] + 2 * _HALO, _HALO))      # input of the stride-1 k5 layer
    lay.append((hs[4], hs[4] + 2, 1))                  # input of conv_post (k3, pad 1)
    lay.append((hs[4], hs[4] + 2, 0))                  # conv_post's output rows
    return lay


def period_flops(B, T, period, channels):
    """(executed, algorithmic) FLOP of one DiscriminatorP forward on B clips of T samples: what the tap-GEMMs run (every row of the
    segment sequence, 6 super-frame taps of which one is zero) against the reference's output frames times kernel taps."""
    lay = period_layout(T, period)
    S = B * period
    ex = al = 0
    cin = 1
    for i, cout in enumerate(channels + [1]):
        seg_in = lay[i][1]
        rows, k_ex, k_al = (seg_in // 3, 6, _K) if i < 4 else ((seg_in, _K, _K) if i == 4 else (seg_in, 3, 3))
        ex += 2 * S * rows * k_ex * cin * cout
        al += 2 * S * lay[i + 1][0] * k_al * cin * cout
        cin = cout
    return ex, al


def segment_view(storage, B, period, H, seg, halo, C):
    """The reference's [B, C, H, period] tensor as a view of segment storage [B*period*seg, C]."""
    return storage.view(B, period, seg, C)[:, :, halo:halo + H].permute(0, 3, 2, 1)


def superframe_weight(w):
    """Conv weight [N, C, 5] (stride 3, pad 2) -> the 2-tap stride-1 conv over super-frames of 3 frames whose first frame sits 2
    before the output's centre: [N, 3C, 2] with W'[n][j*C + c][d] = w[n][c][3d + j] (zero for 3d + j = 5)."""
    n, c, _ = w.shape
    return torch.nn.functional.pad(w, (0, 1)).view(n, c, 2, 3).permute(0, 3, 1, 2).reshape(n, 3 * c, 2)


def superframe_weight_adjoint(g, c):
    """Adjoint of superframe_weight: [N, 3C, 2] -> [N, C, 5] (a gather)."""
    n = g.shape[0]
    return g.reshape(n, 3, c, 2).permute(0, 2, 3, 1).reshape(n, c, 6)[:, :, :_K]


class DiscriminatorP(nn.Module):
    """reference discriminators.py:89-121.  The kernels cover the reference's defaults: weight norm, kernel 5, stride 3, and
    ``hidden`` a positive multiple of 4 (channel quads)."""

    @_record_ctor_args
    def __init__(self, period, kernel_size=5, stride=3, use_spectral_norm=False, hidden=32):
        super().__init__()
        if use_spectral_norm:
            raise NotImplementedError("aero_b200.mpd: spectral norm is not implemented (use_spectral_norm=False)")
        if kernel_size != _K or stride != 3:
            raise NotImplementedError(f"aero_b200.mpd: kernel_size={kernel_size}, stride={stride}: the kernels cover 5 and 3")
        if int(hidden) != hidden or hidden < 4 or hidden % 4:
            raise NotImplementedError(f"aero_b200.mpd: hidden={hidden}: must be a positive multiple of 4")
        if int(period) != period or period < 1:
            raise ValueError(f"aero_b200.mpd: period={period} must be a positive integer")
        self.period = int(period)
        self.channels = [hidden, hidden * 4, hidden * 16, hidden * 32, hidden * 32]
        cin = 1
        convs = []
        for i, cout in enumerate(self.channels):
            convs.append(_wn(nn.Conv2d(cin, cout, (kernel_size, 1), (stride, 1) if i < 4 else 1, padding=(_HALO, 0))))
            cin = cout
        self.convs = nn.ModuleList(convs)
        self.conv_post = _wn(nn.Conv2d(cin, 1, (3, 1), 1, padding=(1, 0)))
        self._precision = 0

    @property
    def train_precision(self):
        """Arithmetic of the convolutions: 0 exact fp32 (SIMT), 1 TF32 on the tensor cores (as aero_b200.Aero).  Mode 3 ("3xTF32") is
        refused: on this model its backward is not fp32-grade (DESIGN.md, section 10)."""
        return self._precision

    @train_precision.setter
    def train_precision(self, v):
        if int(v) == 3:
            raise NotImplementedError("aero_b200.mpd: train_precision=3 (3xTF32) does not reach fp32 accuracy on this model; "
                                      "use 0 (exact fp32) or 1 (TF32)")
        if int(v) not in (0, 1):
            raise ValueError(f"train_precision={v}: 0 (fp32) or 1 (TF32)")
        self._precision = int(v)

    def forward(self, x):
        """x [B, 1, T] fp32 on CUDA -> (logits [B, H5 * period], [five feature maps [B, C, H, period], logits [B, 1, H5, period]])."""
        if x.dim() != 3 or x.shape[1] != 1 or x.dtype != torch.float32:
            raise ValueError(f"aero_b200.mpd: expected fp32 input [B, 1, T], got {tuple(x.shape)} {x.dtype}")
        B, _, T = x.shape
        named = list(self.named_parameters())
        outs = _PeriodFn.apply(x.reshape(B, T), self, [n for n, _ in named], *[p for _, p in named])
        lay = period_layout(T, self.period)
        fmap = [segment_view(o, B, self.period, H, seg, halo, c)
                for o, (H, seg, halo), c in zip(outs, lay[1:], self.channels + [1])]
        return torch.flatten(fmap[-1], 1, -1), fmap


class MultiPeriodDiscriminator(nn.Module):
    """reference discriminators.py:124-147."""

    @_record_ctor_args
    def __init__(self, hidden=32, periods=[2, 3, 5, 7, 11]):
        super().__init__()
        self.discriminators = nn.ModuleList([DiscriminatorP(p, hidden=hidden) for p in periods])

    @property
    def train_precision(self):
        return self.discriminators[0].train_precision

    @train_precision.setter
    def train_precision(self, v):
        for d in self.discriminators:
            d.train_precision = v

    def forward(self, y, y_hat):
        y_d_rs, y_d_gs, fmap_rs, fmap_gs = [], [], [], []
        # real and generated clips never interact: one pass per period over both when their shapes agree
        joint = y.shape == y_hat.shape and y.device == y_hat.device
        B = y.shape[0]
        x = torch.cat([y, y_hat], 0) if joint else None
        for d in self.discriminators:
            if joint:
                logits, fmap = d(x)
                y_d_r, y_d_g, fmap_r, fmap_g = logits[:B], logits[B:], [f[:B] for f in fmap], [f[B:] for f in fmap]
            else:
                (y_d_r, fmap_r), (y_d_g, fmap_g) = d(y), d(y_hat)
            y_d_rs.append(y_d_r)
            y_d_gs.append(y_d_g)
            fmap_rs.append(fmap_r)
            fmap_gs.append(fmap_g)
        return y_d_rs, y_d_gs, fmap_rs, fmap_gs


class _MpdEngine(_DiscEngine):
    """One period's forward and backward on the discriminator's tape machinery (weight norm + tap-GEMM ops of _DiscEngine).

    Per-layer timing: when the module has a list attribute ``layer_events``, each convolution's forward launches and its backward tape
    entries are bracketed by CUDA events, appended there as (layer, "fwd" | "bwd", start, end) (bench_mpd.py reads them)."""

    def _event(self):
        if self._events is None:
            return None
        e = torch.cuda.Event(enable_timing=True)
        e.record(torch.cuda.current_stream(self._device()))
        return e

    def timed_conv(self, name, *a, **k):
        """self.conv, with its forward launches and its tape entries remembered as a span of layer `name`."""
        start, e0 = len(self.tape), self._event()
        y = self.conv(*a, **k)
        if self._events is not None:
            self._events.append((name, "fwd", e0, self._event()))
            self._spans.append((name, start, len(self.tape)))
        return y

    def repack(self, y, S, H, C_, rows, seg, halo):
        """LeakyReLU(0.1) of a convolution's output rows into the next layer's segment layout."""
        a = self._new(S * seg * C_)
        self._check(self.lib.aero_mpd_repack_fwd(_ptr(y), _ptr(a), S, H, C_, rows, seg, halo, _SLOPE, self._stream()))

        def bwd():
            da = self.grad(a)
            if da is None:
                return
            dy = self._new(S * rows * C_)
            self._check(self.lib.aero_mpd_repack_bwd(_ptr(y), _ptr(da), _ptr(dy), S, H, C_, rows, seg, halo, _SLOPE, self._stream()))
            self.acc(y, dy)
        self.tape.append(bwd)
        self.keep.append((y, a))
        return a

    @torch.no_grad()
    def forward(self, x, need_input_grad):
        """x [B, T] fp32 -> the stored tensors of period_layout[1:] (five feature maps, logits), flat."""
        self._reset()
        self._sync_stream()
        mod, lib = self.model, self.lib
        self._events, self._spans = getattr(mod, "layer_events", None), []
        self.params = {k: v.detach().contiguous() for k, v in mod.named_parameters()}
        B, T = x.shape
        P = mod.period
        lay = period_layout(T, P)
        S = B * P
        H, seg, halo = lay[0]
        h = self._new(S * seg)
        self._check(lib.aero_mpd_fold_fwd(_ptr(x), _ptr(h), B, T, P, H, seg, halo, self._stream()))
        self._x_in = x
        if need_input_grad:
            def fold_bwd(h=h):                         # h is rebound to each layer's output below
                dh = self.grad(h)
                if dh is None:
                    return
                dx = self._new(B * T)
                self._check(lib.aero_mpd_fold_bwd(_ptr(dh), _ptr(dx), B, T, P, H, seg, halo, self._stream()))
                self.acc(x, dx)
            self.tape.append(fold_bwd)
        else:
            self.no_grad.update((id(x), id(h)))
        self.keep.append((x, h))
        outs = []
        cin = 1
        for i, cout in enumerate(mod.channels):
            prefix = f"convs.{i}"
            seg_in = lay[i][1]
            w, back = self.wn_weight(prefix, cout, cin * _K)
            if i < 4:                                    # stride 3: 2 taps over super-frames [S * seg_in / 3, 3 * cin]
                rows = seg_in // 3
                y = self.timed_conv(prefix, h, None, 3 * cin, 0, None, prefix + ".bias", _Conv(kt=2), 1, 1, 1, S * rows, cout,
                              w_override=(superframe_weight(w.view(cout, cin, _K)),
                                          lambda g, back=back, cin=cin: back(superframe_weight_adjoint(g, cin).contiguous())))
            else:
                rows = seg_in
                y = self.timed_conv(prefix, h, None, cin, 0, None, prefix + ".bias", _Conv(kt=_K), 1, 1, 1, S * rows, cout,
                              w_override=(w.view(cout, cin, _K), back))
            Ho, seg_o, halo_o = lay[i + 1]
            h = self.repack(y, S, Ho, cout, rows, seg_o, halo_o)
            outs.append(h)
            cin = cout
        w, back = self.wn_weight("conv_post", 1, cin * 3)
        o = self.timed_conv("conv_post", h, None, cin, 0, None, "conv_post.bias", _Conv(kt=3), 1, 1, 1, S * lay[5][1], 1,
                      w_override=(w.view(1, cin, 3), back))
        outs.append(o)
        self._outs = outs
        return outs

    @torch.no_grad()
    def backward(self, grads, grad_sink=None, owned=False):
        """As _DiscEngine.backward: one gradient (or None) per stored output of forward()."""
        self._sync_stream()
        self._sink = grad_sink
        for t, g in zip(self._outs, grads):
            if g is not None:
                self.acc(t, g if owned else g.contiguous().float().reshape(-1).clone())
        ends = {end - 1: (name, start) for name, start, end in self._spans}
        open_ = {}
        for i in range(len(self.tape) - 1, -1, -1):
            if i in ends:
                open_[ends[i][1]] = (ends[i][0], self._event())
            self.tape[i]()
            if i in open_:
                name, e0 = open_.pop(i)
                self._events.append((name, "bwd", e0, self._event()))
        gx = self.g.get(id(self._x_in))
        pg = self.pg
        self._reset()
        return gx, pg


class _PeriodFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, module, names, *params):
        if not x.is_cuda or next(module.parameters()).device != x.device:
            raise RuntimeError("aero_b200.mpd runs on CUDA only (kernels in libaero_b200.so); there is no CPU path")
        with torch.cuda.device(x.device):
            eng = _MpdEngine(module)
            outs = eng.forward(x.detach().contiguous(), ctx.needs_input_grad[0])
        ctx.eng, ctx.names, ctx.dev, ctx.shape = eng, names, x.device, x.shape
        ctx.set_materialize_grads(False)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grads):
        with torch.cuda.device(ctx.dev):
            gx, pg = ctx.eng.backward(grads)
        ctx.eng = None
        return (None if gx is None else gx.view(ctx.shape), None, None, *[pg.get(n) for n in ctx.names])
