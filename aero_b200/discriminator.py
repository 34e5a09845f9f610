"""MelGAN multi-scale discriminator on the CUDA kernels (SURVEY.md section 8f rank 3).

``Discriminator`` mirrors reference ``src/models/discriminators.py:57-78`` (``num_D`` ``NLayerDiscriminator`` scales, ``:14-54``,
joined by ``AvgPool1d(4, 2, 1, count_include_pad=False)``): same constructor arguments, the same ``state_dict`` keys
(``model.disc_i.model.layer_k.{0|1}.{bias, weight_g, weight_v}`` -- the layers are weight-normalised ``WNConv1d``) and the same
return value, a list (scales) of lists (one tensor ``[B, C, T]`` per layer, the last one the logits), so the hinge / feature-matching
losses of ``src/solver.py:475-520`` apply unchanged.

Each scale is ONE ``torch.autograd.Function``: forward and backward run on libaero_b200.so -- the grouped strided convolutions on
``aero_gconv1d_*``, the dense ones on the tap-GEMM, LeakyReLU on ``aero_norm_act_train_*`` (activation only), weight
normalisation on ``aero_weight_norm_*`` -- through the same tape machinery as the generator's training step
(``aero_b200.train_engine.TrainEngine``).  The reflection padding of the first layer and the average pooling between scales act
on the 1-channel waveform and stay ordinary (differentiable) torch calls.  Feature maps are returned as ``[B, C, T]`` VIEWS of
channels-last storage: every consumer in the reference is layout-agnostic (means, L1 distances).
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from . import cabi
from .cabi import NA_LEAKY
from .train_engine import TrainEngine, _Conv, _ptr


def _layer_specs(ndf, n_layers, factor):
    """(name, C_in, C_out, k, stride, pad, groups, leaky) of reference discriminators.py:15-49."""
    specs = [("layer_0.1", 1, ndf, 15, 1, 0, 1, True)]              # after ReflectionPad1d(7)
    nf, stride = ndf, factor
    max_nf = (stride ** (n_layers - 1)) * ndf
    nf_prev = nf
    for n in range(1, n_layers + 1):
        nf_prev = nf
        nf = min(nf * stride, max_nf)
        specs.append((f"layer_{n}.0", nf_prev, nf, stride * 10 + 1, stride, stride * 5, nf_prev // 4, True))
    nf2 = min(nf * 2, max_nf)
    specs.append((f"layer_{n_layers + 1}.0", nf_prev, nf2, 5, 1, 2, 1, True))
    specs.append((f"layer_{n_layers + 2}", nf2, 1, 3, 1, 1, 1, False))
    return specs


class _WN(nn.Module):
    """Parameter holder with torch.nn.utils.weight_norm's names (weight_g [C_out,1,1], weight_v [C_out, C_in/groups, k], bias)."""

    def __init__(self, cin, cout, k, groups):
        super().__init__()
        conv = nn.Conv1d(cin, cout, k, groups=groups)                  # PyTorch's default init, as the reference constructs it
        with torch.no_grad():
            conv.weight.normal_(0.0, 0.02)                               # reference utils.weights_init for "Conv" layers
        self.bias = nn.Parameter(conv.bias.detach().clone())
        self.weight_g = nn.Parameter(conv.weight.detach().flatten(1).norm(dim=1).view(-1, 1, 1).clone())
        self.weight_v = nn.Parameter(conv.weight.detach().clone())


class NLayerDiscriminator(nn.Module):
    def __init__(self, ndf, n_layers, downsampling_factor):
        super().__init__()
        self.specs = _layer_specs(ndf, n_layers, downsampling_factor)
        self.train_precision = 0                                        # 1: dense convolutions in TF32 on the tensor cores
        self.model = nn.ModuleDict()
        for name, cin, cout, k, s, p, g, leaky in self.specs:
            layer, _, idx = name.partition(".")
            if idx:                                                     # Sequential: conv at index `idx`
                seq = nn.Module()
                seq.add_module(idx, _WN(cin, cout, k, g))
                self.model[layer] = seq
            else:
                self.model[layer] = _WN(cin, cout, k, g)

    def forward(self, x):
        xp = torch.nn.functional.pad(x, (7, 7), mode="reflect")         # nn.ReflectionPad1d(7), discriminators.py:19
        names = [n for n, _ in self.named_parameters()]
        outs = _DiscScaleFn.apply(xp, self, names, *[p for _, p in self.named_parameters()])
        return [o.permute(0, 2, 1) for o in outs]                       # [B, C, T] views of channels-last storage


class _DiscEngine(TrainEngine):
    """The generator's tape machinery with the discriminator's two extra ops (weight norm, grouped conv)."""

    def __init__(self, module):
        self.model = module
        self.geom = None
        self.lib = cabi.load()
        self.precision = int(getattr(module, "train_precision", 0))
        self._reset()

    def wn_weight(self, prefix, rows, length):
        """w = g * v / ||v|| for layer `prefix`; returns (w, callback adding d(w) back into weight_g / weight_v gradients)."""
        P = self.params
        v, g = P[prefix + ".weight_v"], P[prefix + ".weight_g"]
        w = torch.empty_like(v)
        self._check(self.lib.aero_weight_norm_fwd(_ptr(v), _ptr(g), _ptr(w), rows, length, self._stream()))

        def back(gw):
            self._check(self.lib.aero_weight_norm_bwd(_ptr(v), _ptr(g), _ptr(gw.contiguous()), _ptr(self.pgrad(prefix + ".weight_v")),
                                                      _ptr(self.pgrad(prefix + ".weight_g")), rows, length, self._stream()))
        return w, back

    def gconv(self, x, prefix, B, Tin, Cin, Cout, k, stride, pad, groups):
        lib = self.lib
        Tout = (Tin + 2 * pad - k) // stride + 1
        w, w_back = self.wn_weight(prefix, Cout, (Cin // groups) * k)
        bias = self.params[prefix + ".bias"]
        y = self._new(B * Tout * Cout)
        args = (B, Tin, Tout, Cin, Cout, groups, k, stride, pad)
        self._check(lib.aero_gconv1d_fwd(_ptr(x), _ptr(w), _ptr(bias), _ptr(y), *args, self._stream()))

        def bwd():
            dy = self.grad(y)
            if dy is None:
                return
            if self.param_grads:
                gw = torch.zeros_like(w)
                self._check(lib.aero_gconv1d_wgrad(_ptr(x), _ptr(dy), _ptr(gw), *args, self._stream()))
                w_back(gw)
                gb = self._new(Cout, zero=True, dtype=torch.float64)
                self._colsum(dy, gb, Cout, B * Tout, Cout)
                self._add_f64(self.pgrad(prefix + ".bias"), gb)
            if id(x) not in self.no_grad:
                dx = self._new(B * Tin * Cin)
                self._check(lib.aero_gconv1d_dgrad(_ptr(dy), _ptr(w), _ptr(dx), *args, self._stream()))
                self.acc(x, dx)
        self.tape.append(bwd)
        self.keep.append((x, y, w))
        return y, Tout

    @torch.no_grad()
    def forward(self, xp, need_input_grad):
        """xp [B, 1, L + 14] (reflection-padded waveform).  Returns the list of layer outputs, channels-last [B, T, C]."""
        self._reset()
        mod = self.model
        self.params = {k: v.detach() for k, v in mod.named_parameters()}
        self.buffers = {}
        B = xp.shape[0]
        h = xp.contiguous().float().view(-1)
        self._x_in = h
        if not need_input_grad:
            self.no_grad.add(id(h))
        T, Cc = xp.shape[-1], 1
        outs = []
        for name, cin, cout, k, s, p, g, leaky in mod.specs:
            prefix = "model." + name
            if g == 1:
                w, w_back = self.wn_weight(prefix, cout, cin * k)
                To = T + 2 * p - k + 1
                y = self.conv(h, None, cin, 0, None, prefix + ".bias", _Conv(kt=k, pad_t=p), B, 1, 1, To, cout, w_override=(w, w_back),
                              T_in=T)
            else:
                y, To = self.gconv(h, prefix, B, T, cin, cout, k, s, p, g)
            if leaky:
                y = self.norm_act(y, NA_LEAKY, B=B, F_in=1, T=To, C_=cout, scope=1, no_norm=True)
            outs.append((y, To, cout))
            h, T, Cc = y, To, cout
        self._outs = outs
        return [y.view(B, To, c) for y, To, c in outs]

    @torch.no_grad()
    def backward(self, grads, grad_sink=None, owned=False):
        """grads: one gradient (or None) per layer output.  grad_sink(name) -> zeroed tensor to accumulate that parameter's gradient
        into (else fresh tensors).  owned: the gradients are flat fp32 buffers the tape may take over and modify (no copy)."""
        self._sync_stream()
        self._sink = grad_sink
        for (y, To, c), gy in zip(self._outs, grads):
            if gy is not None:
                self.acc(y, gy if owned else gy.contiguous().float().reshape(-1).clone())
        for fn in reversed(self.tape):
            fn()
        gx = self.g.get(id(self._x_in))
        pg = self.pg
        self._reset()
        return gx, pg


class _DiscScaleFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xp, module, names, *params):
        if not xp.is_cuda:
            raise RuntimeError("aero_b200.discriminator runs on CUDA only (kernels in libaero_b200.so); there is no CPU path")
        with torch.cuda.device(xp.device):
            eng = _DiscEngine(module)
            outs = eng.forward(xp, ctx.needs_input_grad[0])
        ctx.eng, ctx.names, ctx.dev, ctx.shape = eng, names, xp.device, xp.shape
        ctx.set_materialize_grads(False)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grads):
        with torch.cuda.device(ctx.dev):
            gx, pg = ctx.eng.backward(grads)
        ctx.eng = None
        return (None if gx is None else gx.view(ctx.shape), None, None, *[pg.get(n) for n in ctx.names])


class Discriminator(nn.Module):
    """reference discriminators.py:57-78 (``Discriminator(num_D, ndf, n_layers, downsampling_factor)``)."""

    def __init__(self, num_D=3, ndf=16, n_layers=4, downsampling_factor=4):
        super().__init__()
        self._init_args_kwargs = ((), dict(num_D=num_D, ndf=ndf, n_layers=n_layers, downsampling_factor=downsampling_factor))
        self.model = nn.ModuleDict()
        self.num_D = num_D
        for i in range(num_D):
            self.model[f"disc_{i}"] = NLayerDiscriminator(ndf, n_layers, downsampling_factor)
        self.downsample = nn.AvgPool1d(4, stride=2, padding=1, count_include_pad=False)

    @property
    def train_precision(self):
        return self.model["disc_0"].train_precision

    @train_precision.setter
    def train_precision(self, v):
        for d in self.model.values():
            d.train_precision = int(v)

    def forward(self, x):
        results = []
        for _, disc in self.model.items():
            results.append(disc(x))
            x = self.downsample(x)
        return results
