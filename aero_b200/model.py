"""Drop-in boundary for the AERO generator: ``aero_b200.Aero``.

This class is what ``src.models.aero.Aero`` resolves to in this repo.  It keeps
the reference's Python surface (reference ``src/models/aero.py:223-268`` ctor
kwargs, ``:446`` ``forward(mix, return_spec, return_lr_spec)``, ``:409``
``_spec(x, scale)``, the 331-key ``state_dict`` layout and
``_init_args_kwargs`` used by ``src/model_serializer.py:20``) while the
arithmetic is executed by the sm_90a kernels in ``aero_b200/csrc`` through the
C-ABI library (``include/aero_b200.h``).

The module tree below only *holds parameters*; none of the ``nn`` layers'
``forward`` methods are used on the product path.  The tree is created in the
same order as the reference constructor so that, for a given
``torch.manual_seed``, parameter values are bit-identical to the reference's
(verified in the CPU suite, ``test_..._vs_live_reference_blocks``), which is what lets parity tests seed
both sides instead of shipping 78 MB of weights.
"""
from __future__ import annotations

import functools
import math

import torch
from torch import nn

__all__ = ["Aero", "AeroGeometry", "LayerGeom"]


def _record_ctor_args(init):
    # Same contract as reference src/models/utils.py:7-19: the checkpoint
    # writer re-creates the model from ``_init_args_kwargs``.
    @functools.wraps(init)
    def wrapped(self, *args, **kwargs):
        self._init_args_kwargs = (args, kwargs)
        init(self, *args, **kwargs)

    return wrapped


class _Holder(nn.Module):
    """A parameter container whose forward is never called."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("parameter holder: compute happens in aero_b200.engine")


class _SnakeParam(_Holder):
    # reference src/models/snake.py:45-57: a ~ Exponential(rate 0.1), one per frequency row
    def __init__(self, n):
        super().__init__()
        draw = torch.distributions.exponential.Exponential(torch.tensor([0.1])).rsample([n])
        self.a = nn.Parameter(draw.squeeze())


class _Scale(_Holder):
    # reference src/models/modules.py:130-141 (LayerScale)
    def __init__(self, channels, init):
        super().__init__()
        self.scale = nn.Parameter(torch.full((channels,), float(init)))


class _BiLSTM(_Holder):
    # reference src/models/modules.py:17-30
    def __init__(self, dim, layers, max_steps):
        super().__init__()
        self.max_steps = max_steps
        self.lstm = nn.LSTM(bidirectional=True, num_layers=layers, hidden_size=dim, input_size=dim)
        self.linear = nn.Linear(2 * dim, dim)


class _LocalAttn(_Holder):
    # reference src/models/modules.py:74-92
    def __init__(self, channels, heads, ndecay):
        super().__init__()
        if channels % heads:
            raise AssertionError((channels, heads))
        self.heads, self.ndecay = heads, ndecay
        self.content = nn.Conv1d(channels, channels, 1)
        self.query = nn.Conv1d(channels, channels, 1)
        self.key = nn.Conv1d(channels, channels, 1)
        self.query_decay = nn.Conv1d(channels, heads * ndecay, 1)
        with torch.no_grad():
            self.query_decay.weight.mul_(0.01)
            self.query_decay.bias.fill_(-2.0)
        self.proj = nn.Conv1d(channels, channels, 1)


class _FreqTransform(_Holder):
    # reference src/models/modules.py:279-302 (FTB)
    def __init__(self, nbins, channels, r=5):
        super().__init__()
        self.conv1 = nn.Sequential(nn.Conv2d(channels, r, [1, 1]), nn.BatchNorm2d(r), nn.ReLU())
        self.conv1d = nn.Sequential(nn.Conv1d(r * nbins, channels, 9, padding=4),
                                    nn.BatchNorm1d(channels), nn.ReLU())
        self.freq_fc = nn.Linear(nbins, nbins, bias=False)
        self.conv2 = nn.Sequential(nn.Conv2d(2 * channels, channels, [1, 1]),
                                   nn.BatchNorm2d(channels), nn.ReLU())


def _dconv_act(act_func, nrows):
    # reference src/models/modules.py:194-199,208: 'gelu' -> nn.GELU, 'snake' -> Snake(freq_dim), any other string -> nn.ReLU
    if act_func == "snake":
        return _SnakeParam(nrows)
    return nn.GELU() if act_func == "gelu" else nn.ReLU()


class _ResidualBranch(_Holder):
    # reference src/models/modules.py:152-219 (DConv); always GroupNorm(1, .)
    def __init__(self, channels, compress, depth, init, lstm, attn, nrows, act_func, heads=4, ndecay=4):
        super().__init__()
        hidden = int(channels / compress)
        self.hidden, self.depth = hidden, abs(depth)
        self.layers = nn.ModuleList()
        for d in range(self.depth):
            dil = 2 ** d if depth > 0 else 1
            blk = nn.ModuleDict()
            blk["conv1"] = nn.Sequential(nn.Conv1d(channels, hidden, 3, dilation=dil, padding=dil),
                                         nn.GroupNorm(1, hidden))
            blk["act"] = _dconv_act(act_func, nrows)
            blk["conv2"] = nn.Sequential(nn.Conv1d(hidden, 2 * channels, 1), nn.GroupNorm(1, 2 * channels),
                                         nn.GLU(1), _Scale(channels, init))
            if lstm:
                blk["lstm"] = _BiLSTM(hidden, layers=2, max_steps=200)
            if attn:
                blk["time_attn"] = _LocalAttn(hidden, heads, ndecay)
            self.layers.append(blk)


class _EncLayer(_Holder):
    # reference src/models/aero.py:32-106
    def __init__(self, g: "LayerGeom", norm_groups, dconv_kw):
        super().__init__()
        cin = g.enc_cin
        if g.index == 0:
            self.pre_conv = nn.Conv2d(cin, g.ch, [1, 1])
            cin = g.ch
        if g.ftb:
            self.freq_attn_block = _FreqTransform(g.f_in, cin)
        self.conv = nn.Conv2d(cin, g.ch, [g.kernel, 1], [g.stride, 1], [g.pad, 0])
        self.norm1 = nn.GroupNorm(norm_groups, g.ch) if g.norm else nn.Identity()
        self.rewrite = nn.Conv2d(g.ch, 2 * g.ch, 1, 1, 0)
        self.norm2 = nn.GroupNorm(norm_groups, 2 * g.ch) if g.norm else nn.Identity()
        self.dconv = _ResidualBranch(g.ch, nrows=g.f_out, **dconv_kw) if g.dconv else None


class _DecLayer(_Holder):
    # reference src/models/aero.py:139-187
    def __init__(self, g: "LayerGeom", norm_groups, context):
        super().__init__()
        self.conv_tr = nn.ConvTranspose2d(2 * g.ch, g.dec_cout, [g.kernel, 1], [g.stride, 1])
        self.norm2 = nn.GroupNorm(norm_groups, g.dec_cout) if g.norm else nn.Identity()
        k = 1 + 2 * context
        self.rewrite = nn.Conv2d(2 * g.ch, 4 * g.ch, k, 1, context)
        self.norm1 = nn.GroupNorm(norm_groups, 4 * g.ch) if g.norm else nn.Identity()


class _FreqEmbedding(_Holder):
    # reference src/models/modules.py:252-276 (ScaledEmbedding)
    def __init__(self, n, dim, scale, smooth):
        super().__init__()
        self.embedding = nn.Embedding(n, dim)
        with torch.no_grad():
            if smooth:
                w = torch.cumsum(self.embedding.weight, dim=0)
                w = w / torch.arange(1, n + 1).to(w).sqrt()[:, None]
                self.embedding.weight.copy_(w)
            self.embedding.weight.div_(scale)
        self.scale = scale


class LayerGeom:
    """Static geometry of U-Net level ``index`` (encoder i / decoder depth-1-i)."""

    __slots__ = ("index", "enc_cin", "ch", "dec_cout", "f_in", "f_out", "kernel", "stride", "pad",
                 "norm", "ftb", "lstm", "attn", "dconv")

    def __repr__(self):
        return "LayerGeom(" + ", ".join(f"{k}={getattr(self, k)}" for k in self.__slots__) + ")"


class AeroGeometry:
    """Everything the engine needs to know about shapes, derived from ctor kwargs
    exactly as reference src/models/aero.py:324-407 derives them."""

    def __init__(self, kw):
        self.kw = kw
        self.scale = kw["hr_sr"] / kw["lr_sr"] if kw["spec_upsample"] else 1
        self.nfft = kw["nfft"]
        self.hop_in = int(kw["hop_length"] // self.scale)
        self.win_in = int(self.nfft // self.scale)
        self.hop_out = int(self.hop_in * self.scale)
        self.win_out = int(self.win_in * self.scale)
        self.cac = kw["cac"]
        self.cin0 = kw["in_channels"] * (2 if self.cac else 1)
        self.cout0 = kw["out_channels"] * (2 if self.cac else 1)
        self.layers = []
        ch, f = kw["channels"], self.nfft // 2
        cin = self.cin0
        for i, s in enumerate(kw["strides"]):
            g = LayerGeom()
            g.index, g.enc_cin, g.ch = i, cin, ch
            g.dec_cout = self.cout0 if i == 0 else cin
            freq = i <= kw["freq_ends"]
            if not freq:
                raise NotImplementedError("time-axis (freq=False) layers are not on the AERO path "
                                          "(all shipped configs use freq_ends >= depth-1)")
            g.kernel = f if f < kw["kernel_size"] else kw["kernel_size"]
            g.stride = s
            if s == 1 and g.kernel % 2 == 0 and g.kernel > 1:
                g.kernel -= 1
            g.pad = (g.kernel - s) // 2
            g.f_in, g.f_out = f, f // s
            g.norm = i >= kw["norm_starts"]
            g.ftb = i >= kw["enc_freq_attn"]
            g.lstm = i >= kw["dconv_lstm"]
            g.attn = i >= kw["dconv_time_attn"]
            g.dconv = bool(kw["dconv_mode"] & 1)
            self.layers.append(g)
            cin, ch, f = ch, int(kw["growth"] * ch), f // s
        self.depth = len(self.layers)

    def frames(self, length, scale=False):
        """Number of STFT frames for a length-`length` input (after the hop pad)."""
        hop = self.hop_in
        padded = length + (-length) % hop
        hl = int(hop * self.scale) if scale else hop
        return 1 + padded // hl


_DEFAULTS = dict(
    in_channels=1, out_channels=1, audio_channels=2, channels=48, growth=2,
    nfft=512, hop_length=64, end_iters=0, cac=True,
    rewrite=True, hybrid=False, hybrid_old=False,
    freq_emb=0.2, emb_scale=10, emb_smooth=True,
    kernel_size=8, strides=[4, 4, 2, 2], context=1, context_enc=0, freq_ends=4, enc_freq_attn=4,
    norm_starts=2, norm_groups=4,
    dconv_mode=1, dconv_depth=2, dconv_comp=4, dconv_time_attn=2, dconv_lstm=2, dconv_init=1e-3,
    rescale=0.1, lr_sr=4000, hr_sr=16000, spec_upsample=True, act_func="snake", debug=False,
)


class _AeroTrainFn(torch.autograd.Function):
    """forward = TrainEngine.forward (records a tape), backward = TrainEngine.backward (parameter gradients)."""

    @staticmethod
    def forward(ctx, mix, model, names, *params):
        from .train_engine import TrainEngine
        if not mix.is_cuda or next(model.parameters()).device != mix.device:
            raise RuntimeError("aero_b200.Aero trains on CUDA only (sm_90a kernels in libaero_b200.so); there is no CPU path")
        with torch.cuda.device(mix.device):
            eng = TrainEngine(model)
            wave, spec = eng.forward(mix)
        ctx.eng, ctx.names, ctx.dev = eng, names, mix.device
        ctx.set_materialize_grads(False)
        return wave, spec

    @staticmethod
    def backward(ctx, d_wave, d_spec):
        with torch.cuda.device(ctx.dev):
            grads = ctx.eng.backward(d_wave, d_spec)
        ctx.eng = None
        return (None, None, None, *[grads.get(n) for n in ctx.names])


class Aero(nn.Module):
    """AERO generator (audio super-resolution in the spectral domain), H100-native (sm_90a).

    Constructor kwargs, defaults and attribute names follow reference
    ``src/models/aero.py:223-268`` so that ``Aero(**args.experiment.aero)``
    (reference ``src/models/modelFactory.py:7-8``) works unchanged.
    """

    @_record_ctor_args
    def __init__(self, in_channels=1, out_channels=1, audio_channels=2, channels=48, growth=2,
                 nfft=512, hop_length=64, end_iters=0, cac=True,
                 rewrite=True, hybrid=False, hybrid_old=False,
                 freq_emb=0.2, emb_scale=10, emb_smooth=True,
                 kernel_size=8, strides=[4, 4, 2, 2], context=1, context_enc=0, freq_ends=4,
                 enc_freq_attn=4, norm_starts=2, norm_groups=4,
                 dconv_mode=1, dconv_depth=2, dconv_comp=4, dconv_time_attn=2, dconv_lstm=2,
                 dconv_init=1e-3, rescale=0.1, lr_sr=4000, hr_sr=16000, spec_upsample=True,
                 act_func="snake", debug=False):
        super().__init__()
        kw = {k: v for k, v in locals().items() if k in _DEFAULTS}
        kw["strides"] = list(strides)
        self._check_supported(kw)
        geom = AeroGeometry(kw)
        self.geom = geom

        # attributes the reference exposes (aero.py:305-331)
        self.cac, self.in_channels, self.out_channels = cac, in_channels, out_channels
        self.audio_channels, self.kernel_size, self.context = audio_channels, kernel_size, context
        self.strides, self.depth, self.channels = kw["strides"], geom.depth, channels
        self.lr_sr, self.hr_sr, self.spec_upsample = lr_sr, hr_sr, spec_upsample
        self.scale = geom.scale
        self.nfft = nfft
        self.hop_length = geom.hop_in      # hop of the *input* (low-rate) analysis, aero.py:327
        self.win_length = geom.win_in      # window of the *input* analysis, aero.py:328
        self.end_iters, self.hybrid, self.hybrid_old, self.debug = end_iters, hybrid, hybrid_old, debug
        self.freq_emb = None

        self.act_func = act_func
        dconv_kw = dict(compress=dconv_comp, depth=dconv_depth, init=dconv_init, act_func=act_func)
        self.encoder = nn.ModuleList()
        self.decoder = nn.ModuleList()
        for g in geom.layers:
            self.encoder.append(_EncLayer(g, norm_groups, dict(dconv_kw, lstm=g.lstm, attn=g.attn)))
            self.decoder.insert(0, _DecLayer(g, norm_groups, context))
            if g.index == 0 and freq_emb:
                self.freq_emb = _FreqEmbedding(g.f_out, g.ch, scale=emb_scale, smooth=emb_smooth)
                self.freq_emb_scale = freq_emb
        if rescale:
            self._rescale_1d_convs(rescale)

        self._engine_obj = None
        # training arithmetic of the convolution GEMMs (aero_b200/train_engine.py): 0 = exact fp32 (gradient-parity mode), 1 = TF32 on the
        # tensor cores (what cuDNN does for the reference under torch.backends.cudnn.allow_tf32, PyTorch's default)
        self.train_precision = 0

    # ------------------------------------------------------------------ init helpers
    @staticmethod
    def _check_supported(kw):
        # The reference accepts more combinations than its shipped configs use; the CUDA
        # path covers the spectral ("cac") frequency-only U-Net of conf/experiment/aero_*.yaml,
        # with any DConv activation (act_func) and with or without spectral upsampling (spec_upsample).
        problems = []
        if not kw["cac"]:
            problems.append("cac=False")
        if not kw["rewrite"]:
            problems.append("rewrite=False")
        if kw["dconv_mode"] & 2:
            problems.append("dconv_mode with decoder DConv")
        if kw["context"] != 1 or kw["context_enc"] != 0:
            problems.append("context != 1 or context_enc != 0")
        if kw["nfft"] & (kw["nfft"] - 1) or not 64 <= kw["nfft"] <= 4096:
            problems.append("nfft must be a power of two in [64, 4096]")
        if problems:
            raise NotImplementedError("aero_b200: unsupported configuration: " + ", ".join(problems))

    def _rescale_1d_convs(self, reference):
        # reference aero.py:17-28: only Conv1d/ConvTranspose1d are touched; weight and bias are
        # divided by sqrt(std(weight)/reference).
        with torch.no_grad():
            for sub in self.modules():
                if isinstance(sub, (nn.Conv1d, nn.ConvTranspose1d)):
                    s = (sub.weight.std() / reference) ** 0.5
                    sub.weight.div_(s)
                    if sub.bias is not None:
                        sub.bias.div_(s)

    # ------------------------------------------------------------------ engine plumbing
    def _engine(self):
        if self._engine_obj is None:
            from .engine import AeroEngine
            object.__setattr__(self, "_engine_obj", AeroEngine(self))
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

    # ------------------------------------------------------------------ public surface
    def _spec(self, x, scale=False):
        """Complex spectrogram ``[..., nfft/2, frames]`` (Nyquist bin dropped), reference
        aero.py:409-421.  ``scale=True`` analyses a high-rate signal on the same grid."""
        return self._engine().spec(x, scale=scale)

    def _ispec(self, z):
        """Inverse of the *output-rate* analysis, reference aero.py:423-428."""
        return self._engine().ispec(z)

    def forward(self, mix, return_spec=False, return_lr_spec=False):
        if self.training:
            return self._train_forward(mix, return_spec, return_lr_spec)
        return self._engine().forward(mix, return_spec=return_spec, return_lr_spec=return_lr_spec)

    def _train_forward(self, mix, return_spec, return_lr_spec):
        """Training mode (reference solver.py:305 `self.dmodel(lr)` under autograd): the forward and its backward both run on
        the CUDA kernels (aero_b200/train_engine.py) behind ONE autograd node, so `loss.backward()`, `optimizer.step()`, DDP
        gradient hooks and `return_spec` all behave as with the reference nn.Module."""
        names = [n for n, p in self.named_parameters() if p.requires_grad]
        params = [p for _, p in self.named_parameters() if p.requires_grad]
        wave, spec = _AeroTrainFn.apply(mix, self, names, *params)
        if not return_spec:
            return wave
        B, Fq, T, C2 = spec.shape
        zc = torch.view_as_complex(spec.reshape(B, Fq, T, C2 // 2, 2)).permute(0, 3, 1, 2)
        if not return_lr_spec:
            return wave, zc
        with torch.no_grad():
            was = self.training
            zl = self._engine().spec(mix.detach())
        return wave, zc, zl
