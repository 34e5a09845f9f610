"""Training step of the AERO generator on the CUDA kernels (SURVEY.md section 8f rank 1).

``TrainEngine.forward`` runs ``Aero.forward`` in training mode (reference ``src/models/aero.py:446-523`` with
``model.train()``: batch-statistics BatchNorm in the FTB blocks, nothing folded or fused away) and records a tape;
``TrainEngine.backward`` replays the tape in reverse and returns the gradient of every parameter -- what
``loss.backward()`` does through autograd in the reference (``src/solver.py:602-605``).  Every arithmetic step is a call
into libaero_b200.so (``include/aero_b200.h``, "Training"); PyTorch provides memory, the stream and a few index
shuffles of parameter-sized tensors.  ``aero_b200.model.Aero.forward`` dispatches here when ``self.training`` and wraps the
pair in one ``torch.autograd.Function`` so that ``loss.backward()`` / ``optimizer.step()`` / DDP work unchanged.

Everything is fp32 (exact-fp32 SIMT tap-GEMMs): the bar is 1e-3 relative against reference autograd.
Data gradients of the convolutions run on ``aero_tapgemm_fwd`` itself (the adjoint of a tap-GEMM is a tap-GEMM).

Book-keeping: activations are plain contiguous tensors; every op takes its geometry explicitly (never from a view's shape),
so gradients are keyed by the tensor object and a gradient is just a tensor with the same number of elements.
"""
from __future__ import annotations

import ctypes as C
import math

import torch

from . import cabi, spec
from .cabi import ACT_NONE, NA_GELU, NA_GLU, NA_GLU_SCALE_RES, NA_NO_NORM, NA_NONE, NA_RELU, NA_SNAKE, TAPS_CONV, TAPS_CONVT
from .engine import _ATTN_HEADS, _ATTN_NDECAY, _LSTM_MAX_STEPS, center_groups, dconv_norm_act_op, pack_taps, tf32_round

_FTB_R, _FTB_RP = 5, 8          # FTB squeeze channels (modules.py:286) and their padded count (kernels work on channel quads)


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class _Conv:
    """Geometry of one tap-GEMM layer (forward view)."""

    def __init__(self, kind="conv", kf=1, kt=1, stride_f=1, pad_f=0, dil_t=1, pad_t=0, f_off=0):
        self.kind, self.kf, self.kt, self.stride_f, self.pad_f, self.dil_t, self.pad_t, self.f_off = \
            kind, kf, kt, stride_f, pad_f, dil_t, pad_t, f_off


_C1x1 = _Conv()


class TrainEngine:
    # False: the tape computes data gradients only -- the convolutions skip their weight-gradient GEMMs, bias column sums and
    # derived-weight callbacks (the generator pass of aero_b200.trainer.GanTrainer, whose optimiser does not use them)
    param_grads = True

    def __init__(self, model):
        self.model = model
        self.geom = model.geom
        self.lib = cabi.load()
        # Arithmetic of the convolutions' forward, data-gradient and weight-gradient GEMMs (normalisation, LSTM recurrence, attention and
        # all reductions are fp32 / fp64 in every mode):
        #   0  exact-fp32 SIMT tap-GEMMs (the original gradient-parity mode);
        #   1  TF32 on the tensor cores (what cuDNN does for the reference under PyTorch's default cudnn.allow_tf32);
        #   3  "3xTF32": every operand split into hi + lo TF32 halves, three tensor-core products hi*hi + hi*lo + lo*hi summed in fp32 --
        #      fp32-grade results (~2^-22 per product) at tensor-core speed.
        self.precision = int(getattr(model, "train_precision", 0))
        self._reset()

    def _reset(self):
        self.tape = []
        self.g = {}            # id(activation) -> gradient tensor
        self.pg = {}           # parameter name -> gradient tensor (PyTorch layout)
        self.keep = []         # tensors the tape refers to by id
        self.no_grad = set()   # ids of activations that need no gradient (the input spectrogram)
        self._sink = None      # optional name -> preallocated gradient tensor
        self.marks = []        # (tape length, layer tag) after each encoder / decoder layer of the forward
        self._zpool = {}       # dtype -> [zeroed buffer, bump offset] (see _new)
        self._st = None        # cached stream handle (see _stream)
        self._dev = None

    # ------------------------------------------------------------------ plumbing
    def _device(self):
        d = self._dev
        if d is None:
            d = self._dev = next(self.model.parameters()).device
        return d

    def _stream(self):
        # looked up once per pass (forward / backward each start from _sync_stream): a step makes ~3000 launches and
        # torch.cuda.current_stream() costs more host time than most of them take on the GPU
        st = self._st
        if st is None:
            st = self._st = C.c_void_p(torch.cuda.current_stream(self._device()).cuda_stream)
        return st

    def _sync_stream(self):
        """Re-read the caller's current stream (start of a forward or backward pass)."""
        self._st = None

    def _new(self, *shape, zero=False, dtype=torch.float32):
        if not zero:
            return torch.empty(shape, dtype=dtype, device=self._device())
        # zeroed accumulators (fp64 statistics / column sums, small fp32 gradients): bump-allocated from one buffer zeroed once per step --
        # a step needs ~900 of them, and a memset launch each costs more host time than the kernels that fill them
        n = 1
        for d in shape:
            n *= int(d)
        pool = self._zpool.get(dtype)
        if pool is None and dtype in (torch.float32, torch.float64):
            pool = self._zpool[dtype] = [torch.zeros(1 << 20, dtype=dtype, device=self._device()), 0]
        if pool is None or n > (1 << 18) or pool[1] + n > pool[0].numel():
            return torch.zeros(shape, dtype=dtype, device=self._device())
        t = pool[0][pool[1]:pool[1] + n].view(shape)
        pool[1] += (n + 63) & ~63                                  # 256-byte granules keep every carve-out 16-byte aligned
        return t

    def _add_f64(self, dst, src):
        """dst (fp32 parameter gradient) += src (fp64 sums), one launch."""
        if dst.is_contiguous() and src.is_contiguous() and src.dtype == torch.float64 and dst.numel() == src.numel():
            self._check(self.lib.aero_add_f64(_ptr(dst), _ptr(src), dst.numel(), self._stream()))
        else:
            dst.add_(src.float().view_as(dst))

    def _check(self, rc):
        cabi.check(rc, self.lib)

    def grad(self, t):
        return self.g.get(id(t))

    def acc(self, t, g):
        """Accumulate g into the gradient of activation t (takes ownership of g on first use)."""
        if t is None or g is None or id(t) in self.no_grad:
            return
        cur = self.g.get(id(t))
        if cur is None:
            assert g.numel() == t.numel(), (g.shape, t.shape)
            self.g[id(t)] = g
        else:
            self._check(self.lib.aero_add(_ptr(cur), _ptr(g), cur.numel(), 1.0, self._stream()))

    def pgrad(self, name):
        t = self.pg.get(name)
        if t is None:
            if self._sink is not None:          # caller-owned, zeroed buffer (the trainer's flat gradient buffer)
                t = self._sink(name)
            else:
                t = torch.zeros_like(self.params[name], dtype=torch.float32, memory_format=torch.contiguous_format)
            self.pg[name] = t
        return t

    # ------------------------------------------------------------------ kernel wrappers
    def _tg(self, *, B, F_out, T, N, C1, C2=0, F_in=None, a1_s=None, a2_s=None, o_s=None, mode=TAPS_CONV, kf=1, kt=1, stride_f=1,
            pad_f=0, dil_t=1, pad_t=0, f_off=0, stats_mode=0, groups=1, r_s=None, cs_s=(0, 0), w_sb=0, T_in=None):
        F_in = F_out if F_in is None else F_in
        T_in = T if T_in is None else T_in

        def cl(F, C_):
            return (F * T_in * C_, T_in * C_, C_)
        a1_s = a1_s or (cl(F_in, C1) if C1 else (0, 0, 0))
        a2_s = a2_s or (cl(F_in, C2) if C2 else (0, 0, 0))
        o_s = o_s or (F_out * T * N, T * N, N)
        r_s = r_s or (0, 0, 0)
        return cabi.TapGemmParams(B, F_out, T, N, F_in, T_in, C1, C2, mode, kf, kt, stride_f, pad_f, dil_t, pad_t, f_off,
                                  ACT_NONE, 0, stats_mode, groups, *a1_s, *a2_s, w_sb, *o_s, *r_s, *cs_s, self.precision if self.precision in (1, 3) else 0, 0)

    def _gemm_call(self, p, out, w, a1=None, a2=None, bias=None, residual=None, samp_affine=None, stats=None, colscale=None, halves=None):
        """aero_tapgemm_fwd in the engine's arithmetic mode.  halves: optional dict id(tensor) -> (hi, lo) of operands already split."""
        if p.precision in (1, 3):
            # wgmma path: K-major TF32 twin [taps, pad4(N), K] of the packed weight [taps, K, pad4(N)]; shapes it does not take stay SIMT
            ok = p.w_sb == 0 and colscale is None and w.dim() == 3 and bool(self.lib.aero_tapgemm_tc_eligible(C.byref(p)))
            if ok and p.precision == 3:
                ok = self._splittable(a1, p.C1, p.a1_sb, p.a1_sf, p.a1_st, p) and self._splittable(a2, p.C2, p.a2_sb, p.a2_sf, p.a2_st, p)
            if not ok:
                p.precision = 0
            elif p.precision == 3:
                return self._gemm3(p, out, w, a1, a2, bias, residual, samp_affine, stats, halves)
            else:
                w, _ = self._pack_kmajor(w, False)
        self._launch_gemm(p, out, w, a1, a2, bias, residual, samp_affine, stats, colscale)
        return out

    def _launch_gemm(self, p, out, w, a1, a2, bias, residual, samp_affine, stats, colscale=None):
        self._check(self.lib.aero_tapgemm_fwd(_ptr(a1), _ptr(a2), _ptr(w), _ptr(bias), None, _ptr(colscale), _ptr(residual),
                                              _ptr(samp_affine), _ptr(out), _ptr(stats), C.byref(p), self._stream()))

    def _pack_kmajor(self, w, with_lo):
        wk = torch.empty(w.shape[0], w.shape[2], w.shape[1], device=w.device, dtype=torch.float32)
        wl = torch.empty_like(wk) if with_lo else None
        self._check(self.lib.aero_pack_kmajor_tf32(_ptr(w), _ptr(wk), _ptr(wl), w.shape[0], w.shape[1], w.shape[2], self._stream()))
        return wk, wl

    @staticmethod
    def _splittable(t, C_, sb, sf, st, p):
        """Can operand t (a flat buffer addressed with these strides) be replaced by its element-wise hi / lo copies?"""
        if t is None or C_ == 0:
            return True
        extent = (p.B - 1) * max(sb, 0) + (p.F_in - 1) * max(sf, 0) + (p.T_in - 1) * max(st, 0) + C_
        return t.is_contiguous() and t.dtype == torch.float32 and t.data_ptr() % 16 == 0 and extent <= t.numel()

    def _halves(self, t, cache=None):
        """(hi, lo) with hi = TF32(t), lo = TF32(t - hi), element-wise over the whole buffer."""
        if t is None:
            return None, None
        if cache is not None and id(t) in cache:
            return cache[id(t)]
        hi, lo = torch.empty_like(t), torch.empty_like(t)
        self._check(self.lib.aero_split_tf32(_ptr(t), _ptr(hi), _ptr(lo), t.numel(), self._stream()))
        if cache is not None:
            cache[id(t)] = (hi, lo)
        return hi, lo

    def _gemm3(self, p, out, w, a1, a2, bias, residual, samp_affine, stats, halves):
        """3xTF32: out = A_lo W_hi (+ residual) -> + A_hi W_lo -> + A_hi W_hi + bias, the epilogue (statistics, per-sample affine) on the
        last pass; the small terms go first so that they are not absorbed."""
        p.precision = 1
        wh, wl = self._pack_kmajor(w, True)
        h1, l1 = self._halves(a1, halves)
        h2, l2 = self._halves(a2, halves)
        t1, t2 = torch.empty_like(out), torch.empty_like(out)
        pp = cabi.TapGemmParams.from_buffer_copy(p)
        pp.stats_mode, pp.groups = 0, 1
        if residual is None:
            pp.r_sb = pp.r_sf = pp.r_st = 0
        self._launch_gemm(pp, t1, wh, l1, l2, None, residual, None, None)
        pp.r_sb, pp.r_sf, pp.r_st = p.o_sb, p.o_sf, p.o_st
        self._launch_gemm(pp, t2, wl, h1, h2, None, t1, None, None)
        p.r_sb, p.r_sf, p.r_st = p.o_sb, p.o_sf, p.o_st
        self._launch_gemm(p, out, wh, h1, h2, bias, t2, samp_affine, stats)
        return out

    def _wgrad_call(self, x1, x2, dy, gw, pw, sn, sk, ss, halves=None):
        """aero_tapgemm_wgrad in the engine's arithmetic mode (dW accumulates: the three 3xTF32 products simply add up)."""
        lib = self.lib

        def launch(a, b_, d):
            self._check(lib.aero_tapgemm_wgrad(_ptr(a), _ptr(b_), _ptr(d), _ptr(gw), C.byref(pw), sn, sk, ss, self._stream()))
        if pw.precision == 3:
            pw.precision = 1
            o_ext = (pw.B - 1) * pw.o_sb + (pw.F_out - 1) * pw.o_sf + (pw.T - 1) * pw.o_st + pw.N
            ok = bool(lib.aero_tapgemm_wgrad_tc_eligible(C.byref(pw), _ptr(x1), _ptr(x2), _ptr(dy))) and \
                self._splittable(x1, pw.C1, pw.a1_sb, pw.a1_sf, pw.a1_st, pw) and self._splittable(x2, pw.C2, pw.a2_sb, pw.a2_sf, pw.a2_st, pw) and \
                dy.is_contiguous() and o_ext <= dy.numel()
            if ok:
                h1, l1 = self._halves(x1, halves)
                h2, l2 = self._halves(x2, halves)
                dh, dl = self._halves(dy, halves)
                launch(l1, l2, dh)
                launch(h1, h2, dl)
                launch(h1, h2, dh)
                return
            pw.precision = 0
        launch(x1, x2, dy)

    def _colsum(self, x, out1, N, n_inner, inner_s, z=None, out2=None, n_outer=1, outer_s=0, n_seg=1, seg_sx=0, seg_so=0):
        dbl = (out1 if out1 is not None else out2).dtype == torch.float64
        self._check(self.lib.aero_colsum(_ptr(x), _ptr(z), _ptr(out1), _ptr(out2), 1 if dbl else 0, N, n_inner, inner_s, n_outer,
                                         outer_s, n_seg, seg_sx, seg_so, self._stream()))

    # ------------------------------------------------------------------ conv (tap-GEMM) op
    def conv(self, x1, x2, C1, C2, wname, bname, cv, B, F_in, F_out, T, N, *, wslice=None, residual=None, samp_affine=None,
             stats=None, stats_mode=0, groups=1, w_override=None, b_override=None, o_s=None, T_in=None):
        """out[B,F_out,T,N] = tap-GEMM(cat[x1 (C1 channels), x2 (C2)]) + bias (+ residual) (* samp_affine); records its backward.
        wname / bname: parameter names (PyTorch layout: Conv [N,K,kf,kt] / ConvTranspose [K,N,kf,1]); wslice: slice of the
        weight's input-channel axis actually used (decoder 0 keeps only the skip half).  w_override / b_override =
        (tensor, callback): derived weights (padded / permuted / concatenated parameters); the callback receives the
        gradient of the derived tensor and adds it to the real parameters' gradients.  o_s: output strides (b, f, t)."""
        P = self.params
        K = C1 + C2
        if w_override is not None:
            w, w_back = w_override
        else:
            w, w_back = P[wname], None
            if wslice is not None:
                w = w[:, wslice] if cv.kind == "conv" else w[wslice]
        if b_override is not None:
            bias, b_back = b_override
        else:
            bias, b_back = (P[bname] if bname else None), None
            if stats is not None and bias is not None:
                # the output feeds a GroupNorm: store it without the groups' common bias offset (engine.center_groups).  The
                # shift is piecewise constant in the bias, so the column sums below stay the bias gradient as they are.
                bias = center_groups(bias, groups if stats_mode == 1 else 1)
        if cv.kind == "conv":
            w4 = w.reshape(N, K, cv.kf, cv.kt)
            wp = pack_taps(w4.reshape(N, K, cv.kf * cv.kt))
            mode = TAPS_CONV
        else:
            w4 = w.reshape(K, N, cv.kf, 1)
            wp = pack_taps(w4[:, :, :, 0].permute(1, 0, 2))
            mode = TAPS_CONVT
        os_ = o_s or (F_out * T * N, T * N, N)
        out = self._new(B * F_out * T * N) if o_s is None else self._new(B * os_[0])
        geo = dict(B=B, F_out=F_out, T=T, N=N, C1=C1, C2=C2, F_in=F_in, mode=mode, kf=cv.kf, kt=cv.kt, stride_f=cv.stride_f, pad_f=cv.pad_f,
                   dil_t=cv.dil_t, pad_t=cv.pad_t, f_off=cv.f_off, o_s=os_, T_in=T_in)
        Ti = T if T_in is None else T_in        # input frames (differs from T only for un-padded time kernels: the discriminator's first layer)
        p = self._tg(stats_mode=stats_mode, groups=groups, r_s=os_ if residual is not None else None, **geo)
        self._gemm_call(p, out, wp, a1=x1, a2=x2, bias=bias, residual=residual, samp_affine=samp_affine, stats=stats)

        def bwd():
            dy = self.grad(out)
            if dy is None:
                return
            if samp_affine is not None:                       # out = v * std_b + mean_b  ->  dv = dy * std_b
                d2 = torch.empty_like(dy)
                self._check(self.lib.aero_scale_rows(_ptr(dy), _ptr(d2), _ptr(samp_affine), B, dy.numel() // B, 2, self._stream()))
                dy = d2
            if residual is not None:
                self.acc(residual, dy)
            halves = {} if self.precision == 3 else None          # dy is split once for the weight and the data gradient
            # ---- weight gradient, written in the parameter's own layout
            if self.param_grads:
                direct = w_back is None and wslice is None
                gw = self.pgrad(wname).view(w4.shape) if direct else torch.zeros_like(w4, memory_format=torch.contiguous_format)
                sn, sk = (gw.stride(0), gw.stride(1)) if cv.kind == "conv" else (gw.stride(1), gw.stride(0))
                pw = self._tg(**geo)
                self._wgrad_call(x1, x2, dy, gw, pw, sn, sk, 1, halves)
                if w_back is not None:
                    w_back(gw)
                elif wslice is not None:
                    full = self.pgrad(wname)
                    (full[:, wslice] if cv.kind == "conv" else full[wslice]).add_(gw.view(w.shape))
            # ---- bias gradient: column sums over every output pixel
            if bias is not None and self.param_grads:
                gb = self._new(N, zero=True, dtype=torch.float64)
                self._colsum(dy, gb, N, T, os_[2], n_outer=F_out, outer_s=os_[1], n_seg=B, seg_sx=os_[0], seg_so=0)
                if b_back is not None:
                    b_back(gb.float())
                else:
                    self._add_f64(self.pgrad(bname), gb)
            # ---- data gradients: the adjoint tap-GEMM reads dy (with the forward's output strides)
            for src, lo, cs in ((x1, 0, C1), (x2, C1, C2)):
                if src is None or cs == 0 or id(src) in self.no_grad:
                    continue
                if cv.kind == "conv":
                    ws = w4[:, lo:lo + cs]
                    if cv.stride_f == 1:
                        wd = pack_taps(ws.flip(2, 3).permute(1, 0, 2, 3).reshape(cs, N, cv.kf * cv.kt))
                        pd = self._tg(B=B, F_out=F_in, T=Ti, N=cs, C1=N, F_in=F_out, mode=TAPS_CONV, kf=cv.kf, kt=cv.kt,
                                      pad_f=cv.kf - 1 - cv.pad_f, dil_t=cv.dil_t, pad_t=cv.dil_t * (cv.kt - 1) - cv.pad_t, a1_s=os_, T_in=T)
                    else:
                        assert cv.kt == 1
                        wd = pack_taps(ws[:, :, :, 0].permute(1, 0, 2))
                        pd = self._tg(B=B, F_out=F_in, T=T, N=cs, C1=N, F_in=F_out, mode=TAPS_CONVT, kf=cv.kf, stride_f=cv.stride_f,
                                      f_off=cv.pad_f, a1_s=os_)
                else:
                    wd = pack_taps(w4[lo:lo + cs, :, :, 0])                 # [cs, N, kf] = [N', K', taps]
                    pd = self._tg(B=B, F_out=F_in, T=T, N=cs, C1=N, F_in=F_out, mode=TAPS_CONV, kf=cv.kf, stride_f=cv.stride_f,
                                  pad_f=cv.f_off, a1_s=os_)
                dx = self._new(B * F_in * Ti * cs)
                self._gemm_call(pd, dx, wd, a1=dy, halves=halves)
                self.acc(src, dx)
        self.tape.append(bwd)
        self.keep.append((x1, x2, out, residual))
        return out

    # ------------------------------------------------------------------ normalisation + activation op
    def norm_act(self, x, op, *, B, F_in, T, C_, scope, groups=1, gname=None, bname=None, stats=None, F_out=None, f_off=0, no_norm=False,
                 snake=None, scale=None, residual=None, g_override=None):
        """y = act(norm(x)); stats: fp64 {sum, sumsq} slots of the normalisation (from the producing GEMM or a column sum)."""
        P = self.params
        F_out = F_in if F_out is None else F_out
        glu = op in (NA_GLU, NA_GLU_SCALE_RES)
        Cout = C_ // 2 if glu else C_
        g_back = b_back = gamma = beta = None
        if g_override is not None:
            (gamma, g_back), (beta, b_back) = g_override
        elif not no_norm:
            gamma, beta = P[gname], P[bname]
        sa = P[snake].reshape(-1) if snake else None
        sc = P[scale] if scale else None
        y = self._new(B * F_out * T * Cout)
        p = cabi.NormActParams(B, F_in, F_out, f_off, T, C_, groups, scope, op, 1e-5, NA_NO_NORM if no_norm else 0)
        self._check(self.lib.aero_norm_act_train_fwd(_ptr(x), _ptr(stats), _ptr(gamma), _ptr(beta), _ptr(sa), _ptr(sc), _ptr(residual),
                                                     _ptr(y), C.byref(p), self._stream()))

        def bwd():
            dy = self.grad(y)
            if dy is None:
                return
            # parameter gradients are sums over every pixel whose terms largely cancel: accumulated in fp64 by the kernel
            dgamma = dbeta = dscale = dsn = None
            if not no_norm:
                dgamma, dbeta = self._new(C_, zero=True, dtype=torch.float64), self._new(C_, zero=True, dtype=torch.float64)
            if scale:
                dscale = self._new(Cout, zero=True, dtype=torch.float64)
            if snake:
                dsn = self._new(sa.numel(), zero=True, dtype=torch.float64)
            nslot = B * groups if scope == 1 else (B * F_in if scope == 2 else 1)
            ws = self._new(nslot, 2, zero=True, dtype=torch.float64)
            dx = self._new(x.numel())
            for pas in (1, 2):
                self._check(self.lib.aero_norm_act_train_bwd(_ptr(x), _ptr(stats), _ptr(gamma), _ptr(beta), _ptr(sa), _ptr(sc), _ptr(dy),
                                                             _ptr(dx), _ptr(dgamma), _ptr(dbeta), _ptr(dscale), _ptr(dsn), _ptr(ws), pas,
                                                             C.byref(p), self._stream()))
            if g_back is not None:
                g_back(dgamma.float())
                b_back(dbeta.float())
            elif not no_norm:
                self._add_f64(self.pgrad(gname), dgamma)
                self._add_f64(self.pgrad(bname), dbeta)
            if scale:
                self.pgrad(scale).add_(dscale.float().view_as(self.pgrad(scale)))
            if snake:
                self.pgrad(snake).add_(dsn.float().view_as(self.pgrad(snake)))
            self.acc(x, dx)
            if residual is not None:
                self.acc(residual, dy)
        self.tape.append(bwd)
        self.keep.append((x, y, stats, residual))
        return y

    def _batch_stats(self, x, C_, prefix, nch):
        """Per-channel batch statistics [C][2] fp64 {sum, sumsq} of a channels-last tensor; updates the BatchNorm running
        buffers of `prefix` (momentum 0.1, unbiased variance: nn.BatchNorm train-mode semantics, modules.py:287-300)."""
        n = x.numel() // C_
        s1 = self._new(C_, zero=True, dtype=torch.float64)
        s2 = self._new(C_, zero=True, dtype=torch.float64)
        self._colsum(x, s1, C_, n, C_, z=x, out2=s2)
        st = torch.stack([s1, s2], 1).contiguous()
        Bf = self.buffers
        mean = st[:nch, 0] / n
        var = (st[:nch, 1] / n - mean * mean).clamp_min(0)
        Bf[prefix + ".running_mean"].mul_(0.9).add_(0.1 * mean.float())
        Bf[prefix + ".running_var"].mul_(0.9).add_(0.1 * (var * (n / max(n - 1, 1))).float())
        Bf[prefix + ".num_batches_tracked"].add_(1)
        return st

    # ------------------------------------------------------------------ FTB (modules.py:304-325, train mode)
    def ftb(self, x, p, B, Fq, T, Cc):
        P = self.params
        q = p + ".freq_attn_block"
        dev = self._device()
        r, rp = _FTB_R, _FTB_RP
        # conv1: 1x1 C -> 5 (+BN2d+ReLU), on 8 padded channels, written as [B][T][Fq][8] (conv1d input order f*8+j)
        w8 = torch.zeros(rp, Cc, 1, 1, device=dev)
        w8[:r] = P[q + ".conv1.0.weight"]
        b8 = torch.zeros(rp, device=dev)
        b8[:r] = P[q + ".conv1.0.bias"]
        R_raw = self.conv(x, None, Cc, 0, None, None, _C1x1, B, Fq, Fq, T, rp,
                          w_override=(w8, lambda gw: self.pgrad(q + ".conv1.0.weight").add_(gw.view(rp, Cc, 1, 1)[:r])),
                          b_override=(b8, lambda gb: self.pgrad(q + ".conv1.0.bias").add_(gb[:r])), o_s=(T * Fq * rp, rp, Fq * rp))
        st1 = self._batch_stats(R_raw, rp, q + ".conv1.1", r)
        g8 = torch.ones(rp, device=dev)
        g8[:r] = P[q + ".conv1.1.weight"]
        be8 = torch.zeros(rp, device=dev)
        be8[:r] = P[q + ".conv1.1.bias"]
        R = self.norm_act(R_raw, NA_RELU, B=B, F_in=T, T=Fq, C_=rp, scope=3, stats=st1,
                          g_override=((g8, lambda g_: self.pgrad(q + ".conv1.1.weight").add_(g_[:r])),
                                      (be8, lambda g_: self.pgrad(q + ".conv1.1.bias").add_(g_[:r]))))
        # conv1d over time: 5F -> C, k9 p4, on the [B][1][T][Fq*8] view (reference channel j*F+f -> here f*8+j)
        w1d = P[q + ".conv1d.0.weight"]                                       # [C, 5F, 9]
        w1p = torch.zeros(Cc, Fq, rp, 9, device=dev)
        w1p[:, :, :r] = w1d.view(Cc, r, Fq, 9).permute(0, 2, 1, 3)
        w1p = w1p.view(Cc, Fq * rp, 1, 9)
        G_raw = self.conv(R, None, Fq * rp, 0, None, q + ".conv1d.0.bias", _Conv(kt=9, pad_t=4), B, 1, 1, T, Cc,
                          w_override=(w1p, lambda gw: self.pgrad(q + ".conv1d.0.weight").add_(
                              gw.view(Cc, Fq, rp, 9)[:, :, :r].permute(0, 2, 1, 3).reshape(Cc, r * Fq, 9))))
        st2 = self._batch_stats(G_raw, Cc, q + ".conv1d.1", Cc)
        G = self.norm_act(G_raw, NA_RELU, B=B, F_in=1, T=T, C_=Cc, scope=3, gname=q + ".conv1d.1.weight", bname=q + ".conv1d.1.bias",
                          stats=st2)
        # gated frequency mix: Y[b,f',t,c] = G[b,t,c] * sum_f Wfc[f',f] x[b,f,t,c]
        Wfc = P[q + ".freq_fc.weight"]
        M = T * Cc
        Y = self._freq_mix(x, Wfc, G, B, Fq, M)

        def mix_bwd():
            dY = self.grad(Y)
            if dY is None:
                return
            U = self._freq_mix(x, Wfc, None, B, Fq, M)                         # un-gated mix, recomputed
            dG = self._new(B * M, zero=True)
            self._colsum(dY, None, M, Fq, M, z=U, out2=dG, n_seg=B, seg_sx=Fq * M, seg_so=M)
            self.acc(G, dG)
            self.acc(x, self._freq_mix(dY, Wfc.t().contiguous(), G, B, Fq, M))
            self._check(self.lib.aero_gram(_ptr(dY), _ptr(x), _ptr(G), _ptr(self.pgrad(q + ".freq_fc.weight")), B, Fq, M, Fq * M, Fq * M,
                                           M, self._stream()))
        self.tape.append(mix_bwd)
        self.keep.append((x, G, Y))
        # conv2 on cat([Y, x]) + BN2d + ReLU
        O_raw = self.conv(Y, x, Cc, Cc, q + ".conv2.0.weight", q + ".conv2.0.bias", _C1x1, B, Fq, Fq, T, Cc)
        st3 = self._batch_stats(O_raw, Cc, q + ".conv2.1", Cc)
        self._dbg = dict(R_raw=R_raw, R=R, G_raw=G_raw, G=G, Y=Y, O_raw=O_raw, st3=st3)
        return self.norm_act(O_raw, NA_RELU, B=B, F_in=Fq, T=T, C_=Cc, scope=3, gname=q + ".conv2.1.weight", bname=q + ".conv2.1.bias",
                             stats=st3)

    def _freq_mix(self, x, Wfc, gate, B, Fq, M):
        """out[b][f'][m] = gate[b][m] * sum_f Wfc[f'][f] x[b][f][m]  (a tap-GEMM whose 'weights' are the activations)."""
        out = self._new(B * Fq * M)
        if self.precision == 1 and Fq >= 8 and Fq % 4 == 0 and M % 4 == 0:
            # TF32 mode: contraction over the row axis on the tensor cores, activations as the MN-major operand (AERO_TAPS_MIX, as the
            # inference engine does); the weight is its own K-major form [F', F]
            p = self._tg(B=B, F_out=1, T=M, N=Fq, C1=Fq, mode=cabi.TAPS_MIX, a1_s=(Fq * M, 0, M), o_s=(Fq * M, 0, M),
                         cs_s=(M, 0) if gate is not None else (0, 0))
            p.precision = 1
            self._check(self.lib.aero_tapgemm_fwd(_ptr(x), None, _ptr(tf32_round(Wfc.contiguous())), None, None, _ptr(gate), None, None, _ptr(out),
                                                  None, C.byref(p), self._stream()))
            return out
        p = self._tg(B=B, F_out=1, T=Fq, T_in=Fq, N=M, C1=Fq, a1_s=(0, 0, Fq), w_sb=Fq * M, o_s=(Fq * M, 0, M),
                     cs_s=(M, 0) if gate is not None else (0, 0))
        self._gemm_call(p, out, x, a1=Wfc.contiguous(), colscale=gate)
        return out

    # ------------------------------------------------------------------ BLSTM (modules.py:32-65)
    def blstm(self, h, q, rows, T, H):
        """h [rows][T][H] -> h + Linear(BiLSTM_2(frames(h)))."""
        P, lib = self.params, self.lib
        if T > _LSTM_MAX_STEPS:
            steps, stride = _LSTM_MAX_STEPS, _LSTM_MAX_STEPS // 2
            n_win = math.ceil(T / stride)
        else:
            steps, stride, n_win = T, 0, 1
        n_seq = rows * n_win
        G = 8 * H
        lp = q + ".lstm.lstm."
        x_in, kin, npix = h, H, rows * T
        for layer in range(2):
            names = [f"{lp}weight_ih_l{layer}", f"{lp}weight_ih_l{layer}_reverse"]
            wih = torch.cat([P[n] for n in names], 0).contiguous()                                         # [8H, in]
            bnames = [f"{lp}bias_ih_l{layer}", f"{lp}bias_hh_l{layer}", f"{lp}bias_ih_l{layer}_reverse", f"{lp}bias_hh_l{layer}_reverse"]
            bias = torch.cat([P[bnames[0]] + P[bnames[1]], P[bnames[2]] + P[bnames[3]]]).contiguous()
            whh_names = [f"{lp}weight_hh_l{layer}", f"{lp}weight_hh_l{layer}_reverse"]
            whh = torch.stack([P[n] for n in whh_names]).contiguous()

            def w_back(gw, names=names):
                gw = gw.view(G, -1)
                self.pgrad(names[0]).add_(gw[:4 * H])
                self.pgrad(names[1]).add_(gw[4 * H:])

            def b_back(gb, bnames=bnames):
                for i, n in enumerate(bnames):
                    self.pgrad(n).add_(gb[(i // 2) * 4 * H:(i // 2 + 1) * 4 * H])
            gin = self.conv(x_in, None, kin, 0, None, None, _C1x1, 1, 1, 1, npix, G, w_override=(wih, w_back), b_override=(bias, b_back))
            gates_s, c_s, h_s = self._new(n_seq * steps * G), self._new(n_seq * steps * 2 * H), self._new(n_seq * steps * 2 * H)
            lpar = cabi.LstmParams(rows, T, H, n_win, steps, stride, 1 if layer == 1 else 0, 1 if layer == 0 else 0, 0, 0)
            hout = None if layer == 0 else self._new(rows * T * 2 * H)
            self._check(lib.aero_lstm_train_fwd(_ptr(gin), _ptr(bias), _ptr(whh), _ptr(hout), _ptr(gates_s), _ptr(c_s), _ptr(h_s),
                                                C.byref(lpar), self._stream()))
            out_l = h_s if layer == 0 else hout

            def rec_bwd(layer=layer, gin=gin, whh=whh, whh_names=whh_names, bnames=bnames, gates_s=gates_s, c_s=c_s, h_s=h_s, lpar=lpar,
                        out_l=out_l):
                d_out = self.grad(out_l)
                if d_out is None:
                    return
                dgin_w = self._new(n_seq * steps * G)
                self._check(lib.aero_lstm_bwd(_ptr(d_out), _ptr(gates_s), _ptr(c_s), _ptr(whh), _ptr(dgin_w), C.byref(lpar), self._stream()))
                for d in range(2):
                    # W_hh: dW[g][j] = sum dgates[pos][g] * h[pos -/+ 1][j] inside each window
                    pw = self._tg(B=1, F_out=n_seq, T=steps, N=4 * H, C1=H, F_in=n_seq, a1_s=(0, steps * 2 * H, 2 * H),
                                  o_s=(0, steps * G, G), pad_t=(1 if d == 0 else -1))
                    self._check(lib.aero_tapgemm_wgrad(C.c_void_p(h_s.data_ptr() + 4 * d * H), None,
                                                       C.c_void_p(dgin_w.data_ptr() + 4 * d * 4 * H), _ptr(self.pgrad(whh_names[d])),
                                                       C.byref(pw), H, 1, 1, self._stream()))
                if layer == 0 and n_win > 1:
                    # un-windowed input: sum the overlapping windows back onto the frames; positions beyond T are zero
                    # input with the bias only, so the bias also collects what the fold drops
                    dgin = self._new(rows * T * G)
                    self._check(lib.aero_lstm_fold(_ptr(dgin_w), _ptr(dgin), rows, T, n_win, steps, stride, G, self._stream()))
                    g_all, g_real = self._new(G, zero=True, dtype=torch.float64), self._new(G, zero=True, dtype=torch.float64)
                    self._colsum(dgin_w, g_all, G, n_seq * steps, G)
                    self._colsum(dgin, g_real, G, rows * T, G)
                    extra = (g_all - g_real).float()
                    for i, n in enumerate(bnames):
                        self.pgrad(n).add_(extra[(i // 2) * 4 * H:(i // 2 + 1) * 4 * H])
                else:
                    dgin = dgin_w
                self.acc(gin, dgin)
            self.tape.append(rec_bwd)
            self.keep.append((gin, out_l, gates_s, c_s, h_s))
            x_in, kin, npix = out_l, 2 * H, (n_seq * steps if layer == 0 else rows * T)
        return self.conv(x_in, None, 2 * H, 0, q + ".lstm.linear.weight", q + ".lstm.linear.bias", _C1x1, 1, 1, 1, rows * T, H, residual=h)

    # ------------------------------------------------------------------ LocalState (modules.py:94-127)
    def local_attn(self, h, q, rows, T, H):
        P, lib = self.params, self.lib
        a = q + ".time_attn"
        names = ("query", "key", "content", "query_decay")
        ld = 3 * H + _ATTN_HEADS * _ATTN_NDECAY
        w = torch.cat([P[f"{a}.{n}.weight"] for n in names], 0).contiguous()          # [ld, H, 1]
        b = torch.cat([P[f"{a}.{n}.bias"] for n in names]).contiguous()
        sizes = [H, H, H, _ATTN_HEADS * _ATTN_NDECAY]

        def w_back(gw):
            o = 0
            for n, s_ in zip(names, sizes):
                self.pgrad(f"{a}.{n}.weight").add_(gw.view(ld, H, 1)[o:o + s_])
                o += s_

        def b_back(gb):
            o = 0
            for n, s_ in zip(names, sizes):
                self.pgrad(f"{a}.{n}.bias").add_(gb[o:o + s_])
                o += s_
        qkvd = self.conv(h, None, H, 0, None, None, _C1x1, 1, 1, 1, rows * T, ld, w_override=(w, w_back), b_override=(b, b_back))
        out, lse = self._new(rows * T * H), self._new(rows * _ATTN_HEADS * T)
        ap = cabi.AttnParams(rows, T, H, _ATTN_HEADS, _ATTN_NDECAY, ld, 0)
        self._check(lib.aero_local_attn_train_fwd(_ptr(qkvd), _ptr(out), _ptr(lse), C.byref(ap), self._stream()))

        def bwd():
            dout = self.grad(out)
            if dout is None:
                return
            dq = self._new(rows * T * ld)
            self._check(lib.aero_local_attn_bwd(_ptr(qkvd), _ptr(out), _ptr(lse), _ptr(dout), _ptr(dq), C.byref(ap), self._stream()))
            self.acc(qkvd, dq)
        self.tape.append(bwd)
        self.keep.append((qkvd, out, lse))
        return self.conv(out, None, H, 0, a + ".proj.weight", a + ".proj.bias", _C1x1, 1, 1, 1, rows * T, H, residual=h)

    # ------------------------------------------------------------------ DConv (modules.py:221-249)
    def dconv(self, y, g, B, T):
        kw = self.geom.kw
        Fq, Cc = g.f_out, g.ch
        hid = int(Cc / kw["dconv_comp"])
        rows = B * Fq
        act = dconv_norm_act_op(kw["act_func"])
        for d in range(abs(kw["dconv_depth"])):
            q = f"encoder.{g.index}.dconv.layers.{d}"
            dil = 2 ** d if kw["dconv_depth"] > 0 else 1
            st1 = self._new(rows, 2, zero=True, dtype=torch.float64)
            h_raw = self.conv(y, None, Cc, 0, q + ".conv1.0.weight", q + ".conv1.0.bias", _Conv(kt=3, dil_t=dil, pad_t=dil), B, Fq, Fq, T, hid,
                              stats=st1, stats_mode=2)
            h = self.norm_act(h_raw, act, B=B, F_in=Fq, T=T, C_=hid, scope=2, gname=q + ".conv1.1.weight", bname=q + ".conv1.1.bias",
                              stats=st1, snake=q + ".act.a" if act == NA_SNAKE else None)
            if g.lstm:
                h = self.blstm(h, q, rows, T, hid)
            if g.attn:
                h = self.local_attn(h, q, rows, T, hid)
            st2 = self._new(rows, 2, zero=True, dtype=torch.float64)
            u = self.conv(h, None, hid, 0, q + ".conv2.0.weight", q + ".conv2.0.bias", _C1x1, B, Fq, Fq, T, 2 * Cc, stats=st2, stats_mode=2)
            y = self.norm_act(u, NA_GLU_SCALE_RES, B=B, F_in=Fq, T=T, C_=2 * Cc, scope=2, gname=q + ".conv2.1.weight",
                              bname=q + ".conv2.1.bias", stats=st2, scale=q + ".conv2.3.scale", residual=y)
        return y

    # ------------------------------------------------------------------ encoder / decoder layers
    def encode(self, x, g, B, T):
        """reference aero.py:108-135 (+ the frequency-embedding add aero.py:475-480 for layer 0)."""
        kw = self.geom.kw
        P = self.params
        p = f"encoder.{g.index}"
        Fi, Fo, Cc = g.f_in, g.f_out, g.ch
        cin = g.enc_cin
        ng = kw["norm_groups"]
        if g.index == 0:
            x = self.conv(x, None, cin, 0, p + ".pre_conv.weight", p + ".pre_conv.bias", _C1x1, B, Fi, Fi, T, Cc)
            cin = Cc
        if g.ftb:
            x = self.ftb(x, p, B, Fi, T, cin)
        cv = _Conv(kf=g.kernel, stride_f=g.stride, pad_f=g.pad)
        if g.norm:
            st = self._new(B * ng, 2, zero=True, dtype=torch.float64)
            y_raw = self.conv(x, None, cin, 0, p + ".conv.weight", p + ".conv.bias", cv, B, Fi, Fo, T, Cc, stats=st, stats_mode=1, groups=ng)
            y = self.norm_act(y_raw, NA_GELU, B=B, F_in=Fo, T=T, C_=Cc, scope=1, groups=ng, gname=p + ".norm1.weight", bname=p + ".norm1.bias",
                              stats=st)
        else:
            y_raw = self.conv(x, None, cin, 0, p + ".conv.weight", p + ".conv.bias", cv, B, Fi, Fo, T, Cc)
            y = self.norm_act(y_raw, NA_GELU, B=B, F_in=Fo, T=T, C_=Cc, scope=1, no_norm=True)
        if g.dconv:
            y = self.dconv(y, g, B, T)
        if g.norm:
            st = self._new(B * ng, 2, zero=True, dtype=torch.float64)
            raw = self.conv(y, None, Cc, 0, p + ".rewrite.weight", p + ".rewrite.bias", _C1x1, B, Fo, Fo, T, 2 * Cc, stats=st, stats_mode=1,
                            groups=ng)
            out = self.norm_act(raw, NA_GLU, B=B, F_in=Fo, T=T, C_=2 * Cc, scope=1, groups=ng, gname=p + ".norm2.weight",
                                bname=p + ".norm2.bias", stats=st)
        else:
            raw = self.conv(y, None, Cc, 0, p + ".rewrite.weight", p + ".rewrite.bias", _C1x1, B, Fo, Fo, T, 2 * Cc)
            out = self.norm_act(raw, NA_GLU, B=B, F_in=Fo, T=T, C_=2 * Cc, scope=1, no_norm=True)
        if g.index == 0 and kw["freq_emb"]:
            k = float(kw["emb_scale"] * kw["freq_emb"])
            emb = (P["freq_emb.embedding.weight"] * k).contiguous()
            self._check(self.lib.aero_bcast_add(_ptr(out), _ptr(emb), B, Fo, T, Cc, self._stream()))

            def emb_bwd():
                dy = self.grad(out)
                if dy is None:
                    return
                ge = self._new(Fo * Cc, zero=True, dtype=torch.float64)
                self._colsum(dy, ge, Cc, T, Cc, n_outer=B, outer_s=Fo * T * Cc, n_seg=Fo, seg_sx=T * Cc, seg_so=Cc)
                self.pgrad("freq_emb.embedding.weight").add_((ge.view(Fo, Cc) * k).float())
            self.tape.append(emb_bwd)
        return out

    def decode(self, x, skip, g, j, B, T, last, samp_affine):
        """reference aero.py:189-215."""
        kw = self.geom.kw
        p = f"decoder.{j}"
        Fq, Cc = g.f_out, g.ch
        ng = kw["norm_groups"]
        c1 = 0 if x is None else Cc
        wslice = slice(Cc, 2 * Cc) if x is None else None            # decoder input starts at zero (aero.py:484): only the skip half acts
        cv = _Conv(kf=3, kt=3, pad_f=1, pad_t=1)
        if g.norm:
            st = self._new(B * ng, 2, zero=True, dtype=torch.float64)
            raw = self.conv(x, skip, c1, Cc, p + ".rewrite.weight", p + ".rewrite.bias", cv, B, Fq, Fq, T, 4 * Cc, wslice=wslice, stats=st,
                            stats_mode=1, groups=ng)
            y = self.norm_act(raw, NA_GLU, B=B, F_in=Fq, T=T, C_=4 * Cc, scope=1, groups=ng, gname=p + ".norm1.weight", bname=p + ".norm1.bias",
                              stats=st)
        else:
            raw = self.conv(x, skip, c1, Cc, p + ".rewrite.weight", p + ".rewrite.bias", cv, B, Fq, Fq, T, 4 * Cc, wslice=wslice)
            y = self.norm_act(raw, NA_GLU, B=B, F_in=Fq, T=T, C_=4 * Cc, scope=1, no_norm=True)
        cout = g.dec_cout
        f_full = (Fq - 1) * g.stride + g.kernel
        f_keep = f_full - 2 * g.pad
        if g.norm:
            st = self._new(B * ng, 2, zero=True, dtype=torch.float64)
            raw = self.conv(y, None, 2 * Cc, 0, p + ".conv_tr.weight", p + ".conv_tr.bias", _Conv("convt", kf=g.kernel, stride_f=g.stride),
                            B, Fq, f_full, T, cout, stats=st, stats_mode=1, groups=ng)
            if last:
                raise NotImplementedError("GroupNorm on the last decoder layer (norm_starts=0) is not supported")
            return self.norm_act(raw, NA_GELU, B=B, F_in=f_full, F_out=f_keep, f_off=g.pad, T=T, C_=cout, scope=1, groups=ng,
                                 gname=p + ".norm2.weight", bname=p + ".norm2.bias", stats=st)
        z = self.conv(y, None, 2 * Cc, 0, p + ".conv_tr.weight", p + ".conv_tr.bias",
                      _Conv("convt", kf=g.kernel, stride_f=g.stride, f_off=g.pad), B, Fq, f_keep, T, cout,
                      samp_affine=samp_affine if last else None)
        return z if last else self.norm_act(z, NA_GELU, B=B, F_in=f_keep, T=T, C_=cout, scope=1, no_norm=True)

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, mix):
        """Training-mode forward; returns (waveform [B, C_out, L*scale], output spectrogram [B, Fq, T, 2 C_out] as real pairs)."""
        self._reset()
        model, g, lib = self.model, self.geom, self.lib
        kw = g.kw
        self.params = {k: v.detach() for k, v in model.named_parameters()}
        self.buffers = dict(model.named_buffers())
        for k, v in self.params.items():
            if not v.is_contiguous():
                self.params[k] = v.contiguous()
        if mix.dim() != 3 or mix.shape[1] != kw["in_channels"]:
            raise ValueError(f"expected input [B, {kw['in_channels']}, L], got {tuple(mix.shape)}")
        B, Cin, length = mix.shape
        x = mix.contiguous().float()
        if length % g.hop_in:
            x = torch.nn.functional.pad(x, (0, g.hop_in - length % g.hop_in))
        Lp = x.shape[-1]
        T = 1 + Lp // g.hop_in
        Fq = g.nfft // 2
        C2 = 2 * Cin
        # STFT straight into channels-last [B, F, T, 2*Cin] (aero.py:409-434) + per-sample standardisation (aero.py:462-464)
        z = self._new(B, Fq, T, C2)
        st_in = self._new(B, 2, zero=True, dtype=torch.float64)
        spec.stft_into(x.view(B * Cin, Lp), z, st_in, n_fft=g.nfft, hop=g.hop_in, win=g.win_in, channels=Cin, bins_out=Fq,
                       strides=(Fq * T * C2, 2, T * C2, C2), stream=self._stream())
        xn = self._new(B, Fq, T, C2)
        affine = self._new(B, 2)
        self._check(lib.aero_sample_norm_fwd(_ptr(z), _ptr(st_in), _ptr(xn), _ptr(affine), B, Fq * T * C2, Fq * T * C2, 0, self._stream()))
        self.no_grad.add(id(xn))
        h = xn
        saved = []
        for lg in g.layers:
            h = self.encode(h, lg, B, T)
            saved.append(h)
            self.marks.append((len(self.tape), f"encoder.{lg.index}"))
        h = None
        for j, lg in enumerate(reversed(g.layers)):
            h = self.decode(h, saved.pop(), lg, j, B, T, lg.index == 0, affine)
            self.marks.append((len(self.tape), f"decoder.{j}"))
        Cout = kw["out_channels"]
        out_len = min(int(length * g.scale), g.hop_out * (T - 1))
        y = self._new(B * Cout, out_len)
        spec.istft_into(h, y, n_fft=g.nfft, hop=g.hop_out, win=g.win_out, channels=Cout, frames=T, bins_in=Fq,
                        strides=(Fq * T * 2 * Cout, 2, T * 2 * Cout, 2 * Cout), stream=self._stream())
        self._final = (h, B, Cout, T, Fq, out_len)
        self.keep.append((z, xn, affine, x))
        return y.view(B, Cout, out_len), h.view(B, Fq, T, 2 * Cout)

    # ------------------------------------------------------------------ backward
    @torch.no_grad()
    def istft_adjoint(self, d_wave, B, Cout, T, Fq, out_len):
        """Gradient of the output spectrogram [B, Fq, T, 2 C_out] from the gradient of the waveform (the adjoint of
        aero_istft_fwd, aero_b200.spec.istft_adjoint_into)."""
        g = self.geom
        dz = self._new(B, Fq, T, 2 * Cout)
        spec.istft_adjoint_into(d_wave.reshape(B * Cout, out_len), dz, n_fft=g.nfft, hop=g.hop_out, win=g.win_out, channels=Cout,
                                frames=T, bins=Fq, strides=(Fq * T * 2 * Cout, 2, T * 2 * Cout, 2 * Cout), stream=self._stream())
        return dz

    @torch.no_grad()
    def backward(self, d_wave, d_spec=None, grad_sink=None, on_layer_done=None):
        """d_wave: gradient of the waveform [B, C_out, out_len] (or None); d_spec: gradient of the output spectrogram as real
        pairs [B, Fq, T, 2 C_out] (or None).  Returns {parameter name: gradient}.
        grad_sink(name) -> zeroed tensor to accumulate that parameter's gradient into (else fresh tensors);
        on_layer_done(tag) is called when every gradient of layer `tag` ("decoder.3", ..., "encoder.0") is final."""
        self._sink = grad_sink
        self._sync_stream()
        lib, g = self.lib, self.geom
        h, B, Cout, T, Fq, out_len = self._final
        dz = self.istft_adjoint(d_wave, B, Cout, T, Fq, out_len) if d_wave is not None else None
        if d_spec is not None:
            ds = d_spec.contiguous().float().clone()
            dz = ds if dz is None else dz.add_(ds.view_as(dz))
        if dz is None:
            return {}
        self.acc(h, dz)
        starts = {0: None}
        prev = 0
        for end, tag in self.marks:                       # layer `tag` owns tape[prev:end]; it is done once tape[prev] has run
            starts[prev] = tag
            prev = end
        for i in range(len(self.tape) - 1, -1, -1):
            self.tape[i]()
            if on_layer_done is not None and starts.get(i) is not None:
                on_layer_done(starts[i])
        grads = self.pg
        self._reset()
        return grads
