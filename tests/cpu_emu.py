"""CPU emulation of the libaero_b200 kernel CONTRACTS  --  test infrastructure only.

``EmuEngine`` subclasses the product's ``AeroEngine`` and replaces the seven kernel wrappers with
straightforward torch-CPU statements of what ``include/aero_b200.h`` says each entry point computes
(same argument meaning, strides, window bookkeeping, statistics slots).  Running the *unchanged*
host logic (weight packing, launch sequence, buffer plumbing) on top of it and comparing with the
oracle validates the host side without a GPU.  It is never imported by the product.
"""
import math

import torch
import torch.nn.functional as F

from aero_b200 import cabi
from aero_b200.engine import AeroEngine


def _view(t, sizes, strides):
    return torch.as_strided(t.reshape(-1), sizes, strides, storage_offset=0) if t is not None else None


class EmuEngine(AeroEngine):
    def __init__(self, model):
        self._init_state(model, None)
        self.precision = 0
        self.lstm_tc = False          # the emulation states the recurrence in PyTorch's gate layout
        self.use_graph = False
        self.calls = []

    def _on_device(self):
        import contextlib
        return contextlib.nullcontext()

    def _require(self, x):
        pass

    def _stream(self):
        return None

    # ---- aero_tapgemm_fwd
    def _gemm(self, out, w, *, B, F_out, T, N, C1, a1=None, a2=None, C2=0, F_in=None, T_in=None,
              a1_s=None, a2_s=None, o_s=None, mode=cabi.TAPS_CONV, kf=1, kt=1, stride_f=1, pad_f=0, dil_t=1, pad_t=0,
              f_off=0, bias=None, act=cabi.ACT_NONE, glu=0, stats=None, stats_mode=0, groups=1, addend=None,
              colscale=None, cs_s=(0, 0), residual=None, r_s=None, samp_affine=None, w_sb=0, tag=None, rnd=False):
        self.calls.append(("tapgemm", N, C1 + C2))
        if mode == cabi.TAPS_MIX:
            # out[b][n][m] = colscale[b][m] * sum_k a1[b][k][m] * W[n][k]   (w: K-major twin, rows possibly padded)
            Av = torch.as_strided(a1.reshape(-1), (B, C1, T), (a1_s[0], a1_s[2], 1)).double()
            v = torch.einsum("nk,bkm->bnm", w.reshape(N, -1)[:, :C1].double(), Av)
            if colscale is not None:
                v = v * torch.as_strided(colscale.reshape(-1), (B, 1, T), (cs_s[0], 0, 1)).double()
            torch.as_strided(out.reshape(-1), (B, N, T), (o_s[0], o_s[2], 1)).copy_(v)
            return out
        F_in = F_out if F_in is None else F_in
        T_in = T if T_in is None else T_in
        n_out = N // 2 if glu else N
        K = C1 + C2

        def cl(F_, C_):
            return (F_ * T_in * C_, T_in * C_, C_)
        a1_s = a1_s or (cl(F_in, C1) if a1 is not None else (0, 0, 0))
        a2_s = a2_s or (cl(F_in, C2) if a2 is not None else (0, 0, 0))
        o_s = o_s or (F_out * T * n_out, T * n_out, n_out)
        r_s = r_s or (o_s if residual is not None else (0, 0, 0))
        srcs = []
        if C1:
            srcs.append(_view(a1, (B, F_in, T_in, C1), (*a1_s, 1)))
        if C2:
            srcs.append(_view(a2, (B, F_in, T_in, C2), (*a2_s, 1)))
        A = torch.cat(srcs, -1).double()                                   # [B, F_in, T_in, K]
        ldw = (N + 3) & ~3
        ntaps = kf * kt if mode == cabi.TAPS_CONV else kf // stride_f
        nslab = kf * kt if mode == cabi.TAPS_CONV else kf
        if w_sb:
            Wm = torch.as_strided(w.reshape(-1), (B, nslab, K, N), (w_sb, K * ldw, ldw, 1)).double()
        else:
            Wm = torch.as_strided(w.reshape(-1), (1, nslab, K, N), (0, K * ldw, ldw, 1)).double().expand(B, -1, -1, -1)
        acc = torch.zeros(B, F_out, T, N, dtype=torch.float64, device=A.device)     # runs wherever its inputs live
        for fo in range(F_out):
            for tap in range(ntaps):
                if mode == cabi.TAPS_CONV:
                    jf, jt = divmod(tap, kt)
                    fi, dt, slab = fo * stride_f + jf - pad_f, jt * dil_t - pad_t, tap
                else:
                    fof = fo + f_off
                    fi, dt, slab = fof // stride_f - tap, 0, fof % stride_f + tap * stride_f
                if fi < 0 or fi >= F_in:
                    continue
                lo, hi = max(0, -dt), min(T, T_in - dt)                  # output t with valid input t+dt
                if hi <= lo:
                    continue
                acc[:, fo, lo:hi] += torch.einsum("btk,bkn->btn", A[:, fi, lo + dt:hi + dt], Wm[:, slab])
        v = acc
        if bias is not None:
            v = v + bias.double()[:N]
        if colscale is not None:
            v = v * _view(colscale, (B, 1, T, N), (cs_s[0], 0, cs_s[1], 1)).double()
        if act == cabi.ACT_GELU:
            v = 0.5 * v * (1 + torch.erf(v / math.sqrt(2)))
        elif act == cabi.ACT_RELU:
            v = v.clamp_min(0)
        if glu:
            v = v[..., 0::2] * torch.sigmoid(v[..., 1::2])
        if addend is not None:
            v = v + addend.double().reshape(F_out, n_out)[None, :, None, :]
        if residual is not None:
            v = v + _view(residual, (B, F_out, T, n_out), (*r_s, 1)).double()
        if samp_affine is not None:
            v = v * samp_affine.double()[:, 0].view(B, 1, 1, 1) + samp_affine.double()[:, 1].view(B, 1, 1, 1)
        _view(out, (B, F_out, T, n_out), (*o_s, 1)).copy_(v)              # one rounding, to the output's storage type
        vf = _view(out, (B, F_out, T, n_out), (*o_s, 1))                   # statistics describe the values as stored (FP16 raws)
        if stats_mode == 1:
            g = vf.double().view(B, F_out * T, groups, n_out // groups)
            stats[:, 0] += g.sum((1, 3)).reshape(-1)
            stats[:, 1] += (g * g).sum((1, 3)).reshape(-1)
        elif stats_mode == 2:
            g = vf.double().view(B * F_out, -1)
            stats[:, 0] += g.sum(1)
            stats[:, 1] += (g * g).sum(1)
        return out

    # ---- aero_norm_act_fwd
    def _norm_act(self, x, stats, gamma, beta, y, *, B, F_in, T, C_, groups, scope, op, F_out=None, f_off=0,
                  snake_a=None, scale=None, residual=None, rnd=False):
        self.calls.append(("norm_act", op))
        F_out = F_in if F_out is None else F_out
        xv = x.reshape(B, F_in, T, C_).double()
        gw = C_ // groups
        if scope == 1:
            n = F_in * T * gw
            mean = (stats[:, 0] / n).view(B, 1, 1, groups, 1)
            var = (stats[:, 1] / n).view(B, 1, 1, groups, 1) - mean * mean
        else:
            n = T * C_
            mean = (stats[:, 0] / n).view(B, F_in, 1, 1, 1)
            var = (stats[:, 1] / n).view(B, F_in, 1, 1, 1) - mean * mean
        g = (xv.view(B, F_in, T, groups, gw) - mean) / torch.sqrt(var.clamp_min(0) + 1e-5)
        g = g.view(B, F_in, T, C_) * gamma.double() + beta.double()
        g = g[:, f_off:f_off + F_out]
        if op == cabi.NA_GELU:
            o = 0.5 * g * (1 + torch.erf(g / math.sqrt(2)))
        elif op in (cabi.NA_GLU, cabi.NA_GLU_SCALE_RES):
            o = g[..., :C_ // 2] * torch.sigmoid(g[..., C_ // 2:])
            if op == cabi.NA_GLU_SCALE_RES:
                o = residual.reshape(B, F_out, T, C_ // 2).double() + scale.double() * o
        elif op == cabi.NA_SNAKE:
            a = snake_a.double()[f_off:f_off + F_out].view(1, F_out, 1, 1)
            o = g + torch.sin(g * a) ** 2 / a
        else:
            o = g
        y.reshape(-1)[:o.numel()].copy_(o.float().reshape(-1))
        return y

    # ---- aero_lstm_rec_fwd
    def _lstm_rec(self, gin, bias_pad, whh, hout, *, rows, T, H, n_win, steps, stride, in_windowed, out_windowed,
                  tc=False):
        self.calls.append(("lstm", H))
        G = 4 * H
        n_seq = rows * n_win
        if in_windowed:
            gi = gin.reshape(n_seq, steps, 2, G)
        else:
            g0 = gin.reshape(rows, T, 2 * G)
            pad_len = (n_win - 1) * stride + steps if n_win > 1 else steps
            padded = bias_pad.view(1, 1, 2 * G).expand(rows, pad_len, 2 * G).clone()
            padded[:, :T] = g0
            if n_win > 1:
                gi = padded.unfold(1, steps, stride).permute(0, 1, 3, 2).reshape(n_seq, steps, 2, G)
            else:
                gi = padded.reshape(n_seq, steps, 2, G)
        out = torch.zeros(n_seq, steps, 2, H)
        for d in range(2):
            h = torch.zeros(n_seq, H)
            c = torch.zeros(n_seq, H)
            order = range(steps - 1, -1, -1) if d else range(steps)
            for t in order:
                g = gi[:, t, d] + h @ whh[d].t()
                i, f, gg, o = g.chunk(4, -1)
                c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
                h = torch.sigmoid(o) * torch.tanh(c)
                out[:, t, d] = h
        if out_windowed:
            hout.reshape(-1)[:out.numel()].copy_(out.reshape(-1))
            return
        dst = hout.reshape(rows, T, 2 * H)
        o4 = out.reshape(rows, n_win, steps, 2 * H)
        half = stride // 2
        for k in range(n_win):
            lo = 0 if k == 0 else half
            hi = steps if k == n_win - 1 else steps - half
            f0 = k * stride + lo
            f1 = min(k * stride + hi, T)
            if f1 > f0:
                dst[:, f0:f1] = o4[:, k, lo:lo + (f1 - f0)]

    # ---- aero_local_attn_fwd
    def _attn(self, qkvd, out, *, rows, T, H, heads, ndecay, ld):
        self.calls.append(("attn", H))
        d = H // heads
        m = qkvd.reshape(rows, T, ld).double()
        q = m[..., :H].view(rows, T, heads, d)
        k = m[..., H:2 * H].view(rows, T, heads, d)
        v = m[..., 2 * H:3 * H].view(rows, T, heads, d)
        dq = torch.sigmoid(m[..., 3 * H:3 * H + heads * ndecay].view(rows, T, heads, ndecay)) / 2
        slope = (dq * torch.arange(1, ndecay + 1, dtype=torch.float64)).sum(-1) / math.sqrt(ndecay)   # [rows, s, h]
        idx = torch.arange(T, dtype=torch.float64)
        dist = (idx[:, None] - idx[None, :]).abs()
        sc = torch.einsum("rthc,rshc->rhts", k, q) / math.sqrt(d) - dist * slope.permute(0, 2, 1)[:, :, None, :]
        sc.masked_fill_(torch.eye(T, dtype=torch.bool), -100.0)
        w = torch.softmax(sc, dim=2)
        r = torch.einsum("rhts,rthc->rshc", w, v).reshape(rows * T, H)
        out.reshape(-1)[:r.numel()].copy_(r.float().reshape(-1))

    # ---- aero_sample_norm_fwd
    def _sample_norm(self, x, stats, y, affine, B, per_sample, extent=None, rnd=False):
        self.calls.append(("sample_norm",))
        n = float(per_sample)
        mean = stats[:B, 0] / n
        var = (stats[:B, 1] - n * mean * mean) / (n - 1)
        sd = var.clamp_min(0).sqrt()
        xv = x.reshape(B, -1).double()
        y.reshape(B, -1).copy_(((xv - mean[:, None]) / (1e-5 + sd[:, None])).float())
        affine[:, 0] = sd.float()
        affine[:, 1] = mean.float()

    # ---- aero_freq_mix_small_fwd
    def _freq_mix_small(self, x, Wfc, gate, out, *, B, F, M):
        self.calls.append(("freq_mix_small", F))
        v = torch.einsum("gf,bfm->bgm", Wfc.double(), x.reshape(B, F, M).double()) * gate.reshape(B, 1, M).double()
        out.copy_(v.reshape(out.shape).float())
        return out

    # ---- aero_ftb_lin_squeeze_fwd
    def _ftb_lin_squeeze(self, z, W1p, b1p, R, *, B, F, T, J, r, zrow):
        self.calls.append(("ftb_lin_squeeze",))
        zv = z.reshape(B, F, zrow)[:, :, :T * J].reshape(B, F, T, J).double()
        x = (torch.einsum("nj,bftj->btfn", W1p.double(), zv) + b1p.double()).clamp_min(0)
        R.copy_(x.reshape(B, T, F * r).float())
        return R

    # ---- aero_ftb_lin_out_fwd
    def _ftb_lin_out(self, z, zm, M, s, V, d, out, *, B, F, T, N, J, zrow):
        self.calls.append(("ftb_lin_out",))
        zv = z.reshape(B, F, zrow)[:, :, :T * J].reshape(B, F, T, J).double()
        zmv = zm.reshape(B, F, zrow)[:, :, :T * J].reshape(B, F, T, J).double()
        Mv = M.reshape(B, T, N, J + 1).double()
        x = torch.einsum("btnj,bftj->bftn", Mv[..., :J], zmv) + Mv[..., J][:, None] * s.double()[None, :, None, None]
        x = x + torch.einsum("nj,bftj->bftn", V.double(), zv) + d.double()
        out.copy_(x.clamp_min(0).float())
        return out

    # ---- aero_stft_fwd / aero_istft_fwd
    def stft_into(self, x, z, stats, *, n_fft, hop, win, channels, bins_out, strides):
        self.calls.append(("stft",))
        n_sig, length = x.shape
        w = F.pad(self._window(win), ((n_fft - win) // 2, n_fft - win - (n_fft - win) // 2))
        xp = F.pad(x[:, None], (n_fft // 2, n_fft // 2), mode="reflect")[:, 0]
        fr = xp.unfold(-1, n_fft, hop)
        zz = torch.fft.rfft(fr.double() * w.double(), dim=-1) * n_fft ** -0.5     # [sig, T, bins]
        zz = zz[..., :bins_out].transpose(1, 2)                                     # [sig, bins, T]
        frames = zz.shape[-1]
        B = n_sig // channels
        sb, sc, sk, st = strides
        dst = torch.as_strided(z.reshape(-1), (B, channels, bins_out, frames, 2), (sb, sc, sk, st, 1))
        val = torch.view_as_real(zz).float().view(B, channels, bins_out, frames, 2)
        dst.copy_(val)
        if stats is not None:
            stats[:B, 0] += val.double().sum((1, 2, 3, 4))
            stats[:B, 1] += (val.double() ** 2).sum((1, 2, 3, 4))

    def istft_into(self, z, y, *, n_fft, hop, win, channels, frames, bins_in, strides):
        self.calls.append(("istft",))
        n_sig, out_len = y.shape
        B = n_sig // channels
        sb, sc, sk, st = strides
        src = torch.as_strided(z.reshape(-1), (B, channels, bins_in, frames, 2), (sb, sc, sk, st, 1))
        zc = torch.view_as_complex(src.contiguous()).reshape(n_sig, bins_in, frames).to(torch.complex128)
        zc = F.pad(zc, (0, 0, 0, n_fft // 2 + 1 - bins_in))
        w = F.pad(self._window(win), ((n_fft - win) // 2, n_fft - win - (n_fft - win) // 2)).double()
        fr = torch.fft.irfft(zc.transpose(1, 2) * n_fft ** 0.5, n=n_fft, dim=-1) * w
        total = n_fft + hop * (frames - 1)
        acc = torch.zeros(n_sig, total, dtype=torch.float64)
        env = torch.zeros(total, dtype=torch.float64)
        for t in range(frames):
            acc[:, t * hop:t * hop + n_fft] += fr[:, t]
            env[t * hop:t * hop + n_fft] += w * w
        lo = n_fft // 2
        y.copy_((acc[:, lo:lo + out_len] / env[lo:lo + out_len]).float())


def emulated(model):
    """Attach an EmuEngine to a (CPU) aero_b200.Aero and return the model."""
    object.__setattr__(model, "_engine_obj", EmuEngine(model))
    return model
