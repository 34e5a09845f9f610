"""Ragged batches (AeroEngine.forward_varlen / enhance.enhance_batch) on CPU: the product's host logic (length tables, BiLSTM
framing tables, masking and masked statistics placement) drives torch statements of the new entry points' contracts, and
every clip must come out as the oracle computes it on that clip alone."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cpu_emu import EmuEngine
from util import SEED, rel_l2, trained_like_, white_noise

from aero_b200 import Aero, aero_kwargs, cabi
from aero_b200.enhance import enhance_batch
from aero_b200.engine import lstm_ragged_tables
from oracle import aero_variants_oracle as OV


class RaggedEmuEngine(EmuEngine):
    """EmuEngine plus the contracts of the ragged-batch entry points (include/aero_b200.h, "Ragged batches")."""

    def _frames(self):
        return self._vl.frames_d.tolist()

    # ---- aero_norm_act_fwd with NA_RELU (the `_relu` experiments' DConv activation)
    def _norm_act(self, x, stats, gamma, beta, y, *, op, **kw):
        super()._norm_act(x, stats, gamma, beta, y, op=cabi.NA_NONE if op == cabi.NA_RELU else op, **kw)
        if op == cabi.NA_RELU:
            n = kw["B"] * (kw.get("F_out") or kw["F_in"]) * kw["T"] * kw["C_"]
            y.reshape(-1)[:n].clamp_(min=0)
        return y

    # ---- aero_frame_mask_fwd
    def _frame_mask(self, x):
        self.calls.append(("frame_mask",))
        for b, tb in enumerate(self._frames()):
            x[b, :, tb:] = 0

    # ---- aero_masked_stats_fwd
    def _masked_stats(self, x, stats, *, groups, scope):
        self.calls.append(("masked_stats", scope))
        B, F_, T, C_ = x.shape
        for b, tb in enumerate(self._frames()):
            v = x[b, :, :tb].double()
            k = T / tb
            if scope == 1:
                g = v.reshape(F_, tb, groups, C_ // groups)
                stats[b * groups:(b + 1) * groups, 0] += g.sum((0, 1, 3)) * k
                stats[b * groups:(b + 1) * groups, 1] += (g * g).sum((0, 1, 3)) * k
            else:
                stats[b * F_:(b + 1) * F_, 0] += v.sum((1, 2)) * k
                stats[b * F_:(b + 1) * F_, 1] += (v * v).sum((1, 2)) * k

    # ---- aero_gather_rows_fwd
    def _gather_rows(self, src, dst, idx, fill, n_rows):
        self.calls.append(("gather_rows",))
        width, parts = dst.shape[-1], idx.shape[-1]
        pw = width // parts
        s = src.reshape(-1, width)
        d = dst.reshape(-1, width)
        for q in range(parts):
            j = idx[:n_rows, q].long()
            cols = slice(q * pw, (q + 1) * pw)
            val = s[j.clamp_min(0), cols].float()
            fv = (fill[cols] if fill is not None else torch.zeros(pw)).float().expand_as(val)
            d[:n_rows, cols] = torch.where((j >= 0)[:, None], val, fv).to(d.dtype)

    # ---- aero_sample_norm_varlen_fwd
    def _sample_norm_varlen(self, x, stats, y, affine, B, per_frame, extent, rnd=False):
        self.calls.append(("sample_norm_varlen",))
        for b, tb in enumerate(self._frames()):
            n = float(per_frame * tb)
            mean = stats[b, 0] / n
            sd = ((stats[b, 1] - n * mean * mean) / (n - 1)).clamp_min(0).sqrt()
            y.reshape(B, -1)[b, :extent].copy_(((x.reshape(B, -1)[b, :extent].double() - mean) / (1e-5 + sd)).float())
            affine[b, 0], affine[b, 1] = sd.float(), mean.float()

    # ---- aero_stft_varlen_fwd
    def stft_varlen_into(self, x, lengths, z, stats, *, n_fft, hop, win, channels, bins_out, strides):
        self.calls.append(("stft_varlen",))
        n_sig, length = x.shape
        frames = 1 + length // hop
        B = n_sig // channels
        sb, sc, sk, st = strides
        dst = torch.as_strided(z.reshape(-1), (B, channels, bins_out, frames, 2), (sb, sc, sk, st, 1))
        w = F.pad(self._window(win), ((n_fft - win) // 2, n_fft - win - (n_fft - win) // 2))
        for b, n in enumerate(lengths.tolist()):
            xb = x[b * channels:(b + 1) * channels, :n]
            xb = F.pad(xb, (0, (-n) % hop))
            xp = F.pad(xb[:, None], (n_fft // 2, n_fft // 2), mode="reflect")[:, 0]
            zz = torch.fft.rfft(xp.unfold(-1, n_fft, hop).double() * w.double(), dim=-1) * n_fft ** -0.5
            val = torch.view_as_real(zz[..., :bins_out].transpose(1, 2)).float()      # [channels, bins, T_b, 2]
            tb = val.shape[2]
            dst[b].zero_()
            dst[b, :, :, :tb] = val
            if stats is not None:
                stats[b, 0] += val.double().sum()
                stats[b, 1] += (val.double() ** 2).sum()

    # ---- aero_istft_varlen_fwd
    def istft_varlen_into(self, z, y, frames, out_lens, *, n_fft, hop, win, channels, frames_max, bins_in, strides):
        self.calls.append(("istft_varlen",))
        n_sig, out_len = y.shape
        y.zero_()
        for b, (tb, ol) in enumerate(zip(frames.tolist(), out_lens.tolist())):
            yb = torch.empty(channels, ol)
            sb, sc, sk, st = strides
            zb = torch.as_strided(z.reshape(-1)[b * sb:], (channels, bins_in, tb, 2), (sc, sk, st, 1))
            EmuEngine.istft_into(self, zb.contiguous(), yb, n_fft=n_fft, hop=hop, win=win, channels=channels, frames=tb,
                                 bins_in=bins_in, strides=(channels * bins_in * tb * 2, bins_in * tb * 2, tb * 2, 2))
            y[b * channels:(b + 1) * channels, :ol] = yb

    # ---- aero_local_attn_varlen_fwd
    def _attn(self, qkvd, out, *, rows, T, H, heads, ndecay, ld):
        if self._vl is None:
            return super()._attn(qkvd, out, rows=rows, T=T, H=H, heads=heads, ndecay=ndecay, ld=ld)
        rpc = rows // len(self._frames())
        q3 = qkvd.reshape(rows, T, ld)
        o3 = out.reshape(rows, T, H)
        for b, tb in enumerate(self._frames()):
            sub = q3[b * rpc:(b + 1) * rpc, :tb].contiguous()
            r = torch.empty(rpc * tb, H, dtype=out.dtype)
            super()._attn(sub, r, rows=rpc, T=tb, H=H, heads=heads, ndecay=ndecay, ld=ld)
            o3[b * rpc:(b + 1) * rpc, :tb] = r.view(rpc, tb, H)


def make(exp):
    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs(exp)).eval()
    m.load_state_dict(trained_like_(m.state_dict()))
    object.__setattr__(m, "_engine_obj", RaggedEmuEngine(m))
    return m


def lengths_for_frames(m, frames):
    """Sample counts giving the requested STFT frame counts (not multiples of hop where that is possible)."""
    hop = m.geom.hop_in
    return [max(hop * (t - 1) - (hop // 3 if t > 2 else 0), 1) for t in frames]


def check(m, lengths, seed=3, channels=None):
    C = channels or m.in_channels
    sigs = [white_noise((C, n), seed=seed + i) for i, n in enumerate(lengths)]
    outs = enhance_batch(m, sigs, max_batch=8, return_spec=True, return_lr_spec=True)
    errs = []
    for s, (y, zc, zl) in zip(sigs, outs):
        with torch.no_grad():
            ry, rzc, rzl = OV.aero_forward(m.state_dict(), m.geom, s[None], return_spec=True, return_lr_spec=True)
        assert y.shape == ry[0].shape and zc.shape == rzc[0].shape and zl.shape == rzl[0].shape
        errs.append((rel_l2(y, ry[0]), rel_l2(torch.view_as_real(zc), torch.view_as_real(rzc[0])),
                     rel_l2(torch.view_as_real(zl), torch.view_as_real(rzl[0]))))
    print(m.geom.kw.get("act_func"), lengths, ["%.1e/%.1e/%.1e" % e for e in errs])
    assert max(max(e) for e in errs) < 1e-5, errs
    return m._engine_obj.calls


def test_ragged_frame_counts_around_the_lstm_windows():
    """T of 101, 200, 201, 299, 300, 301 and ~700 frames in one batch: one-sequence clips next to windowed ones, lengths
    that are not multiples of hop."""
    m = make("aero_4-16_512_64")
    calls = check(m, lengths_for_frames(m, [101, 200, 201, 299, 300, 301, 700]))
    kinds = {c[0] for c in calls}
    assert {"stft_varlen", "istft_varlen", "sample_norm_varlen", "masked_stats", "frame_mask", "gather_rows"} <= kinds
    assert "sample_norm" not in kinds and "stft" not in kinds


def test_ragged_shortest_clip_and_short_batch():
    """every clip <= 200 frames (one sequence each, S = the longest clip) including the shortest accepted clip."""
    m = make("aero_4-16_512_256")
    hop = m.geom.hop_in
    shortest = next(n for n in range(1, 4 * m.geom.nfft) if n + (-n) % hop > m.geom.nfft // 2)
    check(m, [shortest, shortest + 7, 1500, 3001])


@pytest.mark.parametrize("exp,C", [("aero_12-48_512_128", 1), ("aero_11-44_512_64", 2), ("aero_4-16_512_64_sinc", 1),
                                   ("aero_4-16_512_64_relu", 1)])
def test_ragged_other_geometries(exp, C):
    m = make(exp)
    check(m, lengths_for_frames(m, [60, 130, 230]), channels=C)


def test_ragged_storage_types_at_precision_2():
    """precision 2 host logic (FP16 buffers, FP16 gathers of LSTM outputs): a one-clip ragged batch equals the ordinary
    forward exactly; in a mixed batch every clip stays within the precision-2 budget against the oracle (1e-3, as
    tests/test_host_logic.py holds the ordinary forward)."""
    m = make("aero_4-16_512_64")
    m._engine_obj.precision = 2
    lengths = lengths_for_frames(m, [90, 250])
    sigs = [white_noise((1, n), seed=11 + i) for i, n in enumerate(lengths)]
    assert rel_l2(enhance_batch(m, sigs[:1])[0], m(sigs[0][None])[0]) == 0
    for s, y in zip(sigs, enhance_batch(m, sigs)):
        with torch.no_grad():
            ref = OV.aero_forward(m.state_dict(), m.geom, s[None])[0]
        assert y.shape == ref.shape and rel_l2(y, ref) < 1e-3


def test_lstm_tables_follow_the_reference_framing():
    """A windowed clip's reassembly picks window 0 for t < 150, then (t - 50) // 100; a short clip keeps its reverse half
    at the end of the S positions; padded frames map to -1."""
    n_seq, S, gin1, h1, gin2, out = lstm_ragged_tables([120, 320], 1, 320)
    assert S == 200 and n_seq == 1 + math.ceil(320 / 100)
    gin1 = gin1.reshape(n_seq, S, 2)
    assert gin1[0, 0, 0] == 0 and gin1[0, 119, 0] == 119 and gin1[0, 120, 0] == -1
    assert gin1[0, S - 120, 1] == 0 and gin1[0, S - 1, 1] == 119 and gin1[0, S - 121, 1] == -1
    assert gin1[4, 0, 0] == 320 + 300 and gin1[4, 20, 0] == -1          # last window of clip 1 starts at frame 300
    o = out.reshape(2, 320, 2)
    assert (o[0, 120:] == -1).all() and o[0, 5, 1] == 5 + S - 120
    assert o[1, 149, 0] == 1 * S + 149 and o[1, 150, 0] == 2 * S + 50 and o[1, 319, 0] == 3 * S + 119


def test_errors_match_the_single_clip_forward():
    m = make("aero_4-16_512_256")
    assert enhance_batch(m, []) == []
    with pytest.raises(ValueError):
        enhance_batch(m, [white_noise((2, 3000))])
    with pytest.raises(cabi.AeroLibraryError, match="reflect padding"):
        enhance_batch(m, [white_noise((1, 3000)), white_noise((1, 200))])
    m.train()
    with pytest.raises(NotImplementedError):
        enhance_batch(m, [white_noise((1, 3000))])
    from aero_b200 import Seanet, seanet_kwargs
    with pytest.raises(NotImplementedError):
        enhance_batch(Seanet(**seanet_kwargs("seanet_4-16")), [white_noise((1, 3000))])
