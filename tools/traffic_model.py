#!/usr/bin/env python
"""Per-launch roofline of one forward: algorithmic HBM bytes (read / written, from the storage types the engine actually
picks) and FLOPs of every launch, from a dry run of the host sequence on CPU (B = 1, scaled), optionally joined with a per-launch
timing list (CSV, see tools/launch_table.py).

    python tools/traffic_model.py launches.csv

Roofline time of a launch = max(read / R, written / W, (read + written) / C, flops / P) with R = W = C = the H100 SXM data-sheet
HBM3 bandwidth (3.35 TB/s) and P = its data-sheet dense FP16 rate (989 TFLOP/s at 700 W): bounds, not measured rates."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402
from aero_b200 import Aero, aero_kwargs, cabi  # noqa: E402
from aero_b200.engine import AeroEngine  # noqa: E402
from launch_table import load as load_launches  # noqa: E402

B_REAL = 32
BW_READ = BW_WRITE = BW_COPY = 3.35e12
P_TENSOR = 989.0e12


def nbytes(t):
    return 0 if t is None else t.numel() * t.element_size()


class DryEngine(AeroEngine):
    """The real host sequence with every kernel wrapper replaced by bookkeeping (no library, no GPU)."""

    def __init__(self, model):
        self._init_state(model, None)
        self.use_graph = False
        self.log = []          # (tag, flops, bytes_read, bytes_written, scales_with_batch_weights_bytes)

    def _on_device(self):
        import contextlib
        return contextlib.nullcontext()

    def _require(self, x): pass
    def _stream(self): return None

    def _gemm(self, out, w, *, B, F_out, T, N, C1, a1=None, a2=None, C2=0, F_in=None, T_in=None, mode=0, kf=1, kt=1, stride_f=1,
              glu=0, residual=None, tag=None, w_sb=0, **kw):
        tag = tag or self._wname.get(w.data_ptr(), "?")
        F_in = F_out if F_in is None else F_in
        T_in = T if T_in is None else T_in
        ea = (a1 if a1 is not None else a2).element_size()
        eo = out.element_size()
        if mode == cabi.TAPS_MIX:
            flops = 2.0 * B * T * N * C1
            rd, wr, wb = ea * B * C1 * T, eo * B * N * T, ea * N * C1
        elif w_sb:                                   # activations as "weights" (fp32 frequency mix)
            flops = 2.0 * B * T * N * C1
            rd, wr, wb = 4.0 * B * C1 * N, eo * B * T * N, 4.0 * T * C1
        else:
            ntaps = kf // stride_f if mode == cabi.TAPS_CONVT else kf * kt
            K, n_out = C1 + C2, (N // 2 if glu else N)
            flops = 2.0 * B * F_out * T * N * K * ntaps
            rd = ea * B * F_in * T_in * K + (eo * B * F_out * T * n_out if residual is not None else 0)
            wr = eo * B * F_out * T * n_out
            wb = ea * K * N * (kf if mode == cabi.TAPS_CONVT else ntaps)
        self.log.append(("gemm:" + tag, flops, rd, wr, wb))
        return out

    def _norm_act(self, x, stats, gamma, beta, y, *, B, F_in, T, C_, groups, scope, op, F_out=None, f_off=0, residual=None, **kw):
        F_out = F_in if F_out is None else F_out
        co = C_ // 2 if op in (cabi.NA_GLU, cabi.NA_GLU_SCALE_RES) else C_
        rd = x.element_size() * B * F_out * T * C_ + (y.element_size() * B * F_out * T * co if residual is not None else 0)
        self.log.append((f"norm_act<{op}>", 0.0, rd, y.element_size() * B * F_out * T * co, 0))
        return y

    def _lstm_rec(self, gin, bias_pad, whh, hout, *, rows, T, H, n_win, steps, **kw):
        self.log.append((f"lstm H={H}", 2.0 * 2 * rows * n_win * steps * 4 * H * H, nbytes(gin), nbytes(hout), nbytes(whh)))

    def _attn(self, qkvd, out, *, rows, T, H, heads, **kw):
        self.log.append((f"attn H={H}", 4.0 * rows * T * T * H, nbytes(qkvd), nbytes(out), 0))

    def _sample_norm(self, x, stats, y, affine, B, per_sample, extent=None, rnd=False):
        self.log.append(("sample_norm", 0.0, 4.0 * B * (extent or per_sample), 4.0 * B * (extent or per_sample), 0))

    def _freq_mix_small(self, x, Wfc, gate, out, *, B, F, M):
        self.log.append((f"freq_mix_small F={F}", 2.0 * B * F * F * M, nbytes(x) + nbytes(gate), nbytes(out), 0))
        return out

    def _ftb_lin_squeeze(self, z, W1p, b1p, R, **kw):
        self.log.append(("ftb_lin_squeeze", 0.0, nbytes(z), nbytes(R), 0))
        return R

    def _ftb_lin_out(self, z, zm, M, s, V, d, out, **kw):
        self.log.append(("ftb_lin_out", 0.0, nbytes(z) + nbytes(zm) + nbytes(M), nbytes(out), 0))
        return out

    def stft_into(self, x, z, stats, **kw):
        self.log.append(("stft", 0.0, nbytes(x), nbytes(z), 0))

    def istft_into(self, z, y, **kw):
        self.log.append(("istft", 0.0, nbytes(z), nbytes(y), 0))


def dry_log(experiment="aero_4-16_512_64", lr_len=8000, precision=2):
    """(tag, flops, bytes read, bytes written, weight bytes) of every launch of one B=1 forward, from a dry run on CPU."""
    kw = aero_kwargs(experiment)
    m = Aero(**kw).eval()
    eng = DryEngine(m)
    eng.precision = precision
    object.__setattr__(m, "_engine_obj", eng)
    m(torch.zeros(1, kw["in_channels"], lr_len))
    return eng.log


def launch_roofline(entry, batch, p_tensor=None):
    """Roofline time (s) and bound of one dry-run entry scaled to `batch` clips."""
    tag, fl, rd, wr, wb = entry
    fl, rd, wr = fl * batch, rd * batch + wb, wr * batch
    cands = {"read": rd / BW_READ, "write": wr / BW_WRITE, "copy": (rd + wr) / BW_COPY, "tensor": fl / (p_tensor or P_TENSOR)}
    bound = max(cands, key=cands.get)
    return cands[bound], bound, fl, rd, wr


def step_roofline(experiment="aero_4-16_512_64", batch=32, lr_len=8000, precision=2, p_tensor=None):
    """Sum over the launches of one forward of each launch's own roofline time: what this launch sequence would cost if every
    kernel ran at its bound (H100 SXM data sheet: 3.35 TB/s HBM3, 989 TFLOP/s dense FP16 unless `p_tensor` is given)."""
    log = dry_log(experiment, lr_len, precision)
    tot, flops, byts = 0.0, 0.0, 0.0
    for e in log:
        t, _, fl, rd, wr = launch_roofline(e, batch, p_tensor)
        tot += t
        flops += fl
        byts += rd + wr
    return {"sum_roofline_ms": tot * 1e3, "launches": len(log), "gflop": flops / 1e9, "hbm_gb": byts / 1e9}


def main():
    log = dry_log()
    meas = None
    if len(sys.argv) > 1:
        rows = [r for r in load_launches(sys.argv[1]) if r[0].startswith("aero::")]
        starts = [i for i, r in enumerate(rows) if "stft512_kernel" in r[0] and "istft" not in r[0]]
        segs = [rows[a:b] for a, b in zip(starts, starts[1:] + [len(rows)])]
        last = [sg for sg in segs if len(sg) == max(len(s_) for s_ in segs)][-1]
        assert len(last) == len(log), (len(last), len(log))
        meas = last
    print("# Per-launch roofline of the forward (aero_4-16_512_64, B=32 x 2 s, engine precision 2), launch list `" + os.path.basename(sys.argv[1]) + "`\n")
    print("Algorithmic bytes / FLOPs per launch from `tools/traffic_model.py` (dry run of the host sequence with the storage types the engine")
    print("picks), measured times from the launch list of the same build.  Roofline time = max(bytes / 3.35 TB/s,")
    print(f"FLOP / {P_TENSOR/1e12:.0f} TFLOP/s): H100 SXM data-sheet figures.  The LSTM rows are latency-bound by construction (200 dependent")
    print("steps), attention is exp/issue-bound.\n")
    print("| # | kernel | op | GFLOP | MB read | MB written | bound | roofline us | measured us | measured / roofline |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    tot_roof = tot_meas = 0.0
    for i, (tag, fl, rd, wr, wb) in enumerate(log):
        fl, rd, wr = fl * B_REAL, rd * B_REAL + wb, wr * B_REAL
        cands = {"read": rd / BW_READ, "write": wr / BW_WRITE, "copy": (rd + wr) / BW_COPY, "tensor": fl / P_TENSOR}
        bound = max(cands, key=cands.get)
        roof = cands[bound] * 1e6
        us = meas[i][2] if meas else float("nan")
        name = meas[i][0].replace("aero::", "") if meas else ""
        tot_roof += roof
        tot_meas += us
        print(f"| {i} | `{name}` | {tag} | {fl/1e9:.1f} | {rd/1e6:.1f} | {wr/1e6:.1f} | {bound} | {roof:.1f} | {us:.1f} | {us/roof:.1f} |")
    print(f"\nSum of per-launch roofline times **{tot_roof/1e3:.2f} ms**; measured **{tot_meas/1e3:.2f} ms** -> the step runs at "
          f"{100*tot_roof/tot_meas:.0f} % of a perfect-kernel bound for this launch sequence.")


if __name__ == "__main__":
    main()
