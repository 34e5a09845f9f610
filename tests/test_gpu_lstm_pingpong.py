"""-m gpu: the wgmma LSTM recurrence (csrc/lstm_tc.cu) with W_hh in registers and two ping-ponged sequence groups per CTA, against
the fp64 recurrence on the kernel's own operands: both benchmark shapes, a last CTA whose second group is partial or empty, one
window (T < 200) and ragged windows (T > 200), fp32 / FP16 gate inputs, fp32 / FP16 outputs, both directions."""
import ctypes as C
import math

import pytest
import torch

from test_gpu_tc_scale import LSTM_BAR, _lstm_run, cdiv, engines, lstm_block_errors, lstm_ref, lstm_whh_from_rows, n_sms, rnd  # noqa: F401

from aero_b200.engine import lstm_gate_reorder, lstm_whh_fp16

pytestmark = pytest.mark.gpu


def lstm_shape(lib, n_seq, H):
    out = (C.c_int32 * 4)()
    assert lib.aero_lstm_tc_shape(n_seq, H, n_sms(), out) == 0
    return dict(S=out[0], nt=out[1], ctas=out[2], tps=out[3])


def rows_for(lib, H, T, last_groups):
    """Smallest row count >= 8 whose last CTA has `last_groups` live groups (1: second group empty, 2: second group partial)."""
    n_win = cdiv(T, 100) if T > 200 else 1
    for rows in range(8, 4000):
        sp = lstm_shape(lib, rows * n_win, H)
        r = rows * n_win - (sp["ctas"] - 1) * 2 * sp["S"]
        if sp["S"] > 1 and ((last_groups == 1 and r <= sp["S"]) or (last_groups == 2 and sp["S"] < r < 2 * sp["S"])):
            return rows
    raise AssertionError("no such row count")


# (H, T, rows): the two recurrences of aero_4-16_512_64 at 32 x 2 s (encoder 2: 8 frequency rows per clip, encoder 3: 4), then the
# ragged last-CTA cases (rows = None: chosen by rows_for)
CASES = [(48, 501, 256, 0), (96, 501, 128, 0),
         (48, 350, None, 1), (48, 150, None, 2), (96, 160, None, 1), (96, 350, None, 2), (64, 120, None, 2), (36, 230, None, 1)]


@pytest.mark.parametrize("gin16", [False, True], ids=["gin32", "gin16"])
@pytest.mark.parametrize("H,T,rows,last_groups", CASES)
def test_lstm_pingpong(engines, H, T, rows, last_groups, gin16):
    gpu, _ = engines
    lib = gpu.lib._lib
    rows = rows or rows_for(lib, H, T, last_groups)
    steps, stride, n_win = (200, 100, cdiv(T, 100)) if T > 200 else (T, 0, 1)
    n_seq = rows * n_win
    sp = lstm_shape(lib, n_seq, H)
    assert 2 * sp["ctas"] <= n_sms() or sp["S"] == min(16 if H <= 80 else 8, 128 // sp["tps"]), sp
    gdt = torch.float16 if gin16 else torch.float32
    gin1 = rnd(rows * T, 8 * H, seed=11).to(gdt)
    gin2 = rnd(n_seq * steps, 8 * H, seed=15).to(gdt)
    b1 = rnd(8 * H, seed=12) * 0.3
    src, ok = lstm_gate_reorder(H)

    def rows_(w):
        return lstm_whh_fp16(torch.cat([torch.where(ok[:, None], w[d][src], torch.zeros(())) for d in range(2)], 0)).cuda()
    whh1r = rows_(rnd(2, 4 * H, H, seed=13, dev="cpu") / math.sqrt(H))
    whh2r = rows_(rnd(2, 4 * H, H, seed=14, dev="cpu") / math.sqrt(H))
    geom = dict(rows=rows, T=T, H=H, n_win=n_win, steps=steps, stride=stride)
    h32 = _lstm_run(gpu, gin1, gin2, b1, whh1r, whh2r, o16=False, prec=1, geom=geom)
    h16 = _lstm_run(gpu, gin1, gin2, b1, whh1r, whh2r, o16=True, prec=2, geom=geom)
    gpu.lib.calls.clear()
    ref1 = lstm_ref(gin1, b1, lstm_whh_from_rows(whh1r, H), in_windowed=0, out_windowed=1, **geom)
    ref2 = lstm_ref(gin2, b1, lstm_whh_from_rows(whh2r, H), in_windowed=1, out_windowed=0, **geom)
    for tag, h, ref in (("fp32 layer-1", h32[0], ref1), ("fp32 layer-2", h32[1], ref2),
                        ("fp16 layer-1", h16[0], ref1), ("fp16 layer-2", h16[1], ref2)):
        assert torch.isfinite(h).all(), tag
        worst, whole = lstm_block_errors(h, ref, steps if "1" in tag else T)
        print(f"lstm ping-pong H={H} T={T} n_seq={n_seq} {sp} {'gin16' if gin16 else 'gin32'} {tag}: worst block {worst:.2e}, "
              f"whole {whole:.2e}")
        assert worst < LSTM_BAR, (tag, worst)
    for a, b in zip(h16, h32):
        assert torch.equal(a, b.half()), "FP16 hout is not the round-to-nearest of the fp32 result"
