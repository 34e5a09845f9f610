"""The wide tap-GEMM tiles (BN = 192 / 256, FP16 operands, long K loops) at multi-wave sizes, against fp64 on the operands the
tensor cores read, checked per output tile (the harness and bars of test_gpu_tc_scale.py).

A wide tile keeps 96 / 128 fp32 accumulators per consumer thread (setmaxnreg moves registers from the producer warpgroup)
and runs its epilogue in 64-column slices of the staging tile, so what these cases cover beyond the narrow widths is the slice
walk: GLU partner columns, residual rows, GroupNorm statistics whose groups straddle slice and tile edges (gw = 192 and 384
against BN = 256), the last n-tile of an N that is not a multiple of the width, both output types and both tile orders.
Every CTA runs >= 3 tiles.  The width rule itself (csrc/tapgemm_tc.cu pick_bn) is mirrored below and checked without a GPU."""
import pytest

import test_gpu_tc_scale as tcs
from aero_b200 import cabi
from test_gpu_tc_scale import cdiv, engines  # noqa: F401  (fixture)

KMAX_BN, KWIDE_BN = 128, 256
WIDE_MIN_KTAPS = 512            # csrc/tapgemm_tc.cu kWideMinKTaps


def pick_bn(N, *, ktaps, precision=2, mix=False, glu=False, groups=None):
    """Tile width of the wgmma tap-GEMM (tapgemm_tc.cu pick_bn; the shared-memory fallback never triggers below N = 8192)."""
    narrow = (cdiv(N, cdiv(N, KMAX_BN)) + 31) & ~31
    if precision != 2 or mix or N < 192 or ktaps < WIDE_MIN_KTAPS:
        return narrow
    bn = 192 if cdiv(N, cdiv(N, KWIDE_BN)) <= 192 else 256
    if groups:
        n_out = N // 2 if glu else N
        if (bn // 2 if glu else bn) // (n_out // groups) + 2 > 8:
            return narrow
    return bn


# long-K geometries (K x taps >= 512): two sources on a 3x3 with the frequency borders of F_out = 3 and the T = 501 tail; a
# strided encoder-style conv; a transposed conv whose rows 10, 11 lie past its natural extent (bias only)
WIDE_GEOMS = {
    "w3x3_two_src": dict(F_in=3, F_out=3, C1=64, C2=32, T=501, kf=3, kt=3, pad_f=1, pad_t=1),
    "wconv_stride2": dict(F_in=8, F_out=4, C1=64, T=333, kf=8, stride_f=2, pad_f=3),
    "wconvt": dict(F_in=4, F_out=12, C1=192, T=270, mode=cabi.TAPS_CONVT, kf=8, stride_f=2),
}


def _ktaps(geom):
    g = WIDE_GEOMS[geom]
    taps = g["kf"] // g["stride_f"] if g.get("mode") == cabi.TAPS_CONVT else g.get("kf", 1) * g.get("kt", 1)
    return (g["C1"] + g.get("C2", 0)) * taps


# (N, GroupNorm groups) per width: N = 768 / 384 fill whole tiles, 480 / 336 leave a ragged last n-tile.  Groups of 384, 192
# and 96 columns against BN = 256, and of 192, 48 and 96 against BN = 192, start inside tiles and slices and straddle their
# edges.  The statistics variants run every shape of their width, the others alternate between the first two.
CASES_N = {256: [dict(N=768, groups=2), dict(N=480, groups=5), dict(N=768, groups=4)],
           192: [dict(N=384, groups=2), dict(N=336, groups=7), dict(N=384, groups=4)]}
# FP16-operand variants of pick_kernel (operand kind, output type, amode, residual, statistics)
VARIANTS = ([("f16", "f32", a, False, False) for a in range(4)] + [("f16", "f32", 0, False, True)] +
            [("f16", "f16", a, False, False) for a in range(4)] + [("f16", "f16", 0, True, False), ("f16", "f16", 0, False, True)])
WIDE = [(bn, v, list(WIDE_GEOMS)[(i + j + k) % len(WIDE_GEOMS)], shape)
        for j, bn in enumerate(CASES_N) for i, v in enumerate(VARIANTS)
        for k, shape in enumerate(CASES_N[bn] if v[4] else [CASES_N[bn][i % 2]])]


@pytest.mark.gpu
@pytest.mark.parametrize("bn,variant,geom,shape", WIDE,
                         ids=[f"bn{bn}-{v[1]}-a{v[2]}{'-res' if v[3] else ''}{'-stats' if v[4] else ''}-{g}-n{s['N']}"
                              for bn, v, g, s in WIDE])
def test_tapgemm_wgmma_wide_multi_wave(engines, monkeypatch, bn, variant, geom, shape):  # noqa: F811
    gpu, emu = engines
    N, glu = shape["N"], variant[2] == 3
    groups = shape["groups"] if variant[4] else None
    ktaps = _ktaps(geom)
    assert pick_bn(N, ktaps=ktaps, glu=glu, groups=groups) == bn
    # the harness of test_gpu_tc_scale.py with this file's geometry and width rule
    monkeypatch.setitem(tcs.GEOMS, geom, WIDE_GEOMS[geom])
    monkeypatch.setattr(tcs, "pick_bn", lambda n: pick_bn(n, ktaps=ktaps, glu=glu, groups=groups))
    res = tcs._run_scale_case(gpu, emu, bn, variant, geom, N, groups=groups)
    for r, order in zip(res, ("forward", "reverse")):
        print(f"{order}: {r['variant']} tiles {r['tiles']}: worst tile {r['err']:.3f} of its bar ({r['rounding'] or 'rel-L2'}), "
              f"stats {r['serr']:.3f}")
        assert r["err"] <= 1.0 and r["serr"] <= 1.0, (order, r)


def test_wide_width_rule():
    """The benchmarked forward's long-K FP16 convolutions take the wide tiles; short-K, TF32 and row-mix launches keep the
    narrow ones; a statistics layout with too many groups per tile falls back."""
    # decoder.{0..3}.rw, decoder.0.ct, encoder.3.conv, encoder.2.conv (aero_4-16_512_64): N, K x taps
    assert pick_bn(1536, ktaps=384 * 9, groups=4) == 256
    assert pick_bn(768, ktaps=384 * 9, groups=4) == 256
    assert pick_bn(384, ktaps=192 * 9, glu=True) == 192
    assert pick_bn(192, ktaps=96 * 9, glu=True) == 192
    assert pick_bn(192, ktaps=768 * 4, groups=4) == 192
    assert pick_bn(384, ktaps=192 * 8, groups=4) == 192
    assert pick_bn(192, ktaps=96 * 8) == 192
    # 1x1 rewrites / LSTM gate inputs (K x taps <= 384), TF32 operands, the row mix: unchanged
    assert pick_bn(768, ktaps=384) == 128
    assert pick_bn(768, ktaps=192) == 128
    assert pick_bn(1536, ktaps=384 * 9, precision=1) == 128
    assert pick_bn(768, ktaps=1024, mix=True) == 128
    assert pick_bn(176, ktaps=1024) == 96
    # 32-column groups: 256 / 32 + 2 > 8 statistics slots per tile, so the narrow width
    assert pick_bn(1536, ktaps=3456, groups=48) == 128
    assert all(_ktaps(g) >= WIDE_MIN_KTAPS for g in WIDE_GEOMS)
