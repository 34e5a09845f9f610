"""Launch shape of the wgmma LSTM recurrence (csrc/lstm_tc.cu, lstm_tc_shape): host logic only, no GPU needed."""
import ctypes as C

import pytest

from aero_b200 import build as build_mod
from aero_b200 import cabi


@pytest.fixture(scope="module")
def lib():
    build_mod.build()
    return cabi.load()


def shape(lib, n_seq, H, sms):
    out = (C.c_int32 * 4)()
    assert lib.aero_lstm_tc_shape(n_seq, H, sms, out) == 0
    return dict(S=out[0], nt=out[1], ctas=out[2], tps=out[3])


def test_benchmark_shapes_fill_one_wave_of_an_h100(lib):
    # aero_4-16_512_64 at 32 x 2 s: encoder 2 (H = 48, 256 rows x 6 windows), encoder 3 (H = 96, 128 rows x 6 windows)
    assert shape(lib, 1536, 48, 132) == dict(S=12, nt=16, ctas=64, tps=8)
    assert shape(lib, 768, 96, 132) == dict(S=6, nt=8, ctas=64, tps=16)


@pytest.mark.parametrize("H", [36, 48, 64, 68, 80, 84, 96])
@pytest.mark.parametrize("sms", [1, 7, 132])
def test_shape_rule(lib, H, sms):
    for n_seq in (1, 2, 15, 16, 17, 131, 132, 133, 640, 768, 1280, 1536, 4000, 20000):
        sp = shape(lib, n_seq, H, sms)
        assert sp["tps"] == -(-(H // 2) // 3)                       # three cell pairs per thread
        assert 1 <= sp["S"] <= min(128 // sp["tps"], 16 if H <= 80 else 8)
        assert sp["S"] <= sp["nt"] and sp["nt"] == (8 if sp["S"] <= 8 else 16)
        assert (sp["ctas"] - 1) * 2 * sp["S"] < n_seq <= sp["ctas"] * 2 * sp["S"]   # every sequence, no empty CTA
        if 2 * sp["ctas"] > max(2, sms - sms % 2):
            assert sp["S"] == min(128 // sp["tps"], 16 if H <= 80 else 8)         # more than one wave only at the cap
        elif sp["S"] > 1:
            assert 2 * -(-n_seq // (2 * (sp["S"] - 1))) > max(2, sms - sms % 2)     # and the narrowest width that fits


def test_unsupported_hidden_sizes(lib):
    out = (C.c_int32 * 4)()
    for H in (32, 12, 50, 100, 128):
        assert lib.aero_lstm_tc_shape(100, H, 132, out) != 0
