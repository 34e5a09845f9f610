"""SEANet on the H100: the forward against the stored reference outputs at every precision, the input stage, the super-frame
convolutions and the reflection halo against fp64 on the operands the kernels read, the production shape, CUDA-graph replay."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from util import SEED, rel_l2
from seanet_util import CASES, case_input, seanet_recipe_state

from aero_b200 import Seanet, cabi
from aero_b200.engine import pack_taps
from aero_b200.seanet import sinc_resample_table, superframe_conv_weight, superframe_convt_weight
from oracle import seanet_oracle as O

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
F = torch.nn.functional


class _Recorder:
    """Library proxy that records the precision every tap-GEMM launch ran at."""

    def __init__(self, lib):
        self._lib, self.precisions = lib, []

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def aero_tapgemm_fwd(self, *a):
        self.precisions.append(a[10]._obj.precision)
        return self._lib.aero_tapgemm_fwd(*a)


def _model(name, precision):
    torch.manual_seed(SEED)
    m = Seanet(**CASES[name][0])
    m.load_state_dict(seanet_recipe_state(m.state_dict()))
    m = m.cuda().eval().use_cuda_graph(False)
    m._engine().precision = precision
    return m


def _std(x, model):
    if not model.normalize:
        return torch.ones(x.shape[0], 1, 1, dtype=torch.float64)
    return x.double().mean(1, keepdim=True).std(-1, keepdim=True)


@pytest.mark.parametrize("precision", [2, 1, 0])
@pytest.mark.parametrize("name", sorted(CASES))
def test_forward_against_golden(name, precision):
    g = np.load(os.path.join(GOLDEN, f"seanet_{name}.npz"))
    m = _model(name, precision)
    x = case_input(name)
    rec = _Recorder(m._engine().lib)
    m._engine().lib = rec
    y = m(x.cuda()).cpu()
    assert tuple(y.shape) == g["y"].shape
    err = rel_l2(y, g["y"])
    # the generated branch: the output divided by std, minus the input skip x0 (which dominates the output)
    target = y.shape[-1]
    branch = y.double() / _std(x, m) - torch.from_numpy(g["x0"][..., :target]).double()
    err_b = rel_l2(branch, g["branch"][..., :target])
    print(f"{name} precision {precision}: out {err:.2e} branch {err_b:.2e}")
    if precision == 0:
        assert set(rec.precisions) == {0}
        assert err <= 1e-5 and err_b <= 1e-5
    else:
        assert precision in rec.precisions          # the wide layers ran on the tensor cores
        assert err <= 1e-3 and err_b <= 2e-3


@pytest.mark.parametrize("name", ["s1", "s3", "s5"])
def test_input_stage_against_oracle(name):
    """aero_seanet_input_fwd alone: normalisation, resampler, zero pad and the reflected halo of x0."""
    m = _model(name, 2)
    x = case_input(name)
    B, Cin, L = x.shape
    lev = m.level_lengths(L)
    Lv, H, fill = lev[0], 9, 3
    if m.upsample:
        filt, width, orig, up = sinc_resample_table(m.lr_sr, m.hr_sr)
        filt, taps = filt.cuda().contiguous(), filt.shape[1]
    else:
        filt, width, orig, up, taps = None, 0, 1, 0, 0
    x0 = torch.full((B, Lv + 2 * H, Cin), float("nan"), device="cuda")
    aff = torch.empty(B, 2, device="cuda")
    p = cabi.ResampleParams(B, Cin, L, orig, up, width, taps, m.hr_length(L), Lv, H, fill, 1, 1e-3)
    xc = x.cuda().contiguous()
    lib = cabi.load()
    cabi.check(lib.aero_seanet_input_fwd(C.c_void_p(xc.data_ptr()), None if filt is None else C.c_void_p(filt.data_ptr()),
                                         C.c_void_p(aff.data_ptr()), C.c_void_p(x0.data_ptr()), C.byref(p), None), lib)
    torch.cuda.synchronize()
    stages = {}
    with torch.no_grad():
        O.seanet_forward({k: v.double() for k, v in m.cpu().state_dict().items()}, m, x.double(), stages)
    ref = F.pad(stages["x0"], (fill, fill), mode="reflect").permute(0, 2, 1)       # [B, Lv + 2 fill, C]
    got = x0[:, H - fill:H + Lv + fill].cpu()
    assert rel_l2(got, ref) <= 1e-6
    assert torch.isnan(x0[:, :H - fill]).all()                                       # nothing outside the requested halo
    assert torch.allclose(aff[:, 0].cpu().double(), _std(x, m).view(-1), rtol=1e-6)


def _engine():
    torch.manual_seed(SEED)
    m = Seanet(**CASES["s6"][0]).cuda().eval()
    eng = m._engine()
    eng.lib = _Recorder(eng.lib)
    return eng


@pytest.mark.parametrize("r,C,N", [(2, 32, 64), (4, 64, 128), (8, 128, 256)])
def test_superframe_conv_and_convt_on_tensor_cores(r, C, N):
    """The strided conv and the transposed conv as 3-tap convs over super-frames, f16 wgmma, against fp64 conv1d /
    conv_transpose1d on the FP16 operands the tensor cores read."""
    eng = _engine()
    g = torch.Generator().manual_seed(r)
    B, T = 3, 97 * r
    p = r // 2 + r % 2
    x = torch.randn(B, T, C, generator=g).half().cuda()
    w = (torch.randn(N, C, 2 * r, generator=g) / (C * r) ** 0.5)
    b = 0.1 * torch.randn(N, generator=g)
    W = eng._add_tc_twins({"down.w": pack_taps(superframe_conv_weight(w, r)).cuda()})
    y = torch.empty(B, T // r, N, dtype=torch.float32, device="cuda")
    eng._gemm(y, W["down.w"], a1=x, B=B, F_out=1, T=T // r, N=N, C1=r * C, kt=3, pad_t=1, a1_s=(T * C, 0, r * C),
              bias=b.cuda())
    assert eng.lib.precisions[-1] == 2
    ref = F.conv1d(x.permute(0, 2, 1).double().cpu(), w.half().double(), b.double(), stride=r, padding=p).permute(0, 2, 1)
    assert rel_l2(y.cpu(), ref) <= 1e-5
    # transposed conv: input [B, T/r, N] -> [B, T, C]
    xt = torch.randn(B, T // r, N, generator=g).half().cuda()
    wt = torch.randn(N, C, 2 * r, generator=g) / (N * 2) ** 0.5
    bt = 0.1 * torch.randn(C, generator=g)
    W = eng._add_tc_twins({"up.w": pack_taps(superframe_convt_weight(wt, r)).cuda()})
    yt = torch.empty(B, T, C, dtype=torch.float32, device="cuda")
    eng._gemm(yt, W["up.w"], a1=xt, B=B, F_out=1, T=T // r, N=r * C, C1=N, kt=3, pad_t=1, o_s=(T * C, 0, r * C),
              bias=bt.repeat(r).cuda())
    assert eng.lib.precisions[-1] == 2
    ref = F.conv_transpose1d(xt.permute(0, 2, 1).double().cpu(), wt.half().double(), bt.double(), stride=r, padding=p,
                             output_padding=r % 2).permute(0, 2, 1)
    assert rel_l2(yt.cpu(), ref) <= 1e-5


@pytest.mark.parametrize("dil", [1, 3, 9])
def test_reflect_halo_and_dilated_conv(dil):
    """LeakyReLU + reflection halo, then the k3 dilated conv reading it with no padding (f16 wgmma, LeakyReLU epilogue),
    against fp64 on the same FP16 operands."""
    eng = _engine()
    g = torch.Generator().manual_seed(dil)
    B, T, C, H = 2, 1000 + dil, 64, 9
    x = torch.randn(B, T, C, generator=g).half().cuda()
    h0 = torch.full((B, T + 2 * H, C), float("nan"), dtype=torch.float16, device="cuda")
    eng._reflect_act(x, h0[:, H:], B=B, T=T, C=C, x_sb=T * C, y_sb=(T + 2 * H) * C, halo=dil)
    ref_h = F.pad(F.leaky_relu(x.permute(0, 2, 1).double().cpu(), 0.2), (dil, dil), mode="reflect")
    got_h = h0[:, H - dil:H + T + dil].permute(0, 2, 1).double().cpu()
    assert torch.equal(got_h, ref_h.half().double())                     # exact: LeakyReLU(0.2) of an FP16 value, rounded once
    w = torch.randn(C, C, 3, generator=g) / (3 * C) ** 0.5
    W = eng._add_tc_twins({"c3.w": pack_taps(w).cuda()})
    y = torch.empty(B, T, C, dtype=torch.float16, device="cuda")
    eng._gemm(y, W["c3.w"], a1=h0[:, H - dil:], B=B, F_out=1, T=T, T_in=T + 2 * dil, N=C, C1=C, kt=3, dil_t=dil,
              a1_s=((T + 2 * H) * C, 0, C), act=cabi.ACT_LEAKY)
    assert eng.lib.precisions[-1] == 2
    ref = F.leaky_relu(F.conv1d(ref_h.half().double(), w.half().double(), dilation=dil), 0.2).permute(0, 2, 1)
    assert rel_l2(y.cpu(), ref) <= 1e-3                                  # FP16 output storage


def test_production_shape_and_graph_replay():
    """32 x 2 s at precision 2 (the benchmarked shape): 4 rows against the oracle; CUDA-graph replay bit-identical to eager."""
    m = _model("s1", 2)
    x = torch.randn(32, 1, 8000, generator=torch.Generator().manual_seed(SEED + 7))
    xc = x.cuda()
    eager = m(xc)
    m.use_cuda_graph(True)
    g1 = m(xc)
    g2 = m(xc)
    torch.cuda.synchronize()
    assert torch.equal(eager, g1) and torch.equal(g1, g2)
    rows = [0, 9, 22, 31]
    with torch.no_grad():
        ref = O.seanet_forward(m.cpu().state_dict(), m, x[rows])
    assert rel_l2(eager[rows].cpu(), ref) <= 1e-3


def test_empty_batch_and_short_input():
    m = _model("s1", 2)
    assert m(torch.zeros(0, 1, 4000, device="cuda")).shape == (0, 1, 16000)
    with pytest.raises(ValueError):
        m(torch.zeros(1, 1, 160, device="cuda"))
    assert m(torch.randn(1, 1, 200, device="cuda")).shape == (1, 1, 800)
