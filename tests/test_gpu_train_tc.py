"""-m gpu: the TF32 tensor-core training mode (TrainEngine.precision = 1): forward, data-gradient and weight-gradient GEMMs of the
convolutions on the tensor cores (csrc/tapgemm_tc.cu, csrc/wgrad_tc.cu) against torch autograd in fp64 on the CPU.

Tolerance: TF32 keeps 10 mantissa bits and the tensor core truncates the operands it reads, so a dot product carries ~1e-3 relative
error; the bar here is 3e-3 relative L2 per tensor (the exact-fp32 mode holds 1e-5 on the same shapes, tests/test_gpu_train_ops.py)."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from util import SEED, rel_l2

from aero_b200 import Aero, aero_kwargs, cabi
from aero_b200.train_engine import TrainEngine, _Conv

pytestmark = pytest.mark.gpu
TOL = 3e-3


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(SEED + seed))


def cl(x):   # NCHW (B,C,F,T) -> channels-last [B,F,T,C]
    return x.permute(0, 2, 3, 1).contiguous()


@pytest.fixture(scope="module")
def eng():
    torch.manual_seed(0)
    m = Aero(**aero_kwargs("aero_4-16_512_256")).cuda().train()
    m.train_precision = 1
    e = TrainEngine(m)
    assert e.precision == 1
    e.params, e.buffers = {}, {}
    return e


def run_backward(e, out, dy):
    e.acc(out, dy.contiguous().cuda().float().reshape(-1))
    for fn in reversed(e.tape):
        fn()
    torch.cuda.synchronize()


# name, conv, K, N, F_in, F_out, T
CONVS = [
    ("dec_3x3", dict(kf=3, kt=3, pad_f=1, pad_t=1), 96, 192, 8, 8, 95),
    ("dec_3x3_wide", dict(kf=3, kt=3, pad_f=1, pad_t=1), 384, 768, 2, 2, 70),          # K > 256: two k-tiles; N: six n-tiles
    ("enc_k8_s4", dict(kf=8, stride_f=4, pad_f=2), 48, 96, 64, 16, 95),
    ("enc_k8_s2", dict(kf=8, stride_f=2, pad_f=3), 96, 192, 16, 8, 61),
    ("dconv_k3_dil2", dict(kt=3, dil_t=2, pad_t=2), 96, 24, 4, 4, 130),
    ("k9", dict(kt=9, pad_t=4), 320, 48, 1, 1, 501),
    ("lstm_ih_like_1x1", dict(), 96, 384, 1, 1, 1000),
    ("ragged_channels", dict(kf=3, kt=3, pad_f=1, pad_t=1), 40, 20, 5, 5, 37),         # K, N not multiples of 32; T not of 32
]


@pytest.mark.parametrize("name,kw,K,N,Fi,Fo,T", CONVS, ids=[c[0] for c in CONVS])
def test_conv_tf32_forward_dgrad_wgrad(eng, name, kw, K, N, Fi, Fo, T):
    e = eng
    e._reset()
    B = 2
    cv = _Conv(**kw)
    x = rnd(B, K, Fi, T, seed=1).double().requires_grad_(True)
    w = (rnd(N, K, cv.kf, cv.kt, seed=2) / math.sqrt(K * cv.kf * cv.kt)).double().requires_grad_(True)
    b = rnd(N, seed=3).double().requires_grad_(True)
    ref = F.conv2d(x, w, b, stride=(cv.stride_f, 1), padding=(cv.pad_f, cv.pad_t), dilation=(1, cv.dil_t))
    assert ref.shape[2] == Fo
    dy = rnd(*ref.shape, seed=4).double()
    ref.backward(dy)
    e.params = {"w": w.detach().float().cuda(), "b": b.detach().float().cuda()}
    xg = cl(x.detach().float()).cuda()
    out = e.conv(xg, None, K, 0, "w", "b", cv, B, Fi, Fo, T, N)
    run_backward(e, out, cl(dy))
    errs = {"out": rel_l2(out.view(B, Fo, T, N).cpu(), cl(ref.detach())), "dw": rel_l2(e.pg["w"].cpu(), w.grad),
            "db": rel_l2(e.pg["b"].cpu(), b.grad), "dx": rel_l2(e.grad(xg).view(B, Fi, T, K).cpu(), cl(x.grad))}
    assert all(v < TOL for v in errs.values()), errs
    assert errs["db"] < 1e-5                                              # reductions stay fp32 / fp64
    assert errs["dw"] > 1e-6 and errs["out"] > 1e-6, ("the tensor-core path did not run", errs)


def test_two_sources_then_transposed_conv_with_crop_tf32(eng):
    e = eng
    e._reset()
    B, T, C1, C2, N, Fq, No = 2, 77, 48, 48, 96, 6, 24
    x1, x2 = rnd(B, C1, Fq, T, seed=1).double().requires_grad_(True), rnd(B, C2, Fq, T, seed=2).double().requires_grad_(True)
    w = (rnd(N, C1 + C2, 3, 3, seed=3) / 30).double().requires_grad_(True)
    b = rnd(N, seed=4).double().requires_grad_(True)
    y = F.conv2d(torch.cat([x1, x2], 1), w, b, padding=1)
    wt = (rnd(N, No, 8, 1, seed=5) / 30).double().requires_grad_(True)       # ConvTranspose2d weight [K, N_out, kf, 1]
    bt = rnd(No, seed=6).double().requires_grad_(True)
    z = F.conv_transpose2d(y, wt, bt, stride=(4, 1))[:, :, 2:-2]
    dz = rnd(*z.shape, seed=7).double()
    z.backward(dz)
    e.params = {"w": w.detach().float().cuda(), "b": b.detach().float().cuda(), "wt": wt.detach().float().cuda(), "bt": bt.detach().float().cuda()}
    a1, a2 = cl(x1.detach().float()).cuda(), cl(x2.detach().float()).cuda()
    yo = e.conv(a1, a2, C1, C2, "w", "b", _Conv(kf=3, kt=3, pad_f=1, pad_t=1), B, Fq, Fq, T, N)
    f_keep = (Fq - 1) * 4 + 8 - 4
    zo = e.conv(yo, None, N, 0, "wt", "bt", _Conv("convt", kf=8, stride_f=4, f_off=2), B, Fq, f_keep, T, No)
    run_backward(e, zo, cl(dz))
    assert rel_l2(zo.view(B, f_keep, T, No).cpu(), cl(z.detach())) < TOL
    for k, r in (("w", w), ("b", b), ("wt", wt), ("bt", bt)):
        assert rel_l2(e.pg[k].cpu(), r.grad) < TOL, k
    assert rel_l2(e.grad(a1).view(B, Fq, T, C1).cpu(), cl(x1.grad)) < TOL and rel_l2(e.grad(a2).view(B, Fq, T, C2).cpu(), cl(x2.grad)) < TOL


def test_wgrad_tc_against_simt_kernel_directly():
    """aero_tapgemm_wgrad with precision 1 (tensor cores) against precision 0 (SIMT) on the same buffers: strided activations (a channel slice
    of a wider tensor), un-padded time kernel (T_in != T) and a pixel count that leaves most split-K slices ragged."""
    lib = cabi.load()
    dev = torch.device("cuda")
    B, Fq, T_in, kt, Cw, C1, N = 3, 5, 83, 5, 64, 32, 48
    T = T_in - (kt - 1)
    xw = rnd(B, Fq, T_in, Cw, seed=11).to(dev)
    x = xw[..., 16:16 + C1]                                                # channel slice: strides of the wide tensor
    dy = rnd(B, Fq, T, N, seed=12).to(dev)
    st = torch.cuda.current_stream().cuda_stream
    outs = []
    for prec in (0, 1):
        p = cabi.TapGemmParams(B, Fq, T, N, Fq, T_in, C1, 0, cabi.TAPS_CONV, 1, kt, 1, 0, 1, 0, 0, cabi.ACT_NONE, 0, 0, 1,
                               Fq * T_in * Cw, T_in * Cw, Cw, 0, 0, 0, 0, Fq * T * N, T * N, N, 0, 0, 0, 0, 0, prec, 0)
        gw = torch.zeros(N, C1, 1, kt, device=dev)
        cabi.check(lib.aero_tapgemm_wgrad(C.c_void_p(x.data_ptr()), None, C.c_void_p(dy.data_ptr()), C.c_void_p(gw.data_ptr()), C.byref(p),
                                          gw.stride(0), gw.stride(1), 1, C.c_void_p(st)), lib)
        outs.append(gw)
    torch.cuda.synchronize()
    ref = torch.einsum("bftn,bftjc->ncj", dy.double(), x.double().unfold(2, kt, 1).permute(0, 1, 2, 4, 3)).view(N, C1, 1, kt)
    assert rel_l2(outs[0].cpu(), ref.cpu()) < 1e-5
    e = rel_l2(outs[1].cpu(), ref.cpu())
    assert 1e-6 < e < TOL, e


@pytest.mark.parametrize("case", ["t1_4-16_hop256", "t3_11-44_stereo"])
def test_generator_gradients_tf32_mode_against_fp64_golden(golden_dir, case):
    """Whole-model gradients in the TF32 mode against the committed fp64 golden of the reference (tests/golden/make_golden_train.py).
    This network's gradient is badly conditioned (GroupNorm / BatchNorm backward subtract projections of nearly equal size, ReLU kinks
    behind BatchNorm: its own fp32 run is 1.3e-3 .. 2.9e-3 from its fp64 run), so 2^-11 operand errors surface as a few percent: measured
    4.9e-2 .. 7.4e-2 for all gradients as one vector, the same as the reference algorithm under PyTorch's default cuDNN TF32 (next test).
    Bars: forward output 2e-3, all gradients together 1e-1, no parameter beyond 0.5 (a wrong kernel gives O(1) on everything upstream)."""
    import os
    import numpy as np
    from util import trained_like_, weights_digest, white_noise
    from test_gpu_train import cotangent, grad_report
    g = np.load(os.path.join(golden_dir, case + ".npz"))
    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs(str(g["exp"])))
    m.load_state_dict(trained_like_(m.state_dict()))
    assert weights_digest(m.state_dict()) == pytest.approx(float(g["digest"]), rel=1e-12)
    m = m.cuda().train()
    m.train_precision = 1
    mix = white_noise((int(g["B"]), m.in_channels, int(g["L"]))).cuda()
    out = m(mix)
    flat = out.detach().reshape(-1).cpu()
    e_out = rel_l2(flat[torch.from_numpy(g["out_idx"].astype(np.int64))], g["out_val"])
    R = cotangent(tuple(out.shape), SEED).cuda()
    ((out * R).sum() / out.numel()).backward()
    torch.cuda.synchronize()
    rows, total = grad_report(m, g)
    print(f"{case} (TF32 training mode): output rel_l2 {e_out:.3e}; all gradients together {total:.3e}; worst:")
    for err, name, rms in rows[:6]:
        print(f"   {err:.3e}  {name}  (ref rms {rms:.3e})")
    assert e_out < 2e-3
    assert total < 1e-1, total
    assert rows[0][0] < 0.5, rows[:5]


def _total_deviation(grads, g):
    """All gradients as one vector against the golden samples (the `total` of test_gpu_train.grad_report), from a name -> tensor map."""
    import numpy as np
    num = den = 0.0
    for name, got_t in grads.items():
        ref = torch.from_numpy(g["g_val/" + name]).double()
        idx = torch.from_numpy(g["g_idx/" + name].astype(np.int64))
        got = got_t.detach().reshape(-1).cpu().double()[idx]
        scale = got_t.numel() / ref.numel()
        num += scale * float((got - ref).pow(2).sum())
        den += scale * float(ref.pow(2).sum())
    return (num / den) ** 0.5


@pytest.mark.parametrize("case", ["t1_4-16_hop256"])
def test_tf32_mode_is_as_accurate_as_the_reference_under_pytorchs_default_tf32(golden_dir, case):
    """Calibration of the TF32 training mode.  The reference trains on a GPU with PyTorch's defaults, i.e. cuDNN convolutions and the
    cuDNN LSTM in TF32 (torch.backends.cudnn.allow_tf32 = True).  The oracle (the reference's algorithm as torch functional code) is run
    here on the GPU under exactly those defaults and its gradients are measured against the fp64 golden; this library's TF32 mode must
    not deviate more than 1.5x as much -- i.e. switching it on costs no more accuracy than the reference's own default arithmetic."""
    import os
    import numpy as np
    from util import trained_like_, white_noise
    from test_gpu_train import cotangent
    from oracle import aero_oracle as O
    g = np.load(os.path.join(golden_dir, case + ".npz"))
    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs(str(g["exp"])))
    m.load_state_dict(trained_like_(m.state_dict()))
    mix = white_noise((int(g["B"]), m.in_channels, int(g["L"]))).cuda()
    R = cotangent(tuple(int(v) for v in g["out_shape"]), SEED).cuda()
    names = [n for n, _ in m.named_parameters()]

    def oracle_grads(allow_tf32):
        sd = {k: (v.clone().cuda().requires_grad_(k in names) if v.dtype.is_floating_point else v.clone().cuda()) for k, v in m.state_dict().items()}
        old = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = allow_tf32
        O.BN_TRAIN = True
        try:
            out = O.aero_forward(sd, m.geom, mix)
            ((out * R).sum() / out.numel()).backward()
        finally:
            O.BN_TRAIN = False
            torch.backends.cudnn.allow_tf32 = old
        return {k: sd[k].grad for k in names if sd[k].grad is not None}

    dev_ref_tf32 = _total_deviation(oracle_grads(True), g)
    dev_ref_fp32 = _total_deviation(oracle_grads(False), g)
    mm = m.cuda().train()
    devs = {}
    for prec in (0, 1):
        mm.train_precision = prec
        mm.zero_grad(set_to_none=True)
        out = mm(mix)
        ((out * R).sum() / out.numel()).backward()
        devs[prec] = _total_deviation({n: p.grad for n, p in mm.named_parameters()}, g)
    torch.cuda.synchronize()
    print(f"{case}: all-gradient deviation from the fp64 golden -- reference algorithm on this GPU: fp32 {dev_ref_fp32:.3e}, PyTorch-default TF32 "
          f"{dev_ref_tf32:.3e}; this library: exact mode {devs[0]:.3e}, TF32 mode {devs[1]:.3e}")
    assert devs[0] < 5e-3
    assert devs[1] < 1.5 * max(dev_ref_tf32, 1e-3) or devs[1] < 1e-2, (devs, dev_ref_tf32)


@pytest.mark.parametrize("Fq,M", [(8, 1504), (16, 3000), (64, 4808), (256, 2004)])
def test_gated_frequency_mix_tf32(eng, Fq, M):
    """FTB's frequency mix out[b][f'][m] = gate[b][m] * sum_f W[f'][f] x[b][f][m] on the tensor cores (AERO_TAPS_MIX) against fp64."""
    e = eng
    e._reset()
    B = 2
    x, Wfc, gate = rnd(B, Fq, M, seed=1), rnd(Fq, Fq, seed=2) / math.sqrt(Fq), rnd(B, M, seed=3)
    ref = torch.einsum("gf,bfm->bgm", Wfc.double(), x.double()) * gate.double()[:, None, :]
    out = e._freq_mix(x.cuda().reshape(-1), Wfc.cuda(), gate.cuda().reshape(-1), B, Fq, M)
    un = e._freq_mix(x.cuda().reshape(-1), Wfc.cuda(), None, B, Fq, M)
    torch.cuda.synchronize()
    err = rel_l2(out.view(B, Fq, M).cpu(), ref)
    assert 1e-6 < err < TOL, err
    assert rel_l2(un.view(B, Fq, M).cpu(), torch.einsum("gf,bfm->bgm", Wfc.double(), x.double())) < TOL


# ------------------------------------------------------------------------------------------------ 3xTF32 (fp32-grade tensor-core mode)
@pytest.fixture(scope="module")
def eng3():
    torch.manual_seed(0)
    m = Aero(**aero_kwargs("aero_4-16_512_256")).cuda().train()
    m.train_precision = 3
    e = TrainEngine(m)
    assert e.precision == 3
    e.params, e.buffers = {}, {}
    return e


@pytest.mark.parametrize("name,kw,K,N,Fi,Fo,T", CONVS, ids=[c[0] for c in CONVS])
def test_conv_3xtf32_is_fp32_grade(eng3, name, kw, K, N, Fi, Fo, T):
    """The same shapes in the 3xTF32 mode: three tensor-core products per GEMM on hi / lo operand halves.  Bar: 3e-5 against fp64 -- the
    operand split is exact to 2^-22, what remains is the tensor core's fp32 accumulation over K (1.1e-5 measured at K = 6912, 1e-6 at
    K = 864; the SIMT kernels hold 1e-5 on every shape) -- and the tensor-core path must have been the one that ran."""
    e = eng3
    e._reset()
    lib = cabi.load()
    B = 2
    cv = _Conv(**kw)
    x = rnd(B, K, Fi, T, seed=1).double().requires_grad_(True)
    w = (rnd(N, K, cv.kf, cv.kt, seed=2) / math.sqrt(K * cv.kf * cv.kt)).double().requires_grad_(True)
    b = rnd(N, seed=3).double().requires_grad_(True)
    ref = F.conv2d(x, w, b, stride=(cv.stride_f, 1), padding=(cv.pad_f, cv.pad_t), dilation=(1, cv.dil_t))
    dy = rnd(*ref.shape, seed=4).double()
    ref.backward(dy)
    e.params = {"w": w.detach().float().cuda(), "b": b.detach().float().cuda()}
    xg = cl(x.detach().float()).cuda()
    n0 = lib.aero_launch_count()
    out = e.conv(xg, None, K, 0, "w", "b", cv, B, Fi, Fo, T, N)
    run_backward(e, out, cl(dy))
    launches = lib.aero_launch_count() - n0
    errs = {"out": rel_l2(out.view(B, Fo, T, N).cpu(), cl(ref.detach())), "dw": rel_l2(e.pg["w"].cpu(), w.grad),
            "db": rel_l2(e.pg["b"].cpu(), b.grad), "dx": rel_l2(e.grad(xg).view(B, Fi, T, K).cpu(), cl(x.grad))}
    assert all(v < 3e-5 for v in errs.values()), errs
    assert launches >= 3 * 3 + 3 + 2, launches        # 9 GEMM passes, 3 operand splits, 2 weight repacks at least


def test_two_sources_then_transposed_conv_3xtf32(eng3):
    e = eng3
    e._reset()
    B, T, C1, C2, N, Fq, No = 2, 77, 48, 48, 96, 6, 24
    x1, x2 = rnd(B, C1, Fq, T, seed=1).double().requires_grad_(True), rnd(B, C2, Fq, T, seed=2).double().requires_grad_(True)
    w = (rnd(N, C1 + C2, 3, 3, seed=3) / 30).double().requires_grad_(True)
    b = rnd(N, seed=4).double().requires_grad_(True)
    y = F.conv2d(torch.cat([x1, x2], 1), w, b, padding=1)
    wt = (rnd(N, No, 8, 1, seed=5) / 30).double().requires_grad_(True)
    bt = rnd(No, seed=6).double().requires_grad_(True)
    z = F.conv_transpose2d(y, wt, bt, stride=(4, 1))[:, :, 2:-2]
    dz = rnd(*z.shape, seed=7).double()
    z.backward(dz)
    e.params = {"w": w.detach().float().cuda(), "b": b.detach().float().cuda(), "wt": wt.detach().float().cuda(), "bt": bt.detach().float().cuda()}
    a1, a2 = cl(x1.detach().float()).cuda(), cl(x2.detach().float()).cuda()
    yo = e.conv(a1, a2, C1, C2, "w", "b", _Conv(kf=3, kt=3, pad_f=1, pad_t=1), B, Fq, Fq, T, N)
    f_keep = (Fq - 1) * 4 + 8 - 4
    zo = e.conv(yo, None, N, 0, "wt", "bt", _Conv("convt", kf=8, stride_f=4, f_off=2), B, Fq, f_keep, T, No)
    run_backward(e, zo, cl(dz))
    assert rel_l2(zo.view(B, f_keep, T, No).cpu(), cl(z.detach())) < 3e-5
    for k, r in (("w", w), ("b", b), ("wt", wt), ("bt", bt)):
        assert rel_l2(e.pg[k].cpu(), r.grad) < 3e-5, k
    assert rel_l2(e.grad(a1).view(B, Fq, T, C1).cpu(), cl(x1.grad)) < 3e-5 and rel_l2(e.grad(a2).view(B, Fq, T, C2).cpu(), cl(x2.grad)) < 3e-5


@pytest.mark.parametrize("case", ["t1_4-16_hop256", "t3_11-44_stereo"])
def test_generator_gradients_3xtf32_against_fp64_golden(golden_dir, case):
    """Whole-model gradients in the 3xTF32 mode against the fp64 golden of the reference.  Measured: all gradients together 5.1e-3 (t1) and
    8.1e-4 (t3), worst parameter 3.3e-3 -- between the exact SIMT mode (9.9e-4 on t1) and plain TF32 (6.5e-2), and within 2x of what the
    reference algorithm gives in PyTorch fp32 on the same GPU (2.6e-3 on t1, calibration test above): the ~1e-6 accumulation error of a
    tensor-core GEMM goes through the same ill-conditioned backward as every other rounding.  Bars: forward 2e-5; all gradients together
    1e-2 (2e-3 for the strict case), a third of the parameters within 1e-3, none beyond 5e-2."""
    import os
    import numpy as np
    from util import trained_like_, weights_digest, white_noise
    from test_gpu_train import GRAD_TOL, STRICT, cotangent, grad_report
    g = np.load(os.path.join(golden_dir, case + ".npz"))
    torch.manual_seed(SEED)
    m = Aero(**aero_kwargs(str(g["exp"])))
    m.load_state_dict(trained_like_(m.state_dict()))
    assert weights_digest(m.state_dict()) == pytest.approx(float(g["digest"]), rel=1e-12)
    m = m.cuda().train()
    m.train_precision = 3
    mix = white_noise((int(g["B"]), m.in_channels, int(g["L"]))).cuda()
    out = m(mix)
    flat = out.detach().reshape(-1).cpu()
    e_out = rel_l2(flat[torch.from_numpy(g["out_idx"].astype(np.int64))], g["out_val"])
    R = cotangent(tuple(out.shape), SEED).cuda()
    ((out * R).sum() / out.numel()).backward()
    torch.cuda.synchronize()
    rows, total = grad_report(m, g)
    ok = sum(1 for r in rows if r[0] < GRAD_TOL)
    print(f"{case} (3xTF32 training mode): output rel_l2 {e_out:.3e}; all gradients together {total:.3e}; {ok}/{len(rows)} within {GRAD_TOL:g}; worst:")
    for err, name, rms in rows[:4]:
        print(f"   {err:.3e}  {name}  (ref rms {rms:.3e})")
    assert e_out < 2e-5
    assert total < (2e-3 if case in STRICT else 1e-2), total
    assert ok >= len(rows) / 3, (ok, len(rows))
    assert rows[0][0] < 5e-2, rows[:5]
