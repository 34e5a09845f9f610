"""-m gpu: the training kernels on the dispatch paths that only production-size launches reach, and FusedAdam against
torch.optim.Adam over many steps.

test_gpu_train_ops.py checks every training op at a few rows against fp64 autograd with one rel-L2 per tensor.  At those sizes
the LSTM training kernels only ever run their NT = 4 bodies (csrc/train_rnn.cu, pick_nt), the attention backward never streams
more than two tiles, and the column-sum kernel (csrc/train.cu, aero_colsum) never reaches its capped grid split.  Here:
  1. BiLSTM training at every <H, NT> instantiation pick_nt can choose, with the sequence counts picked from the device's SM
     count and the instantiation that ran read back from the profiler;
  2. LocalState attention training at every head dim, multi-tile T with partial and one-past last tiles;
  3. aero_colsum, both kernels, float and double outputs, capped splits, carries, unroll tails;
  4. the element-wise training kernels (add, add_f64, bcast_add, scale_rows, gram, lstm_fold);
  5. FusedAdam for 12 steps against torch.optim.Adam in fp64.
Reference principle: fp64 on exactly the fp32 operand values the kernel reads; bars per row / column / slice, so that one bad
CTA or tile cannot be averaged away."""
import copy
import ctypes as C
import io
import math
import re
import warnings

import pytest
import torch
import torch.nn.functional as F

from util import SEED

from aero_b200 import Aero, aero_kwargs, cabi
from aero_b200.train_engine import TrainEngine

pytestmark = pytest.mark.gpu


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(SEED + seed))


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope="module")
def lib():
    return cabi.load()


@pytest.fixture(scope="module")
def eng():
    torch.manual_seed(0)
    m = Aero(**aero_kwargs("aero_4-16_512_256")).cuda().train()
    e = TrainEngine(m)
    e.params, e.buffers = {}, {}
    return e


@pytest.fixture(scope="module")
def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def run_backward(e, out, dy):
    e.acc(out, dy.contiguous().cuda().float().reshape(-1))
    for fn in reversed(e.tape):
        fn()
    torch.cuda.synchronize()


def kernels_launched(fn, needed, tries=3):
    """Names of the CUDA kernels fn launches (torch.profiler, CUPTI activity).  A profiling session does not always record the
    kernels that run right after it starts or right before it stops, so fn is padded with spin kernels on both sides, and fn runs
    again (it must give the same result when repeated) while some kernel named in `needed` is absent from the record.  None when
    no session recorded them all."""
    for _ in range(tries):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            torch.cuda._sleep(1 << 20)
            torch.cuda.synchronize()
            fn()
            torch.cuda._sleep(1 << 20)
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if all(any(k in n for n in names) for k in needed):
            return names
    return None


def instantiations(names, kernel):
    """{(template args)} of kernel among the launched kernel names, e.g. {(48, 8)} for lstm_train_fwd_kernel<48, 8>."""
    pat = re.compile(re.escape(kernel) + r"<([0-9, ]+)>")
    return {tuple(int(v) for v in m.group(1).split(",")) for n in names for m in [pat.search(n)] if m}


def worst_rel(got, ref, dims):
    """Largest per-slice rel-L2 of got against ref, slices indexed by the leading `dims` axes."""
    got, ref = got.double().reshape(*ref.shape[:dims], -1), ref.double().reshape(*ref.shape[:dims], -1)
    e = (got - ref).norm(dim=-1) / ref.norm(dim=-1).clamp_min(1e-30)
    return float(e.max())


# ------------------------------------------------------------------------------------------------ 1. BiLSTM training
_LSTM_STEPS, _LSTM_STRIDE = 200, 100        # reference BLSTM(max_steps=200): windows of 200 frames every 100 frames


def nt_band_rows(nt, n_win, num_sms):
    """Fewest rows whose rows * n_win sequences make pick_nt (csrc/train_rnn.cu) choose nt, plus enough that the last CTA is
    partial.  pick_nt halves from 16 while cdiv(n_seq, nt) * 2 < num_sms."""
    if nt == 4:
        return 3 if n_win > 1 else 5
    lo = nt * (math.ceil(num_sms / 2) - 1) + 1            # the smallest n_seq with cdiv(n_seq, nt) * 2 >= num_sms
    rows = math.ceil(lo / n_win)
    while (rows * n_win) % nt == 0:
        rows += 1
    return rows


def expected_nt(n_seq, nt_max, num_sms):
    nt = nt_max
    while nt > 4 and -(-n_seq // nt) * 2 < num_sms:
        nt //= 2
    return nt


# (H, band NT, T): T > 200 runs the windowed recurrence (T = 501: 6 windows, the production length of a 2 s clip at hop 64),
# T <= 200 one window per row
LSTM_CASES = [(12, 4, 230), (12, 8, 150), (12, 16, 230),
              (24, 4, 77), (24, 8, 501), (24, 16, 180),
              (48, 4, 230), (48, 8, 260), (48, 16, 501),
              (96, 4, 230), (96, 8, 230), (96, 16, 64)]


def blstm_reference(x, lstm, lin):
    """test_gpu_train_ops.test_blstm_block's statement: reference framing + 2-layer BiLSTM + Linear + skip."""
    rows, H, T = x.shape
    if T > _LSTM_STEPS:
        width, stride = _LSTM_STEPS, _LSTM_STRIDE
        n_frames = math.ceil(T / stride)
        xp = F.pad(x, (0, (n_frames - 1) * stride + width - T))
        fr = xp.unfold(-1, width, stride)                     # [rows, H, nF, width]
        nF = fr.shape[2]
        xin = fr.permute(0, 2, 1, 3).reshape(-1, H, width)
    else:
        xin, nF = x, 1
    yl = lstm(xin.permute(2, 0, 1))[0]
    yl = lin(yl).permute(1, 2, 0)
    if T > _LSTM_STEPS:
        frames = yl.reshape(rows, -1, H, width)
        limit = stride // 2
        outp = []
        for k in range(nF):
            if k == 0:
                outp.append(frames[:, k, :, :-limit])
            elif k == nF - 1:
                outp.append(frames[:, k, :, limit:])
            else:
                outp.append(frames[:, k, :, limit:-limit])
        yl = torch.cat(outp, -1)[..., :T]
    return yl + x


@pytest.mark.parametrize("H,nt,T", LSTM_CASES, ids=[f"H{h}_nt{n}_T{t}" for h, n, t in LSTM_CASES])
def test_blstm_every_instantiation(eng, num_sms, H, nt, T):
    e = eng
    e._reset()
    n_win = math.ceil(T / _LSTM_STRIDE) if T > _LSTM_STEPS else 1
    rows = nt_band_rows(nt, n_win, num_sms)
    n_seq = rows * n_win
    assert expected_nt(n_seq, 16, num_sms) == nt and n_seq % nt != 0
    torch.manual_seed(SEED + 1)
    lstm = torch.nn.LSTM(bidirectional=True, num_layers=2, hidden_size=H, input_size=H).double()
    lin = torch.nn.Linear(2 * H, H).double()
    x = rnd(rows, H, T, seed=1).double().requires_grad_(True)
    y = blstm_reference(x, lstm, lin)
    dy = rnd(*y.shape, seed=2).double()
    y.backward(dy)
    q = "enc.dconv.layers.0"
    e.params = {q + ".lstm.lstm." + k: p.detach().float().cuda() for k, p in lstm.named_parameters()}
    e.params.update({q + ".lstm.linear." + k: p.detach().float().cuda() for k, p in lin.named_parameters()})
    hg = x.detach().float().permute(0, 2, 1).contiguous().cuda()           # [rows][T][H]
    res = {}

    def run():
        e._reset()
        res["y"] = e.blstm(hg, q, rows, T, H)
        run_backward(e, res["y"], dy.permute(0, 2, 1))
    names = kernels_launched(run, ("lstm_train_fwd_kernel", "lstm_bwd_kernel"))
    if names is None:
        run()
        warnings.warn(f"H={H} NT={nt}: the profiler recorded no LSTM kernel, the instantiation that ran is unchecked")
    else:
        fwd, bwd = instantiations(names, "lstm_train_fwd_kernel"), instantiations(names, "lstm_bwd_kernel")
        assert fwd == {(H, nt)}, (fwd, n_seq)
        assert bwd == {(H, min(nt, 8 if H == 96 else 16))}, (bwd, n_seq)        # aero_lstm_bwd caps H = 96 at NT = 8
        assert n_win == 1 or any("lstm_fold_kernel" in n for n in names)
    # per row: output and input gradient (every sequence of a row lives in one or two CTAs)
    e_y = worst_rel(res["y"].view(rows, T, H).cpu(), y.detach().permute(0, 2, 1), 1)
    e_dx = worst_rel(e.grad(hg).view(rows, T, H).cpu(), x.grad.permute(0, 2, 1), 1)
    worst = sorted([(worst_rel(e.pg[q + ".lstm.lstm." + k].cpu(), p.grad, 0), k) for k, p in lstm.named_parameters()] +
                   [(worst_rel(e.pg[q + ".lstm.linear." + k].cpu(), p.grad, 0), k) for k, p in lin.named_parameters()], reverse=True)
    print(f"H={H} NT={nt} T={T} rows={rows} n_seq={n_seq}: worst row y {e_y:.2e} dx {e_dx:.2e}; params {worst[0][0]:.2e} ({worst[0][1]})")
    assert e_y < 1e-6 and e_dx < 1e-6, (e_y, e_dx)
    assert worst[0][0] < 1e-5, worst[:4]


def test_lstm_fold_six_windows(lib):
    """aero_lstm_fold at T = 501 (6 windows, the last one covering one real frame) against its fp64 statement."""
    rows, T, steps, stride, Cc = 7, 501, _LSTM_STEPS, _LSTM_STRIDE, 192
    n_win = math.ceil(T / stride)
    w = rnd(rows * n_win, steps, Cc, seed=3)
    ref = torch.zeros(rows, T, Cc, dtype=torch.float64)
    mag = torch.zeros_like(ref)
    w64 = w.double().view(rows, n_win, steps, Cc)
    for k in range(n_win):
        n = min(steps, T - k * stride)
        ref[:, k * stride:k * stride + n] += w64[:, k, :n]
        mag[:, k * stride:k * stride + n] += w64[:, k, :n].abs()
    wg = w.cuda()
    out = torch.full((rows, T, Cc), float("nan"), device="cuda")
    cabi.check(lib.aero_lstm_fold(ptr(wg), ptr(out), rows, T, n_win, steps, stride, Cc, stream()), lib)
    torch.cuda.synchronize()
    err = (out.cpu().double() - ref).abs()
    assert bool(torch.isfinite(out).all())
    assert bool((err <= 2.0 ** -23 * mag).all()), float((err / mag.clamp_min(1e-30)).max())


# ------------------------------------------------------------------------------------------------ 2. attention training
_HEADS, _NDECAY, _TILE = 4, 4, 128          # LocalState(heads=4, ndecay=4); csrc/train_attn.cu streams 128-query / 128-key tiles


def attention_reference(X, H):
    """test_gpu_train_ops.test_local_state_attention_block's core statement, on the [rows][T][ld] buffer the kernels read
    (query | key | content | decay logits).  Returns out [rows][T][H] and lse [rows][heads][T]."""
    R, T, _ = X.shape
    D = H // _HEADS
    q = X[..., :H].reshape(R, T, _HEADS, D).permute(0, 2, 3, 1)
    k = X[..., H:2 * H].reshape(R, T, _HEADS, D).permute(0, 2, 3, 1)
    v = X[..., 2 * H:3 * H].reshape(R, T, _HEADS, D).permute(0, 2, 3, 1)
    dl = X[..., 3 * H:3 * H + _HEADS * _NDECAY].reshape(R, T, _HEADS, _NDECAY).permute(0, 2, 3, 1)
    idx = torch.arange(T)
    delta = idx[:, None] - idx[None, :]
    dots = torch.einsum("bhct,bhcs->bhts", k, q) / math.sqrt(D)
    decays = torch.arange(1, _NDECAY + 1, dtype=torch.float64)
    dk = -decays.view(-1, 1, 1) * delta.abs() / math.sqrt(_NDECAY)
    dots = dots + torch.einsum("fts,bhfs->bhts", dk, torch.sigmoid(dl) / 2)
    dots = dots.masked_fill(torch.eye(T, dtype=torch.bool), -100)
    w = torch.softmax(dots, dim=2)
    out = torch.einsum("bhts,bhct->bhcs", w, v).permute(0, 3, 1, 2).reshape(R, T, H)
    return out, torch.logsumexp(dots, dim=2)


def slices(t, rows, T, H):
    """[rows][T][H'] -> [rows][heads][T][H' / heads]"""
    return t.reshape(rows, T, _HEADS, -1).permute(0, 2, 1, 3)


def tile_worst(got, ref):
    """Largest rel-L2 over (row, head, 128-position tile) of [rows][heads][T][d] tensors; a tile's denominator is floored at a
    tenth of the norm its share of the (row, head) slice would have, so that a one-position tile is held to the slice's scale."""
    rows, heads, T, d = ref.shape
    worst = 0.0
    whole = ref.double().norm(dim=(2, 3))
    for t0 in range(0, T, _TILE):
        n = min(_TILE, T - t0)
        g, r = got[:, :, t0:t0 + n].double(), ref[:, :, t0:t0 + n].double()
        den = torch.maximum(r.norm(dim=(2, 3)), 0.1 * whole * math.sqrt(n / T)).clamp_min(1e-30)
        worst = max(worst, float(((g - r).norm(dim=(2, 3)) / den).max()))
    return worst


ATTN_CASES = [(H, T) for H in (12, 24, 48, 96) for T in (501, 128, 129)]


@pytest.mark.parametrize("H,T", ATTN_CASES, ids=[f"H{h}_T{t}" for h, t in ATTN_CASES])
def test_attention_every_head_dim(lib, num_sms, H, T):
    D = H // _HEADS
    ld = 3 * H + _HEADS * _NDECAY
    tiles = math.ceil(T / _TILE)
    rows = math.ceil(2 * num_sms / (tiles * _HEADS)) + 1              # more than two CTAs per SM
    X = rnd(rows, T, ld, seed=5)
    # decay logits: half the queries near -1 (local attention, as trained), half near -9 (slope ~ 0: every key tile counts)
    far = torch.rand(rows, T, _HEADS, 1, generator=torch.Generator().manual_seed(SEED + 6)) < 0.5
    X[..., 3 * H:] = (X[..., 3 * H:].reshape(rows, T, _HEADS, _NDECAY) + torch.where(far, -9.0, -1.0)).reshape(rows, T, -1)
    dout = rnd(rows, T, H, seed=7)
    Xg, doutg = X.cuda(), dout.cuda()
    out = torch.full((rows, T, H), float("nan"), device="cuda")
    lse = torch.full((rows, _HEADS, T), float("nan"), device="cuda")
    dX = torch.full((rows, T, ld), float("nan"), device="cuda")
    ap = cabi.AttnParams(rows, T, H, _HEADS, _NDECAY, ld, 0)

    # (the head dim selects the instantiation; one that is missing is an error, not a fallback)
    cabi.check(lib.aero_local_attn_train_fwd(ptr(Xg), ptr(out), ptr(lse), C.byref(ap), stream()), lib)
    cabi.check(lib.aero_local_attn_bwd(ptr(Xg), ptr(out), ptr(lse), ptr(doutg), ptr(dX), C.byref(ap), stream()), lib)
    torch.cuda.synchronize()
    # fp64 reference on the same fp32 operands, a few rows at a time (the score tensor is rows x heads x T x T)
    ro, rl, rg = [], [], []
    for r0 in range(0, rows, 4):
        Xr = X[r0:r0 + 4].double().requires_grad_(True)
        o, l_ = attention_reference(Xr, H)
        o.backward(dout[r0:r0 + 4].double())
        ro.append(o.detach())
        rl.append(l_.detach())
        rg.append(Xr.grad)
    ro, rl, rg = torch.cat(ro), torch.cat(rl), torch.cat(rg)
    got, gX = out.cpu(), dX.cpu()
    assert bool(torch.isfinite(got).all() and torch.isfinite(gX).all() and torch.isfinite(lse).all())
    e_lse = float(((lse.cpu().double() - rl).abs() / (1 + rl.abs())).max())
    errs = {"out": tile_worst(slices(got, rows, T, H), slices(ro, rows, T, H))}
    for i, nm in enumerate(("dQ", "dK", "dV")):
        errs[nm] = tile_worst(slices(gX[..., i * H:(i + 1) * H], rows, T, H), slices(rg[..., i * H:(i + 1) * H], rows, T, H))
    errs["dDecay"] = tile_worst(slices(gX[..., 3 * H:], rows, T, H), slices(rg[..., 3 * H:], rows, T, H))
    print(f"H={H} (head dim {D}) T={T} rows={rows}: lse {e_lse:.2e}, worst (row, head, tile) " +
          " ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert e_lse < 1e-5, e_lse
    assert errs["out"] < 5e-6, errs
    assert max(errs["dQ"], errs["dK"], errs["dV"]) < 2e-5, errs
    assert errs["dDecay"] < 5e-5, errs


# ------------------------------------------------------------------------------------------------ 3. column sums
def colsum4_step(N, rows, n_seg):
    """Rows between two reads of one colsum4 thread (aero_colsum's grid-y split, csrc/train.cu)."""
    ys = min(max(-(-rows // 128), 1), 132 * 8 // (-(-N // 128) * n_seg) + 1, 65535)
    return ys * 8


def colsum_step(N, rows, n_seg):
    ys = min(max(-(-rows // 512), 1), 132 * 16 // (-(-N // 32) * n_seg) + 1, 65535)
    return ys * 8


def unroll_tail_rows(step, m=4):
    """Rows at which every colsum4 thread runs m unrolled rounds of 4 rows plus a 1- or 2-row tail."""
    return step * (4 * m + 1) + step // 3


_B, _F, _T = 16, 32, 501
COLSUM_CASES = [
    # name, N, n_inner, inner_s, n_outer, outer_s, n_seg, seg_sx, seg_so, out_double, with_z, outs, misalign
    ("c4_tiny_rows", 48, 5, 48, 1, 0, 1, 0, 0, False, False, "1", False),
    ("c4_capped_unroll_tail_f32", 192, "tail4", 192, 1, 0, 1, 0, 0, False, True, "2", False),
    ("c4_capped_unroll_tail_f64", 48, "tail4", 48, 1, 0, 1, 0, 0, True, True, "12", False),
    ("c4_emb_segments_carry", 48, _T, 48, _B, _F * _T * 48, _F, _T * 48, 48, True, False, "1", False),
    ("c4_outer_carry_small_inner", 96, 100, 96, 3000, 100 * 96 + 8, 1, 0, 0, False, True, "12", False),
    ("c4_segments_z_f32", 384, 1000, 384, 2, 1000 * 384, 3, 2 * 1000 * 384, 384, False, True, "12", False),
    ("scalar_n_mod4_tiny", 45, 7, 45, 1, 0, 1, 0, 0, True, True, "12", False),
    ("scalar_misaligned_prod", 48, 200_000, 48, 1, 0, 1, 0, 0, True, True, "12", True),
    ("scalar_capped_split", 7, 1_100_000, 7, 1, 0, 1, 0, 0, False, False, "1", False),
    ("scalar_segments_outer", 45, 501, 45, 16, 32 * 501 * 45, 32, 501 * 45, 45, False, True, "2", False),
]


@pytest.mark.parametrize("name,N,n_inner,inner_s,n_outer,outer_s,n_seg,seg_sx,seg_so,dbl,with_z,outs,misalign", COLSUM_CASES,
                         ids=[c[0] for c in COLSUM_CASES])
def test_colsum(lib, name, N, n_inner, inner_s, n_outer, outer_s, n_seg, seg_sx, seg_so, dbl, with_z, outs, misalign):
    """aero_colsum takes colsum4_kernel for N % 4 == 0 with 16-byte-aligned rows and strides (`vec`), colsum_kernel otherwise."""
    vec = not misalign and N % 4 == 0
    if n_inner == "tail4":
        n_inner = unroll_tail_rows(colsum4_step(N, 10 ** 9, n_seg))
        assert colsum4_step(N, n_inner, n_seg) == colsum4_step(N, 10 ** 9, n_seg)      # the split is at its cap
    rows = n_inner * n_outer
    step = colsum4_step(N, rows, n_seg) if vec else colsum_step(N, rows, n_seg)
    if "carry" in name:
        assert step % n_inner != 0
    extent = (n_seg - 1) * seg_sx + (n_outer - 1) * outer_s + (n_inner - 1) * inner_s + N
    off = 1 if misalign else 0
    buf = rnd(extent + off, seed=8) + 0.3
    zbuf = rnd(extent + off, seed=9) if with_z else None
    shape, strides = (n_seg, n_outer, n_inner, N), (seg_sx, outer_s, inner_s, 1)
    xv = buf.double().as_strided(shape, strides, off)
    ref1, mag1 = xv.sum((1, 2)), xv.abs().sum((1, 2))
    if with_z:
        zv = zbuf.double().as_strided(shape, strides, off)
        ref2, mag2 = (xv * zv).sum((1, 2)), (xv * zv).abs().sum((1, 2))
    odt = torch.float64 if dbl else torch.float32
    so = seg_so if n_seg > 1 else N
    n_out = (n_seg - 1) * so + N
    pre1, pre2 = rnd(n_out, seed=10).to(odt), rnd(n_out, seed=11).to(odt)       # the kernel accumulates into its outputs
    xg = buf.cuda()
    zg = zbuf.cuda() if with_z else None
    x_ptr = C.c_void_p(xg.data_ptr() + 4 * off)
    z_ptr = C.c_void_p(zg.data_ptr() + 4 * off) if with_z else None
    o1 = pre1.cuda() if "1" in outs else None
    o2 = pre2.cuda() if "2" in outs else None
    cabi.check(lib.aero_colsum(x_ptr, z_ptr, ptr(o1), ptr(o2), int(dbl), N, n_inner, inner_s, n_outer, outer_s, n_seg, seg_sx,
                               so if n_seg > 1 else 0, stream()), lib)
    cols = torch.arange(n_seg)[:, None] * so + torch.arange(N)[None, :]
    worst = 0.0
    for o, pre, ref, mag in ((o1, pre1, ref1, mag1), (o2, pre2, ref2 if with_z else None, mag2 if with_z else None)):
        if o is None:
            continue
        got = o.cpu().double()
        want = pre.double().clone()
        want[cols] += ref
        bar = 1e-5 * (mag + pre.double()[cols].abs())
        err = (got[cols] - want[cols]).abs()
        worst = max(worst, float((err / bar).max()))
        assert bool((err <= bar).all()), (float((err / bar).max()), int((err > bar).sum()))
    print(f"{name}: rows {rows} step {step} ({'colsum4' if vec else 'scalar'}), worst column error {worst:.2e} of the bar")


# ------------------------------------------------------------------------------------------------ 4. element-wise kernels
@pytest.mark.parametrize("n", [1, 3, 4, 5, 4 * 1000 + 3, 3 * (1 << 22) + 1])
@pytest.mark.parametrize("alpha", [1.0, -0.37])
def test_add(lib, n, alpha):
    """aero_add: float4 body + scalar tail; the 8 elements past n are guards that must not change."""
    dst = rnd(n + 8, seed=12)
    src = rnd(n + 8, seed=13)
    dg, sg = dst.cuda(), src.cuda()
    cabi.check(lib.aero_add(ptr(dg), ptr(sg), n, alpha, stream()), lib)
    got = dg.cpu()
    assert torch.equal(got[n:], dst[n:])
    a = torch.tensor(alpha, dtype=torch.float32).double()
    want = a * src[:n].double() + dst[:n].double()                    # the fma, exact in fp64 up to the final rounding
    if alpha == 1.0:
        assert torch.equal(got[:n], dst[:n] + src[:n])
    assert bool(((got[:n].double() - want).abs() <= 2.0 ** -24 * want.abs() * 1.0000001).all())


@pytest.mark.parametrize("n", [1, 5, 3 * (1 << 20) + 7])
def test_add_f64(lib, n):
    dst, src = rnd(n + 4, seed=14), rnd(n + 4, seed=15).double() * 1e-3
    dg, sg = dst.cuda(), src.cuda()
    cabi.check(lib.aero_add_f64(ptr(dg), ptr(sg), n, stream()), lib)
    got = dg.cpu()
    assert torch.equal(got[:n], dst[:n] + src[:n].float()) and torch.equal(got[n:], dst[n:])


@pytest.mark.parametrize("B,Fq,T,Cc", [(2, 3, 5, 4), (16, 128, 501, 48), (3, 7, 11, 12)])
def test_bcast_add(lib, B, Fq, T, Cc):
    x, a = rnd(B, Fq, T, Cc, seed=16), rnd(Fq, Cc, seed=17)
    xg, ag = x.cuda(), a.cuda()
    cabi.check(lib.aero_bcast_add(ptr(xg), ptr(ag), B, Fq, T, Cc, stream()), lib)
    assert torch.equal(xg.cpu(), x + a.view(1, Fq, 1, Cc))


@pytest.mark.parametrize("B,per_sample,s_stride", [(3, 1, 1), (5, 4099, 2), (2, 4096 * 2048 + 1001, 3)])
def test_scale_rows(lib, B, per_sample, s_stride):
    x, s = rnd(B, per_sample, seed=18), rnd(B * s_stride, seed=19)
    xg, sg = x.cuda(), s.cuda()
    y = torch.full((B, per_sample), float("nan"), device="cuda")
    cabi.check(lib.aero_scale_rows(ptr(xg), ptr(y), ptr(sg), B, per_sample, s_stride, stream()), lib)
    assert torch.equal(y.cpu(), x * s[::s_stride].view(B, 1))


@pytest.mark.parametrize("gated", [False, True], ids=["plain", "gated"])
def test_gram_production(lib, gated):
    """aero_gram at the FTB frequency mix's production size (B = 8, F = 256 rows, M = T x C = 501 x 48), chunked with atomics."""
    B, Fq, M = 8, 256, 501 * 48
    Pm, Qm = rnd(B, Fq, M, seed=20), rnd(B, Fq, M, seed=21)
    g = rnd(B, M, seed=22) if gated else None
    pre = rnd(Fq, Fq, seed=23)
    out, Pg, Qg, gg = pre.cuda(), Pm.cuda(), Qm.cuda(), None if g is None else g.cuda()
    cabi.check(lib.aero_gram(ptr(Pg), ptr(Qg), ptr(gg), ptr(out), B, Fq, M, Fq * M, Fq * M, M, stream()), lib)
    got = out.cpu().double()
    # the kernel multiplies P by the gate in fp32 before the product
    P64 = (Pm * g.view(B, 1, M)).double() if gated else Pm.double()
    Q64 = Qm.double()
    want = pre.double() + torch.einsum("bim,bjm->ij", P64, Q64)
    mag = pre.double().abs() + torch.einsum("bim,bjm->ij", P64.abs(), Q64.abs())
    r = float(((got - want).abs() / mag).max())
    print(f"gram (gated={gated}): worst |err| / sum|P Q| {r:.2e}")
    assert r < 1e-5, r


# ------------------------------------------------------------------------------------------------ 5. FusedAdam
def test_fused_adam_matches_torch_adam_over_many_steps():
    """12 steps against torch.optim.Adam (fp64, CPU, same gradients): a parameter spanning three 65536-element chunks, two groups
    with different lr / betas / eps, an lr change at step 6, grad_scale != 1, a parameter whose .grad is None for the first 3
    steps, and at step 8 load_state_dict of a torch.save / torch.load round-trip of the step-4 state, the .grad tensors kept."""
    from aero_b200.optim import FusedAdam
    shapes = [(2 * 65536 + 1234,), (7, 5), (33,), (3, 1000), (17,)]
    groups = [dict(idx=[0, 1, 2], lr=1e-3, betas=(0.9, 0.999), eps=1e-8),
              dict(idx=[3, 4], lr=3e-3, betas=(0.8, 0.99), eps=1e-3)]        # eps ~ |g|: grad_scale is visible
    late, steps, scale = 2, 12, 0.37
    p0 = [1e-3 * rnd(*s, seed=30 + i) for i, s in enumerate(shapes)]
    ours = [t.cuda().requires_grad_(True) for t in p0]
    ref = [t.double().requires_grad_(True) for t in p0]
    opt = FusedAdam([dict(params=[ours[i] for i in g["idx"]], lr=g["lr"], betas=g["betas"], eps=g["eps"]) for g in groups])
    ropt = torch.optim.Adam([dict(params=[ref[i] for i in g["idx"]], lr=g["lr"], betas=g["betas"], eps=g["eps"]) for g in groups],
                            foreach=False)
    gi_of = {i: k for k, g in enumerate(groups) for i in g["idx"]}
    cum_lr = [0.0] * len(shapes)
    held, ckpt = [], None
    for k in range(steps):
        if k == 6:
            for o in (opt, ropt):
                o.param_groups[0]["lr"] = 5e-4
        if k == 4:
            buf = io.BytesIO()
            torch.save(opt.state_dict(), buf)
            ckpt = (buf.getvalue(), copy.deepcopy(ropt.state_dict()))
        if k == 8:
            # keep the moments the optimiser held so far alive: a chunk table that still points at them reads live memory
            held = [t for st in opt.state.values() for t in (st["exp_avg"], st["exp_avg_sq"])]
            opt.load_state_dict(torch.load(io.BytesIO(ckpt[0]), weights_only=True))
            ropt.load_state_dict(ckpt[1])
        for i, s in enumerate(shapes):
            if i == late and k < 3:
                ours[i].grad, ref[i].grad = None, None
                continue
            g = rnd(*s, seed=100 + 10 * k + i) * (1e-3 if gi_of[i] == 1 else 1.0)
            if ours[i].grad is None:
                ours[i].grad = torch.empty_like(ours[i])
            ours[i].grad.copy_(g)                                              # the same .grad storage every step
            ref[i].grad = (g * torch.tensor(scale, dtype=torch.float32)).double()
            cum_lr[i] += opt.param_groups[gi_of[i]]["lr"]
        opt.step(grad_scale=scale)
        ropt.step()
        torch.cuda.synchronize()
        for i in range(len(shapes)):
            d_ours = (ours[i].detach().cpu().double() - p0[i].double())
            d_ref = (ref[i].detach() - p0[i].double())
            bar = 1e-5 * max(cum_lr[i], 1e-30)
            err = float((d_ours - d_ref).abs().max())
            assert err <= bar, (f"step {k + 1}, parameter {i} ({'grad None until step 4' if i == late else shapes[i]}): "
                                f"max |dp - dp_ref| = {err:.3e} > {bar:.3e}")
    for po, pr in zip(ours, ref):
        so, sr = opt.state[po], ropt.state[pr]
        assert int(so["step"]) == int(sr["step"])
        # beta2 reaches the kernel as an fp32 argument: 1 - beta2 carries a relative error up to 2^-24 / (1 - beta2), 6e-5 at 0.999
        for key, tol in (("exp_avg", 1e-5), ("exp_avg_sq", 1e-4)):
            a, b = so[key].cpu().double(), sr[key]
            assert float((a - b).abs().max()) <= tol * float(b.abs().max()), key
    del held
