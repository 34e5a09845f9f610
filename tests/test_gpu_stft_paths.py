"""-m gpu: every kernel the STFT / iSTFT dispatchers can pick, through both entry points.  A ragged batch whose clips all have
the full length is a fixed-length batch, so the ragged-batch kernels must give the fixed-length result bit for bit, on the
n_fft = 512 kernels and on the generic ones.  With ragged lengths the generic kernels are held to the CPU statement of the
contract (tests/test_ragged_host.RaggedEmuEngine)."""
import pytest
import torch

from test_ragged_host import make
from util import rel_l2

from aero_b200 import spec

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n_fft,hop,win", [
    (512, 64, 512),      # n_fft = 512 kernels for both transforms
    (512, 16, 512),      # n_fft = 512 STFT; the iSTFT falls back to the generic kernel (fewer than 8 output hops per CTA)
    (256, 64, 200),      # generic kernels, window shorter than n_fft
    (1024, 128, 600),
])
def test_full_length_ragged_batch_equals_fixed_length(n_fft, hop, win):
    torch.manual_seed(0)
    B, Cc, T = 3, 2, 45
    L, bins = hop * (T - 1), n_fft // 2
    x = torch.randn(B * Cc, L, device="cuda")
    kw = dict(n_fft=n_fft, hop=hop, win=win, channels=Cc, strides=(bins * T * 2 * Cc, 2, T * 2 * Cc, 2 * Cc),
              stream=spec.current_stream())
    per_clip = lambda v: torch.full((B,), v, dtype=torch.int32, device="cuda")
    z = [torch.full((B, bins, T, 2 * Cc), 7.0, device="cuda") for _ in range(2)]
    st = [torch.zeros(B, 2, dtype=torch.float64, device="cuda") for _ in range(2)]
    spec.stft_into(x, z[0], st[0], bins_out=bins, **kw)
    spec.stft_into(x, z[1], st[1], bins_out=bins, lengths=per_clip(L), **kw)
    assert torch.equal(z[1], z[0])
    # each thread sums its moments in fp32, and the generic kernel's two instantiations compile that loop differently: the
    # moments agree to rounding (about 2e-9 relative), not bit for bit
    assert rel_l2(st[1], st[0]) < 1e-6
    y = [torch.full((B * Cc, L), 7.0, device="cuda") for _ in range(2)]
    spec.istft_into(z[0], y[0], frames=T, bins_in=bins, **kw)
    spec.istft_into(z[0], y[1], frames=T, bins_in=bins, clip_frames=per_clip(T), out_lens=per_clip(L), **kw)
    assert torch.equal(y[1], y[0])


def test_generic_ragged_kernels_match_the_contract():
    """n_fft 1024 (no n_fft = 512 kernel) on clips of different lengths, at the tolerances of test_gpu_ragged's contract test."""
    torch.manual_seed(1)
    emu = make("aero_4-16_512_64")._engine_obj
    n_fft, hop, win = 1024, 128, 1024
    lengths = [3001, 128 * 40, 2565]
    frames = [1 + (n + (-n) % hop) // hop for n in lengths]
    T = max(frames)
    Lp = hop * (T - 1)
    x = torch.randn(3, Lp)
    bins = n_fft // 2
    kw = dict(n_fft=n_fft, hop=hop, win=win, channels=1, strides=(bins * T * 2, 0, T * 2, 2))
    za, zb = torch.full((3, bins, T, 2), 7.0), torch.full((3, bins, T, 2), 7.0, device="cuda")
    sa, sb = torch.zeros(3, 2, dtype=torch.float64), torch.zeros(3, 2, dtype=torch.float64, device="cuda")
    emu.stft_varlen_into(x, torch.tensor(lengths), za, sa, bins_out=bins, **kw)
    spec.stft_into(x.cuda(), zb, sb, bins_out=bins, lengths=torch.tensor(lengths, dtype=torch.int32, device="cuda"),
                   stream=spec.current_stream(), **kw)
    assert rel_l2(zb.cpu(), za) < 1e-6 and rel_l2(sb.cpu(), sa) < 1e-6
    for b, tb in enumerate(frames):
        assert (zb[b, :, tb:] == 0).all()
    out_lens = [min(n, hop * (tb - 1)) for n, tb in zip(lengths, frames)]
    wa, wb = torch.empty(3, max(out_lens)), torch.full((3, max(out_lens)), 7.0, device="cuda")
    emu.istft_varlen_into(za, wa, torch.tensor(frames), torch.tensor(out_lens), frames_max=T, bins_in=bins, **kw)
    spec.istft_into(zb, wb, frames=T, bins_in=bins, clip_frames=torch.tensor(frames, dtype=torch.int32, device="cuda"),
                    out_lens=torch.tensor(out_lens, dtype=torch.int32, device="cuda"), stream=spec.current_stream(), **kw)
    assert rel_l2(wb.cpu(), wa) < 1e-5
