"""Ragged SEANet batches on the host (no GPU): the per-clip length tables of SeanetEngine.forward_varlen against the model's own
geometry, and the order in which enhance_batch refuses a SEANet call before it builds an engine or loads the library."""
import pytest
import torch

from util import white_noise
from seanet_util import CASES

from aero_b200 import Seanet
from aero_b200.enhance import enhance_batch
from aero_b200.seanet import seanet_ragged_tables

CONFIGS = {"shipped": CASES["s1"][0], "s3": CASES["s3"][0], "s5": CASES["s5"][0], "s6": CASES["s6"][0]}


def shortest_admissible(m):
    for n in range(2, 1 << 16):
        try:
            m.check_length(n)
            return n
        except ValueError:
            pass
    raise AssertionError("no admissible length")


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_tables_follow_the_model_geometry(name):
    """hr_length, level_lengths (estimate_output_length of the high-rate length, then // ratio per level) and the output length
    min(target, valid) for every length from the shortest admissible one up to a few thousand samples."""
    m = Seanet(**CONFIGS[name])
    lo = shortest_admissible(m)
    lengths = list(range(lo, lo + 3000))
    hr, frames, out_lens = seanet_ragged_tables(m, lengths)
    assert frames.shape == (len(m.ratios) + 1, len(lengths))
    for b, n in enumerate(lengths):
        lev = m.level_lengths(n)
        assert int(hr[b]) == m.hr_length(n)
        assert [int(t) for t in frames[:, b]] == lev
        assert lev[0] == m.estimate_output_length(m.hr_length(n))
        target = n * m.scale_factor if m.upsample else n
        assert int(out_lens[b]) == min(target, lev[0])
    # buffers are sized by the longest clip: every level is monotone in the length
    assert (frames[:, 1:] >= frames[:, :-1]).all()


def test_tables_below_the_admissible_range():
    """The builder itself takes any length (admissibility is check_length's business), down to one sample."""
    m = Seanet(**CONFIGS["shipped"])
    lengths = list(range(1, 400))
    hr, frames, _ = seanet_ragged_tables(m, lengths)
    assert [int(v) for v in hr] == [m.hr_length(n) for n in lengths]
    assert [[int(t) for t in frames[:, b]] for b in range(len(lengths))] == [m.level_lengths(n) for n in lengths]


def test_errors_come_in_order_before_any_engine():
    """Training mode first (whatever else is wrong), then the arguments, then each clip's shape and length, named by its index.
    All of it on CPU tensors and a CPU model: no engine is built and the library is not loaded."""
    m = Seanet(**CONFIGS["shipped"])
    short = shortest_admissible(m) - 1
    good = white_noise((1, 3000))
    with pytest.raises(NotImplementedError):
        enhance_batch(m, [good, white_noise((2, 3000)), white_noise((1, short))], return_spec=True)
    m.eval()
    with pytest.raises(ValueError, match="return_spec"):
        enhance_batch(m, [good], return_spec=True)
    with pytest.raises(ValueError, match="return_spec"):
        enhance_batch(m, [good], return_lr_spec=True)
    with pytest.raises(ValueError, match="max_batch"):
        enhance_batch(m, [good], max_batch=0)
    with pytest.raises(ValueError, match="signal 1"):
        enhance_batch(m, [good, white_noise((2, 3000)), white_noise((1, short))])
    with pytest.raises(ValueError, match="signal 2: .*too short"):
        enhance_batch(m, [good, good, white_noise((1, short))])
    with pytest.raises(ValueError, match="signal 0"):
        enhance_batch(m, [white_noise((3000,))])
    assert enhance_batch(m, []) == []
    assert m._engine_obj is None


def test_stereo_channel_count():
    m = Seanet(**CONFIGS["s5"]).eval()
    with pytest.raises(ValueError, match=r"signal 0: expected \[2, L\]"):
        enhance_batch(m, [white_noise((1, 5000))])
    assert m._engine_obj is None
