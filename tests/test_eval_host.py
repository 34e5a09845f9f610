"""Host logic of test-set scoring (aero_b200.enhance.evaluate_batch, aero_b200.metrics.get_lsd_batch), CPU-only: the
reference's match_signal, the row and frame tables of aero_lsd_varlen_fwd, the non-zero counting rule of reference
evaluate.py and the count-weighted average over two gloo ranks of reference distrib.average."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from aero_b200.enhance import match_signal, nonzero_mean
from aero_b200.metrics import get_lsd_batch, lsd_tables, lsd_varlen

HERE = os.path.dirname(os.path.abspath(__file__))


def _reference_match_signal(signal, ref_len):
    # reference src/utils.py:211-217
    sig_len = signal.shape[-1]
    if sig_len < ref_len:
        signal = torch.nn.functional.pad(signal, (0, ref_len - sig_len))
    elif sig_len > ref_len:
        signal = signal[..., :ref_len]
    return signal


@pytest.mark.parametrize("shape", [(7,), (1, 9), (2, 12), (3, 1, 10)])
@pytest.mark.parametrize("ref_len", [1, 5, 9, 10, 16])
def test_match_signal_is_the_reference_one(shape, ref_len):
    x = torch.randn(shape, generator=torch.Generator().manual_seed(3))
    got, want = match_signal(x, ref_len), _reference_match_signal(x, ref_len)
    assert got.shape == want.shape == (*shape[:-1], ref_len)
    assert torch.equal(got, want)


def test_lsd_tables():
    lengths, row_file = [1025, 1536, 2049, 128000, 3000, 3000], [0, 1, 2, 3, 4, 4]
    tab, max_frames = lsd_tables(lengths, row_file)
    frames = [3, 4, 5, 251, 6, 6]                               # 1 + L // 512
    assert tab.dtype == np.int32 and max_frames == 251
    assert tab.tolist() == lengths + row_file + [0, *np.cumsum(frames).tolist()]


def test_nonzero_counting_rule():
    assert nonzero_mean([0.0, 1.0, 3.0, 0.0]) == (2.0, 2)
    assert nonzero_mean([0.5]) == (0.5, 1)
    assert nonzero_mean([0.0, 0.0]) == (0.0, 0)
    assert nonzero_mean([]) == (0.0, 0)
    assert nonzero_mean(torch.tensor([0.0, 2.0, 4.0]).tolist()) == (3.0, 2)


def test_cpu_tensors_are_refused():
    x = torch.randn(1, 2000)
    with pytest.raises(RuntimeError, match="CUDA"):
        get_lsd_batch([x], [x])
    with pytest.raises(RuntimeError, match="CUDA"):
        lsd_varlen(x, x, [2000], [0], 1)


def _worker(rank, world, port, q):
    sys.path.insert(0, os.path.dirname(HERE))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from aero_b200.parallel import average_over_ranks
    got = (average_over_ranks(*[(1.0, 3), (5.0, 1)][rank]),          # (1*3 + 5*1) / 4
           average_over_ranks(*[(2.0, 2), (0.0, 0)][rank]),          # a rank without a non-zero file adds nothing
           average_over_ranks(0.0, 0))                                # no rank has one
    q.put((rank, got))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_gloo_average_is_weighted_by_count():
    from aero_b200.parallel import average_over_ranks
    assert average_over_ranks(1.25, 7) == 1.25                        # single process: the value itself
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() + 977) % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=240) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank in (0, 1):
        assert res[rank] == (pytest.approx(2.0), pytest.approx(2.0), 0.0)
