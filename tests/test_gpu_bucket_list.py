"""Count-based window calls above 2^26 positions against a direct fold: the bucket path in position ranges.

The wide partition leaves one 32-bit word per item for the bucket update, its position within a range of BKL_RANGE_POS = 2^26
positions and its key within the bucket (wfb_kernels.cuh, bkl_word). A call over more positions is partitioned, updated and queried
range after range, and the multi-GPU destination splits its receive buffer into ranges of receive positions the same way. These
cases put a range boundary inside one call: a few keys, so that every key's open pane and the window groups it fires straddle the
boundary, and batches whose sizes are not whole tiles, so that the last range is partial.

Every window is checked as in tests/test_gpu_ordered_windows.py: the window set, ids and result timestamps against the oracle, and
the order-sensitive hash of tests/cpp/ordered_programs.cu (ordered_program_32p.cu for the step) bit for bit against a direct fold of
every key's surviving items in arrival order. The step also matches the single-GPU operator over the same 80 million tuples byte for
byte. Each case moves a few GB of tuples: host memory for the references, HBM for the call."""
import pytest

import test_gpu_mg_step as mgs
import test_gpu_ordered_windows as ow
from test_gpu_mg_step import prog32p  # noqa: F401  (fixture)
from test_gpu_ordered_windows import progs  # noqa: F401  (fixture)

RANGE_POS = 1 << 26
# 2^26 + 33 545 tuples in batches of 5 000 000 (not whole tiles): the last range is a partial one
N_DIRECT = RANGE_POS + (1 << 15) + 777


def _case(pipelined):
    return ow.Case("above_2p26" + ("_pipelined" if pipelined else ""), 24, 1000, 100, 2, 64, 3, [N_DIRECT], 5_000_000, (),
                   pipelined=pipelined, census=False, seed=21 + int(pipelined))


@pytest.mark.gpu
@pytest.mark.parametrize("pipelined", [False, True], ids=["direct", "pipelined"])
def test_call_above_2p26_positions_matches_direct_fold(wfb, oracle, progs, pipelined):  # noqa: F811
    case = _case(pipelined)
    t, calls = case.stream()
    assert sum(len(tb) for tb, _ in calls[0]) > RANGE_POS
    e, et, h, q, _ = ow._expected(oracle, case, t, calls)
    got, gts, err = ow._run_cb(wfb, wfb._lib.lib(), progs[24], case, calls)
    assert err == 0
    ow._check(got, gts, e, et, h, q, 24)


@pytest.mark.gpu
def test_mg_step_above_2p26_records_matches_direct_fold(wfb, oracle, prog32p):  # noqa: F811
    """A step at one rank of 80 000 000 tuples, 68.6 million of them kept: the destination's receive buffer holds more than 2^26
    records of its single source, so a range boundary falls inside that source's region. A small step before it fires windows of
    every key, so the large step continues open panes and rings."""
    c = mgs.MgCase("above_2p26", 64, 1000, 100, 2, 5, [mgs.S(20_000), mgs.S(41_000_000, 39_000_000), mgs.FLUSH], (), shift=0, seed=23)
    dropped = (80_020_000 - 1 - 3) // 7 - (20_000 - 1 - 3) // 7  # ids in [20 000, 80 020 000) = 3 mod 7: ow.keep_mask drops them
    assert 80_000_000 - dropped > RANGE_POS
    assert mgs.run_case(wfb, oracle, prog32p, c) > 0

