"""k_bidir.cu's PAIR kernels save label scores only, plus the meeting row's blank scores behind the label rows of
the block that holds it.  These cases pin the placements test_bidir_emulation.py does not reach: T <= 8, where
CTA A has no first phase and the meeting row sits in CTA B's single, partial block; a full single block; and PAIR
loss-only calls, whose one phase-2 level reads the meeting row and nothing else."""
import pytest

from tests import util
from tests.test_bidir_emulation import check_one, emu, run  # noqa: F401  (emu: the module's fixture)


@pytest.mark.parametrize("shape", [
    (2, 7, 64, 2),    # T < 8: A has no first phase; the meeting row is row 0 of B's partial block (7 label rows)
    (2, 1, 64, 0),    # T = 1: one level, the meeting row behind a single label row
    (1, 8, 64, 3),    # T = 8: one full block, all of it B's first phase
    (1, 5, 128, 2),   # C = 128 (the NQ = 2 PAIR kernel), T < 8
])
def test_pair_meeting_row_in_b_only_block(emu, oracle, shape):
    from oracle import f64
    B, T, Cn, U = shape
    e, targets = util.bench_inputs(B, T, Cn, U, seed=131 + T)
    check_one(emu, oracle, f64, e, targets, B, T, 1)


@pytest.mark.parametrize("T", [5, 40, 61])
def test_pair_loss_only(emu, oracle, T):
    """PAIR without a gradient: Z from the meeting row (labels and blanks of both CTAs) alone."""
    B, Cn, U = 2, 64, 6
    e, targets = util.bench_inputs(B, T, Cn, U, seed=17 + T)
    loss, grad, status = run(emu, e, targets, want_grad=False, zero_w=1)
    assert grad is None and not status.any()
    for b in range(B):
        lo, _ = oracle.ctc_loss(e[b], targets[b], 0, False)
        assert util.close(loss[b], lo), (b, loss[b], lo)
