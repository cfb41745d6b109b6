"""GPU: CoEx at its evaluation size 540 x 960 (RightTopPad in cfgs/coex/coex_sceneflow_amp.yaml): the regression tail at the
evaluator's batch of 8 against the CPU oracle, and patch() on the reference class, whose last transposed conv returns 136 rows
for a 135-row skip level."""
import pytest
import torch

from oracle import coex as ocx

from test_coex_gpu import REG_BAR, EPE_BAR, distinct_logits, needs_ref, osb, patched_vs_reference, rnd  # noqa: F401  (osb: fixture)

pytestmark = pytest.mark.gpu


def test_regression_b8_540x960(osb):
    _, ops = osb
    cost = distinct_logits(70, 8, 48, 135, 240)
    raw = rnd(71, 8, 9, 540, 960) * 2
    want = ocx.regression(cost, torch.softmax(raw, 1), 2)
    got = ops.coex_regression(cost.cuda(), raw.cuda(), 2, spx_is_logits=True).cpu()
    assert (got - want).abs().max().item() <= REG_BAR


@needs_ref
def test_patch_coex_540x960(osb):
    lib, _ = osb
    epe, std, launches = patched_vs_reference(lib, 2, 540, 960, 72)
    assert launches >= 16 + 3 + 1 + 1 and std > 1 and epe <= EPE_BAR    # + the 136 -> 135 nearest resampling
