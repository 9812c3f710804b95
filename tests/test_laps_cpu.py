"""Host-only checks of tests/laps_ref.py: the grid rules it copies still read as copied, and every batch size of
tests/test_laps_gpu.py runs its kernel's loop a second time on an H100 PCIe (114 SMs) and an H100 SXM (132 SMs)."""
import os

import pytest

import laps_ref as LR


def test_copied_grid_rules_match_their_source_lines():
    for name, line, text in LR.SOURCE:
        with open(os.path.join(LR.CSRC, name)) as f:
            lines = f.read().splitlines()
        assert text in lines[line - 1], f"{name}:{line} is now {lines[line - 1].strip()!r}; laps_ref.py copied {text!r}"


def test_copied_rules_give_the_documented_grids():
    assert [LR.fused_grid(s, 10 ** 6) for s in (114, 132, 148, 400)] == [228, 264, 296, 592]
    assert LR.fused_grid(132, 7) == 7 and LR.l5_grid(132, 10 ** 6) == 264 and LR.l5_grid(400, 10 ** 6) == 800
    assert LR.blocks_for(10 ** 9, 256) == 4736 and LR.blocks_for(0, 64) == 1
    assert LR.grid_for(132, 10 ** 9, 256) == 1056 and LR.grid_for(132, 1, 256) == 1
    # the first batch with a second lap of every batched operator: B * items > 4736 * threads
    first = {op: LR.ops_min_batch(op) for op in LR.OPS}
    assert first == dict(fp_c1=351, bp_output_c1=351, bp_preact_c1=351, apply_step_function=351, bp_weight_c1=2021, fp_s1=2807,
                         bp_output_s1=2807, bp_preact_s1=2807, bp_weight_s1=18945, fp_preact_f=30311, bp_bias_c1=50518,
                         fp_bias_f=60621, makeError_batch=121242, bp_bias_s1=303105, vectorNorm=606209)
    for op, B in first.items():
        assert LR.ops_laps(op, B)[2] == 2 and LR.ops_laps(op, B - 1)[2] == 1, op


@pytest.mark.parametrize("sm_count", [114, 132])
def test_lap_cases_reach_their_regime(sm_count):
    for B, need in LR.eval_batches(sm_count):
        fewest, most = LR.images_per_cta(B, LR.fused_grid(sm_count, B))
        assert most >= need >= 2 and fewest >= 1, (B, fewest, most)
    assert [need for _, need in LR.eval_batches(sm_count)] == [2, 3, 3, 3]
    for B, need in LR.l5_batches(sm_count):
        fewest, most = LR.images_per_cta(B, LR.l5_grid(sm_count, B))
        assert most >= need >= 2 and fewest >= 1, (B, fewest, most)
        assert B <= LR.NB                                      # the gradient cases run the fixture's own digits
    assert LR.images_per_cta(8 * LR.NB, LR.l5_grid(sm_count, 8 * LR.NB))[1] >= 3
    for op in LR.OPS:
        B = LR.ops_batch(op)
        assert LR.ops_laps(op, B)[2] >= 2 and B >= LR.NB, op
    for planes, H, W, k in LR.MAXPOOL_CASES:
        (gf, lf), (gb, lb) = LR.maxpool_laps(sm_count, planes, H, W, k)
        assert lf >= 2 and lb >= 2, (planes, k, lf, lb)
    for B, n in LR.SOFTMAX_CASES:
        assert LR.softmax_laps(sm_count, B)[2] >= 2, (B, n)
        assert B > LR.NB                                       # rows repeat, so tiled rows are compared with their base rows
