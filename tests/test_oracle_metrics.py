"""CPU: the float64 metrics restatement (tests/metrics_oracle.py) against vectors produced by the REAL reference
functions (tests/golden/metrics_vectors.npz, from utils/loss_utils.py l1_loss / ssim and utils/image_utils.py psnr), in
both of the reference's forms: training_report's (the clamped float render) and metrics.py's (the PNG bytes)."""
import os

import numpy as np
import pytest

from tests import metrics_oracle as om

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "metrics_vectors.npz"))
CASES = ["a", "b", "c", "same"]


def _close(got, ref, tol_unit, tol_db):
    for i, t in enumerate((tol_unit, tol_db, tol_db, tol_unit)):
        if np.isinf(ref[i]):
            assert got[i] == ref[i], (i, got[i], ref[i])
        else:
            assert abs(got[i] - ref[i]) <= t, (i, got[i], ref[i])


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("form", ["train", "metrics"])
def test_oracle_reproduces_the_reference_in_float64(case, form):
    render = GOLD[f"{case}_render"] if form == "train" else GOLD[f"{case}_display_u8"]
    if case == "same":   # the float32 render gt/255 equals y only in float32; in float64 the pair is y against y
        render = GOLD["same_gt_u8"].transpose(1, 2, 0)
    got = om.metrics(render, GOLD[f"{case}_gt_u8"])
    _close(got, GOLD[f"{case}_{form}_f64"], 1e-9, 1e-8)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("form", ["train", "metrics"])
def test_reference_float32_noise_floor(case, form):
    """How far the reference's own float32 evaluation sits from its float64 one -- below the bounds the GPU tests
    hold the kernel to (1e-6 on l1 / ssim, 1e-4 dB on the PSNRs)."""
    _close(GOLD[f"{case}_{form}_f32"], GOLD[f"{case}_{form}_f64"], 1e-6, 1e-4)


def test_fixture_covers_the_clamp_the_quantisation_and_ragged_sizes():
    for case in ("a", "b", "c"):
        r = GOLD[f"{case}_render"]
        assert (r < 0).any(), "the clamp of train.py:277 must matter"
        assert case == "c" or (r > 1).any()
        H, W = r.shape[1:]
        assert W % 4 != 0 and GOLD[f"{case}_display_u8"].shape == (H, W, 3)
        assert not np.array_equal(GOLD[f"{case}_train_f64"], GOLD[f"{case}_metrics_f64"])
    assert np.isinf(GOLD["same_train_f64"][1:3]).all() and GOLD["same_train_f64"][3] == 1.0


def test_quantisation_round_trips_every_code():
    """render.py's mul(255).add_(0.5).clamp_(0, 255) of k/255 gives k back (float32): the bytes / 255 of a uint8
    ground truth are exactly what both forms compare against."""
    import torch
    k = torch.arange(256, dtype=torch.uint8)
    assert torch.equal((k.float() / 255).mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8), k)
