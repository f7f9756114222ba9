"""CPU: the float64 LPIPS restatement (tests/lpips_oracle.py) against the real lpipsPyTorch (tests/golden/
lpips_vectors.npz, made by make_golden_lpips.py from seeded weights), for both networks: each network's smallest image,
odd sizes that exercise the stride-4 and pool floors, a layer whose features are exactly zero, an identical pair."""
import os

import numpy as np
import pytest
import torch

from tests import lpips_oracle as ol

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "lpips_vectors.npz"))


@pytest.mark.parametrize("case", sorted(ol.CASES))
def test_oracle_reproduces_the_reference_in_float64(case):
    net, H, W, _, dead, same = ol.CASES[case]
    feats, lin = ol.seeded_weights(net, ol.SEED[net], dead_conv=dead)
    renders, gts = GOLD[f"{case}_render"], GOLD[f"{case}_gt_u8"]
    assert renders.shape == (2, 3, H, W) and gts.shape == (2, 3, H, W)
    for i in range(2):
        if same:   # the identical pair: the ground truth against itself
            x = torch.from_numpy(gts[i]).double()[None] / 255
            got = float(ol.lpips(x, x, net, feats, lin)[0])
        else:
            got = ol.lpips64(renders[i], gts[i], net, feats, lin)
        ref = GOLD[f"{case}_per_image"][i]
        assert abs(got - ref) <= 1e-12 * abs(ref), (case, i, got, ref)
        if same:
            assert got == 0.0 and ref == 0.0


@pytest.mark.parametrize("case", sorted(ol.CASES))
def test_a_batch_call_returns_the_sum_over_its_images(case):
    per, batch = GOLD[f"{case}_per_image"], float(GOLD[f"{case}_batch_sum"])
    assert abs(batch - per.sum()) <= 1e-14 + 1e-12 * abs(batch)


def test_fixture_covers_the_edges():
    assert ol.CASES["alex_min"][1:3] == (31, 31) and ol.CASES["vgg_min"][1:3] == (16, 16)
    assert (GOLD["alex_odd_render"] < 0).any() and (GOLD["alex_odd_render"] > 1).any()   # the clamp matters
    for case in ("alex_dead", "vgg_dead"):   # the dead layer's features are exactly zero at every pixel
        net, H, W, _, dead, _ = ol.CASES[case]
        feats, lin = ol.seeded_weights(net, ol.SEED[net], dead_conv=dead)
        x, _ = ol.inputs(GOLD[f"{case}_render"][0], GOLD[f"{case}_gt_u8"][0])
        f = ol.features(x[None], net, feats)
        assert torch.count_nonzero(f[-1]) == 0 and all(torch.count_nonzero(t) > 0 for t in f[:-1])
        assert GOLD[f"{case}_per_image"].min() > 0


def test_smallest_images_follow_from_the_layer_arithmetic():
    """31 x 31 is AlexNet's smallest input and 16 x 16 VGG-16's: one pixel less and a stage has no output."""
    for net, side in (("alex", 31), ("vgg", 16)):
        feats, lin = ol.seeded_weights(net, 0)
        x = torch.rand(1, 3, side, side, dtype=torch.float64)
        assert torch.isfinite(ol.lpips(x, x.flip(-1), net, feats, lin)).all()
        with pytest.raises(RuntimeError):
            ol.lpips(x[..., :-1, :], x[..., :-1, :], net, feats, lin)
