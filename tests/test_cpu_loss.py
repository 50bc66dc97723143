"""hold_b200.train.Loss against the REFERENCE's own hold/loss.py Loss module: tests/golden/loss/*.pt hold synthetic training
outputs and the loss dict the reference module returned for them (written by `python oracle/ref_harness.py golden_loss` with
$HOLD_REFERENCE naming a checkout of the reference).  Covers the schedules (w_sem, w_sparse at steps 0 / 12 000 / beyond the milestone), the eikonal lower bound
(the term is dropped below 8e-4), the clamped MANO canonical term and the segmentation-id remapping."""
import glob
import os

import pytest
import torch

GOLD = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "loss", "*.pt")))


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p)[:-3] for p in GOLD])
def test_loss_matches_reference_module(path):
    from hold_b200.train import Loss

    rec = torch.load(path)
    ours = Loss()(rec["batch"], rec["outputs"])
    ref = rec["loss"]
    assert set(ours) == set(ref), (sorted(ours), sorted(ref))
    for k, v in ref.items():
        a, b = float(ours[k]), float(v)
        assert abs(a - b) <= 1e-6 * max(1.0, abs(b)), f"{k}: {a} vs reference {b}"


def test_goldens_present():
    assert len(GOLD) == 3
