"""CPU: the fp32 oracle (oracle/gradloss_oracle.py) against the unmodified reference MSGradientLoss (losses.py:11-37,
on the script-compiled pyrdown of utils/generic_utils.py:87-94) and ScaleInvariantLoss (losses.py:39-54, a
ScriptModule), run with the restated kornia filters (``gradloss_oracle.load_reference_losses``): the loss, its
gradient to the prediction and the per-level mask counts, bit for bit (same ops in the same order).  Inputs:
ray-cast room depth with NaN holes, isolated NaNs and a zero-depth patch (one case whose holes cover the whole last
level, so that the reference's loss is NaN and its gradient is not), odd sizes down to 3x3 and a shape whose last
level is one pixel, B = 1 and 3.  The inputs and the reference's outputs are stored in
tests/golden/reference/gradloss_oracle_vs_reference.npz (tests/golden/make_gradloss_reference_golden.py)."""
import pytest
import torch

from oracle import gradloss_oracle as O
from oracle.ref_import import reference_available
from simplerecon_b200.synthetic import make_normals_batch
from tests import refgolden

MODULE = "gradloss_oracle_vs_reference"
# name: (seed, B, H, W, num_scales, holes)
CASES = {
    "room_b2_48x64": (5, 2, 48, 64, 4, True),
    "holes_fill_the_last_level_b3_24x32": (0, 3, 24, 32, 4, True),      # the reference's loss is NaN here
    "odd_b1_17x23_s3": (1, 1, 17, 23, 3, True),
    "wide_b1_9x31_s3": (4, 1, 9, 31, 3, True),
    "small_b3_5x4": (3, 3, 5, 4, 4, False),
    "tiny_b1_3x3_s2": (2, 1, 3, 3, 2, False),
}


def make_inputs(case):
    seed, B, H, W, num_scales, holes = CASES[case]
    t = make_normals_batch(seed, B, H, W, holes=holes)
    return t["depth_gt_b1hw"], t["depth_pred_b1hw"], num_scales


def _step(grad_loss_fn, si_loss_fn, gt, pred):
    """both losses as the training step feeds them (depth_model.py:466, :468) and their gradients"""
    p = pred.clone().requires_grad_(True)
    loss = grad_loss_fn(gt, p)
    loss.backward()
    mask = torch.isfinite(gt) & (gt > 0)
    lg = torch.log(gt[mask]).requires_grad_(True)
    lp = torch.log(pred[mask]).requires_grad_(True)
    si = si_loss_fn(lg, lp)
    si.backward()
    return dict(loss=loss.detach(), grad_depth_pred=p.grad, si_loss=si.detach(), si_grad_gt=lg.grad,
                si_grad_pred=lp.grad)


def reference_outputs() -> dict:
    """runs the unmodified reference classes (needs $SIMPLERECON_REF)"""
    ref = O.load_reference_losses()
    out = {}
    for case in CASES:
        gt, pred, num_scales = make_inputs(case)
        counts = torch.tensor([int(m.sum()) for m in O.level_masks(gt, num_scales)])
        out[case] = dict(depth_gt=gt, depth_pred=pred, num_scales=num_scales, mask_counts=counts,
                         **_step(ref.MSGradientLoss(num_scales), ref.ScaleInvariantLoss(), gt, pred))
    return out


def _oracle(gt, pred, num_scales):
    return _step(lambda a, b: O.ms_gradient_loss(a, b, num_scales), O.scale_invariant_loss, gt, pred)


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_stored_reference(case):
    ref = refgolden.load(MODULE, case)
    gt, pred, num_scales = make_inputs(case)
    assert torch.equal(gt.nan_to_num(-1.0), ref["depth_gt"].nan_to_num(-1.0)) and torch.equal(pred, ref["depth_pred"])
    assert int(ref["num_scales"]) == num_scales
    ours = _oracle(gt, pred, num_scales)
    for name in ("loss", "grad_depth_pred", "si_loss", "si_grad_gt", "si_grad_pred"):
        assert torch.equal(ours[name].nan_to_num(7.0), ref[name].nan_to_num(7.0)), name
    counts = [int(m.sum()) for m in O.level_masks(gt, num_scales)]
    assert counts == ref["mask_counts"].tolist()
    assert bool(torch.isnan(ref["loss"])) == (min(counts) == 0)        # mean over an empty level
    assert torch.isfinite(ref["grad_depth_pred"]).all() and torch.isfinite(ref["si_loss"])
    if CASES[case][5]:
        assert counts[0] < 2 * gt.numel()                              # the holes reach the mask


@pytest.mark.skipif(not reference_available(), reason="needs $SIMPLERECON_REF (the reference tree)")
def test_stored_outputs_are_the_live_reference():
    live = reference_outputs()
    for case, arrays in live.items():
        stored = refgolden.load(MODULE, case)
        for name, v in arrays.items():
            v = torch.as_tensor(v)
            assert torch.equal(v.nan_to_num(7.0), torch.as_tensor(stored[name]).nan_to_num(7.0)), (case, name)
