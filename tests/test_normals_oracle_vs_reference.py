"""CPU: the fp32 normals oracle (oracle/normals_oracle.py) against the unmodified reference NormalGenerator
(utils/geometry_utils.py:92-133, a ScriptModule) and NormalsLoss (losses.py:57-77), run with the restated kornia
filters plugged into its ``kornia.filters`` (``normals_oracle.load_reference_normals``): normals, loss, the loss's
gradients to both normals and the gradient to the predicted depth.  Inputs: ray-cast room depth with NaN holes, isolated NaNs and a zero-depth patch, odd
sizes down to 3x3, B = 1 and 3.  The inputs and the reference's outputs are stored in
tests/golden/reference/normals_oracle_vs_reference.npz (tests/golden/make_normals_reference_golden.py).

Normals and the loss are compared bit for bit (same ops in the same order); the depth gradient within 1e-6 of its
maximum, because autograd through the scripted graph may accumulate the blur's and Sobel's input gradients in
another order than through the eager one.  The all-finite masks are compared exactly."""
import pytest
import torch

from oracle import normals_oracle as O
from oracle.ref_import import reference_available
from simplerecon_b200.synthetic import make_normals_batch
from tests import refgolden

MODULE = "normals_oracle_vs_reference"
# name: (seed, B, H, W, k, sigma, holes)
CASES = {
    "room_b3_24x32": (0, 3, 24, 32, 5, 2.0, True),
    "odd_b1_17x23": (1, 1, 17, 23, 5, 2.0, True),
    "wide_b1_9x31_k7": (4, 1, 9, 31, 7, 3.0, True),
    "small_b3_5x4": (3, 3, 5, 4, 5, 2.0, False),
    "tiny_b1_3x3": (2, 1, 3, 3, 5, 2.0, False),
}


def make_inputs(case):
    seed, B, H, W, k, sigma, holes = CASES[case]
    t = make_normals_batch(seed, B, H, W, holes=holes)
    return t["depth_gt_b1hw"], t["depth_pred_b1hw"], t["invK_b44"], k, sigma


def _step(ng, loss_fn, gt, pred, invK):
    """normals of both depths, the loss, and its gradients to both normals and to the predicted depth"""
    p = pred.clone().requires_grad_(True)
    n_gt = ng(gt, invK).detach().requires_grad_(True)
    n_pred = ng(p, invK)
    n_pred.retain_grad()
    loss = loss_fn(n_gt, n_pred)
    loss.backward()
    return dict(normals_gt=n_gt.detach(), normals_pred=n_pred.detach(), loss=loss.detach(),
                grad_normals_gt=n_gt.grad, grad_normals_pred=n_pred.grad, grad_depth_pred=p.grad)


def reference_outputs() -> dict:
    """runs the unmodified reference modules (needs $SIMPLERECON_REF)"""
    ref = O.load_reference_normals()
    out = {}
    for case in CASES:
        gt, pred, invK, k, sigma = make_inputs(case)
        ng = ref.NormalGenerator(gt.shape[-2], gt.shape[-1], k, sigma)
        out[case] = dict(depth_gt=gt, depth_pred=pred, invK=invK, k=k, sigma=sigma,
                         **_step(ng, ref.NormalsLoss(), gt, pred, invK))
    return out


def _oracle(gt, pred, invK, k, sigma):
    class NG(torch.nn.Module):
        def forward(self, d, K):
            return O.normal_generator(d, K, k, sigma)

    class Loss(torch.nn.Module):
        def forward(self, a, b):
            return O.normals_loss(a, b)

    return _step(NG(), Loss(), gt, pred, invK)


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_stored_reference(case):
    ref = refgolden.load(MODULE, case)
    gt, pred, invK, k, sigma = make_inputs(case)
    assert torch.equal(gt.nan_to_num(-1.0), ref["depth_gt"].nan_to_num(-1.0)) and torch.equal(pred, ref["depth_pred"])
    assert torch.equal(invK, ref["invK"]) and int(ref["k"]) == k and float(ref["sigma"]) == sigma
    ours = _oracle(gt, pred, invK, k, sigma)
    for name in ("normals_gt", "normals_pred"):
        assert torch.equal(O.all_finite(ours[name]), O.all_finite(ref[name])), name
        assert torch.equal(ours[name].nan_to_num(7.0), ref[name].nan_to_num(7.0)), name
    assert torch.equal(ours["loss"].nan_to_num(7.0), ref["loss"].nan_to_num(7.0))
    for name in ("grad_normals_gt", "grad_normals_pred"):
        assert torch.equal(ours[name], ref[name]), name
    g, rg = ours["grad_depth_pred"], ref["grad_depth_pred"]
    assert torch.equal(torch.isfinite(g), torch.isfinite(rg))
    fin = torch.isfinite(rg)
    if fin.any():
        assert (g - rg)[fin].abs().max() <= 1e-6 * rg[fin].abs().max()
    if CASES[case][6]:
        assert (~O.all_finite(ref["normals_gt"])).any() and torch.isfinite(ref["loss"])


@pytest.mark.skipif(not reference_available(), reason="needs $SIMPLERECON_REF (the reference tree)")
def test_stored_outputs_are_the_live_reference():
    live = reference_outputs()
    for case, arrays in live.items():
        stored = refgolden.load(MODULE, case)
        for name, v in arrays.items():
            v = torch.as_tensor(v)
            assert torch.equal(v.nan_to_num(7.0), torch.as_tensor(stored[name]).nan_to_num(7.0)), (case, name)
