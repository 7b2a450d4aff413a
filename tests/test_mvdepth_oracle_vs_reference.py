"""CPU: the multi-view depth-loss oracle against the unmodified reference ``losses.MVDepthLoss``
(losses.py:79-208), value and gradient (stored under tests/golden/reference/, see tests/refgolden.py)."""
import importlib

import pytest
import torch

from oracle import mvdepth_oracle as M
from simplerecon_b200.synthetic import make_mvloss_batch
from tests import refgolden

CASES = [(0, 2, 3, (24, 32)), (1, 1, 7, (30, 40)), (2, 3, 2, (17, 23))]


def _golden(case):
    return refgolden.load("mvdepth_oracle_vs_reference", case)


def _ref_loss(h, w):
    from oracle.ref_import import load_reference
    load_reference()                      # stubs for kornia etc. + sys.path
    losses = importlib.import_module("losses")
    return losses.MVDepthLoss(h, w)


def _mask_args(t, k):
    return (t["cur_depth_b1hw"], t["src_depth_bk1hw"][:, k], t["cur_invK_b44"], t["src_K_bk44"][:, k],
            t["cur_world_T_cam_b44"], t["src_cam_T_world_bk44"][:, k])


def _behind_camera_batch():
    """A (nonsensical) negative prediction at a valid pixel: z_pred <= 0 behind a source camera."""
    t = make_mvloss_batch(7, 1, 2, 16, 20)
    vm, _ = M.valid_mask(*_mask_args(t, 0))
    idx = vm.flatten().nonzero()[0].item()
    p = t["depth_pred_b1hw"].clone()
    p.view(-1)[idx] = -50.0
    return t, p, idx


def reference_outputs():
    """For tests/golden/make_reference_golden.py."""
    out = {}
    for seed, B, K, hw in CASES:
        t = make_mvloss_batch(seed, B, K, *hw)
        p = t["depth_pred_b1hw"].clone().requires_grad_(True)
        loss = _ref_loss(*hw)(**{**t, "depth_pred_b1hw": p})
        loss.backward()
        out[f"loss_{seed}"] = dict(loss=loss.detach(), grad=p.grad)
    t = make_mvloss_batch(5, 2, 2, 20, 28)
    vm, s = _ref_loss(20, 28).get_valid_mask(*_mask_args(t, 1))
    out["mask"] = dict(valid=vm, src=s)
    t, p, _ = _behind_camera_batch()
    p = p.requires_grad_(True)
    loss = _ref_loss(16, 20)(**{**t, "depth_pred_b1hw": p})
    loss.backward()
    out["behind"] = dict(loss=loss.detach(), grad=p.grad)
    return out


@pytest.mark.parametrize("seed,B,K,hw", CASES)
def test_loss_and_gradient_match_live_reference(seed, B, K, hw):
    G = _golden(f"loss_{seed}")
    t = make_mvloss_batch(seed, B, K, *hw)
    p_ora = t["depth_pred_b1hw"].clone().requires_grad_(True)
    l_ora = M.mv_depth_loss(**{**t, "depth_pred_b1hw": p_ora})
    assert torch.isfinite(G["loss"]) and G["loss"].item() > 1e-3
    assert l_ora.item() == G["loss"].item()                  # same ops in the same order: bit-equal
    l_ora.backward()
    assert torch.equal(G["grad"], p_ora.grad) and G["grad"].abs().sum() > 0


def test_valid_mask_matches_live_reference():
    G = _golden("mask")
    t = make_mvloss_batch(5, 2, 2, 20, 28)
    vm_o, s_o = M.valid_mask(*_mask_args(t, 1))
    assert torch.equal(G["valid"], vm_o) and torch.equal(G["src"], s_o)
    assert 0.05 < G["valid"].float().mean().item() < 0.98


def test_prediction_behind_a_source_camera_is_dropped_from_the_mean_but_poisons_its_gradient():
    """z_pred <= 0 makes log() NaN / -inf: nanmean drops NaN terms from the VALUE (losses.py:173); what the
    reference's autograd does with such a pixel is recorded here (the kernel follows it)."""
    G = _golden("behind")
    t, p, idx = _behind_camera_batch()
    p_ora = p.clone().requires_grad_(True)
    l_ora = M.mv_depth_loss(**{**t, "depth_pred_b1hw": p_ora})
    assert torch.isfinite(G["loss"]) and l_ora.item() == G["loss"].item()
    l_ora.backward()
    assert torch.equal(torch.isnan(G["grad"]), torch.isnan(p_ora.grad))
    print("grad at the behind-camera pixel:", G["grad"].view(-1)[idx].item(), "NaNs:", torch.isnan(G["grad"]).sum().item())
