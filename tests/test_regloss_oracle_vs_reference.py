"""CPU: the fp32 oracle (oracle/regloss_oracle.py) against the unmodified reference ``DepthModel.compute_losses``
(experiment_modules/depth_model.py:409-500, imported by ``regloss_oracle.load_reference_depth_model``): the five
regression terms and the gradient of each to every ``log_depth_pred_s{i}`` and to ``depth_pred``, bit for bit, with
NaN at the same places.  Cases: B = 2 at 24x32 with scales at /2^i; an odd 17x23 with 9x12, 5x6 and 3x3 scales; a
scale larger than the ground truth; s1 and s3 absent; an empty mask; an empty inverse-depth mask; predictions at and
below 0.1 with NaN predictions inside the mask; a zero ground truth inside the mask.  Also the whole nine-key dict and
the gradient of ``loss`` to the four scales at 48x64, where the gradient term is finite.  The inputs and the
reference's outputs are stored in tests/golden/reference/regloss_oracle_vs_reference.npz
(tests/golden/make_regloss_reference_golden.py)."""
import types

import pytest
import torch

from oracle import regloss_oracle as R
from oracle import gradloss_oracle, mvdepth_oracle, normals_oracle
from oracle.ref_import import reference_available
from simplerecon_b200 import losses as L
from simplerecon_b200.synthetic import make_training_step_batch
from tests import refgolden

MODULE = "regloss_oracle_vs_reference"
SI_LAMBDA = 0.85
STEP_CASE, STEP_SHAPE = "step_b2_48x64", (2, 48, 64)


def _resized(s0, hw, g, noise=0.03):
    return (torch.nn.functional.adaptive_avg_pool2d(s0, hw) + noise * torch.randn(s0.shape[0], 1, *hw, generator=g))


def make_inputs(case):
    """(depth_gt, mask_b, {scale: log_depth_pred}, depth_pred) of a case, on the CPU, fp32"""
    seed = sorted(CASES).index(case)
    B, H, W, sizes = CASES[case]
    cur, _, out = make_training_step_batch(seed, B, H, W, views=1)
    gt, mask = cur["depth_b1hw"], cur["mask_b_b1hw"]
    s0 = out["log_depth_pred_s0_b1hw"]
    g = torch.Generator().manual_seed(777 + seed)
    lps = {0: s0}
    for i, hw in enumerate(sizes, start=1):
        if hw is not None:
            lps[i] = _resized(s0, hw, g).contiguous()
    dp = out["depth_pred_s0_b1hw"].clone()
    if case == "empty_mask":
        mask = torch.zeros_like(mask)
    elif case == "empty_inv_mask":
        dp = torch.where(torch.rand(dp.shape, generator=g) < 0.5, torch.full_like(dp, 0.1), 0.05 * dp / dp.max())
    elif case == "low_and_nan_preds":
        sel = torch.rand(dp.shape, generator=g)
        dp = torch.where(sel < 0.15, torch.full_like(dp, 0.1), dp)                  # exactly fp32 0.1: not > 0.1
        dp = torch.where((sel >= 0.15) & (sel < 0.3), 0.04 * dp, dp)
        idx = mask.flatten().nonzero()[:, 0]
        lps[0].view(-1)[idx[3]] = float("nan")
        lps[1].view(-1)[0] = float("nan")
        dp.view(-1)[idx[5]] = float("nan")
    elif case == "zero_gt_in_mask":
        idx = mask.flatten().nonzero()[:, 0]
        gt.view(-1)[idx[:4]] = 0.0
    return gt, mask, lps, dp


# name: (B, H, W, sizes of scales 1..3, None = absent)
CASES = {
    "b2_24x32": (2, 24, 32, [(12, 16), (6, 8), (3, 4)]),
    "odd_b1_17x23": (1, 17, 23, [(9, 12), (5, 6), (3, 3)]),
    "scale_larger_than_gt_b1_12x16": (1, 12, 16, [(24, 40), (5, 7), (1, 1)]),
    "s1_s3_absent_b2_24x32": (2, 24, 32, [None, (6, 8), None]),
    "empty_mask": (1, 12, 16, [(6, 8), (3, 4), (2, 2)]),
    "empty_inv_mask": (1, 12, 16, [(6, 8), (3, 4), (2, 2)]),
    "low_and_nan_preds": (2, 16, 20, [(8, 10), (4, 5), (2, 3)]),
    "zero_gt_in_mask": (1, 16, 20, [(8, 10), (4, 5), (2, 3)]),
}


def grads_of_terms(terms_fn, gt, mask, lps, dp):
    """the five terms and the gradient of each to every scale and to depth_pred"""
    leaves = {i: t.clone().requires_grad_(True) for i, t in lps.items()}
    p = dp.clone().requires_grad_(True)
    terms = terms_fn(gt, mask, leaves, p)
    out = {k: terms[k].detach() for k in R.KEYS}
    inputs = [leaves[i] for i in sorted(leaves)] + [p]
    names = [f"s{i}" for i in sorted(leaves)] + ["depth_pred"]
    for k in R.KEYS:
        gs = torch.autograd.grad(terms[k], inputs, retain_graph=True, allow_unused=True)
        for n, x, gr in zip(names, inputs, gs):
            out[f"grad_{k}_{n}"] = gr if gr is not None else torch.zeros_like(x)
    return out


def _stub_model(si_loss):
    """``self`` for the reference's compute_losses when only the regression terms are wanted: the other three loss
    modules return zeros"""
    zero = lambda *a, **k: torch.zeros(())   # noqa: E731
    abs_loss = torch.nn.L1Loss()
    return types.SimpleNamespace(si_loss=si_loss, grad_loss=zero, normals_loss=zero, mv_depth_loss=zero,
                                 abs_loss=abs_loss, ms_loss_fn=abs_loss)


def _reference_terms(dm, model):
    def run(gt, mask, lps, dp):
        B, _, H, W = gt.shape
        eye = torch.eye(4).repeat(B, 1, 1)
        cur = {"depth_b1hw": gt, "mask_b_b1hw": mask, "mask_b1hw": mask.float(), "normals_b3hw": None,
               "invK_s0_b44": eye, "world_T_cam_b44": eye}
        src = {"depth_b1hw": None, "K_s0_b44": None, "cam_T_world_b44": None}
        outputs = {f"log_depth_pred_s{i}_b1hw": t for i, t in lps.items()}
        outputs.update(depth_pred_s0_b1hw=dp, normals_pred_b3hw=None)
        return dm.DepthModel.compute_losses(model, cur, src, outputs)
    return run


def step_outputs(compute, cur, src, out, normal_generator):
    """the step's graph from the four scales (depth_model.py:398-400, :530): depth_pred = exp(s0), normals of it,
    then ``compute`` -> the nine losses and the gradient of ``loss`` to each scale"""
    leaves = {k: v.clone().requires_grad_(True) for k, v in out.items() if k.startswith("log_depth_pred")}
    o = dict(leaves)
    o["depth_pred_s0_b1hw"] = torch.exp(leaves["log_depth_pred_s0_b1hw"])
    o["normals_pred_b3hw"] = normal_generator(o["depth_pred_s0_b1hw"], cur["invK_s0_b44"])
    losses = compute(cur, src, o)
    grads = torch.autograd.grad(losses["loss"], [leaves[f"log_depth_pred_s{i}_b1hw"] for i in range(4)])
    res = {f"{k}": v.detach() for k, v in losses.items()}
    res.update({f"grad_loss_s{i}": g for i, g in enumerate(grads)})
    res["keys"] = torch.tensor([R.STEP_KEYS.index(k) for k in losses])
    return res


def make_step_inputs():
    B, H, W = STEP_SHAPE
    cur, src, out = make_training_step_batch(11, B, H, W, views=3)
    cur["normals_b3hw"] = normals_oracle.normal_generator(cur["depth_b1hw"], cur["invK_s0_b44"])
    return cur, src, out


def reference_outputs() -> dict:
    """runs the unmodified reference (needs $SIMPLERECON_REF)"""
    dm = R.load_reference_depth_model()
    ref_normals = normals_oracle.load_reference_normals()
    res = {}
    run = _reference_terms(dm, _stub_model(dm.ScaleInvariantLoss()))
    for case in CASES:
        gt, mask, lps, dp = make_inputs(case)
        res[case] = dict(depth_gt=gt, mask_b=mask, depth_pred=dp, **{f"log_depth_pred_s{i}": t for i, t in lps.items()},
                         **grads_of_terms(run, gt, mask, lps, dp))
    cur, src, out = make_step_inputs()
    ng = ref_normals.NormalGenerator(STEP_SHAPE[1], STEP_SHAPE[2])
    model = R.reference_model(dm, STEP_SHAPE[1], STEP_SHAPE[2])
    res[STEP_CASE] = step_outputs(lambda c, s, o: dm.DepthModel.compute_losses(model, c, s, o), cur, src, out, ng)
    return res


def _oracle_terms(gt, mask, lps, dp):
    return R.regression_terms(gt, mask, lps, dp, SI_LAMBDA)


def _same(a, b):
    return torch.equal(torch.as_tensor(a).nan_to_num(7.0), torch.as_tensor(b).nan_to_num(7.0)) and \
        torch.equal(torch.as_tensor(a).isnan(), torch.as_tensor(b).isnan())


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_stored_reference(case):
    ref = refgolden.load(MODULE, case)
    gt, mask, lps, dp = make_inputs(case)
    assert _same(gt, ref["depth_gt"]) and torch.equal(mask, ref["mask_b"]) and _same(dp, ref["depth_pred"])
    for i, t in lps.items():
        assert _same(t, ref[f"log_depth_pred_s{i}"])
    ours = grads_of_terms(_oracle_terms, gt, mask, lps, dp)
    assert set(ours) == set(ref) - {"depth_gt", "mask_b", "depth_pred"} - {f"log_depth_pred_s{i}" for i in lps}
    for name, v in ours.items():
        assert _same(v, ref[name]), (case, name)
    n, m = R.masks(gt, mask, dp)
    if case == "empty_mask":
        assert n == 0 and all(torch.isnan(ref[k]) for k in R.KEYS)
    if case == "empty_inv_mask":
        assert n > 0 and m == 0 and torch.isnan(ref["inv_abs_loss"]) and torch.isfinite(ref["ms_loss"])


def test_oracle_step_matches_stored_reference():
    ref = refgolden.load(MODULE, STEP_CASE)
    cur, src, out = make_step_inputs()
    ours = step_outputs(lambda c, s, o: R.compute_losses(c, s, o, SI_LAMBDA), cur, src, out,
                        normals_oracle.normal_generator)
    assert ref["keys"].tolist() == list(range(len(R.STEP_KEYS)))
    for name, v in ours.items():
        assert _same(v, ref[name]), name
    assert all(torch.isfinite(ref[k]) for k in R.STEP_KEYS)


def test_drop_in_compute_losses_through_the_oracle(monkeypatch):
    """losses.compute_losses with the fused call replaced by the oracle: the reference's keys, order and values"""
    monkeypatch.setattr(L, "uses_fused_regression_losses", lambda model, gt: True)
    monkeypatch.setattr(L, "depth_regression_losses", lambda gt, mask, lps, dp, si_lambda: R.regression_terms(
        gt, mask, lps, dp, si_lambda))
    model = types.SimpleNamespace(si_loss=types.SimpleNamespace(si_lambda=SI_LAMBDA),
                                  grad_loss=gradloss_oracle.ms_gradient_loss, normals_loss=normals_oracle.normals_loss,
                                  mv_depth_loss=mvdepth_oracle.mv_depth_loss)
    ref = refgolden.load(MODULE, STEP_CASE)
    cur, src, out = make_step_inputs()
    ours = step_outputs(lambda c, s, o: L.compute_losses(model, c, s, o), cur, src, out, normals_oracle.normal_generator)
    for name, v in ours.items():
        assert _same(v, ref[name]), name


@pytest.mark.skipif(not reference_available(), reason="needs $SIMPLERECON_REF (the reference tree)")
def test_stored_outputs_are_the_live_reference():
    live = reference_outputs()
    for case, arrays in live.items():
        stored = refgolden.load(MODULE, case)
        assert set(arrays) == set(stored), case
        for name, v in arrays.items():
            assert _same(v, stored[name]), (case, name)
