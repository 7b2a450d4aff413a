"""Oracle for the regression-loss kernels (DESIGN §4.15): the five regression terms of the reference's
``DepthModel.compute_losses`` (experiment_modules/depth_model.py:447-474) in the reference's operation order —
``F.interpolate`` (nearest), boolean indexing, ``nn.L1Loss`` and the ``ScaleInvariantLoss`` arithmetic — and the whole
nine-key ``compute_losses`` composed from the oracles of every term.

TEST INFRASTRUCTURE — never imported by the product package.

Everything runs in the dtype of its inputs: fp32 is the reference's computation, fp64 the yardstick for the kernels.
The one constant, the ``depth_pred > 0.1`` limit, is PyTorch's fp32 rounding of 0.1 in both modes, so that the fp64
mode selects the pixels the fp32 computation does.

``load_reference_depth_model()`` imports the unmodified experiment_modules/depth_model.py.  It needs pytorch_lightning,
matplotlib and moviepy, none of which this project depends on or uses on the loss path: inert stand-ins are
registered for them (``LightningModule = nn.Module``), together with the restated kornia filters of
``gradloss_oracle`` and ``normals_oracle``.
"""
from __future__ import annotations

import importlib
import sys
import types

import torch
import torch.nn.functional as F
from torch import Tensor, nn

from oracle import gradloss_oracle, mvdepth_oracle, normals_oracle

KEYS = ("ms_loss", "abs_loss", "si_loss", "inv_abs_loss", "log_l1_loss")
# the reference's key order (depth_model.py:489-499)
STEP_KEYS = ("loss", "si_loss", "grad_loss", "abs_loss", "normals_loss", "ms_loss", "inv_abs_loss", "log_l1_loss",
             "mv_loss")
INV_DEPTH_LIMIT = float(torch.tensor(0.1, dtype=torch.float32))


def regression_terms(depth_gt: Tensor, mask_b: Tensor, log_depth_preds: dict, depth_pred: Tensor,
                     si_lambda: float = 0.85) -> dict:
    """depth_model.py:447-474 with ``ms_loss_fn = abs_loss = nn.L1Loss()``; ``log_depth_preds`` maps a scale index to
    ``log_depth_pred_s{i}_b1hw``"""
    l1 = nn.L1Loss()
    log_depth_pred = log_depth_preds[0]
    log_depth_gt = torch.log(depth_gt)
    ms_loss = 0
    for i in range(4):
        if i in log_depth_preds:
            log_depth_pred_resized = F.interpolate(log_depth_preds[i], size=depth_gt.shape[-2:], mode="nearest")
            ms_loss += l1(log_depth_gt[mask_b], log_depth_pred_resized[mask_b]) / 2 ** i
    abs_loss = l1(depth_gt[mask_b], depth_pred[mask_b])
    si_loss = gradloss_oracle.scale_invariant_loss(log_depth_gt[mask_b], log_depth_pred[mask_b], si_lambda)
    mask_b_limit = torch.logical_and(mask_b, depth_pred > INV_DEPTH_LIMIT)
    inv_abs_loss = l1(1 / depth_gt[mask_b_limit], 1 / depth_pred[mask_b_limit])
    log_l1_loss = l1(log_depth_gt[mask_b], log_depth_pred[mask_b])
    return dict(ms_loss=ms_loss, abs_loss=abs_loss, si_loss=si_loss, inv_abs_loss=inv_abs_loss,
                log_l1_loss=log_l1_loss)


def masks(depth_gt: Tensor, mask_b: Tensor, depth_pred: Tensor) -> tuple[int, int]:
    """(n, m): the pixels of mask_b and of mask_b & depth_pred > 0.1"""
    return int(mask_b.sum()), int((mask_b & (depth_pred.float() > INV_DEPTH_LIMIT)).sum())


def compute_losses(cur_data: dict, src_data: dict, outputs: dict, si_lambda: float = 0.85) -> dict:
    """DepthModel.compute_losses (depth_model.py:409-500) from the oracles of every term: the nine losses in the
    reference's key order"""
    depth_gt, depth_pred = cur_data["depth_b1hw"], outputs["depth_pred_s0_b1hw"]
    log_preds = {i: outputs[f"log_depth_pred_s{i}_b1hw"] for i in range(4) if f"log_depth_pred_s{i}_b1hw" in outputs}
    t = regression_terms(depth_gt, cur_data["mask_b_b1hw"], log_preds, depth_pred, si_lambda)
    grad_loss = gradloss_oracle.ms_gradient_loss(depth_gt, depth_pred)
    normals_loss = normals_oracle.normals_loss(cur_data["normals_b3hw"], outputs["normals_pred_b3hw"])
    mv_loss = mvdepth_oracle.mv_depth_loss(depth_pred, depth_gt, src_data["depth_b1hw"], cur_data["invK_s0_b44"],
                                           src_data["K_s0_b44"], cur_data["world_T_cam_b44"],
                                           src_data["cam_T_world_b44"])
    loss = t["ms_loss"] + 1.0 * grad_loss + 1.0 * normals_loss + 0.2 * mv_loss
    out = dict(loss=loss, grad_loss=grad_loss, normals_loss=normals_loss, mv_loss=mv_loss, **t)
    return {k: out[k] for k in STEP_KEYS}


def _stand_ins() -> None:
    """inert modules for the imports of depth_model.py and utils/visualization_utils.py that the loss path never uses"""
    for name in ("pytorch_lightning", "matplotlib", "matplotlib.pyplot", "moviepy", "moviepy.editor"):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    pl = sys.modules["pytorch_lightning"]
    if not hasattr(pl, "LightningModule"):
        pl.LightningModule = nn.Module
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    sys.modules["moviepy"].editor = sys.modules["moviepy.editor"]


def load_reference_depth_model() -> types.ModuleType:
    """The unmodified reference ``experiment_modules/depth_model.py`` (needs ``$SIMPLERECON_REF``), imported after
    the restated kornia filters are in place (``gradloss_oracle.load_reference_losses``,
    ``normals_oracle.load_reference_normals``) and with the stand-ins above."""
    gradloss_oracle.load_reference_losses()
    normals_oracle.load_reference_normals()
    _stand_ins()
    return importlib.import_module("experiment_modules.depth_model")


def reference_model(depth_model: types.ModuleType, height: int, width: int) -> types.SimpleNamespace:
    """What ``DepthModel.compute_losses`` reads from ``self``: the loss modules ``DepthModel.__init__`` builds
    (depth_model.py:139-151), from the names ``depth_model`` bound at import"""
    abs_loss = nn.L1Loss()
    return types.SimpleNamespace(si_loss=depth_model.ScaleInvariantLoss(), grad_loss=depth_model.MSGradientLoss(),
                                 abs_loss=abs_loss, ms_loss_fn=abs_loss, normals_loss=depth_model.NormalsLoss(),
                                 mv_depth_loss=depth_model.MVDepthLoss(height, width))
