"""Oracle for the gradient-loss kernels (DESIGN §4.14): MSGradientLoss (reference losses.py:11-37, with
``pyrdown`` of utils/generic_utils.py:87-94) and ScaleInvariantLoss (losses.py:39-54), in the reference's
operation order.

TEST INFRASTRUCTURE — never imported by the product package.

The reference pins kornia 0.6.7 (simplerecon_env.yml:19), which is not a dependency of this project, so
``blur_pool2d`` is restated here from its definition (``_blur_pool_by_kernel2d``): a depthwise ``conv2d`` with
the normalised Pascal kernel ([1,2,1] x [1,2,1] / 16 for size 3), stride 2 and ZERO padding (k - 1) // 2, so
the output is ceil(h / 2) and the border outputs are darkened.  ``spatial_gradient`` is the restatement of
``oracle.normals_oracle``.  No test can compare these against the live kornia; the restatement is this project's
definition.  ``blur_pool2d`` is TorchScript-compilable: the reference's ``pyrdown`` is ``@torch.jit.script``-
compiled when utils/generic_utils.py is imported and keeps whatever ``kornia.filters.blur_pool2d`` existed then, and
``oracle.ref_import`` registers an ``avg_pool2d`` placeholder under that name (nothing on its paths executes it).
``load_reference_losses`` therefore puts this function into the stand-in ``kornia.filters`` and has the unmodified
utils/generic_utils.py compiled against it, so the unmodified reference ``MSGradientLoss`` runs on it.

Everything runs in the dtype of its inputs: fp32 is the reference's computation, fp64 the yardstick for the
kernels.
"""
from __future__ import annotations

import importlib
import sys
import types
from typing import List

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle.normals_oracle import spatial_gradient


def blur_pool2d(input: Tensor, kernel_size: int, stride: int = 2) -> Tensor:
    """kornia.filters.blur_pool2d (0.6.7): get_pascal_kernel_2d(kernel_size, norm=True), then
    F.conv2d(input, kernel, padding=(k - 1) // 2, stride=stride, groups=C)"""
    row = torch.ones(1)
    for _ in range(kernel_size - 1):
        row = F.pad(row, [1, 0]) + F.pad(row, [0, 1])
    kernel = row.unsqueeze(1) * row.unsqueeze(0)
    kernel = (kernel / kernel.sum()).to(dtype=input.dtype, device=input.device)
    c = input.size(1)
    pad = (kernel_size - 1) // 2
    return F.conv2d(input, kernel.unsqueeze(0).unsqueeze(0).repeat(c, 1, 1, 1), padding=[pad, pad],
                    stride=[stride, stride], groups=c)


def pyrdown(input_tensor: Tensor, num_scales: int = 4) -> List[Tensor]:
    """utils/generic_utils.py:87-94"""
    output = [input_tensor]
    for _ in range(num_scales - 1):
        output.append(blur_pool2d(output[-1], 3))
    return output


def level_masks(depth_gt: Tensor, num_scales: int = 4) -> List[Tensor]:
    """the masks MSGradientLoss selects with, one per level: (B, 1, 2, h, w) bool, per gradient component"""
    return [spatial_gradient(g).isfinite().all(dim=1, keepdim=True) for g in pyrdown(depth_gt, num_scales)]


def ms_gradient_loss(depth_gt: Tensor, depth_pred: Tensor, num_scales: int = 4) -> Tensor:
    """MSGradientLoss.forward (losses.py:17-37)"""
    grad_loss = torch.tensor(0, dtype=depth_gt.dtype, device=depth_gt.device)
    for pred_down, gtn_down in zip(pyrdown(depth_pred, num_scales), pyrdown(depth_gt, num_scales)):
        gtn_grad = spatial_gradient(gtn_down)
        mask = gtn_grad.isfinite().all(dim=1, keepdim=True)
        pred_grad = spatial_gradient(pred_down).masked_select(mask)
        grad_error = torch.abs(pred_grad - gtn_grad.masked_select(mask))
        grad_loss = grad_loss + torch.mean(grad_error)
    return grad_loss


def scale_invariant_loss(log_depth_gt: Tensor, log_depth_pred: Tensor, si_lambda: float = 0.85) -> Tensor:
    """ScaleInvariantLoss.forward (losses.py:46-54)"""
    log_diff = log_depth_gt - log_depth_pred
    return torch.sqrt((log_diff ** 2).mean() - si_lambda * (log_diff.mean() ** 2))


def _kornia_stand_in() -> None:
    """``kornia.filters`` as the reference will see it: a real kornia if one is importable, else a stand-in module
    (the one ``oracle.ref_import`` registered, or one registered here, which ``ref_import`` then leaves alone) that
    carries the restated ``blur_pool2d`` and ``spatial_gradient``."""
    if "kornia" not in sys.modules:
        kornia, filters = types.ModuleType("kornia"), types.ModuleType("kornia.filters")
        kornia.filters = filters
        sys.modules["kornia"], sys.modules["kornia.filters"] = kornia, filters
    filters = sys.modules["kornia.filters"]
    if getattr(sys.modules["kornia"], "__file__", None) is None:
        filters.blur_pool2d = blur_pool2d
        if not hasattr(filters, "spatial_gradient"):
            filters.spatial_gradient = spatial_gradient


def load_reference_losses() -> types.SimpleNamespace:
    """The unmodified reference ``MSGradientLoss`` and ``ScaleInvariantLoss`` (losses.py), needs
    ``$SIMPLERECON_REF``.  ``pyrdown`` is compiled at the import of utils/generic_utils.py; if that happened
    earlier in this process against ``ref_import``'s ``avg_pool2d`` placeholder (its graph shows it), the module is
    reloaded, which compiles the same unmodified source against the restatement, and ``losses`` is handed the
    recompiled function under the name it imported."""
    from oracle.ref_import import load_reference
    _kornia_stand_in()
    load_reference()
    generic_utils = importlib.import_module("utils.generic_utils")
    if "avg_pool2d" in str(generic_utils.pyrdown.inlined_graph):
        generic_utils = importlib.reload(generic_utils)
    losses = importlib.import_module("losses")
    losses.pyrdown = generic_utils.pyrdown
    return types.SimpleNamespace(MSGradientLoss=losses.MSGradientLoss, ScaleInvariantLoss=losses.ScaleInvariantLoss,
                                 losses=losses)
