"""Oracle for the normals kernels (DESIGN §4.13): NormalGenerator (reference utils/geometry_utils.py:92-133)
and NormalsLoss (losses.py:57-77), in the reference's operation order.

TEST INFRASTRUCTURE — never imported by the product package.

The reference pins kornia 0.6.7 (simplerecon_env.yml:19), which is not a dependency of this project, so its
three filters are restated from their definitions with ``F.pad`` + ``conv2d``:
  - ``gaussian_blur2d(x, (k, k), (s, s))``: separable, an x pass then a y pass, each a cross-correlation
    with 'reflect' padding; the 1-D taps are kornia's ``gaussian(k, s)`` in fp32, cast to the input;
  - ``spatial_gradient(x)``: Sobel, normalised by the sum of absolute weights (8), 'replicate' padding,
    (B, C, 2, H, W) with the x derivative first.
No test can compare these against the live kornia.  They are TorchScript-compilable: the reference's
``NormalGenerator`` is a ``ScriptModule`` that scripts the kornia calls, and ``load_reference_normals`` plugs
them into the stand-in ``kornia.filters`` that ``oracle.ref_import`` registers, so the unmodified reference
module runs on them.

``normal_generator`` / ``normals_loss`` run in the dtype of their inputs: fp32 is the reference's
computation, fp64 (same fp32 taps, upcast) the yardstick for the kernels.
"""
from __future__ import annotations

import importlib
import sys
import types
from typing import Tuple

import torch
import torch.nn.functional as F
from torch import Tensor


def gaussian(window_size: int, sigma: float) -> Tensor:
    """kornia.filters.kernels.gaussian (0.6.7)"""
    x = torch.arange(window_size) - window_size // 2
    if window_size % 2 == 0:
        x = x + 0.5
    gauss = torch.exp(-x.pow(2.0) / float(2 * sigma ** 2))
    return gauss / gauss.sum()


def gaussian_blur2d(input: Tensor, kernel_size: Tuple[int, int], sigma: Tuple[float, float],
                    border_type: str = "reflect", separable: bool = True) -> Tensor:
    """kornia.filters.gaussian_blur2d (0.6.7): separable_filter2d = filter2d with the (1, kx) kernel, then
    filter2d with the (ky, 1) kernel, each padding 'same' with ``border_type``; depthwise cross-correlation."""
    c = input.shape[1]
    kx = gaussian(kernel_size[1], sigma[1]).to(input)
    ky = gaussian(kernel_size[0], sigma[0]).to(input)
    px, py = kernel_size[1] // 2, kernel_size[0] // 2
    out = F.pad(input, [px, px, 0, 0], mode=border_type)
    out = F.conv2d(out, kx.reshape(1, 1, 1, -1).expand(c, 1, 1, kernel_size[1]), groups=c)
    out = F.pad(out, [0, 0, py, py], mode=border_type)
    return F.conv2d(out, ky.reshape(1, 1, -1, 1).expand(c, 1, kernel_size[0], 1), groups=c)


def sobel_kernel(dtype: torch.dtype, device: torch.device) -> Tensor:
    """(2, 3, 3): kornia's get_sobel_kernel2d / normalize_kernel2d (x derivative first)"""
    kx = torch.tensor([[-1.0, 0.0, 1.0], [-2.0, 0.0, 2.0], [-1.0, 0.0, 1.0]])
    k = torch.stack([kx, kx.transpose(0, 1)])
    k = k / k.abs().sum(-1).sum(-1).unsqueeze(-1).unsqueeze(-1)
    return k.to(dtype=dtype, device=device)


def spatial_gradient(input: Tensor, mode: str = "sobel", order: int = 1, normalized: bool = True) -> Tensor:
    """kornia.filters.spatial_gradient (0.6.7), Sobel, first order, normalised: (B, C, 2, H, W)"""
    b, c, h, w = input.shape
    k = sobel_kernel(input.dtype, input.device).unsqueeze(1)
    padded = F.pad(input.reshape(b * c, 1, h, w), [1, 1, 1, 1], mode="replicate")
    return F.conv2d(padded, k).view(b, c, 2, h, w)


def pix_coords(height: int, width: int) -> Tensor:
    """BackprojectDepth.pix_coords_13N (geometry_utils.py:34-44): (1, 3, H*W) fp32, pixel centres, xy order"""
    xx, yy = torch.meshgrid(torch.arange(width), torch.arange(height), indexing="xy")
    pix = torch.stack((xx, yy), dim=0) + 0.5
    return torch.cat([pix, torch.ones_like(pix[:1])], 0).flatten(1).unsqueeze(0)


def normal_generator(depth_b1hw: Tensor, invK_b44: Tensor, kernel_size: int = 5, std: float = 2.0) -> Tensor:
    """NormalGenerator.forward (geometry_utils.py:107-133) in the dtype of the depth"""
    _, _, h, w = depth_b1hw.shape
    smooth = gaussian_blur2d(depth_b1hw, (kernel_size, kernel_size), (std, std))
    cam = torch.matmul(invK_b44[:, :3, :3], pix_coords(h, w).to(depth_b1hw))
    cam = smooth.flatten(start_dim=2) * cam
    points = cam.view(-1, 3, h, w)
    g = spatial_gradient(points)
    return F.normalize(torch.cross(g[:, :, 0], g[:, :, 1], dim=1), dim=1)


def normals_loss(normals_gt_b3hw: Tensor, normals_pred_b3hw: Tensor) -> Tensor:
    """NormalsLoss.forward (losses.py:58-77)"""
    mask = torch.logical_and(normals_gt_b3hw.isfinite().all(dim=1, keepdim=True),
                             normals_pred_b3hw.isfinite().all(dim=1, keepdim=True))
    pred = normals_pred_b3hw.masked_fill(~mask, 1.0)
    gt = normals_gt_b3hw.masked_fill(~mask, 1.0)
    dot = 0.5 * (1.0 - torch.einsum("bchw, bchw -> bhw", pred, gt)).unsqueeze(1)
    return dot.masked_select(mask).mean()


def all_finite(normals_b3hw: Tensor) -> Tensor:
    """the per-pixel mask NormalsLoss uses: (B, H, W) bool"""
    return normals_b3hw.isfinite().all(dim=1)


def load_reference_normals() -> types.SimpleNamespace:
    """The unmodified reference ``NormalGenerator`` (utils/geometry_utils.py) and ``NormalsLoss`` (losses.py),
    needs ``$SIMPLERECON_REF``.  ``oracle.ref_import`` registers a stand-in ``kornia.filters`` that carries only
    ``blur_pool2d``; the restated ``gaussian_blur2d`` and ``spatial_gradient`` are added to it here, before a
    ``NormalGenerator`` is built (its script methods resolve the names when an instance is first created).
    A real kornia, if one is importable, is left alone."""
    from oracle.ref_import import load_reference
    ref = load_reference()
    filters = sys.modules["kornia.filters"]
    for name, fn in (("gaussian_blur2d", gaussian_blur2d), ("spatial_gradient", spatial_gradient)):
        if not hasattr(filters, name):
            setattr(filters, name, fn)
    losses = importlib.import_module("losses")
    return types.SimpleNamespace(NormalGenerator=ref.geometry.NormalGenerator, NormalsLoss=losses.NormalsLoss,
                                 geometry=ref.geometry, losses=losses)
