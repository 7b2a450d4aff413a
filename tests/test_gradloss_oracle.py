"""CPU: the restated blur_pool2d / pyrdown and the two losses of oracle/gradloss_oracle.py against their
definitions: the Pascal kernel's analytic border values, the ceil output size, how NaN holes dilate down the
pyramid, the per-component mask, the NaN of an empty level, and TorchScript-compilability (the reference's
pyrdown is script-compiled on top of blur_pool2d)."""
import math

import pytest
import torch

from oracle import gradloss_oracle as O
from oracle.normals_oracle import spatial_gradient


def test_blur_pool_of_a_constant_image():
    out = O.blur_pool2d(torch.ones(2, 1, 8, 10), 3)
    assert out.shape == (2, 1, 4, 5)
    assert torch.all(out[:, :, 1:, 1:] == 1.0)                        # every tap inside the map
    assert torch.all(out[:, :, 0, 0] == 9.0 / 16.0)                   # the corner loses a row and a column of taps
    assert torch.all(out[:, :, 0, 1:] == 0.75) and torch.all(out[:, :, 1:, 0] == 0.75)


def test_blur_pool_is_the_pascal_kernel_at_stride_two():
    x = torch.arange(35, dtype=torch.float64).reshape(1, 1, 5, 7) ** 1.5
    out = O.blur_pool2d(x, 3)
    k = torch.tensor([1.0, 2.0, 1.0], dtype=torch.float64)
    padded = torch.nn.functional.pad(x, [1, 1, 1, 1])
    for y in range(3):
        for xx in range(4):
            want = (padded[0, 0, 2 * y:2 * y + 3, 2 * xx:2 * xx + 3] * (k[:, None] * k[None]) / 16).sum()
            assert abs(out[0, 0, y, xx] - want) <= 1e-12 * abs(want) + 1e-15


@pytest.mark.parametrize("H,W", [(5, 4), (17, 23), (24, 32), (3, 3), (1, 1)])
def test_level_sizes_are_ceil(H, W):
    pyr = O.pyrdown(torch.rand(2, 1, H, W), 4)
    assert len(pyr) == 4
    h, w = H, W
    for lvl in pyr:
        assert lvl.shape == (2, 1, h, w)
        h, w = math.ceil(h / 2), math.ceil(w / 2)


def test_nan_holes_dilate_down_the_pyramid():
    x = torch.rand(1, 1, 16, 16)
    x[0, 0, 5, 6] = float("nan")                                      # odd row, even column
    l0, l1, l2 = O.pyrdown(x, 3)
    # level-1 output Y reads rows 2Y-1..2Y+1: row 5 is read by Y = 2 and 3, column 6 by X = 3 only
    assert torch.isnan(l1).nonzero()[:, 2:].tolist() == [[2, 3], [3, 3]]
    # level-2 output reads 2Y-1..2Y+1 of level 1: rows 2, 3 by Y = 1 (both) and Y = 2 (row 3); column 3 by X = 1, 2
    assert torch.isnan(l2).nonzero()[:, 2:].tolist() == [[1, 1], [1, 2], [2, 1], [2, 2]]
    # the mask drops a component when any of its nine clamped window values is NaN: the zero taps count
    m0 = O.level_masks(x, 1)[0]
    assert m0.shape == (1, 1, 2, 16, 16) and m0.dtype == torch.bool
    assert torch.equal(m0[0, 0, 0], m0[0, 0, 1])
    assert (~m0[0, 0, 0]).nonzero().tolist() == [[y, xx] for y in (4, 5, 6) for xx in (5, 6, 7)]


def test_mask_is_per_gradient_component():
    gt = torch.rand(3, 1, 9, 11)
    masks = O.level_masks(gt, 4)
    assert [tuple(m.shape) for m in masks] == [(3, 1, 2, 9, 11), (3, 1, 2, 5, 6), (3, 1, 2, 3, 3), (3, 1, 2, 2, 2)]
    assert all(m.all() for m in masks)
    loss = O.ms_gradient_loss(gt, gt + 0.0)
    assert loss.item() == 0.0


def test_loss_is_the_sum_of_the_levels_means():
    g = torch.Generator().manual_seed(3)
    gt, pred = torch.rand(2, 1, 12, 10, generator=g).double(), torch.rand(2, 1, 12, 10, generator=g).double()
    want = sum((spatial_gradient(p) - spatial_gradient(q)).abs().mean()
               for p, q in zip(O.pyrdown(pred, 3), O.pyrdown(gt, 3)))
    assert abs(O.ms_gradient_loss(gt, pred, 3) - want) <= 1e-14


def test_an_empty_level_gives_nan_and_a_finite_gradient():
    gt = torch.rand(1, 1, 5, 4)
    gt[0, 0, 2, 1] = float("nan")                                     # reaches every value of the 2x1 and 1x1 levels
    counts = [int(m.sum()) for m in O.level_masks(gt, 4)]
    assert counts[0] > 0 and counts[-1] == 0
    pred = torch.rand(1, 1, 5, 4, requires_grad=True)
    loss = O.ms_gradient_loss(gt, pred)
    assert torch.isnan(loss)
    loss.backward()
    assert torch.isfinite(pred.grad).all() and pred.grad.abs().max() > 0


def test_scale_invariant_loss():
    d = torch.tensor([0.5, -0.25, 1.0], dtype=torch.float64)
    want = math.sqrt((d ** 2).mean().item() - 0.85 * d.mean().item() ** 2)
    assert abs(O.scale_invariant_loss(d, torch.zeros(3, dtype=torch.float64)).item() - want) <= 1e-15
    assert torch.isnan(O.scale_invariant_loss(torch.empty(0), torch.empty(0)))
    assert torch.isnan(O.scale_invariant_loss(torch.ones(4), torch.zeros(4), si_lambda=1.5))   # negative radicand


def test_blur_pool_and_pyrdown_compile_to_torchscript():
    x = torch.rand(2, 1, 9, 7)
    x[0, 0, 3, 3] = float("nan")
    scripted = torch.jit.script(O.pyrdown)
    for a, b in zip(scripted(x, 4), O.pyrdown(x, 4)):
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0))
