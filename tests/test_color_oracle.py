"""CPU: the colour oracle's pixel rule is PyTorch's `nearest` resize followed by the depth pixel's sample
(what Open3DFuser does, tools/fusers_helper.py:127-132), and its values / weights are tsdf_oracle's."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import color_oracle as CO
from oracle import tsdf_oracle as T
from simplerecon_b200.synthetic import make_color_tsdf_case


@pytest.mark.parametrize("hw,chw", [((48, 64), (72, 96)), ((48, 64), (96, 128)), ((48, 64), (24, 32)),
                                    ((48, 64), (37, 53)), ((192, 256), (480, 640))])
def test_colour_pixel_is_nearest_resize(hw, chw):
    H, W = hw
    Hc, Wc = chw
    img = torch.arange(3 * Hc * Wc, dtype=torch.float32).reshape(1, 3, Hc, Wc)
    resized = F.interpolate(img, size=(H, W))
    sy, sx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    cx = torch.clamp(torch.floor(sx * torch.tensor(np.float32(Wc) / np.float32(W))), max=Wc - 1).long()
    cy = torch.clamp(torch.floor(sy * torch.tensor(np.float32(Hc) / np.float32(H))), max=Hc - 1).long()
    assert torch.equal(img[0][:, cy, cx], resized[0])


def test_values_and_weights_are_the_plain_oracles():
    c = make_color_tsdf_case(seed=2, frames=3, voxel_size=0.1, height=48, width=64, color_hw=(60, 80), masked=True)
    tv, tw, origin = T.new_volume(c["bounds"], 0.1)
    pv, pw = tv.clone(), tw.clone()
    tc = torch.zeros((3, *tv.shape))
    CO.integrate(tv, tw, tc, origin, 0.1, c["depth"], c["cam_T_world"], c["K"], c["color"], c["mask"], max_depth=3.0)
    T.integrate(pv, pw, origin, 0.1, c["depth"], c["cam_T_world"], c["K"], c["mask"], max_depth=3.0)
    assert torch.equal(tv, pv) and torch.equal(tw, pw) and int((tw > 0).sum()) > 300
    assert torch.equal(tw > 0, tc.sum(0) > 0)
    assert float(tc.min()) >= 0.0 and float(tc.max()) <= 1.0


def test_imagenet_round_trip():
    """The synthetic frames are ImageNet-normalised; reverse_imagenet_normalize's constants undo it."""
    c = make_color_tsdf_case(seed=3, frames=1, voxel_size=0.2, height=24, width=32, color_hw=(30, 40))
    m = torch.tensor(CO.REVERSE_MEAN).view(1, 3, 1, 1)
    s = torch.tensor(CO.REVERSE_STD).view(1, 3, 1, 1)
    assert (((c["color"] - m) / s) - c["color_raw"]).abs().max() < 1e-6
