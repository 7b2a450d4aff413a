"""GPU: colour fusion (DESIGN §4.11) — the colour integration kernel and the vertex-colour pass on an H100,
bit for bit against the float32 oracle at larger sizes, deterministic, and at OurFuser's default 504^3."""
import numpy as np
import pytest
import torch

import simplerecon_b200 as S
from oracle import color_oracle as CO
from simplerecon_b200 import _native
from simplerecon_b200.synthetic import make_color_tsdf_case, room_wall_color

pytestmark = pytest.mark.gpu


def _cuda(c):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in c.items()}


@pytest.mark.parametrize("zcut,color_hw,frames", [(None, (144, 192), 4), (None, (240, 320), 18), (61, (48, 64), 3)])
def test_integrate_matches_oracle_bitwise(cuda_device, zcut, color_hw, frames):
    voxel = 0.05
    c = make_color_tsdf_case(seed=31, frames=frames, voxel_size=voxel, height=96, width=128, color_hw=color_hw,
                             masked=True)
    vol = S.TSDF.from_bounds(c["bounds"], voxel, color=True)
    plain = S.TSDF.from_bounds(c["bounds"], voxel)
    if zcut is not None:
        cut = lambda t: t[..., :zcut].contiguous()
        vol = S.TSDF(cut(vol.tsdf_values), cut(vol.tsdf_weights), voxel, vol.origin, cut(vol.tsdf_colors))
        plain = S.TSDF(cut(plain.tsdf_values), cut(plain.tsdf_weights), voxel, plain.origin)
    g = _cuda(c)
    S.TSDFFuser(vol, max_depth=3.0).integrate_depth(g["depth"], g["cam_T_world"], g["K"], g["mask"], color_b3hw=g["color"])
    assert _native.last_variant() == "tsdf_integrate_color_f16"
    S.TSDFFuser(plain, max_depth=3.0).integrate_depth(g["depth"], g["cam_T_world"], g["K"], g["mask"])
    tv, tw, tc = vol.tsdf_values.cpu().clone(), vol.tsdf_weights.cpu().clone(), vol.tsdf_colors.cpu().clone()
    tv.fill_(-1), tw.zero_(), tc.zero_()
    CO.integrate(tv, tw, tc, vol.origin, voxel, c["depth"], c["cam_T_world"], c["K"], c["color"], c["mask"],
                 max_depth=3.0)
    assert int((tw > 0).sum()) > 10000
    assert torch.equal(vol.tsdf_values.cpu(), plain.tsdf_values.cpu()) and torch.equal(vol.tsdf_weights.cpu(), plain.tsdf_weights.cpu())
    assert torch.equal(vol.tsdf_values.cpu(), tv) and torch.equal(vol.tsdf_weights.cpu(), tw)
    assert torch.equal(vol.tsdf_colors.cpu().view(torch.int32), tc.view(torch.int32))
    for single in (False, True):
        v, f, n, col = vol.extract_mesh(single_mesh=single, with_colors=True)
        pv, pf, pn = plain.extract_mesh(single_mesh=single)
        assert torch.equal(v, pv) and torch.equal(f, pf) and torch.equal(n, pn) and len(f) > 5000
        ref = CO.vertex_colors(tv, tw, tc, single_mesh=single)
        assert np.array_equal(col.cpu().numpy().view(np.int32), ref.view(np.int32))


def test_deterministic(cuda_device):
    c = _cuda(make_color_tsdf_case(seed=32, frames=6, voxel_size=0.04, height=120, width=160, color_hw=(240, 320)))
    outs = []
    for _ in range(2):
        vol = S.TSDF.from_bounds(c["bounds"], 0.04, color=True)
        S.TSDFFuser(vol, max_depth=3.0).integrate_depth(c["depth"], c["cam_T_world"], c["K"], color_b3hw=c["color"])
        outs.append((vol.tsdf_colors.clone(), *vol.extract_mesh(with_colors=True)))
    for x, y in zip(*outs):
        assert torch.equal(x, y)


def test_full_size_volume(cuda_device):
    """OurFuser's default volume (±10 m at 4 cm: 504^3) with colour: 1.54 GB of colour planes."""
    c = _cuda(make_color_tsdf_case(seed=21, frames=8, voxel_size=0.04, height=240, width=320, color_hw=(480, 640),
                                   room=(6.0, 5.0, 3.0)))
    bounds = {k: (-10.0 if k.endswith("min") else 10.0) for k in ("xmin", "xmax", "ymin", "ymax", "zmin", "zmax")}
    vol = S.TSDF.from_bounds(bounds, 0.04, color=True)
    assert vol.tsdf_colors.shape == (3, 504, 504, 504) and vol.tsdf_colors.is_cuda
    assert vol.tsdf_colors.numel() * 4 == 3 * 4 * 504 ** 3
    S.TSDFFuser(vol, max_depth=3.0).integrate_depth(c["depth"], c["cam_T_world"], c["K"], color_b3hw=c["color"])
    v, f, n, col = vol.extract_mesh(with_colors=True)
    pv, pf, pn = S.TSDF(vol.tsdf_values, vol.tsdf_weights, 0.04, vol.origin).extract_mesh()
    assert len(v) == len(pv) and len(f) == len(pf) and len(f) > 100000
    assert bool(((col >= 0) & (col <= 1)).all())
    # the room's walls (6 x 5 x 3 m from the origin) keep their analytic colour
    v1, f1, n1, c1 = vol.extract_mesh(single_mesh=True, with_colors=True)
    rgb, _, edge, line = room_wall_color(v1.cpu().double(), room=(6.0, 5.0, 3.0))
    keep = (edge > 0.08) & (line > 0.08)
    err = (c1.cpu().double()[keep] - rgb[keep]).abs().max(1).values
    assert int(keep.sum()) > 10000 and float((err <= 1e-4).double().mean()) >= 0.9 and float(err.max()) <= 0.1
