"""GPU: the voxel-block hashed volume (SparseTSDF, DESIGN §4.16) on an H100 — bitwise equal to a dense TSDF on the
same lattice after the same frames (values, weights, colours) and the same mesh, on the synthetic room and on
random poses whose frusta leave the room, overlap only partly and cross the image border and max_depth; no host
synchronisation while integrating; capacity overflow as a Python error; the allocation bounded by the frusta."""
import math

import pytest
import torch

import simplerecon_b200 as S
from simplerecon_b200 import _native, tsdf as tsdf_mod
from simplerecon_b200.synthetic import make_color_tsdf_case
from tests.sparse_tsdf_cases import (assert_meshes_equal, assert_volumes_equal, covering_bounds, fuse_pair,
                                     random_pose_case)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("color,batch,frames", [(False, None, 6), (True, None, 6), (False, 1, 4), (True, 2, 18)])
def test_room_matches_dense_bitwise(cuda_device, color, batch, frames):
    voxel = 0.04
    c = make_color_tsdf_case(seed=41, frames=frames, voxel_size=voxel, height=96, width=128, color_hw=(144, 192),
                             masked=True)
    b = covering_bounds()
    dense, sparse = fuse_pair(c, b, voxel, color, cuda_device, batch=batch, max_blocks=1 << 15)
    assert_volumes_equal(dense, sparse, b, min_touched=50000)
    assert_meshes_equal(dense, sparse, color, min_faces=20000)


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("color", [False, True])
def test_random_poses_match_dense_bitwise(cuda_device, seed, color):
    voxel = 0.05
    c = random_pose_case(seed, frames=5, height=72, width=96, color_hw=(72, 96), voxel=voxel)
    dense, sparse = fuse_pair(c, c["bounds"], voxel, color, cuda_device, batch=2 if seed else None,
                              max_blocks=1 << 16)
    assert_volumes_equal(dense, sparse, c["bounds"], min_touched=5000)
    assert_meshes_equal(dense, sparse, color, min_faces=1000)


def test_integrate_does_not_synchronise(cuda_device):
    c = make_color_tsdf_case(seed=42, frames=4, voxel_size=0.04, height=96, width=128, color_hw=(96, 128))
    g = {k: (v.to(cuda_device) if torch.is_tensor(v) else v) for k, v in c.items()}
    plain = S.SparseTSDF(0.04, max_blocks=1 << 14)
    colored = S.SparseTSDF(0.04, max_blocks=1 << 14, color=True)
    fp, fc = S.TSDFFuser(plain, max_depth=3.0), S.TSDFFuser(colored, max_depth=3.0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(2):
            fp.integrate_depth(g["depth"], g["cam_T_world"], g["K"], g["mask"])
            fc.integrate_depth(g["depth"], g["cam_T_world"], g["K"], g["mask"], color_b3hw=g["color"])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert plain.allocated_blocks == colored.allocated_blocks > 0


def test_capacity_overflow_is_a_python_error(cuda_device):
    c = make_color_tsdf_case(seed=43, frames=4, voxel_size=0.04, height=96, width=128, color_hw=(96, 128))
    g = {k: (v.to(cuda_device) if torch.is_tensor(v) else v) for k, v in c.items()}
    full = S.SparseTSDF(0.04, max_blocks=1 << 15)
    S.TSDFFuser(full, max_depth=3.0).integrate_depth(g["depth"], g["cam_T_world"], g["K"])
    need = full.allocated_blocks
    small = S.SparseTSDF(0.04, max_blocks=need // 4)
    S.TSDFFuser(small, max_depth=3.0).integrate_depth(g["depth"], g["cam_T_world"], g["K"])
    with pytest.raises(tsdf_mod.SparseCapacityError, match=f"max_blocks >= {need}"):
        small.to_mesh()
    # the device is fine: the full volume meshes afterwards
    torch.cuda.synchronize()
    assert len(full.extract_mesh()[1]) > 1000


def _frustum_bound(c, voxel, max_depth):
    """Blocks a frame can need, from its frustum alone: the volume of the frustum (0 .. max_depth + trunc, image
    widened by the allocation margins) in block volumes, plus the blocks its surface can cut (area / block face
    times a factor of 3 for the blocks a face crosses diagonally)."""
    K = c["K"][0].double()
    H, W = c["depth"].shape[-2:]
    mx, my = 2 + 0.01 * W + 8, 2 + 0.01 * H + 8
    z = (max_depth * 1.01 + 0.01) + 8 * voxel
    wx, wy = (W + 2 * mx) / K[0, 0] * z, (H + 2 * my) / K[1, 1] * z
    vol = wx * wy * z / 3
    area = wx * wy + 2 * (wx + wy) * math.hypot(z, max(wx, wy) / 2)
    blk = 8 * voxel
    return vol / blk ** 3 + 3 * area / blk ** 2


def test_room_at_2cm_uses_far_less_memory_than_the_dense_cube(cuda_device):
    voxel = 0.02
    c = make_color_tsdf_case(seed=44, frames=8, voxel_size=voxel, height=192, width=256, color_hw=(192, 256))
    g = {k: (v.to(cuda_device) if torch.is_tensor(v) else v) for k, v in c.items()}
    vol = S.SparseTSDF(voxel, max_blocks=1 << 17)
    S.TSDFFuser(vol, max_depth=3.0).integrate_depth(g["depth"], g["cam_T_world"], g["K"])
    n = vol.allocated_blocks
    assert 0 < n <= 8 * _frustum_bound(c, voxel, 3.0)
    dense_bytes = 4 * math.ceil(20.0 / voxel / 8) ** 3 * 8 ** 3        # the ±10 m cube: fp16 value + weight
    assert vol.state.numel() * 4 < dense_bytes                       # the whole state, pool capacity included
    assert n * 8 ** 3 * 4 * 100 < dense_bytes                          # what is allocated: < 1 % of the cube
    assert len(vol.extract_mesh()[1]) > 10000
