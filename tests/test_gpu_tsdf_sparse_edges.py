"""GPU: the voxel-block TSDF (SparseTSDF, DESIGN §4.16) on an H100 where its lattice arithmetic can go wrong:
negative and mixed-sign voxel and block indices, the ends of the 21-bit key range and past them, lattices 100 m to
10 km from the world origin, exact pool capacity, a full hash table, more than 16 frames per call, and ragged, thin
and 2048-pixel-wide images.  Volumes are compared bit for bit with a dense TSDF or the oracle on the same lattice
(tests/sparse_tsdf_edge_cases.py has the shifted-lattice argument), meshes with the dense mesh."""
import numpy as np
import pytest
import torch

from simplerecon_b200 import _native, tsdf as tsdf_mod
from simplerecon_b200.synthetic import make_color_tsdf_case
from tests.sparse_tsdf_cases import (assert_meshes_equal, assert_volumes_equal, covering_bounds, fuse_pair,
                                     random_pose_case)
from tests.sparse_tsdf_edge_cases import (BLOCK_HI, BLOCK_LO, assert_shifted_meshes_equal, block_coords,
                                          boundary_blocks, fuse_shifted, hash_slots, integrate_chunks, lattice_shift,
                                          oracle_box, read_box_raw, snap_bounds, translate_case)

pytestmark = pytest.mark.gpu

ROOM_CENTRE = (2.0, 1.5, 1.3125)


def room(seed=41, frames=6, voxel=0.0625, h=72, w=96, color_hw=(90, 120)):
    return make_color_tsdf_case(seed=seed, frames=frames, voxel_size=voxel, height=h, width=w, color_hw=color_hw,
                                masked=True)


@pytest.mark.parametrize("voxel", [2.0 ** -4, 2.0 ** -5])
@pytest.mark.parametrize("color", [False, True])
def test_mixed_sign_room(cuda_device, voxel, color):
    c = room(voxel=voxel)
    b = covering_bounds(pad=0.625)
    dense, sparse = fuse_shifted(c, b, voxel, color, cuda_device, ROOM_CENTRE, chunks=[2, 4], max_blocks=1 << 16)
    blocks = block_coords(sparse)
    assert (blocks.min(0) < 0).all() and (blocks.max(0) > 0).all()
    assert_volumes_equal(dense, sparse, b, min_touched=20000)
    assert_shifted_meshes_equal(dense, sparse, lattice_shift(dense.origin, ROOM_CENTRE, voxel), color, min_faces=5000)


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("color", [False, True])
def test_mixed_sign_random_poses(cuda_device, seed, color):
    voxel = 2.0 ** -4
    c = random_pose_case(seed, frames=5, height=72, width=96, color_hw=(72, 96), voxel=voxel, box=(-2.0, 2.0))
    b = snap_bounds(c["bounds"], voxel)
    dense, sparse = fuse_shifted(c, b, voxel, color, cuda_device, (0.0, 0.0, 0.0), chunks=[2, 3], max_blocks=1 << 16)
    blocks = block_coords(sparse)
    assert (blocks.min(0) < 0).all() and (blocks.max(0) >= 0).all()
    assert_volumes_equal(dense, sparse, b, min_touched=3000)
    assert_shifted_meshes_equal(dense, sparse, lattice_shift(dense.origin, (0.0, 0.0, 0.0), voxel), color,
                                min_faces=500)


@pytest.mark.parametrize("color", [False, True])
def test_oracle_on_a_negative_box(cuda_device, color):
    """0.04 m voxels: to_dense of a box at negative lattice indices equals the oracle on that box."""
    voxel = 0.04
    c = room(seed=42, frames=3, voxel=voxel, h=48, w=64, color_hw=(48, 64))
    origin = (2.0, 1.5, 1.3)
    sparse = tsdf_mod.SparseTSDF(voxel, origin=list(origin), device=cuda_device, color=color, max_blocks=1 << 15)
    integrate_chunks(tsdf_mod.TSDFFuser(sparse, max_depth=c["max_depth"]), c, cuda_device, color, [3])
    box = sparse.to_dense(covering_bounds())
    lo = np.rint((box.origin.double().numpy() - np.float32(origin)) / np.float32(voxel)).astype(np.int64)
    assert (lo < 0).all()
    v, w, col = oracle_box(c, origin, voxel, lo, box.tsdf_values.shape, color, c["max_depth"])
    assert int((w > 0).sum()) > 20000
    assert torch.equal(box.tsdf_values.cpu().view(torch.int16), v.view(torch.int16))
    assert torch.equal(box.tsdf_weights.cpu().view(torch.int16), w.view(torch.int16))
    if color:
        assert torch.equal(box.tsdf_colors.cpu().view(torch.int32), col.view(torch.int32))
    assert_shifted_meshes_equal(box, sparse, -lo, color, min_faces=5000)


def edge_origin(c, b, voxel, axis, block, low, device):
    """The sparse origin that puts the lowest (``low``) or highest allocated block on ``axis`` at ``block``."""
    _, ref = fuse_pair(c, b, voxel, False, device, max_blocks=1 << 15)
    blocks = block_coords(ref)
    k = block - (blocks[:, axis].min() if low else blocks[:, axis].max())
    o = [b["xmin"], b["ymin"], b["zmin"]]
    o[axis] -= 8 * int(k) * voxel
    return o


@pytest.mark.parametrize("axis,block,low", [(0, BLOCK_LO, True), (1, BLOCK_HI, False), (2, BLOCK_LO, True)])
@pytest.mark.parametrize("color", [False, True])
def test_lattice_edges(cuda_device, axis, block, low, color):
    """Fused blocks at the lowest (highest) allocatable block: bit-for-bit volume, no range flag, and a mesh (at
    |x| near 2^23 fp32 keeps no sub-voxel position, so the normals and face topology, positions to an ulp)."""
    voxel = 2.0 ** -4
    c, b = room(seed=43, frames=4), covering_bounds(pad=0.625)
    o = edge_origin(c, b, voxel, axis, block, low, cuda_device)
    dense, sparse = fuse_shifted(c, b, voxel, color, cuda_device, o, max_blocks=1 << 15)
    blocks = block_coords(sparse)
    assert (blocks[:, axis].min() if low else blocks[:, axis].max()) == block
    assert sparse.header()[_native.SPARSE_HDR_RANGE] == 0
    assert_volumes_equal(dense, sparse, b, min_touched=20000)
    assert_shifted_meshes_equal(dense, sparse, lattice_shift(dense.origin, o, voxel), color, min_faces=5000,
                                positions=False)
    assert sparse.header()[_native.SPARSE_HDR_RANGE] == 0
    assert_volumes_equal(dense, sparse, b, min_touched=20000)


def test_lowest_packable_block_is_refused_at_integration(cuda_device):
    voxel = 2.0 ** -4
    c, b = room(seed=43, frames=4), covering_bounds(pad=0.625)
    o = edge_origin(c, b, voxel, 0, BLOCK_LO - 1, True, cuda_device)
    dense, sparse = fuse_shifted(c, b, voxel, False, cuda_device, o, max_blocks=1 << 15)
    if sparse.header()[_native.SPARSE_HDR_RANGE]:
        with pytest.raises(RuntimeError, match="outside voxel indices"):
            sparse.to_dense(b)
        return
    sparse.extract_mesh(scale_to_world=False)
    assert sparse.header()[_native.SPARSE_HDR_RANGE] == 0


@pytest.mark.parametrize("axis,block,low", [(0, BLOCK_HI + 1, False), (1, BLOCK_LO - 1, True),
                                            (2, BLOCK_LO - 3, True)])
def test_past_the_edges(cuda_device, axis, block, low):
    voxel = 2.0 ** -4
    c, b = room(seed=44, frames=1, h=24, w=32), covering_bounds(pad=0.625)
    o = edge_origin(c, b, voxel, axis, block, low, cuda_device)
    sparse = tsdf_mod.SparseTSDF(voxel, origin=o, device=cuda_device, max_blocks=1 << 15)
    integrate_chunks(tsdf_mod.TSDFFuser(sparse, max_depth=c["max_depth"]), c, cuda_device, False, [1])
    for call in (lambda: sparse.to_dense(b), sparse.extract_mesh, sparse.to_mesh):
        with pytest.raises(RuntimeError, match="outside voxel indices"):
            call()
    blocks = block_coords(sparse)
    assert len(blocks) > 0 and blocks.min() >= BLOCK_LO and blocks.max() <= BLOCK_HI
    lo, hi = 8 * blocks.min(0), 8 * blocks.max(0) + 8
    lo[axis], hi[axis] = (8 * BLOCK_HI, 8 * BLOCK_HI + 8) if low else (-8 * (BLOCK_HI + 1), -8 * BLOCK_HI)
    v, w = read_box_raw(sparse, lo, hi - lo)
    assert bool((v == -1).all()) and bool((w == 0).all())


@pytest.mark.parametrize("far", [100.0, 1000.0, 10000.0])
def test_far_from_the_world_origin(cuda_device, far):
    voxel = 0.0625
    T = (far, -0.7 * far, 0.4 * far)
    c = translate_case(room(seed=45, frames=4, voxel=voxel), T)
    over = translate_case(room(seed=46, frames=1, voxel=voxel), (3e4, 0.0, 0.0))
    c = {k: torch.cat([c[k], over[k]]) if torch.is_tensor(c[k]) else c[k] for k in c}
    P = (c["K"][-1].half().float() @ c["cam_T_world"][-1].half().float()).half()
    assert not bool(torch.isfinite(P[:3]).all())
    pad = 1.0 + far / 2048 * 2
    b = {k: v + T["xyz".index(k[0])] for k, v in covering_bounds(pad=pad).items()}
    dense, sparse = fuse_pair(c, b, voxel, True, cuda_device, max_blocks=1 << 17)
    assert sparse.header()[1:3] == [0, 0]
    # at 10 km every frame's translation overflows fp16 (fx * 10^4 > 65504): nothing is fused, in either volume
    assert_volumes_equal(dense, sparse, b, min_touched=0 if far > 5000 else 5000)


def test_exact_capacity(cuda_device):
    """max_blocks == need fuses bit for bit with the hash table near its 50 % design load; need - 1 names need;
    need + boundary meshes and need + boundary - 1 refuses the mesh but keeps the volume; a one-block pool fills
    the hash table (LOST) and stays an error, also after integrating again."""
    voxel, b = 0.025, covering_bounds()
    best = 0.0
    for seed in range(47, 51):          # the room views whose block count is nearest below a power of two > 1024
        for frames in range(2, 9):
            case = room(seed=seed, frames=frames, voxel=voxel)
            _, probe = fuse_pair(case, b, voxel, False, cuda_device, max_blocks=1 << 16)
            n = probe.allocated_blocks
            if n > 1024 and n / hash_slots(n) > best:
                c, roomy, best = case, probe, n / hash_slots(n)
    need = roomy.allocated_blocks
    assert best > 0.45, (need, best)
    boundary = boundary_blocks(roomy)
    dense, exact = fuse_pair(c, b, voxel, False, cuda_device, max_blocks=need)
    assert exact.header()[:3] == [need, 0, 0]
    assert_volumes_equal(dense, exact, b, min_touched=20000)
    _, short = fuse_pair(c, b, voxel, False, cuda_device, max_blocks=need - 1)
    with pytest.raises(tsdf_mod.SparseCapacityError) as e:
        short.to_dense(b)
    assert e.value.needed == need
    _, meshable = fuse_pair(c, b, voxel, False, cuda_device, max_blocks=need + boundary)
    assert_meshes_equal(dense, meshable, False, min_faces=5000)
    _, tight = fuse_pair(c, b, voxel, False, cuda_device, max_blocks=need + boundary - 1)
    with pytest.raises(tsdf_mod.SparseCapacityError, match="boundary blocks"):
        tight.extract_mesh()
    assert_volumes_equal(dense, tight, b, min_touched=20000)
    _, one = fuse_pair(c, b, voxel, False, cuda_device, max_blocks=1)
    for _ in range(2):
        assert one.header()[_native.SPARSE_HDR_LOST] > 0
        with pytest.raises(tsdf_mod.SparseCapacityError):
            one.to_dense(b)
        integrate_chunks(tsdf_mod.TSDFFuser(one, max_depth=c["max_depth"]), c, cuda_device, False,
                         [c["depth"].shape[0]])
    torch.cuda.synchronize()


@pytest.mark.parametrize("color", [False, True])
def test_more_than_16_frames_per_call(cuda_device, color):
    voxel = 0.0625
    c, b = room(seed=48, frames=33, voxel=voxel, h=48, w=64, color_hw=(60, 80)), covering_bounds(pad=0.625)
    o = [b["xmin"], b["ymin"], b["zmin"]]
    dense, one_call = fuse_shifted(c, b, voxel, color, cuda_device, o, max_blocks=1 << 15)
    assert_volumes_equal(dense, one_call, b, min_touched=20000)
    _, chunked = fuse_shifted(c, b, voxel, color, cuda_device, o, chunks=[1, 16, 16], max_blocks=1 << 15)
    assert_volumes_equal(dense, chunked, b, min_touched=20000)


@pytest.mark.parametrize("h,w,color_hw", [(61, 83, (61, 83)), (1, 96, (3, 100)), (72, 1, (70, 2)),
                                          (48, 2048, (40, 1500)), (61, 83, (200, 300))])
def test_image_shapes(cuda_device, h, w, color_hw):
    """Ragged 8-pixel tiles, one-pixel rows and columns, the 2048-pixel width the margin argument is made for,
    and colour images of another size than the depth."""
    voxel = 0.05
    c = random_pose_case(5, frames=4, height=h, width=w, color_hw=color_hw, voxel=voxel, box=(0.0, 4.0))
    dense, sparse = fuse_pair(c, c["bounds"], voxel, True, cuda_device, batch=3, max_blocks=1 << 17)
    assert_volumes_equal(dense, sparse, c["bounds"], min_touched=50 if min(h, w) == 1 else 3000)
    if min(h, w) > 1:
        assert_meshes_equal(dense, sparse, True, min_faces=300)
