"""CPU: the voxel-block TSDF (SparseTSDF, DESIGN §4.16) under the host emulation (tests/emu) where its lattice
arithmetic can go wrong: negative and mixed-sign voxel and block indices, the ends of the 21-bit key range, volumes
past those ends, lattices far from the world origin, exact pool capacity, a full hash table, and more than 16
frames per call.  Every volume is compared bit for bit with a dense TSDF or the oracle on the same lattice
(tests/sparse_tsdf_edge_cases.py has the shifted-lattice argument), every mesh with the dense mesh."""
import numpy as np
import pytest
import torch

from simplerecon_b200 import _native, tsdf as tsdf_mod
from simplerecon_b200.synthetic import make_color_tsdf_case
from tests.sparse_tsdf_cases import (assert_meshes_equal, assert_volumes_equal, covering_bounds, fuse_pair,
                                     random_pose_case)
from tests.sparse_tsdf_edge_cases import (BLOCK_HI, BLOCK_LO, assert_shifted_meshes_equal, block_coords,
                                          boundary_blocks, fuse_shifted, integrate_chunks, lattice_shift, oracle_box,
                                          read_box_raw, snap_bounds, translate_case)
from tests.test_emu_tsdf_sparse import emulated  # noqa: F401  (the fixture)

ROOM_CENTRE = (2.0, 1.5, 1.25)
# the pool of every volume here: a little above what these scenes need (the emulated reset costs time per pool block)
POOL = 512


def small_room(seed=5, frames=3, voxel=0.125, h=20, w=28):
    return make_color_tsdf_case(seed=seed, frames=frames, voxel_size=voxel, height=h, width=w, color_hw=(h + 4, w - 4),
                                masked=True)


def test_mixed_sign_room(emulated):
    """The sparse origin at the room's centre: voxel and block indices cross zero on all three axes."""
    voxel, color = 2.0 ** -3, True
    c = small_room(voxel=voxel)
    b = covering_bounds(pad=0.625)
    dense, sparse = fuse_shifted(c, b, voxel, color, "cpu", ROOM_CENTRE, max_blocks=POOL)
    blocks = block_coords(sparse)
    assert (blocks.min(0) < 0).all() and (blocks.max(0) > 0).all()
    assert_volumes_equal(dense, sparse, b, min_touched=500)
    assert_shifted_meshes_equal(dense, sparse, lattice_shift(dense.origin, ROOM_CENTRE, voxel), color, min_faces=100)


def test_mixed_sign_random_poses(emulated):
    voxel = 2.0 ** -2
    c = random_pose_case(3, frames=3, height=20, width=28, color_hw=(20, 28), voxel=voxel, box=(-2.0, 2.0),
                         max_depth=2.0)
    b = snap_bounds(c["bounds"], voxel)
    dense, sparse = fuse_shifted(c, b, voxel, True, "cpu", (0.0, 0.0, 0.0), chunks=[2, 1], max_blocks=POOL)
    blocks = block_coords(sparse)
    assert (blocks.min(0) < 0).all() and (blocks.max(0) >= 0).all()
    assert_volumes_equal(dense, sparse, b, min_touched=100)
    assert_shifted_meshes_equal(dense, sparse, lattice_shift(dense.origin, (0.0, 0.0, 0.0), voxel), True, min_faces=20)


def test_oracle_on_a_negative_box(emulated):
    """An ordinary voxel size: to_dense of a box at negative lattice indices equals the oracle on that box."""
    voxel = 0.15
    c = small_room(seed=6, frames=2, voxel=voxel)
    origin = (2.0, 1.5, 1.3)
    sparse = tsdf_mod.SparseTSDF(voxel, origin=list(origin), device="cpu", color=True, max_blocks=POOL)
    integrate_chunks(tsdf_mod.TSDFFuser(sparse, max_depth=c["max_depth"]), c, "cpu", True, [2])
    b = covering_bounds()
    box = sparse.to_dense(b)
    lo = np.rint((box.origin.double().numpy() - np.float32(origin)) / np.float32(voxel)).astype(np.int64)
    assert (lo < 0).all()
    v, w, col = oracle_box(c, origin, voxel, lo, box.tsdf_values.shape, True, c["max_depth"])
    assert int((w > 0).sum()) > 300
    assert torch.equal(box.tsdf_values.view(torch.int16), v.view(torch.int16))
    assert torch.equal(box.tsdf_weights.view(torch.int16), w.view(torch.int16))
    assert torch.equal(box.tsdf_colors.view(torch.int32), col.view(torch.int32))
    assert_shifted_meshes_equal(box, sparse, -lo, True, min_faces=50)


def edge_origin(c, b, voxel, axis: int, block: int, low: bool):
    """The sparse origin that puts the case's lowest (``low``) or highest allocated block on ``axis`` at ``block``:
    the allocation measured with the sparse lattice on the dense one, then shifted by whole blocks (exact at a
    power-of-two voxel size, so the allocation shifts with it)."""
    _, ref = fuse_pair(c, b, voxel, False, "cpu", max_blocks=POOL)
    blocks = block_coords(ref)
    k = block - (blocks[:, axis].min() if low else blocks[:, axis].max())
    o = [b["xmin"], b["ymin"], b["zmin"]]
    o[axis] -= 8 * int(k) * voxel
    return o


def edge_case(voxel=0.125):
    return small_room(seed=7, frames=1, voxel=voxel), covering_bounds(pad=0.625)


@pytest.mark.parametrize("axis,block,low", [(0, BLOCK_LO, True), (1, BLOCK_HI, False)])
def test_lattice_edges(emulated, axis, block, low):
    """The fused blocks reach the lowest (highest) allocatable block on one axis: the volume reads back bit for bit,
    no range flag, and it meshes (voxel coordinates near 2^23: fp32 keeps no sub-voxel position there, so the
    vertices are compared as the normals and the face topology, positions to one ulp) and stays readable."""
    voxel = 0.125
    c, b = edge_case(voxel)
    o = edge_origin(c, b, voxel, axis, block, low)
    dense, sparse = fuse_shifted(c, b, voxel, False, "cpu", o, max_blocks=POOL)
    blocks = block_coords(sparse)
    assert (blocks[:, axis].min() if low else blocks[:, axis].max()) == block
    assert sparse.header()[_native.SPARSE_HDR_RANGE] == 0
    assert_volumes_equal(dense, sparse, b, min_touched=100)
    assert_shifted_meshes_equal(dense, sparse, lattice_shift(dense.origin, o, voxel), False, min_faces=50,
                                positions=False)
    assert sparse.header()[_native.SPARSE_HDR_RANGE] == 0
    assert_volumes_equal(dense, sparse, b, min_touched=100)


def test_lowest_packable_block_is_refused_at_integration(emulated):
    """A block at -2^20 packs, but the boundary block meshing needs below it does not.  Either such a volume
    meshes and stays whole, or the frame is refused when it is integrated; a volume that fused must never raise the
    range error from its first mesh on (and poison every later read)."""
    voxel = 0.125
    c, b = edge_case(voxel)
    o = edge_origin(c, b, voxel, 0, BLOCK_LO - 1, True)
    dense, sparse = fuse_shifted(c, b, voxel, False, "cpu", o, max_blocks=POOL)
    if sparse.header()[_native.SPARSE_HDR_RANGE]:
        with pytest.raises(RuntimeError, match="outside voxel indices"):
            sparse.to_dense(b)
        return
    sparse.extract_mesh(scale_to_world=False)
    assert sparse.header()[_native.SPARSE_HDR_RANGE] == 0


@pytest.mark.parametrize("axis,block,low", [(0, BLOCK_HI + 1, False), (2, BLOCK_LO - 2, True)])
def test_past_the_edges(emulated, axis, block, low):
    """A frame whose frusta straddle the end of the key range raises the range error at the next host-visible
    point; every block that went in is in range, and the blocks a wrapped key would alias (the opposite end of the
    axis) read -1 / 0."""
    voxel = 0.125
    c, b = edge_case(voxel)
    o = edge_origin(c, b, voxel, axis, block, low)
    sparse = tsdf_mod.SparseTSDF(voxel, origin=o, device="cpu", max_blocks=POOL)
    integrate_chunks(tsdf_mod.TSDFFuser(sparse, max_depth=c["max_depth"]), c, "cpu", False, [1])
    for call in (lambda: sparse.to_dense(b), sparse.extract_mesh):
        with pytest.raises(RuntimeError, match="outside voxel indices"):
            call()
    blocks = block_coords(sparse)
    assert len(blocks) > 0 and blocks.min() >= BLOCK_LO and blocks.max() <= BLOCK_HI
    lo, hi = 8 * blocks.min(0), 8 * blocks.max(0) + 8
    lo[axis], hi[axis] = (8 * BLOCK_HI, 8 * BLOCK_HI + 8) if low else (-8 * (BLOCK_HI + 1), -8 * BLOCK_HI)
    v, w = read_box_raw(sparse, lo, hi - lo)
    assert bool((v == -1).all()) and bool((w == 0).all())


@pytest.mark.parametrize("far", [100.0, 1000.0])
def test_far_from_the_world_origin(emulated, far):
    """Cameras and lattice ``far`` metres out on every axis: the fp16 voxel coordinates collapse (their ulp is
    0.06 m at 100 m, 0.5 m at 1 km), and the 2^-10 world margin still covers every voxel the dense volume changes.
    A last frame 30 km out overflows the fp16 projection's translation: it changes no voxel in either volume."""
    voxel = 0.125
    c = translate_case(small_room(seed=8, frames=2, voxel=voxel), (far, -0.7 * far, 0.4 * far))
    over = translate_case(small_room(seed=9, frames=1, voxel=voxel), (3e4, 0.0, 0.0))
    c = {k: torch.cat([c[k], over[k]]) if torch.is_tensor(c[k]) and k != "K" else c[k] for k in c}
    c["K"] = torch.cat([c["K"], over["K"]])
    P = (c["K"][-1].half().float() @ c["cam_T_world"][-1].half().float()).half()
    assert not bool(torch.isfinite(P[:3]).all())
    b = {k: v + (far, -0.7 * far, 0.4 * far)["xyz".index(k[0])] for k, v in covering_bounds(pad=1.5).items()}
    dense, sparse = fuse_pair(c, b, voxel, True, "cpu", max_blocks=POOL)
    assert sparse.header()[1:3] == [0, 0]
    assert_volumes_equal(dense, sparse, b, min_touched=300)


def test_exact_capacity(emulated):
    """max_blocks == need fuses bit for bit with the hash table near its 50 % design load; need - 1 names need;
    need + boundary meshes and need + boundary - 1 refuses the mesh but keeps the volume; a one-block pool is an
    error, also after integrating again (the GPU test fills its hash table)."""
    voxel = 0.125
    c, b = small_room(seed=1, frames=2, voxel=voxel), covering_bounds()
    _, roomy = fuse_pair(c, b, voxel, False, "cpu", max_blocks=POOL)
    need = roomy.allocated_blocks
    boundary = boundary_blocks(roomy)
    dense, exact = fuse_pair(c, b, voxel, False, "cpu", max_blocks=need)
    assert exact.header()[:3] == [need, 0, 0]
    assert_volumes_equal(dense, exact, b, min_touched=500)
    _, short = fuse_pair(c, b, voxel, False, "cpu", max_blocks=need - 1)
    with pytest.raises(tsdf_mod.SparseCapacityError) as e:
        short.to_dense(b)
    assert e.value.needed == need
    _, meshable = fuse_pair(c, b, voxel, False, "cpu", max_blocks=need + boundary)
    assert_meshes_equal(dense, meshable, False, min_faces=100)
    _, tight = fuse_pair(c, b, voxel, False, "cpu", max_blocks=need + boundary - 1)
    with pytest.raises(tsdf_mod.SparseCapacityError, match="boundary blocks"):
        tight.extract_mesh()
    assert_volumes_equal(dense, tight, b, min_touched=500)
    _, one = fuse_pair(c, b, voxel, False, "cpu", max_blocks=1)
    for _ in range(2):
        with pytest.raises(tsdf_mod.SparseCapacityError):
            one.to_dense(b)
        integrate_chunks(tsdf_mod.TSDFFuser(one, max_depth=c["max_depth"]), c, "cpu", False, [2])


def test_more_than_16_frames_per_call(emulated):
    """33 frames in one call (chunks of 16, 16 and 1 inside) and the same frames as 1 + 16 + 16 calls both equal a
    dense volume fed them in one call."""
    voxel = 0.25
    c, b = small_room(seed=2, frames=33, voxel=voxel, h=12, w=16), covering_bounds(pad=1.5)
    dense, one_call = fuse_shifted(c, b, voxel, False, "cpu", [b["xmin"], b["ymin"], b["zmin"]], max_blocks=POOL)
    assert_volumes_equal(dense, one_call, b, min_touched=300)
    _, chunked = fuse_shifted(c, b, voxel, False, "cpu", [b["xmin"], b["ymin"], b["zmin"]], chunks=[1, 16, 16],
                              max_blocks=POOL)
    assert_volumes_equal(dense, chunked, b, min_touched=300)
