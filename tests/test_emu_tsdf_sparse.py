"""CPU: the voxel-block hashed volume (SparseTSDF, DESIGN §4.16) under the host emulation (tests/emu): after the
same frames it reads back bitwise equal to a dense TSDF on the same lattice — values, weights, colours — and
meshes to the same mesh; capacity overflow is an ordinary Python error; the C ABI refuses bad arguments."""
import contextlib
import ctypes as C
import sys
import types

import pytest
import torch

from simplerecon_b200 import _native, tsdf as tsdf_mod
from simplerecon_b200.synthetic import make_color_tsdf_case
from tests import emu
from tests.sparse_tsdf_cases import (assert_meshes_equal, assert_volumes_equal, covering_bounds, fuse_pair,
                                     random_pose_case)


@pytest.fixture()
def emulated(monkeypatch):
    lib = emu.load_or_skip()
    monkeypatch.setattr(_native, "_lib", lib)
    monkeypatch.setattr(tsdf_mod, "_require_cuda", lambda t: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev=None: types.SimpleNamespace(cuda_stream=0))
    real_empty = torch.empty

    def aligned_empty(*size, **kw):
        if kw.get("dtype") is torch.uint8 and len(size) == 1 and isinstance(size[0], int):
            buf = real_empty(size[0] + 256, **kw)
            off = (-buf.data_ptr()) % 256
            return buf[off:off + size[0]]
        return real_empty(*size, **kw)

    monkeypatch.setattr(torch, "empty", aligned_empty)
    return lib


@pytest.mark.parametrize("color,batch", [(False, None), (True, 1)])
def test_room_matches_dense_bitwise(emulated, color, batch):
    voxel = 0.15
    c = make_color_tsdf_case(seed=1, frames=3, voxel_size=voxel, height=24, width=32, color_hw=(30, 40), masked=True)
    b = covering_bounds()
    dense, sparse = fuse_pair(c, b, voxel, color, "cpu", batch=batch, max_blocks=1024)
    assert _native.last_variant() == ("sparse_tsdf_integrate_color_f16" if color else "sparse_tsdf_integrate_f16")
    assert_volumes_equal(dense, sparse, b, min_touched=1000)
    assert_meshes_equal(dense, sparse, color, min_faces=400)


@pytest.mark.parametrize("seed", [0, 1])
def test_random_poses_match_dense_bitwise(emulated, seed):
    voxel = 0.25
    c = random_pose_case(seed, frames=4, height=20, width=28, color_hw=(20, 28), voxel=voxel, box=(0.0, 4.0))
    dense, sparse = fuse_pair(c, c["bounds"], voxel, True, "cpu", batch=2, max_blocks=1024)
    assert_volumes_equal(dense, sparse, c["bounds"], min_touched=200)
    assert_meshes_equal(dense, sparse, True, min_faces=50)


def test_lattice_box_and_repeated_meshing(emulated):
    """to_dense of a box off the origin and smaller than the touched region reads the lattice sub-box; meshing
    twice gives the same mesh and leaves the block count as it was."""
    voxel = 0.15
    c = make_color_tsdf_case(seed=2, frames=2, voxel_size=voxel, height=24, width=32, color_hw=(24, 32))
    b = covering_bounds()
    dense, sparse = fuse_pair(c, b, voxel, False, "cpu", max_blocks=1024)
    n = sparse.allocated_blocks
    m1 = sparse.extract_mesh()
    m2 = sparse.extract_mesh(single_mesh=True)
    m3 = sparse.extract_mesh()
    assert sparse.allocated_blocks == n and all(torch.equal(a, b_) for a, b_ in zip(m1, m3))
    sub = {"xmin": 1.0, "xmax": 2.5, "ymin": 0.55, "ymax": 1.6, "zmin": -0.3, "zmax": 1.0}
    box = sparse.to_dense(sub)
    lo = [int(torch.floor((torch.tensor(sub[a + "min"], dtype=torch.float32) - dense.origin[i]) / voxel + 1e-6))
          for i, a in enumerate("xyz")]
    X, Y, Z = box.tsdf_values.shape
    ref = dense.tsdf_values[lo[0]:lo[0] + X, lo[1]:lo[1] + Y, lo[2]:lo[2] + Z]
    assert torch.equal(box.tsdf_values, ref) and int((box.tsdf_weights > 0).sum()) > 50
    assert len(m2[1]) > 0


def test_capacity_overflow_raises_at_host_visible_points(emulated, tmp_path, monkeypatch):
    monkeypatch.setitem(sys.modules, "trimesh", types.SimpleNamespace(Trimesh=lambda **kw: kw))
    voxel = 0.15
    c = make_color_tsdf_case(seed=3, frames=2, voxel_size=voxel, height=24, width=32, color_hw=(24, 32))
    _, full = fuse_pair(c, covering_bounds(), voxel, False, "cpu", max_blocks=1024)
    need = full.allocated_blocks
    small = tsdf_mod.SparseTSDF.from_bounds(covering_bounds(), voxel, device="cpu", max_blocks=need // 3)
    tsdf_mod.TSDFFuser(small, max_depth=c["max_depth"]).integrate_depth(c["depth"], c["cam_T_world"], c["K"])
    assert small.header()[_native.SPARSE_HDR_BLOCKS] == need          # the counter kept counting: the size needed
    for call in (small.extract_mesh, small.to_mesh, lambda: small.save(str(tmp_path), "m.bin"),
                 lambda: small.to_dense(covering_bounds())):
        with pytest.raises(tsdf_mod.SparseCapacityError, match=f"max_blocks >= {need}") as e:
            call()
        assert e.value.needed == need
    # room for the volume but not for the mesh's boundary blocks
    tight = tsdf_mod.SparseTSDF.from_bounds(covering_bounds(), voxel, device="cpu", max_blocks=need)
    tsdf_mod.TSDFFuser(tight, max_depth=c["max_depth"]).integrate_depth(c["depth"], c["cam_T_world"], c["K"])
    tight.to_dense(covering_bounds())
    with pytest.raises(tsdf_mod.SparseCapacityError, match="boundary blocks"):
        tight.extract_mesh()
    assert tight.header()[:2] == [need, 0]                          # the volume itself is still whole


def test_argument_checks(emulated):
    lib = emulated
    voxel = 0.1
    c = make_color_tsdf_case(seed=4, frames=1, voxel_size=voxel, height=24, width=32, color_hw=(24, 32))
    plain = tsdf_mod.SparseTSDF(voxel, device="cpu", max_blocks=64)
    colored = tsdf_mod.SparseTSDF(voxel, device="cpu", max_blocks=64, color=True)
    assert torch.equal(plain.origin, torch.tensor([-10.0, -10.0, -10.0]))
    with pytest.raises(ValueError, match="without colour"):
        tsdf_mod.TSDFFuser(plain).integrate_depth(c["depth"], c["cam_T_world"], c["K"], color_b3hw=c["color"])
    with pytest.raises(ValueError, match="needs color_b3hw"):
        tsdf_mod.TSDFFuser(colored).integrate_depth(c["depth"], c["cam_T_world"], c["K"])
    with pytest.raises(ValueError, match="with_colors"):
        plain.extract_mesh(with_colors=True)
    with pytest.raises(ValueError, match="max_blocks"):
        tsdf_mod.SparseTSDF(voxel, device="cpu", max_blocks=0)
    d = plain._desc()
    assert lib.srcv_sparse_tsdf_reset(None, None) == 1
    bad = _native.SparseTsdf.from_buffer_copy(d)
    bad.state = d.state + 8
    assert lib.srcv_sparse_tsdf_reset(C.byref(bad), None) == 4
    bad = _native.SparseTsdf.from_buffer_copy(d)
    bad.voxel_size = 0.0
    assert lib.srcv_sparse_tsdf_reset(C.byref(bad), None) == 2
    assert lib.srcv_sparse_tsdf_mesh_begin(C.byref(d), 65, None) == 2
    lo, dims = (C.c_int32 * 3)(0, 0, 0), (C.c_int32 * 3)(0, 4, 4)
    out = torch.empty(64, dtype=torch.float16)
    assert lib.srcv_sparse_tsdf_read_box(C.byref(d), lo, dims, C.c_void_p(out.data_ptr()),
                                         C.c_void_p(out.data_ptr()), None, None) == 2
    col = torch.empty(3 * 64)
    dims = (C.c_int32 * 3)(4, 4, 4)
    assert lib.srcv_sparse_tsdf_read_box(C.byref(d), lo, dims, C.c_void_p(out.data_ptr()), C.c_void_p(out.data_ptr()),
                                         C.c_void_p(col.data_ptr()), None) == 4        # no colour planes
    n0 = lib.srcv_launch_count()
    tsdf_mod.TSDFFuser(plain).integrate_depth(c["depth"], c["cam_T_world"], c["K"])
    assert lib.srcv_launch_count() - n0 == 4
