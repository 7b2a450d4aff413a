"""Shared by the SparseTSDF tests (CPU emulation and GPU): a dense TSDF and a SparseTSDF on one lattice fed the
same frames, and the comparisons DESIGN §4.16 promises between them."""
from __future__ import annotations

import numpy as np
import torch

from simplerecon_b200 import tsdf as tsdf_mod
from simplerecon_b200.synthetic import _axis_angle, make_color_tsdf_case


def covering_bounds(room=(4.0, 3.0, 2.6), pad=0.6) -> dict:
    """Bounds around the synthetic room with a margin wider than the truncation band plus a pixel's footprint:
    every voxel a frame inside the room can update lies inside, with untouched voxels all around."""
    return {"xmin": -pad, "xmax": room[0] + pad, "ymin": -pad, "ymax": room[1] + pad, "zmin": -pad, "zmax": room[2] + pad}


def random_pose_case(seed: int, frames: int, height: int, width: int, color_hw, voxel: float, box=(-1.0, 5.0),
                     max_depth: float = 3.0) -> dict:
    """make_color_tsdf_case with each camera moved to a random place in the cube ``box`` and turned to a random
    orientation: frusta that leave the room, overlap only partly, and cross the image border and max_depth at
    every angle.  The depth maps stay the room's (a different scene per frame is fine for the comparison).
    ``bounds`` covers every frustum up to max_depth plus the truncation band, with a margin."""
    c = make_color_tsdf_case(seed=seed, frames=frames, voxel_size=voxel, height=height, width=width,
                             color_hw=color_hw, masked=True)
    g = torch.Generator().manual_seed(777 + seed)
    Es = []
    for _ in range(frames):
        axis = torch.randn(3, generator=g, dtype=torch.float64)
        R = _axis_angle((axis / axis.norm())[None], torch.rand(1, generator=g, dtype=torch.float64) * 6.28)[0]
        pos = torch.rand(3, generator=g, dtype=torch.float64) * (box[1] - box[0]) + box[0]
        E = torch.eye(4, dtype=torch.float64)
        E[:3, :3] = R.T
        E[:3, 3] = -(R.T @ pos)
        Es.append(E.float())
    reach = max_depth * 1.5 + 4 * voxel
    bounds = {f"{a}{m}": (box[0] - reach if m == "min" else box[1] + reach) for a in "xyz" for m in ("min", "max")}
    return dict(c, cam_T_world=torch.stack(Es), max_depth=max_depth, bounds=bounds)


def fuse_pair(c: dict, bounds: dict, voxel: float, color: bool, device, batch=None, max_blocks=1 << 14,
              max_depth=None):
    """(dense, sparse) after the same frames, in batches of ``batch`` frames (all at once if None)."""
    dense = tsdf_mod.TSDF.from_bounds(bounds, voxel, device=device, color=color)
    sparse = tsdf_mod.SparseTSDF.from_bounds(bounds, voxel, device=device, color=color, max_blocks=max_blocks)
    md = c["max_depth"] if max_depth is None else max_depth
    fd, fs = tsdf_mod.TSDFFuser(dense, max_depth=md), tsdf_mod.TSDFFuser(sparse, max_depth=md)
    n = c["depth"].shape[0]
    step = n if batch is None else batch
    for b0 in range(0, n, step):
        sl = slice(b0, b0 + step)
        args = [c["depth"][sl].to(device), c["cam_T_world"][sl].to(device), c["K"][sl].to(device),
                c["mask"][sl].to(device) if c.get("mask") is not None else None]
        kw = dict(color_b3hw=c["color"][sl].to(device)) if color else {}
        fd.integrate_depth(*args, **kw)
        fs.integrate_depth(*args, **kw)
    return dense, sparse


def assert_volumes_equal(dense, sparse, bounds: dict, min_touched: int = 100) -> None:
    back = sparse.to_dense(bounds)
    assert torch.equal(back.origin, dense.origin) and back.tsdf_values.shape == dense.tsdf_values.shape
    assert int((dense.tsdf_weights > 0).sum()) >= min_touched
    assert torch.equal(back.tsdf_values.view(torch.int16), dense.tsdf_values.view(torch.int16))
    assert torch.equal(back.tsdf_weights.view(torch.int16), dense.tsdf_weights.view(torch.int16))
    if dense.tsdf_colors is not None:
        assert torch.equal(back.tsdf_colors.view(torch.int32), dense.tsdf_colors.view(torch.int32))
    # the dense volume's border is untouched: the comparison covered every voxel any frame updated
    w = dense.tsdf_weights
    assert not bool((w[[0, -1]] > 0).any() or (w[:, [0, -1]] > 0).any() or (w[:, :, [0, -1]] > 0).any())


def canonical_mesh(mesh) -> tuple:
    """Vertex records (position, normal and colour bits) sorted; each face as its three vertex records, rotated to
    start at the smallest (orientation kept), faces sorted.  Records rather than indices: a vertex at an exact
    zero of the volume sits on a lattice point that several edges share, so positions repeat."""
    arrs = [t.detach().cpu().numpy() for t in mesh]
    verts, faces, rest = arrs[0], arrs[1].astype(np.int64), [a for i, a in enumerate(arrs) if i != 1]
    key = np.concatenate([a.astype(np.float32).view(np.int32).reshape(len(verts), -1) for a in rest], 1)
    rank = np.unique(key, axis=0, return_inverse=True)[1].reshape(-1)      # equal records, equal rank
    f = rank[faces].reshape(-1, 3)
    r = np.argmin(f, 1)
    f = np.stack([f[np.arange(len(f)), (r + k) % 3] for k in range(3)], 1)
    return key[np.lexsort(key.T[::-1])], np.unique(key, axis=0), f[np.lexsort(f.T[::-1])]


def assert_meshes_equal(dense, sparse, color: bool, min_faces: int = 100) -> None:
    for single in (False, True):
        for world in (False, True):
            for with_colors in ((False, True) if color else (False,)):
                md = dense.extract_mesh(scale_to_world=world, single_mesh=single, with_colors=with_colors)
                ms = sparse.extract_mesh(scale_to_world=world, single_mesh=single, with_colors=with_colors)
                assert len(md) == len(ms) and len(md[1]) >= (1 if single else min_faces)
                kd, ud, fd = canonical_mesh(md)
                ks, us, fs = canonical_mesh(ms)
                assert np.array_equal(kd, ks) and np.array_equal(ud, us) and np.array_equal(fd, fs), \
                    (single, world, with_colors)
