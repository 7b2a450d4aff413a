"""Shared by the SparseTSDF edge tests (tests/test_emu_tsdf_sparse_edges.py, tests/test_gpu_tsdf_sparse_edges.py): the
volume at any lattice offset, next to tests/sparse_tsdf_cases.py's same-lattice builders.

With voxel_size = 2^-k and origins that are multiples of it, origin + i * voxel_size is exact in fp32 for every
|i| < 2^24 whose result is representable.  A SparseTSDF at origin o_s and a dense TSDF at o_d = o_s + L * voxel_size
then compute the same world coordinates, so sparse voxel i is dense voxel i - L, bit for bit.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from simplerecon_b200 import tsdf as tsdf_mod

KEY_BIAS = 1 << 20            # block coordinates -2^20 .. 2^20 - 1 pack into the 21-bit keys (srcv_block_hash.cuh)
BLOCK_LO, BLOCK_HI = -KEY_BIAS + 1, KEY_BIAS - 1    # the allocatable blocks: meshing packs the block below each one


def lattice_shift(dense_origin, sparse_origin, voxel: float) -> np.ndarray:
    """The shift with dense index = sparse index + shift, (sparse_origin - dense_origin) / voxel; asserts that the
    two origins lie on one lattice exactly."""
    d = (np.asarray(sparse_origin, np.float64) - np.asarray(dense_origin, np.float64)) / voxel
    L = np.rint(d).astype(np.int64)
    assert np.array_equal(d, L.astype(np.float64)), (dense_origin, sparse_origin, voxel)
    return L


def translate_case(c: dict, T) -> dict:
    """The same scene moved by T in the world: every camera moved with it (extrinsics rebuilt in fp64, stored in
    fp32 as the cases store them), ``bounds`` moved too when the case has them."""
    T = torch.as_tensor(T, dtype=torch.float64)
    E = c["cam_T_world"].double().clone()
    E[:, :3, 3] = E[:, :3, 3] - (E[:, :3, :3] @ T)
    out = dict(c, cam_T_world=E.float())
    if "bounds" in c:
        out["bounds"] = {k: v + float(T["xyz".index(k[0])]) for k, v in c["bounds"].items()}
    return out


def snap_bounds(bounds: dict, voxel: float) -> dict:
    """``bounds`` widened to multiples of ``voxel``: a dense origin on every power-of-two lattice of that pitch."""
    return {k: float((np.floor if k.endswith("min") else np.ceil)(v / voxel) * voxel) for k, v in bounds.items()}


def integrate_chunks(fuser, c: dict, device, color: bool, chunks) -> None:
    """Feed the case's frames to ``fuser`` in order, ``chunks`` frames per integrate_depth call."""
    b0 = 0
    for n in chunks:
        sl = slice(b0, b0 + n)
        args = [c["depth"][sl].to(device), c["cam_T_world"][sl].to(device), c["K"][sl].to(device),
                c["mask"][sl].to(device) if c.get("mask") is not None else None]
        kw = dict(color_b3hw=c["color"][sl].to(device)) if color else {}
        fuser.integrate_depth(*args, **kw)
        b0 += n
    assert b0 == c["depth"].shape[0]


def fuse_shifted(c: dict, bounds: dict, voxel: float, color: bool, device, sparse_origin, chunks=None,
                 max_blocks=1 << 14, max_depth=None):
    """(dense over ``bounds``, sparse at ``sparse_origin``) after the same frames; the dense volume gets them all in
    one call, the sparse one in ``chunks`` (one call if None)."""
    dense = tsdf_mod.TSDF.from_bounds(bounds, voxel, device=device, color=color)
    sparse = tsdf_mod.SparseTSDF(voxel, origin=list(sparse_origin), device=device, color=color, max_blocks=max_blocks)
    md = c["max_depth"] if max_depth is None else max_depth
    n = c["depth"].shape[0]
    integrate_chunks(tsdf_mod.TSDFFuser(dense, max_depth=md), c, device, color, [n])
    integrate_chunks(tsdf_mod.TSDFFuser(sparse, max_depth=md), c, device, color, chunks or [n])
    return dense, sparse


def hash_slots(max_blocks: int) -> int:
    """The hash table's size for max_blocks (sparse_hash_slots in srcv_tsdf_sparse.cuh)."""
    h = 1024
    while h < 2 * max_blocks:
        h <<= 1
    return h


def block_coords(sparse) -> np.ndarray:
    """(n, 3) int: the coordinates of the allocated blocks, read from the state (header, keys, slots, coords; each
    section 256-byte aligned, as carve_sparse lays them out)."""
    al = lambda n: (n + 255) // 256 * 256
    H = hash_slots(sparse.max_blocks)
    off = 256 + al(8 * H) + al(4 * H)
    n = sparse.allocated_blocks
    return sparse.state[off:off + 16 * n].view(torch.int32).reshape(n, 4)[:, :3].cpu().numpy().astype(np.int64)


def read_box_raw(sparse, lo, dims):
    """(values, weights) of the lattice box at ``lo`` straight from the C ABI, without the header check that
    ``to_dense`` makes first: the read-back of a volume whose range flag is up."""
    lib = tsdf_mod._native.load()
    dev = sparse.state.device
    values = torch.empty(tuple(dims), dtype=torch.float16, device=dev)
    weights = torch.empty(tuple(dims), dtype=torch.float16, device=dev)
    with torch.cuda.device(dev):
        tsdf_mod._native.check(lib.srcv_sparse_tsdf_read_box(
            C.byref(sparse._desc()), (C.c_int32 * 3)(*map(int, lo)), (C.c_int32 * 3)(*map(int, dims)),
            C.c_void_p(values.data_ptr()), C.c_void_p(weights.data_ptr()), None, sparse._stream()))
    return values, weights


def boundary_blocks(sparse) -> int:
    """How many boundary blocks meshing inserts: mesh_begin, the header, mesh_end (the volume is left as it was)."""
    lib = tsdf_mod._native.load()
    n = sparse.allocated_blocks
    desc = sparse._desc()
    with torch.cuda.device(sparse.state.device):
        tsdf_mod._native.check(lib.srcv_sparse_tsdf_mesh_begin(C.byref(desc), n, sparse._stream()))
        total = sparse.header()[tsdf_mod._native.SPARSE_HDR_BLOCKS]
        tsdf_mod._native.check(lib.srcv_sparse_tsdf_mesh_end(C.byref(desc), n, sparse._stream()))
    assert sparse.header()[:3] == [n, 0, 0]
    return total - n


def oracle_box(c: dict, origin, voxel: float, lo, dims, color: bool, max_depth: float):
    """oracle.tsdf_oracle / color_oracle after all of the case's frames, on the lattice box of indices lo .. lo + dims
    - 1 of the lattice at ``origin``: (values, weights, colours or None), CPU."""
    from oracle import color_oracle, tsdf_oracle
    values = -torch.ones(tuple(dims), dtype=torch.float16)
    weights = torch.zeros(tuple(dims), dtype=torch.float16)
    o = torch.as_tensor(origin, dtype=torch.float32)
    mask = c["mask"].bool() if c.get("mask") is not None else None
    if color:
        colors = torch.zeros((3, *dims), dtype=torch.float32)
        color_oracle.integrate(values, weights, colors, o, voxel, c["depth"], c["cam_T_world"], c["K"], c["color"],
                               mask, max_depth=max_depth, lo=tuple(lo))
        return values, weights, colors
    tsdf_oracle.integrate(values, weights, o, voxel, c["depth"], c["cam_T_world"], c["K"], mask, max_depth=max_depth,
                          lo=tuple(lo))
    return values, weights, None


def _mesh_arrays(mesh):
    a = [t.detach().cpu().numpy() for t in mesh]
    records = np.concatenate([a[2].astype(np.float32).view(np.int32)] +
                             ([a[3].astype(np.float32).view(np.int32)] if len(a) > 3 else []), 1)
    return a[0].astype(np.float64), a[1].astype(np.int64), records


def _canonical_faces(rank: np.ndarray, faces: np.ndarray) -> np.ndarray:
    f = rank[faces].reshape(-1, 3)
    r = np.argmin(f, 1)
    f = np.stack([f[np.arange(len(f)), (r + k) % 3] for k in range(3)], 1)       # rotated, orientation kept
    return f[np.lexsort(f.T[::-1])]


def assert_meshes_match_shifted(md, ms, shift, positions: bool = True, ulps: float = 4.0) -> None:
    """The sparse mesh ``ms`` equals the dense mesh ``md`` on a lattice shifted by ``shift`` (dense index = sparse
    index + shift), both in voxel coordinates (scale_to_world=False).

    Faces, normals and colours depend only on the volume's values, so they must match exactly.  A vertex position
    is fl(x + t) at lattice coordinate x, so the two differ by the rounding at each one's x: after the shift a
    sparse vertex must lie within ``ulps`` ulp of |x| + 1 (of both meshes) of a dense vertex with the same normal
    and colour bits, and the faces through that matching must be the dense faces.  ``positions=False`` is for
    |x| near 2^23, where fp32 keeps no sub-voxel position: the normals and colours as multisets, the faces as
    triples of them, and each coordinate's sorted positions within one ulp."""
    vd, fd, rd = _mesh_arrays(md)
    vs, fs, rs = _mesh_arrays(ms)
    assert len(vd) == len(vs) and len(fd) == len(fs) and rd.shape == rs.shape
    assert np.array_equal(rd[np.lexsort(rd.T[::-1])], rs[np.lexsort(rs.T[::-1])])
    ps = vs + np.asarray(shift, np.float64)
    if not positions:
        both = np.unique(np.concatenate([rd, rs]), axis=0, return_inverse=True)[1].reshape(-1)
        assert np.array_equal(_canonical_faces(both[:len(rd)], fd), _canonical_faces(both[len(rd):], fs))
        tol = np.spacing(np.abs(vs).astype(np.float32).max(0) + 1).astype(np.float64) + 1e-3
        for a in range(3):
            assert np.abs(np.sort(ps[:, a]) - np.sort(vd[:, a])).max() <= tol[a], a
        return
    from scipy.spatial import cKDTree
    tol = ulps * (np.spacing(np.abs(vs).astype(np.float32) + 1).astype(np.float64) +
                  np.spacing(np.abs(vd).astype(np.float32).max() + 1))
    k = min(8, len(vd))
    _, idx = cKDTree(vd).query(ps, k=k, distance_upper_bound=float(tol.max()) * 2)
    idx = idx.reshape(len(ps), k)
    found = idx < len(vd)
    cand = np.where(found, idx, 0)
    ok = found & np.all(np.abs(vd[cand] - ps[:, None]) <= tol[:, None], -1) & np.all(rd[cand] == rs[:, None], -1)
    assert ok.any(1).all(), f"{int((~ok.any(1)).sum())} of {len(vs)} sparse vertices have no dense match"
    match = cand[np.arange(len(cand)), np.argmax(ok, 1)]
    key = np.concatenate([vd.astype(np.float32).view(np.int32), rd], 1)
    rank = np.unique(key, axis=0, return_inverse=True)[1].reshape(-1)       # equal records, equal rank
    assert np.array_equal(_canonical_faces(rank, fd), _canonical_faces(rank[match], fs))


def assert_shifted_meshes_equal(dense, sparse, shift, color: bool, min_faces: int = 100, positions: bool = True):
    """assert_meshes_match_shifted for single_mesh False and True, with colours when the volumes have them."""
    for single in (False, True):
        for with_colors in ((False, True) if color else (False,)):
            md = dense.extract_mesh(scale_to_world=False, single_mesh=single, with_colors=with_colors)
            ms = sparse.extract_mesh(scale_to_world=False, single_mesh=single, with_colors=with_colors)
            assert len(md[1]) >= (1 if single else min_faces), (single, len(md[1]))
            assert_meshes_match_shifted(md, ms, shift, positions=positions)
