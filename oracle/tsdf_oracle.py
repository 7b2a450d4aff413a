"""CPU restatement of the reference's dense-grid TSDF integration — TEST INFRASTRUCTURE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this.

Follows ``TSDFFuser.integrate_depth`` / ``project_to_camera`` of the reference
(tools/tsdf.py:221-320, :204-219) as it is driven by ``OurFuser.fuse_frames``
(tools/fusers_helper.py:64-71): depth maps, intrinsics and extrinsics arrive as **fp16** and
the whole update runs in fp16 tensors, i.e. every elementwise op rounds its result to half
(PyTorch evaluates a half op in fp32 and rounds once).  The restatement spells that rounding
out — ``r16`` after every operation, in the reference's operation order — so that the CUDA
kernel has an exact arithmetic to match; it is pinned bit-for-bit against the imported
reference class in tests/test_tsdf_oracle_vs_reference.py.

Volume layout: (X, Y, Z) half arrays, z fastest, as TSDF.from_bounds builds them
(tools/tsdf.py:70-97).  Batched frames are applied one after the other (:298).
"""
from __future__ import annotations

import numpy as np
import torch

VOX_MOD = 8            # tools/tsdf.py:17
TRUNCATION_VOXELS = 3.0  # TSDFFuser.truncation_size, :181
MAX_W = 100.0          # TSDFFuser.maxW, :182


def r16(x: torch.Tensor) -> torch.Tensor:
    """round to fp16, keep computing in fp32 (what a half op in PyTorch does)"""
    return x.half().float()


def volume_dims(bounds: dict, voxel_size: float):
    """tools/tsdf.py:78-83: voxel counts rounded up to multiples of 8."""
    return tuple(int(np.ceil((bounds[a + "max"] - bounds[a + "min"]) / voxel_size / VOX_MOD)) * VOX_MOD
                 for a in "xyz")


def voxel_coords(origin: torch.Tensor, dims, voxel_size: float, lo=(0, 0, 0)) -> torch.Tensor:
    """(3,X,Y,Z) fp16 world coordinates: origin + index * voxel_size evaluated in fp32, then
    .half() (tools/tsdf.py:99-110, :92).  ``lo`` offsets the indices: the box of lattice indices
    lo .. lo + dims - 1 of the lattice at ``origin`` (any sign; a SparseTSDF's lattice is unbounded)."""
    grid = torch.meshgrid([torch.arange(l, l + d) for l, d in zip(lo, dims)], indexing="ij")
    return (origin.float().view(3, 1, 1, 1) + torch.stack(grid, 0) * voxel_size).half()


def new_volume(bounds: dict, voxel_size: float):
    """(tsdf_values, tsdf_weights, origin): -1 / 0 initialised (tools/tsdf.py:94-95)."""
    dims = volume_dims(bounds, voxel_size)
    origin = torch.tensor([bounds["xmin"], bounds["ymin"], bounds["zmin"]], dtype=torch.float32)
    return (-torch.ones(dims, dtype=torch.float16), torch.zeros(dims, dtype=torch.float16), origin)


def project(K_b44: torch.Tensor, cam_T_world_b44: torch.Tensor, coords_3xyz: torch.Tensor):
    """tools/tsdf.py:204-219 in fp16: P = (K @ E)[:, :3] rounded to half; cam = P @ (x,y,z,1)
    accumulated in fp32 over k = 0..3 and rounded to half; x, y divided by z (half)."""
    Kf, Ef = K_b44.half().float(), cam_T_world_b44.half().float()
    P = r16(torch.matmul(Kf, Ef))[:, :3]                                   # :211
    pts = torch.cat([coords_3xyz.float().reshape(3, -1), torch.ones(1, coords_3xyz[0].numel())], 0)
    cam = r16(torch.einsum("bik,kn->bin", P, pts))                        # :216 (fp32 accumulation, one rounding)
    xy = r16(cam[:, :2] / cam[:, 2:3])                                     # :217
    return xy, cam[:, 2:3]


def sample_nearest(depth_b1hw: torch.Tensor, xy_b2N: torch.Tensor):
    """:249-263: 2 p / size - 1 in half, then grid_sample(nearest, zeros, align_corners=False),
    whose index arithmetic also runs in half for a half grid: ((g + 1) size - 1) / 2, each op
    rounded, then round-half-to-even."""
    B, _, H, W = depth_b1hw.shape
    size = torch.tensor([W, H], dtype=torch.float32).view(1, 2, 1)
    g = r16(r16(r16(2.0 * xy_b2N) / size) - 1.0)                           # :249
    ix = r16(r16(r16(r16(g + 1.0) * size) - 1.0) / 2.0)
    ix = torch.round(ix)                                                   # nearbyint: half to even
    x, y = ix[:, 0], ix[:, 1]
    ok = (x >= 0) & (x <= W - 1) & (y >= 0) & (y <= H - 1)
    xi = x.clamp(0, W - 1).long()
    yi = y.clamp(0, H - 1).long()
    flat = depth_b1hw.float().reshape(B, H * W)
    out = torch.gather(flat, 1, yi * W + xi)
    return torch.where(ok, out, torch.zeros_like(out)).unsqueeze(1)        # zeros padding


def overflow_voxels(origin: torch.Tensor, dims, voxel_size: float, cam_T_world_b44, K_b44, hw) -> torch.Tensor:
    """(X,Y,Z) bool: voxels whose normalised sampling coordinate overflows fp16 (|x / z| > 65504:
    voxels next to a camera's principal plane) in ANY frame of the batch.  grid_sample's
    float -> integer conversion of an infinite coordinate is undefined behaviour: the reference
    run on a CPU returns pixel (0,0) there, the reference run on a GPU (use_gpu=True, its default)
    saturates to an out-of-range index and returns the zeros padding.  The oracle and the kernel
    take the padding (the GPU behaviour); comparisons against a CPU run of the reference exclude
    these voxels."""
    xy, _ = project(K_b44, cam_T_world_b44, voxel_coords(origin, dims, voxel_size))
    H, W = hw
    size = torch.tensor([W, H], dtype=torch.float32).view(1, 2, 1)
    g = r16(r16(r16(2.0 * xy) / size) - 1.0)
    return (~torch.isfinite(g)).any(1).any(0).reshape(dims)


def integrate(tsdf_values: torch.Tensor, tsdf_weights: torch.Tensor, origin: torch.Tensor, voxel_size: float,
              depth_b1hw: torch.Tensor, cam_T_world_b44: torch.Tensor, K_b44: torch.Tensor,
              depth_mask_b1hw: torch.Tensor | None = None, min_depth: float = 0.5, max_depth: float = 5.0,
              lo=(0, 0, 0)):
    """In-place update of (tsdf_values, tsdf_weights) (fp16, (X,Y,Z)) with a batch of depth maps.
    tools/tsdf.py:221-320.  ``lo``: the volume holds lattice indices lo .. lo + dims - 1 (voxel_coords)."""
    dims = tuple(tsdf_values.shape)
    coords = voxel_coords(origin, dims, voxel_size, lo)
    trunc = TRUNCATION_VOXELS * voxel_size                                 # :200-202
    depth = depth_b1hw.half()
    if depth_mask_b1hw is not None:                                        # :251-253
        depth = depth.clone()
        depth[~depth_mask_b1hw] = -1
    xy, vz = project(K_b44, cam_T_world_b44, coords)                       # :240-242
    ds = sample_nearest(depth, xy)                                         # :256-261
    # A python scalar meeting a half tensor: ARITHMETIC keeps the scalar in fp32 (PyTorch evaluates
    # reduced-precision binary ops with a scalar operand in the op-math type, CPU and CUDA alike),
    # COMPARISONS cast it to half first.
    f = lambda v: float(torch.tensor(v, dtype=torch.float32))
    h = lambda v: float(torch.tensor(v, dtype=torch.float16))
    conf = r16(torch.clamp(r16(1.0 - r16(r16(ds - f(min_depth)) / f(max_depth - min_depth))), 0.0, 1.0) ** 2)  # :264-266
    dist = r16(ds - vz)                                                    # :269
    tv = torch.clamp(r16(dist / f(trunc)), -1.0, 1.0)                      # :270
    valid = (vz > 0) & (dist > -h(trunc)) & (ds > 0) & (vz < h(max_depth)) & (conf > 0)   # :273-275
    tvals = tsdf_values.reshape(-1)
    wvals = tsdf_weights.reshape(-1)
    for b in range(depth.shape[0]):                                        # :298 sequential over the batch
        m = valid[b, 0]
        old_t, old_w = tvals[m].float(), wvals[m].float()
        new_t, c = tv[b, 0][m], conf[b, 0][m]
        rate = torch.where(c < old_w, torch.tensor(2.0), torch.tensor(5.0))  # :310
        new_w = r16(r16(c * rate) / MAX_W)                                 # :313
        total = r16(old_w + new_w)                                         # :314
        tvals[m] = r16(r16(r16(old_t * old_w) + r16(new_t * new_w)) / total).half()   # :317
        wvals[m] = torch.clamp(total, max=1.0).half()                      # :318
    return tsdf_values, tsdf_weights
