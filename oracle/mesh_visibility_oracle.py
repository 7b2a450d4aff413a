"""numpy restatement of the visibility rule of mesh evaluation (csrc/srcv_mesh_visibility.cuh, DESIGN §4.18), and
the same rule as a PyTorch op sequence — test and measurement infrastructure, never imported by the package.

Both evaluate elementwise in fp64 from the fp32 inputs, in the kernel's order, with no matmul (a BLAS sums in its
own order): x = ((E00 px + E01 py) + E02 pz) + E03 (likewise y, z), U = (K00 x + K01 y) + K02 z (likewise V),
ix = rint(U / z - 0.5), iy = rint(V / z - 0.5) rounding half to even; the point is observed when 0 < z < max_depth,
0 <= ix < W, 0 <= iy < H, and d = depth[iy, ix] has 0 < d < max_depth and d - z > -margin.  A frame with a
non-finite entry in E's rows 0..2 or in K[:2, :3] observes nothing."""
from __future__ import annotations

import math

import numpy as np


def _frames(depths, K, cam_T_world):
    d = np.asarray(depths, np.float32)
    if d.ndim == 4:
        d = d[:, 0]
    F = d.shape[0]
    E = np.asarray(cam_T_world, np.float32).astype(np.float64)
    Kd = np.asarray(K, np.float32).astype(np.float64)
    if Kd.ndim == 2:
        Kd = np.broadcast_to(Kd, (F, 4, 4))
    return d, Kd, E


def observation_counts(points, depths, K, cam_T_world, margin: float = 0.05, max_depth: float = math.inf) -> np.ndarray:
    """(N,) int32: the frames that observe each point of ``points`` (N, 3)."""
    p = np.asarray(points, np.float32).astype(np.float64)
    d, Kd, E = _frames(depths, K, cam_T_world)
    F, H, W = d.shape
    px, py, pz = p[:, 0], p[:, 1], p[:, 2]
    counts = np.zeros(len(p), np.int32)
    with np.errstate(all="ignore"):
        for f in range(F):
            e, k = E[f], Kd[f]
            if not (np.isfinite(e[:3]).all() and np.isfinite(k[:2, :3]).all()):
                continue
            x, y, z = (((e[r, 0] * px + e[r, 1] * py) + e[r, 2] * pz) + e[r, 3] for r in range(3))
            U = (k[0, 0] * x + k[0, 1] * y) + k[0, 2] * z
            V = (k[1, 0] * x + k[1, 1] * y) + k[1, 2] * z
            ix = np.rint(U / z - 0.5)
            iy = np.rint(V / z - 0.5)
            ok = (z > 0) & (z < max_depth) & (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
            dd = np.zeros(len(p))
            dd[ok] = d[f, iy[ok].astype(np.int64), ix[ok].astype(np.int64)]
            ok &= (dd > 0) & (dd < max_depth) & ((dd - z) > -margin)
            counts += ok
    return counts


def observation_counts_torch(points, depths, K, cam_T_world, margin: float = 0.05, max_depth: float = math.inf,
                             chunk: int = 1 << 22):
    """The same counts as a PyTorch op sequence on the tensors' device (fp64 elementwise transform, round, gather,
    compare), ``chunk`` points at a time: the baseline the kernel is measured against, and a fast device oracle."""
    import torch
    dev = points.device
    p = points.to(torch.float64)
    d = depths[:, 0] if depths.dim() == 4 else depths
    d = d.to(torch.float32).contiguous()
    F, H, W = d.shape
    E = cam_T_world.to(torch.float32).to(torch.float64)
    Kd = K.to(torch.float32).to(torch.float64)
    if Kd.dim() == 2:
        Kd = Kd.expand(F, 4, 4)
    good = (torch.isfinite(E[:, :3]).flatten(1).all(1) & torch.isfinite(Kd[:, :2, :3]).flatten(1).all(1)).tolist()
    Eh, Kh = E.cpu().tolist(), Kd.cpu().tolist()        # python floats: scalars of the elementwise ops, exact in fp64
    counts = torch.zeros(len(p), dtype=torch.int32, device=dev)
    flat = d.reshape(F, H * W)
    for i0 in range(0, len(p), chunk):
        px, py, pz = p[i0:i0 + chunk].unbind(1)
        acc = torch.zeros(len(px), dtype=torch.int32, device=dev)
        for f in range(F):
            if not good[f]:
                continue
            e, k = Eh[f], Kh[f]
            x, y, z = (((px * e[r][0] + py * e[r][1]) + pz * e[r][2]) + e[r][3] for r in range(3))
            U = (x * k[0][0] + y * k[0][1]) + z * k[0][2]
            V = (x * k[1][0] + y * k[1][1]) + z * k[1][2]
            ix = torch.round(U / z - 0.5)
            iy = torch.round(V / z - 0.5)
            ok = (z > 0) & (z < max_depth) & (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
            idx = torch.where(ok, iy * W + ix, torch.zeros_like(ix)).to(torch.int64)
            dd = flat[f][idx].to(torch.float64)
            ok &= (dd > 0) & (dd < max_depth) & ((dd - z) > -margin)
            acc += ok.to(torch.int32)
        counts[i0:i0 + chunk] = acc
    return counts
