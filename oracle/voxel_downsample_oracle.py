"""numpy restatement of voxel down-sampling (csrc/srcv_voxel_downsample.cuh, DESIGN §4.19), and the same rule as a
PyTorch op sequence — test and measurement infrastructure, never imported by the package.

The rule (Open3D's VoxelDownSample, restated from its documented behaviour), in fp64 from the fp32 points and the
voxel size s: b = min_i p_i - 0.5 s per axis; point p lies in voxel v = floor((p - b) / s) (IEEE subtraction and
division); each occupied voxel gives the fp64 sum of its points, accumulated in input order from 0.0, divided by the
count and rounded once to fp32; colours likewise (uint8 as c / 255.0 in fp64, floats as given).  Voxels in ascending
(vx, vy, vz) order.

The sums are sequential on purpose: np.sum / np.add.reduce sum pairwise.  Points of rank r within their voxel (in
input order) are added for every voxel at once, rank after rank; a voxel with more than ``long_run`` points is summed
with np.add.accumulate (np.cumsum) after a leading 0.0, which is the same left-to-right sum, so a cloud in one voxel
does not cost one numpy call per point."""
from __future__ import annotations

import numpy as np

MAX_EXTENT = 1 << 21


def voxel_keys(points, voxel_size: float):
    """(N, 3) int64 voxel coordinates of the rule; raises ValueError for an extent of 2^21 voxels or more."""
    p = np.asarray(points, np.float32).astype(np.float64)
    s = float(voxel_size)
    b = p.min(0) - 0.5 * s
    v = np.floor((p - b) / s)
    if not np.all(v.max(0) + 1 < MAX_EXTENT):
        raise ValueError("extent of 2^21 or more voxels")
    return v.astype(np.int64)


def _colors64(colors):
    c = np.asarray(colors)
    return c.astype(np.float64) / 255.0 if c.dtype == np.uint8 else c.astype(np.float64)


def _sequential_sums(values, inv, order, starts, counts, long_run):
    """Per voxel, the left-to-right sum from 0.0 of values[order[starts[j] : starts[j] + counts[j]]]."""
    M = len(counts)
    acc = np.zeros((M, values.shape[1]))
    short = counts <= long_run
    for r in range(int(min(counts.max(), long_run))):
        j = np.nonzero(short & (counts > r))[0]
        acc[j] += values[order[starts[j] + r]]
    for j in np.nonzero(~short)[0]:
        run = values[order[starts[j]:starts[j] + counts[j]]]
        acc[j] = np.cumsum(np.concatenate([np.zeros((1, values.shape[1])), run]), axis=0)[-1]
    return acc


def voxel_down_sample(points, voxel_size: float, colors=None, long_run: int = 256):
    """(points (M,3) float32, colors (M,3) float32 or None, counts (M,) int32) of the rule."""
    p = np.asarray(points, np.float32)
    v = voxel_keys(p, voxel_size)
    n = v.max(0) + 1
    key = (v[:, 0] * n[1] + v[:, 1]) * n[2] + v[:, 2]     # ascending key <=> ascending (vx, vy, vz)
    _, inv, counts = np.unique(key, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    order = np.argsort(inv, kind="stable")                # each voxel's points, in input order
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    sums = _sequential_sums(p.astype(np.float64), inv, order, starts, counts, long_run)
    out = (sums / counts[:, None]).astype(np.float32)
    out_c = None
    if colors is not None:
        csum = _sequential_sums(_colors64(colors), inv, order, starts, counts, long_run)
        out_c = (csum / counts[:, None]).astype(np.float32)
    return out, out_c, counts.astype(np.int32)


def voxel_down_sample_torch(points, voxel_size: float, colors=None):
    """The same rule as a PyTorch op sequence on the tensors' device: fp64 keys, a stable sort, then the sums rank by
    rank (one indexed add per rank, each voxel at most once per add, so the order is input order).  The baseline the
    kernel is measured against; its loop takes one step per point of the most crowded voxel."""
    import torch
    p = points.to(torch.float32).to(torch.float64)
    s = float(voxel_size)
    b = p.min(0).values - 0.5 * s
    v = torch.floor((p - b) / s).to(torch.int64)
    n = v.max(0).values + 1
    if not bool((n < MAX_EXTENT).all()):
        raise ValueError("extent of 2^21 or more voxels")
    key = (v[:, 0] * n[1] + v[:, 1]) * n[2] + v[:, 2]
    skey, order = torch.sort(key, stable=True)
    head = torch.ones_like(skey, dtype=torch.bool)
    head[1:] = skey[1:] != skey[:-1]
    vid = torch.cumsum(head.to(torch.int64), 0) - 1
    M = int(vid[-1]) + 1
    starts = torch.nonzero(head).reshape(-1)
    rank = torch.arange(len(skey), device=p.device) - starts[vid]
    counts = torch.bincount(vid, minlength=M)
    vals = [p]
    if colors is not None:
        vals.append(colors.to(torch.float64) / 255.0 if colors.dtype == torch.uint8 else colors.to(torch.float64))
    x = torch.cat(vals, 1)[order]
    by_rank = torch.argsort(rank, stable=True)
    rank_counts = torch.bincount(rank, minlength=int(counts.max())).tolist()
    acc = torch.zeros(M, x.shape[1], dtype=torch.float64, device=p.device)
    i0 = 0
    for c in rank_counts:
        sel = by_rank[i0:i0 + c]
        j = vid[sel]
        acc[j] = acc[j] + x[sel]
        i0 += c
    mean = (acc / counts[:, None].to(torch.float64)).to(torch.float32)
    return mean[:, :3], (mean[:, 3:] if colors is not None else None), counts.to(torch.int32)
