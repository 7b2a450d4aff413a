"""float32 restatement of the TSDF colour fusion and the vertex colours (DESIGN §4.11) — TEST INFRASTRUCTURE.

Colour is this library's definition (the reference's OurFuser has none), so this oracle pins the kernels
(csrc/srcv_tsdf.cu, csrc/srcv_mesh.cuh) to the documented rule bit for bit:
  - integration: tsdf_oracle's projection and nearest depth sample pick each (voxel, frame) update and its
    depth pixel (sx, sy); the colour pixel is (min(floor(sx * f32(Wc/W)), Wc-1), min(floor(sy * f32(Hc/H)),
    Hc-1)), rgb = clamp((x - mean) / std, 0, 1), and c = (c * tw + rgb * nw) / total with that update's
    fp16 old weight tw, nw and total — separately rounded fp32 ops;
  - vertices: the crossing edges re-enumerated in the §4.10 order (owner in linear order, then axis),
    t = (0 - va) / (vb - va) in fp32, and the colour ca + t (cb - ca) when both endpoints have weight,
    the weighted endpoint's colour when one has, grey 0.7 when none has.
Values and weights are tsdf_oracle.integrate's, step for step.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import tsdf_oracle as T

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)
# reverse_imagenet_normalize (reference utils/generic_utils.py:153-159)
REVERSE_MEAN = (-2.11790393, -2.03571429, -1.80444444)
REVERSE_STD = (4.36681223, 4.46428571, 4.44444444)
GREY = np.float32(0.7)


def sample_index(xy_b2N: torch.Tensor, H: int, W: int):
    """tsdf_oracle.sample_nearest's pixel index (sx, sy) and its in-image flag."""
    size = torch.tensor([W, H], dtype=torch.float32).view(1, 2, 1)
    g = T.r16(T.r16(T.r16(2.0 * xy_b2N) / size) - 1.0)
    ix = torch.round(T.r16(T.r16(T.r16(T.r16(g + 1.0) * size) - 1.0) / 2.0))
    x, y = ix[:, 0], ix[:, 1]
    return x, y, (x >= 0) & (x <= W - 1) & (y >= 0) & (y <= H - 1)


def integrate(tsdf_values, tsdf_weights, tsdf_colors, origin, voxel_size, depth_b1hw, cam_T_world_b44, K_b44,
              color_b3hw, depth_mask_b1hw=None, min_depth: float = 0.5, max_depth: float = 5.0,
              mean=REVERSE_MEAN, std=REVERSE_STD, lo=(0, 0, 0)):
    """In-place update of values / weights (fp16 (X,Y,Z)) and colours (fp32 (3,X,Y,Z)); ``lo`` as in
    tsdf_oracle.integrate (the volume holds lattice indices lo .. lo + dims - 1)."""
    dims = tuple(tsdf_values.shape)
    B, _, H, W = depth_b1hw.shape
    Hc, Wc = color_b3hw.shape[-2:]
    coords = T.voxel_coords(origin, dims, voxel_size, lo)
    trunc = T.TRUNCATION_VOXELS * voxel_size
    depth = depth_b1hw.half()
    if depth_mask_b1hw is not None:
        depth = depth.clone()
        depth[~depth_mask_b1hw] = -1
    xy, vz = T.project(K_b44, cam_T_world_b44, coords)
    ds = T.sample_nearest(depth, xy)
    f = lambda v: float(torch.tensor(v, dtype=torch.float32))
    h = lambda v: float(torch.tensor(v, dtype=torch.float16))
    conf = T.r16(torch.clamp(T.r16(1.0 - T.r16(T.r16(ds - f(min_depth)) / f(max_depth - min_depth))), 0.0, 1.0) ** 2)
    dist = T.r16(ds - vz)
    tv = torch.clamp(T.r16(dist / f(trunc)), -1.0, 1.0)
    valid = (vz > 0) & (dist > -h(trunc)) & (ds > 0) & (vz < h(max_depth)) & (conf > 0)
    # colour pixel of each (frame, voxel): PyTorch's nearest rule on the depth pixel, fp32 scale in / out
    sx, sy, _ = sample_index(xy, H, W)
    scale_x = torch.tensor(np.float32(Wc) / np.float32(W))
    scale_y = torch.tensor(np.float32(Hc) / np.float32(H))
    cx = torch.clamp(torch.floor(sx * scale_x), max=Wc - 1).clamp_min(0).long()
    cy = torch.clamp(torch.floor(sy * scale_y), max=Hc - 1).clamp_min(0).long()
    img = color_b3hw.float()
    m32 = torch.tensor(mean, dtype=torch.float32).view(3, 1)
    s32 = torch.tensor(std, dtype=torch.float32).view(3, 1)
    tvals, wvals = tsdf_values.reshape(-1), tsdf_weights.reshape(-1)
    cvals = tsdf_colors.reshape(3, -1)
    for b in range(B):
        m = valid[b, 0]
        old_t, old_w = tvals[m].float(), wvals[m].float()
        new_t, c = tv[b, 0][m], conf[b, 0][m]
        rate = torch.where(c < old_w, torch.tensor(2.0), torch.tensor(5.0))
        new_w = T.r16(T.r16(c * rate) / T.MAX_W)
        total = T.r16(old_w + new_w)
        rgb = img[b][:, cy[b][m], cx[b][m]]                                   # (3, n)
        rgb = torch.clamp((rgb - m32) / s32, 0.0, 1.0)
        cvals[:, m] = (cvals[:, m] * old_w + rgb * new_w) / total
        tvals[m] = T.r16(T.r16(T.r16(old_t * old_w) + T.r16(new_t * new_w)) / total).half()
        wvals[m] = torch.clamp(total, max=1.0).half()
    return tsdf_values, tsdf_weights, tsdf_colors


def _emitted_edges(inside: np.ndarray, weighted: np.ndarray, single_mesh: bool) -> np.ndarray:
    """(3,X,Y,Z) bool: the edge along axis a from each voxel crosses the level and is emitted (§4.10)."""
    X, Y, Z = inside.shape
    ok = np.ones((X - 1, Y - 1, Z - 1), bool)
    if single_mesh:
        for c in range(8):
            dx, dy, dz = c & 1, (c >> 1) & 1, c >> 2
            ok &= weighted[dx:X - 1 + dx, dy:Y - 1 + dy, dz:Z - 1 + dz]
    okp = np.zeros((X + 1, Y + 1, Z + 1), bool)                    # okp[i+1, j+1, k+1] = cube (i,j,k) processed
    okp[1:X, 1:Y, 1:Z] = ok
    emit = np.zeros((3, X, Y, Z), bool)
    for a in range(3):
        lo, hi = [slice(None)] * 3, [slice(None)] * 3
        lo[a], hi[a] = slice(0, -1), slice(1, None)
        cross = inside[tuple(lo)] != inside[tuple(hi)]
        b, c = [k for k in range(3) if k != a]
        anyok = np.zeros(cross.shape, bool)
        for db in (0, 1):
            for dc in (0, 1):
                start = [1, 1, 1]
                start[b] -= db
                start[c] -= dc
                anyok |= okp[tuple(slice(start[k], start[k] + cross.shape[k]) for k in range(3))]
        emit[a][tuple(lo)] = cross & anyok
    return emit


def vertex_colors(values, weights, colors, single_mesh: bool = False) -> np.ndarray:
    """(V,3) float32 vertex colours in srcv_mesh_extract's vertex order."""
    v32 = np.clip(torch.as_tensor(values).float().cpu().numpy(), np.float32(-1), np.float32(1))
    w = torch.as_tensor(weights).float().cpu().numpy() > 0
    col = torch.as_tensor(colors).float().cpu().numpy()
    emit = _emitted_edges(v32 < 0, w, single_mesh)
    owners = np.argwhere(np.transpose(emit, (1, 2, 3, 0)))         # (V, 4) x, y, z, axis in vertex order
    a = owners[:, :3]
    b = a + np.eye(3, dtype=np.int64)[owners[:, 3]]
    va, vb = v32[a[:, 0], a[:, 1], a[:, 2]], v32[b[:, 0], b[:, 1], b[:, 2]]
    t = (np.float32(0) - va) / (vb - va)
    wa, wb = w[a[:, 0], a[:, 1], a[:, 2]], w[b[:, 0], b[:, 1], b[:, 2]]
    ca = col[:, a[:, 0], a[:, 1], a[:, 2]].T
    cb = col[:, b[:, 0], b[:, 1], b[:, 2]].T
    mix = ca + t[:, None] * (cb - ca)
    out = np.where((wa & wb)[:, None], mix, np.where(wa[:, None], ca, np.where(wb[:, None], cb, GREY)))
    return out.astype(np.float32)
