"""Marching-cubes oracle of the TSDF mesh extraction (csrc/srcv_mesh.cuh, DESIGN §4.10), in numpy fp64.

A restatement of the documented semantics, independent of the kernel's structure: the vertex set
and order (one vertex per emitted crossing edge, ordered by owning voxel = the edge's lower endpoint
in linear order, then axis x, y, z), the face order (cube by cube in linear order, then table
order), the single-mesh rule and the degenerate-face rule.  The triangulation is read from the
generated header the kernel compiles.  Positions and normals are fp64; the degenerate-face decision
is made, as documented, on the fp32 index-space positions.  Test infrastructure only.
"""
from __future__ import annotations

import re
from pathlib import Path

import numpy as np
import torch

HEADER = Path(__file__).resolve().parents[1] / "simplerecon_b200" / "csrc" / "srcv_mc_table.h"


def read_table() -> np.ndarray:
    """(256, kMaxTris, 3) int edge triples, -1 padded."""
    text = HEADER.read_text()
    maxt = int(re.search(r"kMaxTris = (\d+);", text).group(1))
    body = text[text.index("kTris[256]"):]
    rows = re.findall(r"\{([-0-9, ]+)\},\s*//", body)
    assert len(rows) == 256
    return np.array([[int(v) for v in r.split(",")] for r in rows], dtype=np.int64).reshape(256, maxt, 3)


_TABLE = None


def table() -> np.ndarray:
    global _TABLE
    if _TABLE is None:
        _TABLE = read_table()
    return _TABLE


def edge_geometry():
    """(lower-corner offset (12,3), axis (12,))."""
    off, axis = np.zeros((12, 3), np.int64), np.zeros(12, np.int64)
    for e in range(12):
        a, j = divmod(e, 4)
        b, c = [k for k in range(3) if k != a]
        off[e, b], off[e, c], axis[e] = j & 1, j >> 1, a
    return off, axis


def _np(t) -> np.ndarray:
    return t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)


def extract(values, weights=None, scale_to_world: bool = False, single_mesh: bool = False,
            origin=(0.0, 0.0, 0.0), voxel_size: float = 1.0):
    """values / weights: (X,Y,Z) fp16 volumes.  Returns (verts (V,3) f64, faces (F,3) int64,
    normals (V,3) f64).  ``origin`` is used as given (the caller rounds it to fp16)."""
    v32 = np.clip(_np(values).astype(np.float32), -1.0, 1.0)
    v = v32.astype(np.float64)
    X, Y, Z = v.shape
    inside = v < 0
    # processed cubes (anchored at their lowest corner)
    if single_mesh:
        w = _np(weights).astype(np.float32) > 0
        ok = np.ones((X - 1, Y - 1, Z - 1), bool)
        for dx in (0, 1):
            for dy in (0, 1):
                for dz in (0, 1):
                    ok &= w[dx:X - 1 + dx, dy:Y - 1 + dy, dz:Z - 1 + dz]
    else:
        ok = np.ones((X - 1, Y - 1, Z - 1), bool)
    okp = np.zeros((X + 1, Y + 1, Z + 1), bool)          # okp[i+1, j+1, k+1] = ok[i, j, k], False outside
    okp[1:X, 1:Y, 1:Z] = ok
    # emitted crossing edges, per axis, on the full (X,Y,Z) grid of owners
    emit = np.zeros((3, X, Y, Z), bool)
    t64 = np.zeros((3, X, Y, Z))
    t32 = np.zeros((3, X, Y, Z), np.float32)
    for a in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[a], hi[a] = slice(0, -1), slice(1, None)
        lo, hi = tuple(lo), tuple(hi)
        cross = inside[lo] != inside[hi]
        b, c = [k for k in range(3) if k != a]
        anyok = np.zeros(cross.shape, bool)
        for db in (0, 1):
            for dc in (0, 1):
                shape = list(cross.shape)
                start = [1, 1, 1]
                start[b] -= db
                start[c] -= dc
                sl = tuple(slice(start[k], start[k] + shape[k]) for k in range(3))
                anyok |= okp[sl]
        emit[a][lo] = cross & anyok
        with np.errstate(divide="ignore", invalid="ignore"):
            t64[a][lo] = np.where(cross, -v[lo] / (v[hi] - v[lo]), 0.0)
            t32[a][lo] = np.where(cross, np.float32(0) - v32[lo], np.float32(0)) / \
                np.where(cross, v32[hi] - v32[lo], np.float32(1))
    # vertex ids: owner linear index major, axis minor
    order = np.transpose(emit, (1, 2, 3, 0)).reshape(-1)
    vid = np.full(order.shape, -1, np.int64)
    vid[order] = np.arange(int(order.sum()))
    vid = vid.reshape(X, Y, Z, 3)
    owners = np.argwhere(np.transpose(emit, (1, 2, 3, 0)))           # (V, 4): x, y, z, axis, in vertex order
    ox, oy, oz, ax = owners.T
    base = owners[:, :3].astype(np.float64)
    t = t64[ax, ox, oy, oz]
    verts = base.copy()
    verts[np.arange(len(ax)), ax] += t
    p32 = owners[:, :3].astype(np.float32)
    p32[np.arange(len(ax)), ax] += t32[ax, ox, oy, oz]
    # normals: central differences (one-sided at the border), interpolated with t, normalised
    g = np.stack(np.gradient(v), -1) if min(X, Y, Z) >= 2 else np.zeros((X, Y, Z, 3))
    ga = g[ox, oy, oz]
    step = np.eye(3, dtype=np.int64)[ax]
    gb = g[ox + step[:, 0], oy + step[:, 1], oz + step[:, 2]]
    n = ga + t[:, None] * (gb - ga)
    ln = np.linalg.norm(n, axis=1, keepdims=True)
    normals = np.where(ln > 0, n / np.where(ln > 0, ln, 1.0), 0.0)
    # faces
    corner = np.array([[c & 1, (c >> 1) & 1, (c >> 2) & 1] for c in range(8)], np.int64)
    case = np.zeros((X - 1, Y - 1, Z - 1), np.int64)
    for c in range(8):
        dx, dy, dz = corner[c]
        case |= inside[dx:X - 1 + dx, dy:Y - 1 + dy, dz:Z - 1 + dz].astype(np.int64) << c
    act = ok & (case != 0) & (case != 255)
    cubes = np.argwhere(act)                                          # linear order
    tris = table()[case[act]]                                         # (n, maxt, 3)
    eoff, eax = edge_geometry()
    valid = tris[..., 0] >= 0
    cidx, slot = np.nonzero(valid)                                     # cube-major, table order
    edges = tris[cidx, slot]                                           # (m, 3)
    own = cubes[cidx][:, None, :] + eoff[edges]                        # (m, 3, 3)
    faces = vid[own[..., 0], own[..., 1], own[..., 2], eax[edges]]
    assert (faces >= 0).all()
    fp = p32[faces]                                                    # (m, 3, 3) fp32 positions
    degen = (np.all(fp[:, 0] == fp[:, 1], -1) | np.all(fp[:, 1] == fp[:, 2], -1) |
             np.all(fp[:, 0] == fp[:, 2], -1))
    faces = faces[~degen]
    if scale_to_world:
        verts = np.asarray(origin, np.float64)[None] + verts * float(voxel_size)
    return verts, faces.astype(np.int64), normals


def crossing_edges_torch(values) -> int:
    """Crossing edges of the clamped volume, counted independently with three torch comparisons."""
    ins = values.float().clamp(-1, 1) < 0
    return int((ins[1:] != ins[:-1]).sum() + (ins[:, 1:] != ins[:, :-1]).sum() + (ins[:, :, 1:] != ins[:, :, :-1]).sum())
