"""numpy / scipy restatement of the mesh evaluation (csrc/srcv_mesh_eval.cuh, DESIGN §4.17) — test
infrastructure, never imported by the package.

Distances are an fp64 KD-tree over the fp32 coordinates taken to fp64 (``scipy.spatial.cKDTree``); the sampler
reproduces the kernel's counter hash bit for bit and its triangle choice and barycentric map in fp64, with the
area CDF as a sequential ``np.cumsum`` (the kernel's is a tiled tree, so a draw that lands within rounding of a
CDF boundary may pick the neighbouring triangle)."""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

KEYS = ("acc", "comp", "chamfer", "precision", "recall", "fscore")
_M64 = (1 << 64) - 1


def uniforms(seed: int, index: np.ndarray, draw: int) -> np.ndarray:
    """U(seed, i, draw) in [0, 1): x = seed * 0x9e3779b97f4a7c15 + (3 i + draw + 1) * 0xd1b54a32d192ed03 mod 2^64,
    splitmix64's finaliser, then the top 53 bits / 2^53."""
    i = np.asarray(index, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = np.uint64(seed & _M64) * np.uint64(0x9E3779B97F4A7C15) + \
            (np.uint64(3) * i + np.uint64(draw + 1)) * np.uint64(0xD1B54A32D192ED03)
        x ^= x >> np.uint64(30)
        x *= np.uint64(0xBF58476D1CE4E5B9)
        x ^= x >> np.uint64(27)
        x *= np.uint64(0x94D049BB133111EB)
        x ^= x >> np.uint64(31)
    return (x >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def triangle_areas(verts: np.ndarray, faces: np.ndarray) -> np.ndarray:
    v = np.asarray(verts, dtype=np.float32).astype(np.float64)
    f = np.asarray(faces, dtype=np.int64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    return 0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1)


def sample_surface(verts: np.ndarray, faces: np.ndarray, num_samples: int, seed: int = 0,
                   return_faces: bool = False):
    """The kernel's stratified area-uniform samples (N, 3) fp32 (and the triangle of each)."""
    v = np.asarray(verts, dtype=np.float32).astype(np.float64)
    f = np.asarray(faces, dtype=np.int64)
    cdf = np.cumsum(triangle_areas(verts, faces))
    total = cdf[-1]
    i = np.arange(num_samples, dtype=np.uint64)
    u0, u1, u2 = (uniforms(seed, i, k) for k in range(3))
    t = (i.astype(np.float64) + u0) / float(num_samples) * total
    t = np.where(t < total, t, total * (1.0 - 2.0 ** -52))
    tri = np.minimum(np.searchsorted(cdf, t, side="right"), len(f) - 1)
    s = np.sqrt(u1)
    wa, wb, wc = 1.0 - s, s * (1.0 - u2), s * u2
    fa, fb, fc = (v[f[tri, k]] for k in range(3))
    pts = (wa[:, None] * fa + wb[:, None] * fb + wc[:, None] * fc).astype(np.float32)
    return (pts, tri) if return_faces else pts


def nearest_distances(queries: np.ndarray, points: np.ndarray) -> np.ndarray:
    """fp64 KD-tree distances from the fp32 coordinates."""
    q = np.asarray(queries, dtype=np.float32).astype(np.float64)
    p = np.asarray(points, dtype=np.float32).astype(np.float64)
    return cKDTree(p).query(q, k=1, workers=-1)[0]


def brute_distances(queries: np.ndarray, points: np.ndarray) -> np.ndarray:
    """The same minimum by exhaustive search (small sets)."""
    q = np.asarray(queries, dtype=np.float32).astype(np.float64)
    p = np.asarray(points, dtype=np.float32).astype(np.float64)
    return np.sqrt(((q[:, None, :] - p[None, :, :]) ** 2).sum(-1).min(1))


def metrics_from_distances(d_pred: np.ndarray, d_gt: np.ndarray, threshold: float = 0.05) -> dict:
    acc, comp = float(np.mean(d_pred)), float(np.mean(d_gt))
    precision = float(np.count_nonzero(d_pred < threshold)) / len(d_pred)
    recall = float(np.count_nonzero(d_gt < threshold)) / len(d_gt)
    fscore = 2 * precision * recall / (precision + recall) if precision + recall > 0 else 0.0
    return dict(zip(KEYS, (acc, comp, 0.5 * (acc + comp), precision, recall, fscore)))


def mesh_metrics(pred_points: np.ndarray, gt_points: np.ndarray, threshold: float = 0.05) -> dict:
    """The six metrics of two point sets (already sampled)."""
    return metrics_from_distances(nearest_distances(pred_points, gt_points), nearest_distances(gt_points, pred_points),
                                  threshold)


def box_mesh(size=(4.0, 3.0, 2.6), origin=(0.0, 0.0, 0.0)):
    """The closed axis-aligned box [origin, origin + size] as 8 vertices and 12 triangles."""
    o, s = np.asarray(origin, np.float64), np.asarray(size, np.float64)
    verts = np.array([[(i >> 2) & 1, (i >> 1) & 1, i & 1] for i in range(8)], np.float64) * s + o
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    faces = [f for a, b, c, d in quads for f in ((a, b, c), (a, c, d))]
    return verts.astype(np.float32), np.asarray(faces, np.int32)
