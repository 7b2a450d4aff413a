"""Mesh evaluation on the GPU (csrc/srcv_mesh_eval.cuh, DESIGN §4.17): accuracy, completeness, Chamfer distance,
precision, recall and F-score of a fused mesh or point cloud against the ground truth.

These are the "Mesh Metrics" of the reference README's tables (Acc, Comp, Chamfer, Precision, Recall,
F-Score).  The reference scores meshes with TransformerFusion's ``eval.py`` (and a point cloud through the
same code), which needs open3d or trimesh and a CPU KD-tree.  Here every step runs on the GPU: a seeded
area-uniform surface sampler, an exact nearest-neighbour search (a hashed uniform grid with a brute-force
queue for far queries) and a fixed-order fp64 reduction.

Parity with TransformerFusion's or NeuralRecon's scripts is not claimed: their code is not part of the
reference, and they may apply visibility masks or voxel down-sampling in ways this module does not reproduce.
``mesh_metrics(..., down_sample=s)`` voxel-down-samples both point sets at voxel size ``s`` before scoring them
(``point_cloud_fusion.voxel_down_sample``, csrc/srcv_voxel_downsample.cuh, DESIGN §4.19), which approximates the
2 cm down-sampling NeuralRecon's evaluation is commonly run with.

Visibility culling (csrc/srcv_mesh_visibility.cuh, DESIGN §4.18): given the depth frames of the scan
(``Views``), ``observation_counts`` counts the frames that observe each point, and ``mesh_metrics(..., views=)``
scores only the points of each side that at least one frame observes.  A point is observed by a frame when fusing
that frame's depth map would update a voxel at the point (the reference fuser's validity rule, with the
truncation replaced by ``margin``); see ``observation_counts`` for the exact arithmetic.

With P the predicted points, G the ground-truth points (metres) and d(x, S) = min over s in S of |x - s|,
evaluated in fp64 from the fp32 coordinates:

    acc = mean d(p, G)    comp = mean d(g, P)    chamfer = (acc + comp) / 2
    precision = share of p with d(p, G) < threshold    recall = share of g with d(g, P) < threshold
    fscore = 2 precision recall / (precision + recall), 0 when both are 0

Inputs are CUDA tensors, or numpy arrays, which are moved to the current CUDA device.  Coordinates may be
fp32 or fp64 and are taken to fp32; faces may be int32 or int64.  There is no CPU path: a CPU tensor raises.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Any, NamedTuple

import numpy as np
import torch

from . import _native

KEYS = ("acc", "comp", "chamfer", "precision", "recall", "fscore")
# samples drawn from each side given as a mesh (10^6: a room-sized scene at about one sample per cm^2)
DEFAULT_NUM_SAMPLES = 1_000_000
_MAX_POINTS = 1 << 28
_FLAG_NAMES = ((_native.MESH_EVAL_BAD_FACE, "a face index outside [0, V)"),
               (_native.MESH_EVAL_NONFINITE, "a non-finite (NaN or inf) coordinate"),
               (_native.MESH_EVAL_ZERO_AREA, "a mesh of zero total area"),
               (_native.MESH_EVAL_BAD_VIEW, "a non-finite entry in a view's K or cam_T_world"),
               (_native.VOXEL_NONFINITE_COLOR, "a non-finite (NaN or inf) colour"),
               (_native.VOXEL_EXTENT, "an extent of 2^21 or more voxels on an axis (the voxel size is too small)"))
_COLOR_TYPES = {torch.uint8: _native.COLORS_U8, torch.float32: _native.COLORS_F32, torch.float64: _native.COLORS_F64}


def _require_cuda(t: torch.Tensor) -> None:
    """The device gate (tests/ patch exactly this to drive the host-emulated library)."""
    if t.device.type != "cuda":
        raise RuntimeError("simplerecon_b200 mesh evaluation runs on CUDA (sm_90a) only; there is no CPU fallback")


def _default_device() -> torch.device:
    """Where numpy inputs go: the current CUDA device."""
    if not torch.cuda.is_available():
        raise RuntimeError("simplerecon_b200 mesh evaluation needs a CUDA device; there is no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


def _lib():
    return _native.load()


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _tensor(x, what: str) -> torch.Tensor:
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(np.ascontiguousarray(x)).to(_default_device())
    if not torch.is_tensor(x):
        raise TypeError(f"{what} must be a torch tensor or a numpy array, got {type(x).__name__}")
    _require_cuda(x)
    return x


def _coords(x, what: str) -> torch.Tensor:
    t = _tensor(x, what)
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"{what} must be (N, 3), got {tuple(t.shape)}")
    if t.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"{what} must be float32 or float64, got {t.dtype}")
    if t.shape[0] == 0:
        raise ValueError(f"{what} is empty")
    if t.shape[0] > _MAX_POINTS:
        raise ValueError(f"{what} has {t.shape[0]} points; at most 2^28 are supported")
    return t.detach().to(torch.float32).contiguous()


def _faces(x, num_verts: int) -> torch.Tensor:
    t = _tensor(x, "faces")
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"faces must be (F, 3), got {tuple(t.shape)}")
    if t.dtype not in (torch.int32, torch.int64):
        raise ValueError(f"faces must be int32 or int64, got {t.dtype}")
    if t.shape[0] == 0:
        raise ValueError("the mesh has no faces")
    if num_verts >= 1 << 31 or t.shape[0] >= 1 << 31:
        raise ValueError("meshes are limited to 2^31 - 1 vertices and faces")
    # int64 indices outside int32 stay outside [0, V) (and raise the device flag) instead of wrapping
    return t.detach().clamp(-1, num_verts).to(torch.int32).contiguous()


def _args(flags, num_faces=0, num_queries=0, num_points=0, stats=None) -> _native.MeshEvalArgs:
    return _native.MeshEvalArgs(num_faces, num_queries, num_points, flags.data_ptr(),
                                stats.data_ptr() if stats is not None else None)


def _workspace(args, dev) -> torch.Tensor:
    n = _lib().srcv_mesh_eval_workspace_bytes(C.byref(args))
    if n == 0:
        raise ValueError("unsupported mesh-evaluation sizes")
    return torch.empty(n, dtype=torch.uint8, device=dev)


def _sample(verts, faces, num_samples: int, seed: int, flags) -> torch.Tensor:
    dev = verts.device
    args = _args(flags, num_faces=faces.shape[0])
    ws = _workspace(args, dev)
    out = torch.empty(num_samples, 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _native.check(_lib().srcv_mesh_sample_f32(
            C.byref(args), C.c_void_p(verts.data_ptr()), verts.shape[0], C.c_void_p(faces.data_ptr()), num_samples,
            seed % (1 << 64), C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(), _stream(dev)))
    return out


def _distances(queries, points, flags, stats=None) -> torch.Tensor:
    dev = queries.device
    if points.device != dev:
        raise ValueError(f"queries on {dev} and points on {points.device}")
    args = _args(flags, num_queries=queries.shape[0], num_points=points.shape[0], stats=stats)
    ws = _workspace(args, dev)
    out = torch.empty(queries.shape[0], dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _native.check(_lib().srcv_nearest_distances_f32(
            C.byref(args), C.c_void_p(queries.data_ptr()), C.c_void_p(points.data_ptr()), C.c_void_p(out.data_ptr()),
            C.c_void_p(ws.data_ptr()), ws.numel(), _stream(dev)))
    return out


def _check_count(num_samples: int) -> int:
    n = int(num_samples)
    if not 1 <= n <= _MAX_POINTS:
        raise ValueError(f"num_samples must be in 1 .. 2^28, got {num_samples}")
    return n


def sample_surface(verts, faces, num_samples: int, seed: int = 0) -> torch.Tensor:
    """``num_samples`` points (N, 3) fp32 drawn uniformly by area from the mesh ``(verts (V,3), faces (F,3))``.

    Sample i is stratified: its triangle is the first whose area CDF exceeds (i + u0) / N of the total area, so
    the samples come out in triangle order; within it the point is (1 - sqrt u1) a + sqrt u1 (1 - u2) b +
    sqrt u1 u2 c.  u0, u1, u2 come from a counter hash of (seed, i, draw) (DESIGN §4.17): the same inputs and
    seed give bitwise the same samples.  A face index outside [0, V), a non-finite coordinate or a zero total
    area makes every sample NaN (``mesh_metrics`` names the condition).  No host synchronisation."""
    n = _check_count(num_samples)
    v = _coords(verts, "verts")
    f = _faces(faces, v.shape[0])
    if f.device != v.device:
        raise ValueError(f"verts on {v.device} and faces on {f.device}")
    flags = torch.zeros(1, dtype=torch.int32, device=v.device)
    return _sample(v, f, n, int(seed), flags)


def nearest_distances(queries, points) -> torch.Tensor:
    """(Nq,) fp64: the distance from each query to its nearest point of ``points`` (N, 3), evaluated in fp64
    from the fp32 coordinates, exactly (the same minimum a fp64 KD-tree finds).  A non-finite coordinate makes
    every distance NaN.  No host synchronisation."""
    q = _coords(queries, "queries")
    p = _coords(points, "points")
    flags = torch.zeros(1, dtype=torch.int32, device=q.device)
    return _distances(q, p, flags)


def _device_of(x, what: str) -> torch.device:
    probe = x[0] if isinstance(x, (tuple, list)) else x
    return _default_device() if isinstance(probe, np.ndarray) else _tensor(probe, what).device


def _side(x, what: str, num_samples: int, seed: int, flags) -> torch.Tensor:
    if isinstance(x, (tuple, list)):
        if len(x) != 2:
            raise ValueError(f"{what} must be (verts, faces) or an (N, 3) point set")
        v = _coords(x[0], f"{what} verts")
        f = _faces(x[1], v.shape[0])
        return _sample(v, f, num_samples, seed, flags)
    return _coords(x, f"{what} points")


class Views(NamedTuple):
    """The depth frames that decide which points ``mesh_metrics`` scores (DESIGN §4.18).

    ``depths`` (F, 1, H, W) as the reference passes ``depth_b1hw``, or (F, H, W), metres; ``K`` (F, 4, 4)
    intrinsics at that resolution, or one (4, 4) for every frame; ``cam_T_world`` (F, 4, 4) world -> camera.
    A point is observed by a frame when 0 < z < ``max_depth``, it projects into the image and the depth d read
    there satisfies 0 < d < ``max_depth`` and d - z > -``margin`` (metres)."""
    depths: Any
    K: Any
    cam_T_world: Any
    margin: float = 0.05
    max_depth: float = math.inf


def _frames(x, what: str, shape: tuple, dev) -> torch.Tensor:
    t = _tensor(x, what)
    if t.device != dev:
        raise ValueError(f"{what} on {t.device}, points on {dev}")
    if not t.is_floating_point():
        raise ValueError(f"{what} must be floating point, got {t.dtype}")
    if tuple(t.shape) not in shape:
        raise ValueError(f"{what} must be {' or '.join(map(str, shape))}, got {tuple(t.shape)}")
    return t.detach().to(torch.float32).contiguous()


def _views(views, dev, tile_cull: bool = True):
    """(the C struct, the tensors it points into) for ``views`` on device ``dev``."""
    if not isinstance(views, Views):
        views = Views(*views)
    margin, max_depth = float(views.margin), float(views.max_depth)
    if not (math.isfinite(margin) and margin >= 0.0):
        raise ValueError(f"margin must be finite and >= 0, got {views.margin}")
    if not max_depth > 0.0:
        raise ValueError(f"max_depth must be > 0, got {views.max_depth}")
    d = _tensor(views.depths, "depths")
    if d.dim() == 4 and d.shape[1] == 1:
        d = d[:, 0]
    if d.dim() != 3 or min(d.shape) == 0:
        raise ValueError(f"depths must be (F, 1, H, W) or (F, H, W) and not empty, got {tuple(_tensor(views.depths, 'depths').shape)}")
    F, H, W = d.shape
    if H * W >= 1 << 31 or F >= 1 << 31:
        raise ValueError(f"depth frames of {H} x {W} (x {F}) are too large: H W < 2^31")
    d = _frames(d, "depths", ((F, H, W),), dev)
    K = _frames(views.K, "K", ((4, 4), (F, 4, 4)), dev)
    E = _frames(views.cam_T_world, "cam_T_world", ((F, 4, 4),), dev)
    s = _native.MeshViews(d.data_ptr(), K.data_ptr(), E.data_ptr(), F, H, W, int(K.dim() == 2), margin, max_depth,
                          int(tile_cull))
    return s, (d, K, E)


def _count(points, vs, counts, flags, stats=None) -> None:
    dev = points.device
    args = _args(flags, num_points=points.shape[0], stats=stats)
    with torch.cuda.device(dev):
        _native.check(_lib().srcv_observation_counts_f32(C.byref(args), C.byref(vs), C.c_void_p(points.data_ptr()),
                                                         C.c_void_p(counts.data_ptr()), _stream(dev)))


def _compact(points, counts, flags, num_kept) -> torch.Tensor:
    """The points with count > 0 in input order, at the head of an (N, 3) buffer; their number goes to num_kept."""
    dev = points.device
    args = _args(flags, num_points=points.shape[0])
    ws = _workspace(args, dev)
    out = torch.empty_like(points)
    with torch.cuda.device(dev):
        _native.check(_lib().srcv_compact_observed_f32(
            C.byref(args), C.c_void_p(points.data_ptr()), C.c_void_p(counts.data_ptr()), C.c_void_p(out.data_ptr()),
            C.c_void_p(num_kept.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(), _stream(dev)))
    return out


def _check_voxel_size(voxel_size) -> float:
    s = float(voxel_size)
    if not (math.isfinite(s) and s > 0.0):
        raise ValueError(f"voxel_size must be finite and > 0, got {voxel_size}")
    return s


def _colors(x, points) -> torch.Tensor:
    """(N, 3) uint8, float32 or float64 colours on the points' device, as given (no conversion)."""
    t = _tensor(x, "colors")
    if t.device != points.device:
        raise ValueError(f"colors on {t.device} and points on {points.device}")
    if tuple(t.shape) != (points.shape[0], 3):
        raise ValueError(f"colors must be ({points.shape[0]}, 3) like the points, got {tuple(t.shape)}")
    if t.dtype not in _COLOR_TYPES:
        raise ValueError(f"colors must be uint8, float32 or float64, got {t.dtype}")
    return t.detach().contiguous()


def _down_sample(points, voxel_size: float, flags, colors=None, num_out=None):
    """Launches the voxel down-sampling of ``points`` (fp32 (N, 3) on the device): returns (points (N, 3) fp32,
    colours (N, 3) fp32 or None, counts (N,) int32, num_out (1,) int64), of which the first num_out rows are the
    result.  No host synchronisation."""
    dev = points.device
    n = points.shape[0]
    lib = _lib()
    ws = torch.empty(lib.srcv_voxel_down_sample_workspace_bytes(n), dtype=torch.uint8, device=dev)
    out = torch.empty(n, 3, dtype=torch.float32, device=dev)
    out_c = torch.empty(n, 3, dtype=torch.float32, device=dev) if colors is not None else None
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    if num_out is None:
        num_out = torch.zeros(1, dtype=torch.int64, device=dev)
    ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None   # noqa: E731
    with torch.cuda.device(dev):
        _native.check(lib.srcv_voxel_down_sample_f32(
            ptr(points), n, float(voxel_size), ptr(colors),
            _native.COLORS_NONE if colors is None else _COLOR_TYPES[colors.dtype], ptr(out), ptr(out_c), ptr(counts),
            ptr(num_out), ptr(flags), ptr(ws), ws.numel(), _stream(dev)))
    return out, out_c, counts, num_out


def _observation_counts(points, depths, K, cam_T_world, margin=0.05, max_depth=math.inf, counts=None,
                        tile_cull: bool = True, stats=None) -> torch.Tensor:
    p = _coords(points, "points")
    vs, keep = _views(Views(depths, K, cam_T_world, margin, max_depth), p.device, tile_cull)
    if counts is None:
        counts = torch.zeros(p.shape[0], dtype=torch.int32, device=p.device)
    elif not (torch.is_tensor(counts) and counts.dtype == torch.int32 and tuple(counts.shape) == (p.shape[0],)
              and counts.device == p.device and counts.is_contiguous()):
        raise ValueError(f"counts must be a contiguous int32 ({p.shape[0]},) tensor on {p.device}")
    flags = torch.zeros(1, dtype=torch.int32, device=p.device)
    _count(p, vs, counts, flags, stats)
    return counts


def observation_counts(points, depths, K, cam_T_world, margin: float = 0.05, max_depth: float = math.inf,
                       counts=None) -> torch.Tensor:
    """(N,) int32 on the device: how many of the F depth frames observe each point of ``points`` (N, 3).

    ``depths`` (F, 1, H, W) or (F, H, W) metres, ``K`` (F, 4, 4) or one (4, 4), ``cam_T_world`` (F, 4, 4) world ->
    camera, as ``Views`` describes.  Evaluated in fp64 from the fp32 inputs, in this order: x = ((E00 px + E01 py)
    + E02 pz) + E03 (likewise y, z), U = (K00 x + K01 y) + K02 z (likewise V), ix = rint(U / z - 0.5) and
    iy = rint(V / z - 0.5) rounding half to even (``grid_sample(mode="nearest")``); the point is observed when
    0 < z < max_depth, 0 <= ix < W, 0 <= iy < H, and d = depths[f, iy, ix] has 0 < d < max_depth and
    d - z > -margin.  A point with a non-finite coordinate, and a frame with a non-finite K or cam_T_world entry,
    observe nothing (``mesh_metrics`` raises for them).  With ``counts`` (int32 (N,) on the same device) the
    counts are added into it in place and it is returned, so frames can be fed in chunks or batch by batch.
    Bitwise deterministic; no host synchronisation."""
    return _observation_counts(points, depths, K, cam_T_world, margin, max_depth, counts)


def mesh_metrics(pred, gt, threshold: float = 0.05, num_samples: int = DEFAULT_NUM_SAMPLES, seed: int = 0,
                 views: Views | None = None, down_sample: float | None = None) -> dict:
    """{acc, comp, chamfer, precision, recall, fscore} (Python floats, in that order) of ``pred`` against ``gt``.

    Each side is a mesh ``(verts, faces)``, replaced by ``num_samples`` area-uniform surface samples
    (``sample_surface`` with ``seed`` for ``pred`` and ``seed + 1`` for ``gt``; default 10^6 per side), or a
    point set ``(N, 3)`` used as given.  ``threshold`` is in metres (default 5 cm).  The result is deterministic:
    the same inputs and seed give bitwise the same metrics.  One host synchronisation, at the end; a face index
    outside [0, V), a non-finite coordinate or a mesh of zero total area raises ``ValueError``.

    With ``views`` (``Views``), each side's points that no frame observes (``observation_counts`` == 0) are
    dropped before the distances; the call then synchronises twice, and a side left with no point, or a view with
    a non-finite K or cam_T_world entry, raises ``ValueError``.

    With ``down_sample`` (a voxel size in metres, e.g. 0.02), each side's points (its samples, or the point set as
    given) are replaced by their voxel down-sampling (``point_cloud_fusion.voxel_down_sample``) before the views and
    the distances; this adds one host synchronisation, and a side whose extent is 2^21 voxels or more raises
    ``ValueError``.  ``None`` (the default) scores the points as they are."""
    if not threshold > 0:
        raise ValueError(f"threshold must be positive, got {threshold}")
    n = _check_count(num_samples)
    voxel = None if down_sample is None else _check_voxel_size(down_sample)
    flags = torch.zeros(1, dtype=torch.int32, device=_device_of(pred, "pred"))
    P = _side(pred, "pred", n, int(seed), flags)
    G = _side(gt, "gt", n, int(seed) + 1, flags)
    if P.device != G.device:
        raise ValueError(f"pred on {P.device} and gt on {G.device}")
    dev = P.device
    if voxel is not None:
        num_out = torch.zeros(2, dtype=torch.int64, device=dev)
        ds = [_down_sample(X, voxel, flags, num_out=num_out[k:k + 1])[0] for k, X in enumerate((P, G))]
        n_pred, n_gt, bad = torch.cat([num_out, flags.to(torch.int64)]).tolist()   # the extra host synchronisation
        _raise_flags(bad)
        P, G = ds[0][:n_pred], ds[1][:n_gt]
    if views is not None:
        vs, keep = _views(views, dev)
        num_kept = torch.zeros(2, dtype=torch.int64, device=dev)
        sides = []
        for k, X in enumerate((P, G)):
            counts = torch.zeros(X.shape[0], dtype=torch.int32, device=dev)
            _count(X, vs, counts, flags)
            sides.append(_compact(X, counts, flags, num_kept[k:k + 1]))
        n_pred, n_gt, bad = torch.cat([num_kept, flags.to(torch.int64)]).tolist()   # the extra host synchronisation
        _raise_flags(bad)
        for name, m in (("pred", n_pred), ("gt", n_gt)):
            if m == 0:
                raise ValueError(f"mesh_metrics: no point of {name} is observed by the views")
        P, G = sides[0][:n_pred], sides[1][:n_gt]
    d_pred = _distances(P, G, flags)
    d_gt = _distances(G, P, flags)
    args = _args(flags, num_queries=P.shape[0], num_points=G.shape[0])
    ws = _workspace(args, dev)
    out = torch.empty(8, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _native.check(_lib().srcv_mesh_metrics_f64(
            C.byref(args), C.c_void_p(d_pred.data_ptr()), C.c_void_p(d_gt.data_ptr()), float(threshold),
            C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(), _stream(dev)))
    vals = out.tolist()                                   # the one host synchronisation
    _raise_flags(int(vals[6]))
    return dict(zip(KEYS, vals[:6]))


def _raise_flags(bad: int, who: str = "mesh_metrics") -> None:
    if bad:
        raise ValueError(f"{who}: the input has " + " and ".join(name for bit, name in _FLAG_NAMES if bad & bit))
