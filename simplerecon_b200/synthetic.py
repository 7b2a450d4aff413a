"""Synthetic frame tuples shaped like the reference's dataloader output.

There is no dataset or checkpoint in this environment, so every test and
benchmark runs on seeded synthetic tuples that follow SURVEY.md §8(d):

* matching features ~ N(0,1) fp32 — the reference's matching encoder ends in an
  affine-free ``InstanceNorm2d(16)`` (reference ``modules/networks.py:201``), so
  zero-mean / unit-variance per channel is the true marginal.  ``smooth=True``
  box-filters and re-standardises them (closer to real, spatially correlated
  feature maps).
* intrinsics: the ScanNet depth camera (reference ``README.md:175-182``) scaled the
  way ``datasets/scannet_dataset.py:460-470`` does it, to the matching resolution.
* poses: small rigid motions in the DVMVS keyframe range
  (reference ``tools/keyframe_buffer.py:12-22``): rotation about a random axis by
  up to 0.15 rad, translation of 5–30 cm; sources sorted by ascending
  ``pose_distance`` like ``datasets/generic_mvs_dataset.py:643-659``.
* depth range 0.25–5 m (reference ``options.py:133-134``).

Generated on the CPU from a ``torch.Generator`` so the CPU oracle and the GPU
kernels see bit-identical inputs.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

SCANNET_FX, SCANNET_FY, SCANNET_CX, SCANNET_CY = 570.924255, 570.924316, 319.5, 239.5
MIN_DEPTH, MAX_DEPTH = 0.25, 5.0


@dataclass
class Workload:
    """One BASELINE.json configuration, at feature-map resolution."""
    name: str
    kind: str          # "dot" | "mlp"
    batch: int
    views: int         # K source views
    height: int        # matching feature-map H (= image_h / 4)
    width: int
    planes: int        # D
    channels: int = 16


# BASELINE.json `configs`, in order (image size -> feature map = image/4,
# reference experiment_modules/depth_model.py:171-172).
CONFIGS = [
    Workload("cfg0_dot_256x192_D16_K2_B1", "dot", 1, 2, 48, 64, 16),
    Workload("cfg1_dot_640x480_D64_K7_B4", "dot", 4, 7, 120, 160, 64),
    Workload("cfg2_hero_640x480_D64_K7_B8", "mlp", 8, 7, 120, 160, 64),
    Workload("cfg3_hero_640x480_D96_K7_B16", "mlp", 16, 7, 120, 160, 96),
    Workload("cfg4_hero_640x480_D64_K7_B64", "mlp", 64, 7, 120, 160, 64),
]


# Stress shape of SURVEY.md §8: the FEATURE MAP itself is 480x640 (16x the pixels of the
# BASELINE configs; 137 MB of source features per frame, larger than L2).  Not a BASELINE
# config — `bench.py --workload stress_dot` / `stress_hero` report it for context.
STRESS = [
    Workload("stress_dot_480x640map_D64_K7_B1", "dot", 1, 7, 480, 640, 64),
    Workload("stress_hero_480x640map_D64_K7_B1", "mlp", 1, 7, 480, 640, 64),
]


def matching_intrinsics(height: int, width: int) -> torch.Tensor:
    """4x4 K at the matching resolution for a (4*height)x(4*width) frame of a
    640x480 ScanNet-like camera."""
    sx, sy = width / 640.0, height / 480.0
    K = torch.eye(4, dtype=torch.float64)
    K[0, 0], K[1, 1] = SCANNET_FX * sx, SCANNET_FY * sy
    K[0, 2], K[1, 2] = SCANNET_CX * sx, SCANNET_CY * sy
    return K


def _axis_angle(axis: torch.Tensor, theta: torch.Tensor) -> torch.Tensor:
    """Rodrigues, float64.  axis (...,3) unit, theta (...)."""
    x, y, z = axis.unbind(-1)
    zero = torch.zeros_like(x)
    Kx = torch.stack([zero, -z, y, z, zero, -x, -y, x, zero], -1).reshape(*axis.shape[:-1], 3, 3)
    s = torch.sin(theta)[..., None, None]
    c = torch.cos(theta)[..., None, None]
    I = torch.eye(3, dtype=axis.dtype).expand_as(Kx)
    return I + s * Kx + (1 - c) * (Kx @ Kx)


def _pose_distance(pose: torch.Tensor) -> torch.Tensor:
    tr = pose[..., :3, :3].diagonal(dim1=-2, dim2=-1).sum(-1)
    r = torch.sqrt(2 * (1 - torch.clamp(tr, max=3.0) / 3))
    t = pose[..., :3, 3].norm(dim=-1)
    return torch.sqrt(t * t + r * r)


def make_tuple(batch: int, views: int, height: int, width: int, channels: int = 16,
               seed: int = 1234, smooth: bool = False, max_angle: float = 0.15,
               t_range=(0.05, 0.30)) -> dict:
    """Returns the keyword arguments of ``CostVolumeManager.forward`` (CPU, fp32)."""
    g = torch.Generator().manual_seed(seed)
    B, K, C, H, W = batch, views, channels, height, width
    cur = torch.randn(B, C, H, W, generator=g)
    src = torch.randn(B, K, C, H, W, generator=g)
    if smooth:
        def sm(x):
            shp = x.shape
            y = torch.nn.functional.avg_pool2d(x.reshape(-1, 1, H, W), 5, 1, 2)
            y = y.reshape(shp)
            mu = y.mean((-2, -1), keepdim=True)
            sd = y.std((-2, -1), keepdim=True)
            return (y - mu) / sd
        cur, src = sm(cur), sm(src)
    axis = torch.randn(B, K, 3, generator=g, dtype=torch.float64)
    axis = axis / axis.norm(dim=-1, keepdim=True)
    theta = torch.rand(B, K, generator=g, dtype=torch.float64) * max_angle
    tdir = torch.randn(B, K, 3, generator=g, dtype=torch.float64)
    tdir = tdir / tdir.norm(dim=-1, keepdim=True)
    tnorm = t_range[0] + torch.rand(B, K, generator=g, dtype=torch.float64) * (t_range[1] - t_range[0])
    E = torch.eye(4, dtype=torch.float64).repeat(B, K, 1, 1)      # src_cam_T_cur_cam
    E[..., :3, :3] = _axis_angle(axis, theta)
    E[..., :3, 3] = tdir * tnorm[..., None]
    P = torch.linalg.inv(E)                                         # cur_cam_T_src_cam
    order = torch.argsort(_pose_distance(P), dim=1)                 # ascending, like the dataloader
    gather = lambda x: torch.gather(x, 1, order[..., None, None].expand_as(x))
    E, P = gather(E), gather(P)
    Kmat = matching_intrinsics(H, W)
    return dict(
        cur_feats=cur.contiguous(),
        src_feats=src.contiguous(),
        src_extrinsics=E.float().contiguous(),
        src_poses=P.float().contiguous(),
        src_Ks=Kmat.float().repeat(B, K, 1, 1).contiguous(),
        cur_invK=torch.linalg.inv(Kmat).float().repeat(B, 1, 1).contiguous(),
        min_depth=torch.tensor(MIN_DEPTH).view(1, 1, 1, 1),
        max_depth=torch.tensor(MAX_DEPTH).view(1, 1, 1, 1),
    )


def make_workload_tuple(w: Workload, seed_offset: int = 0, batch: int | None = None, **kw) -> dict:
    idx = [c.name for c in CONFIGS].index(w.name) if w in CONFIGS else 99
    return make_tuple(batch or w.batch, w.views, w.height, w.width, w.channels,
                      seed=1234 + idx + 1000 * seed_offset, **kw)


def mlp_state(views: int = 7, channels: int = 16, hidden=(128, 128), seed: int = 0) -> dict:
    """Seeded default-``nn.Linear``-init weights under the reference's state_dict
    keys (``mlp.net.{0,2,4}.{weight,bias}``; reference modules/networks.py:134-147)."""
    f_in = channels * (views + 1) + 10 * views + 4                  # reference modules/cost_volume.py:420-435
    dims = [f_in, *hidden, 1]
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for i, (a, b) in enumerate(zip(dims[:-1], dims[1:])):
        bound = 1.0 / math.sqrt(a)
        sd[f"mlp.net.{2 * i}.weight"] = (torch.rand(b, a, generator=g) * 2 - 1) * bound
        sd[f"mlp.net.{2 * i}.bias"] = (torch.rand(b, generator=g) * 2 - 1) * bound
    return sd


def to_device(tup: dict, device) -> dict:
    return {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in tup.items()}


def make_tsdf_case(seed: int = 0, frames: int = 2, voxel_size: float = 0.04, height: int = 192, width: int = 256,
                   room=(4.0, 3.0, 2.6), masked: bool = False) -> dict:
    """A synthetic fusion step for the dense-grid TSDF integration (reference tools/tsdf.py:221-320):
    `frames` depth maps of a box-shaped room seen from inside (ray-cast analytically, plus noise),
    intrinsics of a ScanNet-like camera at (height, width), world->camera extrinsics, and the
    volume bounds OurFuser would take from a mesh of that room (tools/tsdf.py:52-67)."""
    g = torch.Generator().manual_seed(4321 + seed)
    rx, ry, rz = room
    fx = SCANNET_FX * width / 640.0
    fy = SCANNET_FY * height / 480.0
    K = torch.eye(4, dtype=torch.float64)
    K[0, 0], K[1, 1], K[0, 2], K[1, 2] = fx, fy, SCANNET_CX * width / 640.0, SCANNET_CY * height / 480.0
    v, u = torch.meshgrid(torch.arange(height, dtype=torch.float64) + 0.5,
                          torch.arange(width, dtype=torch.float64) + 0.5, indexing="ij")
    rays_cam = torch.stack([(u - K[0, 2]) / fx, (v - K[1, 2]) / fy, torch.ones_like(u)], -1)   # z = 1
    depths, Es = [], []
    for _ in range(frames):
        pos = torch.tensor([rx, ry, rz], dtype=torch.float64) * (0.3 + 0.4 * torch.rand(3, generator=g, dtype=torch.float64))
        axis = torch.randn(3, generator=g, dtype=torch.float64)
        axis = axis / axis.norm()
        Rwc = _axis_angle(axis[None], (torch.rand(1, generator=g, dtype=torch.float64) * 3.0))[0]   # camera -> world
        d = rays_cam @ Rwc.T                                                 # ray directions in the world
        lo, hi = -pos, torch.tensor([rx, ry, rz], dtype=torch.float64) - pos
        t = torch.where(d > 0, hi / d.clamp_min(1e-12), lo / d.clamp_max(-1e-12))   # exit distance per axis
        depth = t.min(-1).values                                            # along z = 1 rays: depth itself
        depth = depth + 0.01 * torch.randn(depth.shape, generator=g, dtype=torch.float64)
        depths.append(depth.float())
        E = torch.eye(4, dtype=torch.float64)                                # world -> camera
        E[:3, :3] = Rwc.T
        E[:3, 3] = -(Rwc.T @ pos)
        Es.append(E.float())
    depth = torch.stack(depths)[:, None]
    mask = (torch.rand(depth.shape, generator=g) > 0.1) if masked else None
    pad = 3 * voxel_size
    bounds = {"xmin": -pad, "xmax": rx + pad, "ymin": -pad, "ymax": ry + pad, "zmin": -pad, "zmax": rz + pad}
    return dict(depth=depth, cam_T_world=torch.stack(Es), K=K.float().repeat(frames, 1, 1), mask=mask,
                bounds=bounds, voxel_size=voxel_size, max_depth=3.0)


def make_mvs_scene(seed: int = 0, frames: int = 8, height: int = 96, width: int = 128, room=(4.0, 3.0, 2.6),
                   noise: float = 0.005) -> dict:
    """A synthetic scan for the multi-view depth-consistency fusion (reference
    tools/torch_point_cloud_fusion.py): `frames` views of a box-shaped room from nearby poses (so the
    frusta overlap), each with its analytically ray-cast depth map (pixel (x, y) is the ray through
    integer coordinates, as the fuser's un-projection assumes, :29-35), 3x3 intrinsics, world->camera
    poses and random uint8 images.  A few depth pixels are zeroed (invalid predictions)."""
    g = torch.Generator().manual_seed(9876 + seed)
    rx, ry, rz = room
    fx, fy = SCANNET_FX * width / 640.0, SCANNET_FY * height / 480.0
    K = torch.eye(3, dtype=torch.float64)
    K[0, 0], K[1, 1], K[0, 2], K[1, 2] = fx, fy, SCANNET_CX * width / 640.0, SCANNET_CY * height / 480.0
    v, u = torch.meshgrid(torch.arange(height, dtype=torch.float64), torch.arange(width, dtype=torch.float64),
                          indexing="ij")
    rays_cam = torch.stack([(u - K[0, 2]) / fx, (v - K[1, 2]) / fy, torch.ones_like(u)], -1)
    centre = torch.tensor([rx, ry, rz], dtype=torch.float64) * 0.5
    base_axis = torch.randn(3, generator=g, dtype=torch.float64)
    base_axis = base_axis / base_axis.norm()
    base_R = _axis_angle(base_axis[None], torch.rand(1, generator=g, dtype=torch.float64) * 3.0)[0]
    depths, Ps = [], []
    for _ in range(frames):
        pos = centre + 0.35 * (torch.rand(3, generator=g, dtype=torch.float64) - 0.5) * torch.tensor([rx, ry, rz])
        ax = torch.randn(3, generator=g, dtype=torch.float64)
        Rwc = base_R @ _axis_angle((ax / ax.norm())[None], torch.rand(1, generator=g, dtype=torch.float64) * 0.35)[0]
        d = rays_cam @ Rwc.T
        lo, hi = -pos, torch.tensor([rx, ry, rz], dtype=torch.float64) - pos
        t = torch.where(d > 0, hi / d.clamp_min(1e-12), lo / d.clamp_max(-1e-12))
        depth = t.min(-1).values + noise * torch.randn(height, width, generator=g, dtype=torch.float64)
        depth[torch.rand(height, width, generator=g) < 0.02] = 0.0
        depths.append(depth.float())
        E = torch.eye(4, dtype=torch.float64)
        E[:3, :3] = Rwc.T
        E[:3, 3] = -(Rwc.T @ pos)
        Ps.append(E.float())
    images = torch.randint(0, 256, (frames, height, width, 3), generator=g, dtype=torch.uint8)
    return dict(depths=torch.stack(depths), cam_T_world=torch.stack(Ps), K=K.float().repeat(frames, 1, 1),
                images=images)


def make_mvloss_batch(seed: int = 0, batch: int = 2, views: int = 3, height: int = 48, width: int = 64,
                      pred_noise: float = 0.05) -> dict:
    """Inputs of the multi-view depth regression loss (reference losses.py:180-190, called from
    experiment_modules/depth_model.py:477-485): per batch item a reference frame with its ground-truth
    depth and `views` source frames of the same synthetic room scan, 4x4 intrinsics / poses, and a
    predicted depth = ground truth x exp(noise) (positive, as the model's exp head produces)."""
    g = torch.Generator().manual_seed(4242 + seed)
    cur_d, src_d, invK, srcK, wTc, scTw, pred = [], [], [], [], [], [], []
    for b in range(batch):
        sc = make_mvs_scene(seed=seed * 131 + b, frames=views + 1, height=height, width=width)
        K4 = torch.eye(4).repeat(views + 1, 1, 1)
        K4[:, :3, :3] = sc["K"]
        cur_d.append(sc["depths"][0][None])
        src_d.append(sc["depths"][1:][:, None])
        invK.append(torch.inverse(K4[0]))
        srcK.append(K4[1:])
        wTc.append(torch.inverse(sc["cam_T_world"][0]))
        scTw.append(sc["cam_T_world"][1:])
        pred.append((sc["depths"][0].clamp_min(0.05) * torch.exp(pred_noise * torch.randn(height, width, generator=g)))[None])
    return dict(depth_pred_b1hw=torch.stack(pred), cur_depth_b1hw=torch.stack(cur_d), src_depth_bk1hw=torch.stack(src_d),
                cur_invK_b44=torch.stack(invK), src_K_bk44=torch.stack(srcK), cur_world_T_cam_b44=torch.stack(wTc),
                src_cam_T_world_bk44=torch.stack(scTw))


# one base colour per wall of the ray-cast room: x = 0, x = rx, y = 0, y = ry, z = 0, z = rz
ROOM_WALL_COLORS = ((0.85, 0.25, 0.20), (0.20, 0.70, 0.30), (0.25, 0.35, 0.90),
                    (0.90, 0.80, 0.20), (0.70, 0.30, 0.80), (0.20, 0.80, 0.85))
ROOM_CHECKER_M = 0.5          # checker cell size in world metres
IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def room_wall_color(points: torch.Tensor, room=(4.0, 3.0, 2.6)):
    """Analytic colour of the room's walls at world points (N,3) (float64): the nearest wall's base colour
    times a world-space checker (1.0 / 0.6) in the wall's two in-plane coordinates.  Returns (rgb (N,3),
    wall index (N,), distance to the nearest wall edge (N,), distance to the nearest checker line (N,))."""
    p = points.double()
    ext = torch.tensor(room, dtype=torch.float64)
    d = torch.cat([p, ext - p], 1).abs()                                  # distance to walls 0..5 (x0, y0, z0, x1, ...)
    wall6 = d.argmin(1)
    axis = wall6 % 3
    wall = 2 * axis + wall6 // 3                                          # ROOM_WALL_COLORS order
    other = torch.stack([torch.tensor([1, 2]), torch.tensor([0, 2]), torch.tensor([0, 1])])[axis]   # (N, 2)
    q = torch.gather(p, 1, other)                                         # in-plane coordinates
    qe = torch.gather(ext.expand_as(p), 1, other)
    edge = torch.minimum(q, qe - q).abs().min(1).values
    cell = torch.floor(q / ROOM_CHECKER_M)
    checker = torch.where((cell.sum(1) % 2) == 0, 1.0, 0.6).double()
    frac = q / ROOM_CHECKER_M - cell
    line = (torch.minimum(frac, 1 - frac) * ROOM_CHECKER_M).min(1).values
    rgb = torch.tensor(ROOM_WALL_COLORS, dtype=torch.float64)[wall] * checker[:, None]
    return rgb, wall, edge, line


def make_color_tsdf_case(seed: int = 0, frames: int = 2, voxel_size: float = 0.04, height: int = 192,
                         width: int = 256, color_hw=(288, 384), room=(4.0, 3.0, 2.6), masked: bool = False) -> dict:
    """make_tsdf_case (same depth maps, poses and RNG stream) plus colour frames of the same views at
    ``color_hw``: each pixel's ray through its centre hits a wall whose analytic colour is
    room_wall_color.  ``color`` is ImageNet-normalised as the dataloader hands images out (B,3,Hc,Wc);
    ``color_raw`` is the same in [0, 1]."""
    c = make_tsdf_case(seed=seed, frames=frames, voxel_size=voxel_size, height=height, width=width, room=room,
                       masked=masked)
    Hc, Wc = color_hw
    fx, fy = SCANNET_FX * Wc / 640.0, SCANNET_FY * Hc / 480.0
    cx, cy = SCANNET_CX * Wc / 640.0, SCANNET_CY * Hc / 480.0
    v, u = torch.meshgrid(torch.arange(Hc, dtype=torch.float64) + 0.5, torch.arange(Wc, dtype=torch.float64) + 0.5,
                          indexing="ij")
    rays = torch.stack([(u - cx) / fx, (v - cy) / fy, torch.ones_like(u)], -1).reshape(-1, 3)
    ext = torch.tensor(room, dtype=torch.float64)
    imgs = []
    for E in c["cam_T_world"].double():
        Rwc = E[:3, :3].T
        pos = -(Rwc @ E[:3, 3])
        d = rays @ Rwc.T
        t = torch.where(d > 0, (ext - pos) / d.clamp_min(1e-12), -pos / d.clamp_max(-1e-12)).min(-1).values
        rgb, _, _, _ = room_wall_color(pos + t[:, None] * d, room)
        imgs.append(rgb.reshape(Hc, Wc, 3).permute(2, 0, 1).float())
    raw = torch.stack(imgs)
    mean = torch.tensor(IMAGENET_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD).view(1, 3, 1, 1)
    return dict(c, color=((raw - mean) / std).contiguous(), color_raw=raw.contiguous())
