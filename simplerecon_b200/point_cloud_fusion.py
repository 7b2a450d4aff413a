"""Multi-view depth-consistency point-cloud fusion, backed by the sm_90a kernel.

Mirrors the reference's ``tools/torch_point_cloud_fusion.py`` — ``process_depth`` (:12-97) and
``process_scene`` (:100-118), the 3DVNet-style fuser ``pc_fusion.py:158`` calls — with the same
names, argument meaning and return values (numpy arrays of the consistent points, their colours
and the per-pixel validity), so ``pc_fusion.py`` can import this module in its place.

One launch per reference frame walks every source frame in registers (the reference materialises
(n_src, 3, H*W) tensors several times over per batch of 100 sources).  CUDA tensors on an sm_90
device, or an exception: there is no CPU path.

``voxel_down_sample`` is the last step of ``pc_fusion.py`` (:166-169, Open3D's ``voxel_down_sample``) on the
GPU (csrc/srcv_voxel_downsample.cuh, DESIGN §4.19), and ``fuse_point_cloud`` runs ``pc_fusion.py:158-169`` —
the consistency of every frame, then the down-sampling — on the device, with two host synchronisations.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _native
from . import mesh_eval as _me


def _require_cuda(t: torch.Tensor) -> None:
    """The device gate (tests/ patch exactly this to drive the host-emulated library)."""
    if t.device.type != "cuda":
        raise RuntimeError("simplerecon_b200 point-cloud fusion runs on CUDA (sm_90a) only; there is no CPU fallback")


class _Scan:
    """Device-resident scan: depths, intrinsics, poses and their inverses (inverted ONCE per scan;
    the reference inverts per reference frame, :25-27), plus the kernel's staged workspace."""

    def __init__(self, depths_nhw, poses_n44, K_n33, device):
        f = lambda t: t.to(device=device, dtype=torch.float32).contiguous()
        self.depths, self.P, self.K = f(depths_nhw), f(poses_n44), f(K_n33)
        self.K_inv, self.P_inv = torch.inverse(self.K).contiguous(), torch.inverse(self.P).contiguous()
        self.N, self.H, self.W = (int(x) for x in self.depths.shape)
        self.desc = _native.MvsScan(self.depths.data_ptr(), self.K.data_ptr(), self.K_inv.data_ptr(),
                                    self.P.data_ptr(), self.P_inv.data_ptr(), self.N, self.H, self.W)
        lib = _native.load()
        n = lib.srcv_mvs_workspace_bytes(C.byref(self.desc))
        self.ws = torch.empty(n, device=device, dtype=torch.uint8)
        self.ws_bytes = n
        self.staged = False

    def consistency(self, ref_index: int, z_thresh: float, n_consistent_thresh: int):
        """-> pts_avg (H*W,3) fp32, n_valid (H*W) int32, valid (H,W) bool — device tensors."""
        dev = self.depths.device
        pts = torch.empty(self.H * self.W, 3, device=dev, dtype=torch.float32)
        nv = torch.empty(self.H * self.W, device=dev, dtype=torch.int32)
        valid = torch.empty(self.H * self.W, device=dev, dtype=torch.uint8)
        self.consistency_into(ref_index, z_thresh, n_consistent_thresh, pts, nv, valid)
        return pts, nv, valid.view(self.H, self.W).bool()

    def consistency_into(self, ref_index: int, z_thresh: float, n_consistent_thresh: int, pts, nv, valid) -> None:
        """The consistency of frame ``ref_index`` into contiguous device views pts (H*W,3) fp32, nv (H*W) int32
        and valid (H*W) uint8.  No host synchronisation."""
        lib = _native.load()
        dev = self.depths.device
        with torch.cuda.device(dev):
            _native.check(lib.srcv_mvs_consistency_f32(
                C.byref(self.desc), int(ref_index), float(z_thresh), int(n_consistent_thresh),
                C.c_void_p(pts.data_ptr()), C.c_void_p(nv.data_ptr()), C.c_void_p(valid.data_ptr()),
                C.c_void_p(self.ws.data_ptr()), self.ws_bytes, int(self.staged),
                C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        self.staged = True


def process_depth(ref_depth, ref_image, src_depths, src_images, ref_P, src_Ps, ref_K, src_Ks, z_thresh=0.1,
                  n_consistent_thresh=3):
    """reference :12-97.  ``src_images`` is accepted and unused, as in the reference."""
    _require_cuda(ref_depth if ref_depth.is_cuda else src_depths)
    dev = ref_depth.device if ref_depth.is_cuda else src_depths.device
    scan = _Scan(torch.cat([ref_depth.to(dev)[None], src_depths.to(dev)], 0),
                 torch.cat([ref_P.to(dev)[None], src_Ps.to(dev)], 0),
                 torch.cat([ref_K.to(dev)[None], src_Ks.to(dev)], 0), dev)
    pts, _, valid = scan.consistency(0, z_thresh, n_consistent_thresh)
    pts_filtered = pts[valid.reshape(-1)].cpu().numpy()
    rgb_filtered = ref_image.to(dev)[valid].view(-1, 3).cpu().numpy()
    return pts_filtered, rgb_filtered, valid.cpu().numpy()


def process_scene(depth_preds, images, poses, K, z_thresh, n_consistent_thresh):
    """reference :100-118: every frame of the scan against all the others."""
    dev = depth_preds.device
    _require_cuda(depth_preds)
    scan = _Scan(depth_preds, poses, K, dev)
    images = images.to(dev)
    fused_pts, fused_rgb, all_valid = [], [], []
    for ref_idx in range(scan.N):
        pts, _, valid = scan.consistency(ref_idx, z_thresh, n_consistent_thresh)
        fused_pts.append(pts[valid.reshape(-1)].cpu().numpy())
        fused_rgb.append(images[ref_idx][valid].view(-1, 3).cpu().numpy())
        all_valid.append(valid.cpu().numpy())
    return np.concatenate(fused_pts, axis=0), np.concatenate(fused_rgb, axis=0), np.stack(all_valid, axis=0)


def voxel_down_sample(points, voxel_size: float, colors=None):
    """Open3D's ``PointCloud.voxel_down_sample`` on the GPU: ``(points (M,3) fp32, colors (M,3) fp32 or None,
    counts (M,) int32)``, device tensors that are slices of (N, ...) buffers.

    ``points`` (N,3) float32 or float64 (taken to fp32), ``colors`` None or (N,3) uint8, float32 or float64, CUDA
    tensors or numpy arrays (moved to the current CUDA device).  In fp64 from the fp32 points and the voxel size s:
    per axis b = min_i p_i - 0.5 s, and point p lies in voxel v = floor((p - b) / s) (an IEEE subtraction and
    division).  Each occupied voxel gives one point, the fp64 sum of its points accumulated in input order from 0.0,
    divided by their count and rounded once to fp32, and its point count; colours are averaged the same way, uint8
    taken as c / 255.0 in fp64 (what ``pc_fusion.py`` hands Open3D) and floats as given.  Voxels come out in
    ascending (vx, vy, vz) order, so the result is bitwise deterministic and does not depend on the input order
    beyond the order of each voxel's sum.  Parity with Open3D holds for this rule, as sets: Open3D's order is that
    of a hash map.

    ``ValueError`` for: a voxel size that is not finite or not > 0; no point, or more than 2^28; ``colors`` not
    (N,3); a non-finite coordinate or colour; 2^21 or more voxels along an axis.  One host synchronisation, which
    reads M with the device's flag word."""
    s = _me._check_voxel_size(voxel_size)
    p = _me._coords(points, "points")
    c = None if colors is None else _me._colors(colors, p)
    flags = torch.zeros(1, dtype=torch.int32, device=p.device)
    out, out_c, counts, num_out = _me._down_sample(p, s, flags, c)
    m, bad = torch.cat([num_out, flags.to(torch.int64)]).tolist()   # the one host synchronisation
    _me._raise_flags(bad, "voxel_down_sample")
    return out[:m], (out_c[:m] if out_c is not None else None), counts[:m]


def fuse_point_cloud(depth_preds, images, poses, K, z_thresh=0.04, n_consistent_thresh=3, voxel_size=0.02):
    """``pc_fusion.py:158-169`` on the device: ``process_scene``'s consistency for every frame, then
    ``voxel_down_sample`` at ``voxel_size`` of the consistent points and their colours.  Returns
    ``(points (M,3) fp32, colors (M,3) fp32, counts (M,) int32)`` as device tensors, bitwise equal to
    ``voxel_down_sample`` of ``process_scene``'s concatenated points and colours.

    ``images`` (N,H,W,3) uint8 (taken as c / 255, as ``pc_fusion.py`` does) or float32 (as given).  Each frame's
    consistent points are gathered in pixel order with the in-order compaction of mesh evaluation, frames in
    order, into one device buffer: no per-frame host copy.  Two host synchronisations: the gathered count, and
    the down-sampling's."""
    s = _me._check_voxel_size(voxel_size)
    _require_cuda(depth_preds)
    dev = depth_preds.device
    scan = _Scan(depth_preds, poses, K, dev)
    images = images.to(dev)
    if tuple(images.shape) != (scan.N, scan.H, scan.W, 3):
        raise ValueError(f"images must be ({scan.N}, {scan.H}, {scan.W}, 3), got {tuple(images.shape)}")
    if images.dtype not in (torch.uint8, torch.float32):
        raise ValueError(f"images must be uint8 or float32, got {images.dtype}")
    HW = scan.H * scan.W
    chunk = max(1, _me._MAX_POINTS // HW)                  # frames per compaction (at most 2^28 pixels)
    flags = torch.zeros(1, dtype=torch.int32, device=dev)
    num_kept = torch.zeros(2 * ((scan.N + chunk - 1) // chunk), dtype=torch.int64, device=dev)
    nv = torch.empty(HW, dtype=torch.int32, device=dev)
    kept = []
    for k, f0 in enumerate(range(0, scan.N, chunk)):
        nf = min(chunk, scan.N - f0)
        pts = torch.empty(nf * HW, 3, dtype=torch.float32, device=dev)
        valid = torch.empty(nf * HW, dtype=torch.uint8, device=dev)
        for f in range(nf):
            scan.consistency_into(f0 + f, z_thresh, n_consistent_thresh, pts[f * HW:(f + 1) * HW], nv,
                                  valid[f * HW:(f + 1) * HW])
        counts = valid.to(torch.int32)
        rgb = images[f0:f0 + nf].reshape(nf * HW, 3).to(torch.float32)   # uint8 values are exact in fp32
        kept.append((_me._compact(pts, counts, flags, num_kept[2 * k:2 * k + 1]),
                     _me._compact(rgb, counts, flags, num_kept[2 * k + 1:2 * k + 2])))
    m = num_kept.tolist()                                  # host synchronisation 1
    P = torch.cat([p[:m[2 * k]] for k, (p, _) in enumerate(kept)])
    rgb = torch.cat([c[:m[2 * k]] for k, (_, c) in enumerate(kept)])
    if images.dtype == torch.uint8:
        rgb = rgb.to(torch.uint8)
    return voxel_down_sample(P, s, rgb)                    # host synchronisation 2
