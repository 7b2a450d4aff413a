"""Multi-view depth-consistency point-cloud fusion, backed by the sm_90a kernel.

Mirrors the reference's ``tools/torch_point_cloud_fusion.py`` — ``process_depth`` (:12-97) and
``process_scene`` (:100-118), the 3DVNet-style fuser ``pc_fusion.py:158`` calls — with the same
names, argument meaning and return values (numpy arrays of the consistent points, their colours
and the per-pixel validity), so ``pc_fusion.py`` can import this module in its place.

One launch per reference frame walks every source frame in registers (the reference materialises
(n_src, 3, H*W) tensors several times over per batch of 100 sources).  CUDA tensors on an sm_90
device, or an exception: there is no CPU path.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _native


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
        lib = _native.load()
        dev = self.depths.device
        with torch.cuda.device(dev):
            pts = torch.empty(self.H * self.W, 3, device=dev, dtype=torch.float32)
            nv = torch.empty(self.H * self.W, device=dev, dtype=torch.int32)
            valid = torch.empty(self.H * self.W, device=dev, dtype=torch.uint8)
            _native.check(lib.srcv_mvs_consistency_f32(
                C.byref(self.desc), int(ref_index), float(z_thresh), int(n_consistent_thresh),
                C.c_void_p(pts.data_ptr()), C.c_void_p(nv.data_ptr()), C.c_void_p(valid.data_ptr()),
                C.c_void_p(self.ws.data_ptr()), self.ws_bytes, int(self.staged),
                C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        self.staged = True
        return pts, nv, valid.view(self.H, self.W).bool()


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
