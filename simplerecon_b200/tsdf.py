"""Dense-grid TSDF fusion of predicted depth maps, backed by the sm_90a kernel.

Mirrors the reference's ``tools/tsdf.py`` — ``TSDF`` (:11-170, the volume and its bounds
arithmetic) and ``TSDFFuser`` (:173-320, ``integrate_depth``) — as ``OurFuser.fuse_frames``
uses them (``tools/fusers_helper.py:22-71``): same constructor / method names, argument
meaning and fp16 state, so ``test.py:321-373`` can fuse through this class unchanged.  Mesh
extraction (marching cubes, trimesh export, :132-169) is host post-processing and stays the
reference's.

Differences, by design: ``voxel_coords`` is not stored (the kernel recomputes the 6 bytes per
voxel from the grid index; the property materialises it on demand), a batch of frames is ONE
launch (frames are applied in order inside the kernel), and there is no CPU path: CUDA tensors
on an sm_90 device, or an exception.
"""
from __future__ import annotations

import ctypes as C
from typing import Tuple

import numpy as np
import torch

from . import _native


class TSDF:
    """Volume container (reference tools/tsdf.py:11-130)."""

    VOX_MOD = 8   # final voxel volume dimensions are multiples of 8 (:17)

    def __init__(self, tsdf_values: torch.Tensor, tsdf_weights: torch.Tensor, voxel_size: float,
                 origin: torch.Tensor):
        self.tsdf_values = tsdf_values.half().contiguous()
        self.tsdf_weights = tsdf_weights.half().contiguous()
        self.voxel_size = float(voxel_size)
        self.origin = origin.float()          # kept in fp32: the coordinates are built in fp32 and then halved (:99-110, :92)

    @classmethod
    def from_bounds(cls, bounds: dict, voxel_size: float, device="cuda"):
        """-1 / 0 initialised volume covering ``bounds`` (:70-97)."""
        for key in ("xmin", "xmax", "ymin", "ymax", "zmin", "zmax"):
            if key not in bounds:
                raise KeyError("Provided bounds dict need to have keys 'xmin', 'xmax', 'ymin', 'ymax', 'zmin', 'zmax'!")
        dims = tuple(int(np.ceil((bounds[a + "max"] - bounds[a + "min"]) / voxel_size / cls.VOX_MOD)) * cls.VOX_MOD
                     for a in "xyz")
        origin = torch.tensor([bounds["xmin"], bounds["ymin"], bounds["zmin"]], dtype=torch.float32)
        values = -torch.ones(dims, dtype=torch.float16, device=device)
        weights = torch.zeros(dims, dtype=torch.float16, device=device)
        return cls(values, weights, voxel_size, origin)

    @classmethod
    def generate_voxel_coords(cls, origin: torch.Tensor, volume_dims: Tuple[int, int, int], voxel_size: float):
        """World coordinates of every voxel, (3,X,Y,Z) (:99-110)."""
        grid = torch.meshgrid([torch.arange(vd, device=origin.device) for vd in volume_dims], indexing="ij")
        return origin.view(3, 1, 1, 1) + torch.stack(grid, 0) * voxel_size

    @property
    def voxel_coords(self) -> torch.Tensor:
        """fp16 (3,X,Y,Z), materialised on demand (the kernel does not read it)."""
        return self.generate_voxel_coords(self.origin.to(self.tsdf_values.device), tuple(self.tsdf_values.shape),
                                          self.voxel_size).half()

    def cuda(self):
        self.tsdf_values = self.tsdf_values.cuda()
        self.tsdf_weights = self.tsdf_weights.cuda()
        return self

    def cpu(self):
        self.tsdf_values = self.tsdf_values.cpu()
        self.tsdf_weights = self.tsdf_weights.cpu()
        return self


def _require_cuda(t: torch.Tensor) -> None:
    """The device gate of the fuser (tests/ patch exactly this to drive the host-emulated library)."""
    if t.device.type != "cuda":
        raise RuntimeError("simplerecon_b200 TSDF fusion runs on CUDA (sm_90a) only; there is no CPU fallback")


class TSDFFuser:
    """Fuses depth maps into a TSDF volume (reference tools/tsdf.py:173-320)."""

    def __init__(self, tsdf: TSDF, min_depth: float = 0.5, max_depth: float = 5.0, use_gpu: bool = True):
        if not use_gpu:
            raise RuntimeError("use_gpu=False: this fuser has no CPU path")
        self.tsdf = tsdf
        self.min_depth = min_depth
        self.max_depth = max_depth
        self.use_gpu = use_gpu
        self.truncation_size = 3.0
        self.maxW = 100.0

    voxel_coords = property(lambda self: self.tsdf.voxel_coords)
    tsdf_values = property(lambda self: self.tsdf.tsdf_values)
    tsdf_weights = property(lambda self: self.tsdf.tsdf_weights)
    voxel_size = property(lambda self: self.tsdf.voxel_size)
    shape = property(lambda self: self.tsdf.tsdf_values.shape)
    truncation = property(lambda self: self.truncation_size * self.voxel_size)

    @torch.no_grad()
    def integrate_depth(self, depth_b1hw: torch.Tensor, cam_T_world_T_b44: torch.Tensor, K_b44: torch.Tensor,
                        depth_mask_b1hw: torch.Tensor | None = None) -> None:
        """In-place update of the volume with a batch of depth maps, applied in order (:221-320).
        Inputs are taken to fp16 as ``OurFuser.fuse_frames`` does (fusers_helper.py:64-71)."""
        values, weights = self.tsdf.tsdf_values, self.tsdf.tsdf_weights
        _require_cuda(values)
        dev = values.device
        lib = _native.load()
        B, _, H, W = depth_b1hw.shape
        depth = depth_b1hw.to(dev).half().contiguous()
        E = cam_T_world_T_b44.to(dev).half().contiguous()
        K = K_b44.to(dev).half().contiguous()
        mask = None
        if depth_mask_b1hw is not None:
            mask = depth_mask_b1hw.to(dev).to(torch.uint8).contiguous()
        vol = _native.TsdfVolume()
        vol.tsdf_values, vol.tsdf_weights = values.data_ptr(), weights.data_ptr()
        vol.X, vol.Y, vol.Z = (int(d) for d in values.shape)
        for i in range(3):
            vol.origin[i] = float(self.tsdf.origin[i])
        vol.voxel_size, vol.truncation_voxels, vol.max_weight = self.voxel_size, self.truncation_size, self.maxW
        fr = _native.TsdfFrames(depth.data_ptr(), E.data_ptr(), K.data_ptr(),
                                mask.data_ptr() if mask is not None else None, B, H, W,
                                float(self.min_depth), float(self.max_depth))
        with torch.cuda.device(dev):
            n = lib.srcv_tsdf_workspace_bytes(C.byref(fr))
            ws = torch.empty(n, device=dev, dtype=torch.uint8)
            _native.check(lib.srcv_tsdf_integrate_f16(
                C.byref(vol), C.byref(fr), C.c_void_p(ws.data_ptr()), n,
                C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
