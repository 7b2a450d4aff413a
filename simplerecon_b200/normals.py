"""Surface normals from depth and the normals loss, backed by the sm_90a kernels
(csrc/srcv_normals.cuh, DESIGN §4.13).

Mirrors ``NormalGenerator`` of the reference's ``utils/geometry_utils.py`` (:92-133) and ``NormalsLoss`` of
its ``losses.py`` (:57-77): same constructors, same ``forward`` signatures, and ``NormalGenerator`` owns a
``backproject`` submodule, so the ``state_dict`` keys of a ``DepthModel`` (``compute_normals.backproject.
pix_coords_13N``) are unchanged and reference checkpoints load strictly.  ``NormalGenerator`` is one launch
forward and two backward (the backward recomputes from the depth, nothing but the inputs is saved);
``NormalsLoss`` is two launches forward and one backward, with no host synchronisation.

CUDA tensors on an sm_90 device, or an exception: there is no CPU path.  fp16 / bf16 depth (Lightning
``precision=16``) is computed in fp32 and the normals and gradients come back in the input dtype; the loss
is fp32, as the reference computes it with autocast off.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from . import _native
from .geometry import BackprojectDepth


def _require_cuda(t: torch.Tensor) -> None:
    """The device gate (tests/ patch exactly this to drive the host-emulated library)."""
    if t.device.type != "cuda":
        raise RuntimeError("simplerecon_b200 normals run on CUDA (sm_90a) only; there is no CPU fallback")


def _lib():
    return _native.load()


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _f32c(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.float32).contiguous()


def gaussian_taps(kernel_size: int, sigma: float) -> torch.Tensor:
    """kornia 0.6.7 ``gaussian(window_size, sigma)`` (the 1-D taps of ``gaussian_blur2d``), fp32, by its
    exact expression, so that the kernel blurs with the reference's bits."""
    x = torch.arange(kernel_size) - kernel_size // 2
    if kernel_size % 2 == 0:
        x = x + 0.5
    gauss = torch.exp(-x.pow(2.0) / float(2 * sigma ** 2))
    return gauss / gauss.sum()


class _NormalsCall:
    def __init__(self, depth, invK, taps, k):
        B, H, W = int(depth.shape[0]), int(depth.shape[-2]), int(depth.shape[-1])
        self.depth, self.invK = depth, invK
        self.taps = taps
        self.B, self.H, self.W = B, H, W
        self.args = _native.NormalsArgs(depth.data_ptr(), invK.data_ptr(), taps.data_ptr(), B, H, W, int(k))
        self.device = depth.device

    def forward(self) -> torch.Tensor:
        dev = self.device
        out = torch.empty(self.B, 3, self.H, self.W, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            _native.check(_lib().srcv_normals_forward_f32(C.byref(self.args), C.c_void_p(out.data_ptr()),
                                                          _stream(dev)))
        return out

    def backward(self, grad_normals: torch.Tensor) -> torch.Tensor:
        dev = self.device
        g = _f32c(grad_normals)
        out = torch.empty(self.B, 1, self.H, self.W, device=dev, dtype=torch.float32)
        n = _lib().srcv_normals_workspace_bytes(C.byref(self.args))
        ws = torch.empty(n, device=dev, dtype=torch.uint8)
        with torch.cuda.device(dev):
            _native.check(_lib().srcv_normals_backward_f32(
                C.byref(self.args), C.c_void_p(g.data_ptr()), C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()),
                n, _stream(dev)))
        return out


class _NormalsFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth, invK, taps, k):
        d, K = _f32c(depth), _f32c(invK)
        normals = _NormalsCall(d, K, taps, k).forward()
        ctx.save_for_backward(d, K, taps)     # the backward recomputes the chain from the depth
        ctx.k = k
        ctx.depth_dtype = depth.dtype
        return normals.to(depth.dtype)

    @staticmethod
    def backward(ctx, grad_normals):
        d, K, taps = ctx.saved_tensors
        g = _NormalsCall(d, K, taps, ctx.k).backward(grad_normals)
        return g.to(ctx.depth_dtype), None, None, None


class NormalGenerator(nn.Module):
    """reference utils/geometry_utils.py:92-133"""

    def __init__(self, height: int, width: int, smoothing_kernel_size: int = 5, smoothing_kernel_std: float = 2.0):
        super().__init__()
        self.height = height
        self.width = width
        # unused by the kernel (it forms the pixel rays itself); kept for the reference's state_dict keys
        self.backproject = BackprojectDepth(self.height, self.width)
        self.kernel_size = smoothing_kernel_size
        self.std = smoothing_kernel_std
        self.register_buffer("taps", gaussian_taps(smoothing_kernel_size, smoothing_kernel_std), persistent=False)

    def forward(self, depth_b1hw: torch.Tensor, invK_b44: torch.Tensor) -> torch.Tensor:
        _require_cuda(depth_b1hw)
        if depth_b1hw.dim() != 4 or depth_b1hw.shape[1] != 1 or \
                tuple(depth_b1hw.shape[-2:]) != (self.height, self.width):
            raise ValueError(f"depth_b1hw must be (B, 1, {self.height}, {self.width}), got {tuple(depth_b1hw.shape)}")
        B = depth_b1hw.shape[0]
        if tuple(invK_b44.shape) != (B, 4, 4):
            raise ValueError(f"invK_b44 must be ({B}, 4, 4), got {tuple(invK_b44.shape)}")
        if invK_b44.device != depth_b1hw.device:
            raise ValueError(f"depth on {depth_b1hw.device}, invK on {invK_b44.device}")
        taps = self.taps if self.taps.device == depth_b1hw.device else self.taps.to(depth_b1hw.device)
        return _NormalsFunction.apply(depth_b1hw, invK_b44, taps, self.kernel_size)


class _NormalsLossFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, normals_gt, normals_pred):
        gt, pred = _f32c(normals_gt), _f32c(normals_pred)
        B, _, H, W = gt.shape
        dev = gt.device
        n = _lib().srcv_normals_loss_workspace_bytes(B, H, W)
        if n == 0:
            raise ValueError(f"unsupported normals shape {tuple(gt.shape)}")
        ws = torch.empty(n, device=dev, dtype=torch.uint8)
        loss = torch.empty((), device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            _native.check(_lib().srcv_normals_loss_forward_f32(
                C.c_void_p(gt.data_ptr()), C.c_void_p(pred.data_ptr()), B, H, W, C.c_void_p(loss.data_ptr()),
                C.c_void_p(ws.data_ptr()), n, _stream(dev)))
        ctx.save_for_backward(gt, pred, ws)     # the workspace keeps the masked-pixel count
        ctx.dtypes = (normals_gt.dtype, normals_pred.dtype)
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        gt, pred, ws = ctx.saved_tensors
        B, _, H, W = gt.shape
        dev = gt.device
        g = _f32c(grad_loss).reshape(1)
        g_pred = torch.empty_like(pred)
        g_gt = torch.empty_like(gt) if ctx.needs_input_grad[0] else None
        with torch.cuda.device(dev):
            _native.check(_lib().srcv_normals_loss_backward_f32(
                C.c_void_p(gt.data_ptr()), C.c_void_p(pred.data_ptr()), B, H, W, C.c_void_p(g.data_ptr()),
                C.c_void_p(g_pred.data_ptr()), C.c_void_p(g_gt.data_ptr() if g_gt is not None else 0),
                C.c_void_p(ws.data_ptr()), ws.numel(), _stream(dev)))
        return (g_gt.to(ctx.dtypes[0]) if g_gt is not None else None), g_pred.to(ctx.dtypes[1])


class NormalsLoss(nn.Module):
    """reference losses.py:57-77"""

    def forward(self, normals_gt_b3hw: torch.Tensor, normals_pred_b3hw: torch.Tensor) -> torch.Tensor:
        _require_cuda(normals_pred_b3hw)
        if normals_gt_b3hw.dim() != 4 or normals_gt_b3hw.shape[1] != 3 or \
                normals_gt_b3hw.shape != normals_pred_b3hw.shape:
            raise ValueError(f"normals must both be (B, 3, H, W), got {tuple(normals_gt_b3hw.shape)} and "
                             f"{tuple(normals_pred_b3hw.shape)}")
        if normals_gt_b3hw.device != normals_pred_b3hw.device:
            raise ValueError(f"normals on {normals_gt_b3hw.device} and {normals_pred_b3hw.device}")
        return _NormalsLossFunction.apply(normals_gt_b3hw, normals_pred_b3hw)
