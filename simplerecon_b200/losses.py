"""Multi-view depth regression loss, backed by the sm_90a kernel.

Mirrors ``MVDepthLoss`` of the reference's ``losses.py`` (:79-208) — constructor ``(height, width)``,
``forward`` with the reference's keyword names (``experiment_modules/depth_model.py:477-485`` calls it
by keyword), ``get_valid_mask`` (:90-135) and ``get_error_for_pair`` (:138-178) — so ``depth_model``
can construct it in place of the reference class.  The loss is differentiable w.r.t.
``depth_pred_b1hw`` (the only input the reference's training graph reaches; the ground-truth depths
and the cameras are data).

One forward launch (+ a fixed-order finalize) walks all source views per pixel in registers; the
backward is one launch that recomputes the geometry.  CUDA tensors on an sm_90 device, or an
exception: there is no CPU path.  Half / bfloat16 inputs (Lightning ``precision=16``) are computed in
fp32, the gradient is returned in the prediction's dtype.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from . import _native


def _require_cuda(t: torch.Tensor) -> None:
    """The device gate (tests/ patch exactly this to drive the host-emulated library)."""
    if t.device.type != "cuda":
        raise RuntimeError("simplerecon_b200 MVDepthLoss runs on CUDA (sm_90a) only; there is no CPU fallback")


def _lib():
    return _native.load()


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _f32c(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.float32).contiguous()


class _Call:
    """The dense fp32 copies of one call's inputs and its C descriptor (kept alive together)."""

    def __init__(self, depth_pred, cur_depth, src_depth, cur_invK, src_K, cur_world_T_cam, src_cam_T_world):
        if src_depth.dim() == 4:          # one pair: (B,1,H,W) source depth, (B,4,4) matrices
            src_depth, src_K, src_cam_T_world = src_depth[:, None], src_K[:, None], src_cam_T_world[:, None]
        B, K = int(src_depth.shape[0]), int(src_depth.shape[1])
        H, W = int(cur_depth.shape[-2]), int(cur_depth.shape[-1])
        if tuple(depth_pred.shape) != (B, 1, H, W) or tuple(cur_depth.shape) != (B, 1, H, W) or \
                tuple(src_depth.shape) != (B, K, 1, H, W):
            raise ValueError(f"depth shapes do not agree: pred {tuple(depth_pred.shape)}, cur {tuple(cur_depth.shape)}, "
                             f"src {tuple(src_depth.shape)}")
        for name, m, shp in (("cur_invK_b44", cur_invK, (B, 4, 4)), ("src_K_bk44", src_K, (B, K, 4, 4)),
                             ("cur_world_T_cam_b44", cur_world_T_cam, (B, 4, 4)),
                             ("src_cam_T_world_bk44", src_cam_T_world, (B, K, 4, 4))):
            if tuple(m.shape) != shp:
                raise ValueError(f"{name} must be {shp}, got {tuple(m.shape)}")
        tensors = (depth_pred, cur_depth, src_depth, cur_invK, src_K, cur_world_T_cam, src_cam_T_world)
        if any(x.device != depth_pred.device for x in tensors):
            raise ValueError("MVDepthLoss inputs live on different devices: " + ", ".join(str(x.device) for x in tensors))
        self.t = [_f32c(x) for x in tensors]
        self.B, self.K, self.H, self.W = B, K, H, W
        self.args = _native.MvLossArgs(*[C.c_void_p(x.data_ptr()) for x in self.t], B, K, H, W)
        self.device = self.t[0].device
        n = _lib().srcv_mvloss_workspace_bytes(C.byref(self.args))
        self.ws = torch.empty(n, device=self.device, dtype=torch.uint8)

    def forward(self, want_masks: bool = False):
        dev = self.device
        loss = torch.empty((), device=dev, dtype=torch.float32)
        valid = torch.empty(self.B, self.K, self.H, self.W, device=dev, dtype=torch.uint8) if want_masks else None
        sampled = torch.empty(self.B, self.K, self.H, self.W, device=dev, dtype=torch.float32) if want_masks else None
        with torch.cuda.device(dev):
            _native.check(_lib().srcv_mvloss_forward_f32(
                C.byref(self.args), C.c_void_p(loss.data_ptr()),
                C.c_void_p(valid.data_ptr() if want_masks else 0), C.c_void_p(sampled.data_ptr() if want_masks else 0),
                C.c_void_p(self.ws.data_ptr()), self.ws.numel(), _stream(dev)))
        return loss, valid, sampled

    def backward(self, grad_loss: torch.Tensor) -> torch.Tensor:
        dev = self.device
        g = _f32c(grad_loss).reshape(1)
        out = torch.empty(self.B, 1, self.H, self.W, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            _native.check(_lib().srcv_mvloss_backward_f32(
                C.byref(self.args), C.c_void_p(g.data_ptr()), C.c_void_p(out.data_ptr()),
                C.c_void_p(self.ws.data_ptr()), self.ws.numel(), _stream(dev)))
        return out


class _MvLossFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth_pred, cur_depth, src_depth, cur_invK, src_K, cur_world_T_cam, src_cam_T_world):
        call = _Call(depth_pred, cur_depth, src_depth, cur_invK, src_K, cur_world_T_cam, src_cam_T_world)
        loss, _, _ = call.forward()
        ctx.call = call                     # dense fp32 inputs + the workspace with the per-view counts
        ctx.pred_dtype = depth_pred.dtype
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        g = ctx.call.backward(grad_loss)
        return g.to(ctx.pred_dtype), None, None, None, None, None, None


class MVDepthLoss(nn.Module):
    """reference losses.py:79-208"""

    def __init__(self, height, width):
        super().__init__()
        self.height = height
        self.width = width

    def get_valid_mask(self, cur_depth_b1hw, src_depth_b1hw, cur_invK_b44, src_K_b44, cur_world_T_cam_b44,
                       src_cam_T_world_b44):
        """reference :90-135 -> (valid_mask_b1hw bool, src_depth_sampled_b1hw)"""
        _require_cuda(cur_depth_b1hw)
        call = _Call(cur_depth_b1hw, cur_depth_b1hw, src_depth_b1hw, cur_invK_b44, src_K_b44, cur_world_T_cam_b44,
                     src_cam_T_world_b44)
        _, valid, sampled = call.forward(want_masks=True)
        return valid.bool(), sampled.to(src_depth_b1hw.dtype)

    def get_error_for_pair(self, depth_pred_b1hw, cur_depth_b1hw, src_depth_b1hw, cur_invK_b44, src_K_b44,
                           cur_world_T_cam_b44, src_cam_T_world_b44):
        """reference :138-178: the loss of ONE source view"""
        _require_cuda(depth_pred_b1hw)
        return _MvLossFunction.apply(depth_pred_b1hw, cur_depth_b1hw, src_depth_b1hw, cur_invK_b44, src_K_b44,
                                     cur_world_T_cam_b44, src_cam_T_world_b44)

    def forward(self, depth_pred_b1hw, cur_depth_b1hw, src_depth_bk1hw, cur_invK_b44, src_K_bk44,
                cur_world_T_cam_b44, src_cam_T_world_bk44):
        """reference :180-208: mean over the source views of the per-view whole-batch nanmean"""
        _require_cuda(depth_pred_b1hw)
        return _MvLossFunction.apply(depth_pred_b1hw, cur_depth_b1hw, src_depth_bk1hw, cur_invK_b44, src_K_bk44,
                                     cur_world_T_cam_b44, src_cam_T_world_bk44)
