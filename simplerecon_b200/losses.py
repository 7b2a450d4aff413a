"""The training losses of the reference's ``losses.py``, backed by the sm_90a kernels: ``MVDepthLoss`` (below),
``MSGradientLoss`` and ``ScaleInvariantLoss`` (csrc/srcv_gradloss.cuh, DESIGN §4.14; at the end of this module).
``NormalsLoss`` lives in ``normals.py`` with the generator it consumes.

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
        raise RuntimeError("simplerecon_b200 losses run on CUDA (sm_90a) only; there is no CPU fallback")


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


def _msgrad_forward(depth_gt: torch.Tensor, depth_pred: torch.Tensor, num_scales: int):
    """(loss, workspace) of dense fp32 inputs.  The workspace starts with the four int64 counts of masked
    gradient components per level and keeps both pyramids for the backward (include/srcv_b200.h)."""
    B, _, H, W = depth_gt.shape
    dev = depth_gt.device
    n = _lib().srcv_msgrad_workspace_bytes(B, H, W, num_scales)
    if n == 0:
        raise ValueError(f"unsupported depth shape {tuple(depth_gt.shape)} (B <= 65535, B H W < 2^30)")
    ws = torch.empty(n, device=dev, dtype=torch.uint8)
    loss = torch.empty((), device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _native.check(_lib().srcv_msgrad_forward_f32(
            C.c_void_p(depth_gt.data_ptr()), C.c_void_p(depth_pred.data_ptr()), B, H, W, num_scales,
            C.c_void_p(loss.data_ptr()), C.c_void_p(ws.data_ptr()), n, _stream(dev)))
    return loss, ws


class _MsGradFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth_gt, depth_pred, num_scales):
        gt, pred = _f32c(depth_gt), _f32c(depth_pred)
        loss, ws = _msgrad_forward(gt, pred, num_scales)
        ctx.save_for_backward(gt, pred, ws)     # the workspace keeps the pyramids and the per-level counts
        ctx.num_scales = num_scales
        ctx.pred_dtype = depth_pred.dtype
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        gt, pred, ws = ctx.saved_tensors
        B, _, H, W = gt.shape
        dev = gt.device
        g = _f32c(grad_loss).reshape(1)
        out = torch.empty_like(pred)
        with torch.cuda.device(dev):
            _native.check(_lib().srcv_msgrad_backward_f32(
                C.c_void_p(gt.data_ptr()), C.c_void_p(pred.data_ptr()), B, H, W, ctx.num_scales,
                C.c_void_p(g.data_ptr()), C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                _stream(dev)))
        return None, out.to(ctx.pred_dtype), None


class MSGradientLoss(nn.Module):
    """reference losses.py:11-37 (Equation 3 of the paper): the sum over ``num_scales`` blur-pool pyramid levels
    of the mean absolute difference of the Sobel gradients, over the gradient components whose ground-truth
    window is finite.  Differentiable w.r.t. ``depth_pred`` only: ``depth_gt`` is data, as in ``MVDepthLoss``.
    Three launches forward, ``num_scales`` backward, no host synchronisation.  Half / bfloat16 inputs are
    computed in fp32; the loss is fp32 and the gradient comes back in the prediction's dtype."""

    MAX_SCALES = 4

    def __init__(self, num_scales: int = 4):
        super().__init__()
        if not 1 <= num_scales <= self.MAX_SCALES:
            raise ValueError(f"num_scales must be in [1, {self.MAX_SCALES}] (the pyramid kernel's depth), "
                             f"got {num_scales}")
        self.num_scales = num_scales

    def forward(self, depth_gt: torch.Tensor, depth_pred: torch.Tensor) -> torch.Tensor:
        _require_cuda(depth_pred)
        if depth_gt.dim() != 4 or depth_gt.shape[1] != 1 or depth_gt.shape != depth_pred.shape:
            raise ValueError(f"depths must both be (B, 1, H, W), got {tuple(depth_gt.shape)} and "
                             f"{tuple(depth_pred.shape)}")
        if depth_gt.device != depth_pred.device:
            raise ValueError(f"depths on {depth_gt.device} and {depth_pred.device}")
        return _MsGradFunction.apply(depth_gt, depth_pred, self.num_scales)


class _SiLossFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, log_depth_gt, log_depth_pred, si_lambda):
        gt, pred = _f32c(log_depth_gt), _f32c(log_depth_pred)
        dev, count = gt.device, gt.numel()
        n = _lib().srcv_si_loss_workspace_bytes(count)
        if n == 0:
            raise ValueError(f"unsupported input size {count} (at most 2^31 - 1 elements)")
        ws = torch.empty(n, device=dev, dtype=torch.uint8)
        loss = torch.empty((), device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            _native.check(_lib().srcv_si_loss_forward_f32(
                C.c_void_p(gt.data_ptr()), C.c_void_p(pred.data_ptr()), count, si_lambda,
                C.c_void_p(loss.data_ptr()), C.c_void_p(ws.data_ptr()), n, _stream(dev)))
        ctx.save_for_backward(gt, pred, ws)     # the workspace keeps mean(d) and the loss
        ctx.si_lambda = si_lambda
        ctx.dtypes = (log_depth_gt.dtype, log_depth_pred.dtype)
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        gt, pred, ws = ctx.saved_tensors
        dev = gt.device
        g = _f32c(grad_loss).reshape(1)
        g_gt = torch.empty_like(gt) if ctx.needs_input_grad[0] else None
        g_pred = torch.empty_like(pred) if ctx.needs_input_grad[1] else None
        with torch.cuda.device(dev):
            _native.check(_lib().srcv_si_loss_backward_f32(
                C.c_void_p(gt.data_ptr()), C.c_void_p(pred.data_ptr()), gt.numel(), ctx.si_lambda,
                C.c_void_p(g.data_ptr()), C.c_void_p(g_gt.data_ptr() if g_gt is not None else 0),
                C.c_void_p(g_pred.data_ptr() if g_pred is not None else 0), C.c_void_p(ws.data_ptr()), ws.numel(),
                _stream(dev)))
        return (g_gt.to(ctx.dtypes[0]) if g_gt is not None else None,
                g_pred.to(ctx.dtypes[1]) if g_pred is not None else None, None)


class ScaleInvariantLoss(nn.Module):
    """reference losses.py:39-54: ``sqrt(mean(d^2) - si_lambda mean(d)^2)`` with ``d = log_depth_gt -
    log_depth_pred``, any equal shape (the caller passes the 1-D ``x[mask_b]``, depth_model.py:468).  ``d`` is
    fp32, the sums and the formula fp64; NaN for a negative radicand or an empty input, as ``torch.sqrt`` and
    ``mean`` give.  Differentiable in both inputs.  Two launches forward, one backward."""

    def __init__(self, si_lambda: float = 0.85):
        super().__init__()
        self.si_lambda = si_lambda

    def forward(self, log_depth_gt: torch.Tensor, log_depth_pred: torch.Tensor) -> torch.Tensor:
        _require_cuda(log_depth_pred)
        if log_depth_gt.shape != log_depth_pred.shape:
            raise ValueError(f"shapes differ: {tuple(log_depth_gt.shape)} and {tuple(log_depth_pred.shape)}")
        if log_depth_gt.device != log_depth_pred.device:
            raise ValueError(f"inputs on {log_depth_gt.device} and {log_depth_pred.device}")
        return _SiLossFunction.apply(log_depth_gt, log_depth_pred, float(self.si_lambda))
