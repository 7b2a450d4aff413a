"""The training losses of the reference's ``losses.py``, backed by the sm_90a kernels: ``MVDepthLoss`` (below),
``MSGradientLoss`` and ``ScaleInvariantLoss`` (csrc/srcv_gradloss.cuh, DESIGN §4.14).  ``NormalsLoss`` lives in
``normals.py`` with the generator it consumes.  At the end of this module, the regression terms the reference
computes inline in ``DepthModel.compute_losses`` (``depth_regression_losses``, csrc/srcv_regloss.cuh, DESIGN §4.15)
and a drop-in ``compute_losses`` built on all of them.

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


# ---- the regression terms of compute_losses (csrc/srcv_regloss.cuh, DESIGN §4.15) ---------------------------------

REGRESSION_KEYS = ("ms_loss", "abs_loss", "si_loss", "inv_abs_loss", "log_l1_loss")   # the kernel's output order
NUM_SCALES = 4                                                                         # log_depth_pred_s0..s3


def _regloss_call(gt, mask, depth_pred, log_preds, si_lambda):
    """(args, workspace) of dense inputs: fp32 depths, uint8 mask, log_preds a list of four fp32 tensors or None."""
    B, _, H, W = gt.shape
    hs = [int(t.shape[-2]) if t is not None else 0 for t in log_preds]
    ws_ = [int(t.shape[-1]) if t is not None else 0 for t in log_preds]
    args = _native.RegLossArgs(
        C.c_void_p(gt.data_ptr()), C.c_void_p(mask.data_ptr()), C.c_void_p(depth_pred.data_ptr()),
        (C.c_void_p * 4)(*[t.data_ptr() if t is not None else None for t in log_preds]),
        (C.c_int32 * 4)(*hs), (C.c_int32 * 4)(*ws_), B, H, W, si_lambda)
    n = _lib().srcv_regloss_workspace_bytes(C.byref(args))
    if n == 0:
        raise ValueError(f"unsupported shapes: depth {tuple(gt.shape)}, scales "
                         f"{[tuple(t.shape) if t is not None else None for t in log_preds]} "
                         "(B <= 65535, B H W < 2^30, every scale at least 1x1)")
    return args, torch.empty(n, device=gt.device, dtype=torch.uint8)


class _RegLossFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, depth_gt, mask_b, depth_pred, si_lambda, *log_preds):
        gt, dp = _f32c(depth_gt), _f32c(depth_pred)
        mask = mask_b.detach().contiguous().view(torch.uint8)
        lps = [_f32c(t) if t is not None else None for t in log_preds]
        args, ws = _regloss_call(gt, mask, dp, lps, si_lambda)
        dev = gt.device
        out = torch.empty(len(REGRESSION_KEYS), device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            _native.check(_lib().srcv_regloss_forward_f32(C.byref(args), C.c_void_p(out.data_ptr()),
                                                          C.c_void_p(ws.data_ptr()), ws.numel(), _stream(dev)))
        ctx.set_materialize_grads(False)     # an output autograd did not reach passes NULL: it adds nothing
        ctx.save_for_backward(gt, mask, dp, ws, *lps)   # the workspace keeps n, m, mean(d) and si
        ctx.args = args
        ctx.dtypes = (depth_pred.dtype, [t.dtype if t is not None else None for t in log_preds])
        return tuple(out.unbind(0))

    @staticmethod
    def backward(ctx, *grads):
        gt, mask, dp, ws, *lps = ctx.saved_tensors
        dev = gt.device
        ups = [_f32c(g) if g is not None else None for g in grads]
        want = ctx.needs_input_grad
        g_lp = [torch.empty_like(t) if t is not None and want[4 + i] else None for i, t in enumerate(lps)]
        g_dp = torch.empty_like(dp) if want[2] else None
        ptr = lambda t: t.data_ptr() if t is not None else None   # noqa: E731
        with torch.cuda.device(dev):
            _native.check(_lib().srcv_regloss_backward_f32(
                C.byref(ctx.args), (C.c_void_p * 5)(*map(ptr, ups)), (C.c_void_p * 4)(*map(ptr, g_lp)),
                C.c_void_p(ptr(g_dp)), C.c_void_p(ws.data_ptr()), ws.numel(), _stream(dev)))
        dp_dtype, lp_dtypes = ctx.dtypes
        return (None, None, g_dp.to(dp_dtype) if g_dp is not None else None, None,
                *[g.to(d) if g is not None else None for g, d in zip(g_lp, lp_dtypes)])


def depth_regression_losses(depth_gt_b1hw: torch.Tensor, mask_b_b1hw: torch.Tensor, log_depth_preds: dict,
                            depth_pred_b1hw: torch.Tensor, si_lambda: float = 0.85) -> dict:
    """The regression terms of the reference's ``DepthModel.compute_losses`` (experiment_modules/depth_model.py:
    447-474) in one fused call: ``dict(ms_loss, abs_loss, si_loss, inv_abs_loss, log_l1_loss)`` of fp32 0-d tensors.

    ``log_depth_preds`` maps a scale index (0..3) to ``log_depth_pred_s{i}_b1hw``; scale 0 is required and has the
    ground truth's (B, 1, H, W) shape, the others may be absent or any size (each is nearest-resampled to the ground
    truth, as ``F.interpolate`` does).  ``mask_b_b1hw`` is the boolean ``mask_b``.  ``ms_loss`` is the sum over the
    present scales i of the masked mean of ``|log gt - log_depth_pred_s{i}|`` / 2^i; ``si_loss`` uses ``si_lambda``;
    ``inv_abs_loss`` is over ``mask_b & (depth_pred > 0.1)``.  An empty mask gives NaN, as the mean of an empty
    tensor does.  Differentiable w.r.t. every ``log_depth_pred_s{i}`` and ``depth_pred`` (separate inputs, as in the
    reference, where ``depth_pred = exp(log_depth_pred_s0)`` is its own autograd node); the ground truth is data.
    Two launches forward, one backward, no host synchronisation.  Half / bfloat16 inputs are computed in fp32; the
    losses are fp32 and gradients come back in each input's dtype."""
    _require_cuda(depth_gt_b1hw)
    if depth_gt_b1hw.dim() != 4 or depth_gt_b1hw.shape[1] != 1:
        raise ValueError(f"depth_gt_b1hw must be (B, 1, H, W), got {tuple(depth_gt_b1hw.shape)}")
    shape = depth_gt_b1hw.shape
    if set(log_depth_preds) - set(range(NUM_SCALES)):
        raise ValueError(f"scale indices must be in 0..{NUM_SCALES - 1}, got {sorted(log_depth_preds)}")
    if 0 not in log_depth_preds:
        raise ValueError("log_depth_preds needs scale 0")
    for name, t in (("mask_b_b1hw", mask_b_b1hw), ("depth_pred_b1hw", depth_pred_b1hw), ("scale 0", log_depth_preds[0])):
        if t.shape != shape:
            raise ValueError(f"{name} must have the ground truth's shape {tuple(shape)}, got {tuple(t.shape)}")
    if mask_b_b1hw.dtype != torch.bool:
        raise ValueError(f"mask_b_b1hw must be bool, got {mask_b_b1hw.dtype}")
    lps = [log_depth_preds.get(i) for i in range(NUM_SCALES)]
    for i, t in enumerate(lps):
        if t is not None and (t.dim() != 4 or t.shape[:2] != shape[:2] or t.numel() == 0):
            raise ValueError(f"scale {i} must be (B, 1, h, w) with B = {shape[0]} and h, w >= 1, got {tuple(t.shape)}")
    tensors = [depth_gt_b1hw, mask_b_b1hw, depth_pred_b1hw, *[t for t in lps if t is not None]]
    if any(t.device != depth_gt_b1hw.device for t in tensors):
        raise ValueError("inputs live on different devices: " + ", ".join(str(t.device) for t in tensors))
    outs = _RegLossFunction.apply(depth_gt_b1hw, mask_b_b1hw, depth_pred_b1hw, float(si_lambda), *lps)
    return dict(zip(REGRESSION_KEYS, outs))


def uses_fused_regression_losses(model, depth_gt) -> bool:
    """Whether ``compute_losses`` runs the fused kernels for this model and ground truth: CUDA ground truth, and the
    multi-scale loss being the model's ``abs_loss``, a mean-reduced ``nn.L1Loss`` (``loss_type == "log_l1"``,
    depth_model.py:142, :150-151).  Anything else goes to the reference's original."""
    abs_loss = getattr(model, "abs_loss", None)
    return (torch.is_tensor(depth_gt) and depth_gt.is_cuda and getattr(model, "ms_loss_fn", None) is abs_loss
            and isinstance(abs_loss, nn.L1Loss) and abs_loss.reduction == "mean")


def compute_losses(self, cur_data, src_data, outputs):
    """Drop-in ``DepthModel.compute_losses`` (experiment_modules/depth_model.py:409-500), assigned to the class by
    ``install(regression_losses=True)``: the same nine losses under the same keys in the same order.  ``ms_loss``,
    ``abs_loss``, ``si_loss``, ``inv_abs_loss`` and ``log_l1_loss`` come from one ``depth_regression_losses`` call;
    ``grad_loss``, ``normals_loss`` and ``mv_loss`` from the model's own ``grad_loss``, ``normals_loss`` and
    ``mv_depth_loss`` modules with the reference's arguments (kernel-backed when those were installed too).  When
    ``uses_fused_regression_losses`` is false the call goes to the reference's saved original."""
    depth_gt = cur_data["depth_b1hw"]
    if not uses_fused_regression_losses(self, depth_gt):
        from .install import saved_original
        return saved_original("experiment_modules.depth_model", "DepthModel.compute_losses")(
            self, cur_data, src_data, outputs)
    log_preds = {i: outputs[f"log_depth_pred_s{i}_b1hw"] for i in range(NUM_SCALES)
                 if f"log_depth_pred_s{i}_b1hw" in outputs}
    if not log_preds:
        raise Exception("Could not find a valid scale to compute si loss!")
    depth_pred = outputs["depth_pred_s0_b1hw"]
    log_preds[0] = outputs["log_depth_pred_s0_b1hw"]      # a KeyError without scale 0, as the reference's :444
    terms = depth_regression_losses(depth_gt, cur_data["mask_b_b1hw"], log_preds, depth_pred,
                                    si_lambda=float(self.si_loss.si_lambda))
    grad_loss = self.grad_loss(depth_gt, depth_pred)
    normals_loss = self.normals_loss(cur_data["normals_b3hw"], outputs["normals_pred_b3hw"])
    mv_loss = self.mv_depth_loss(
        depth_pred_b1hw=depth_pred,
        cur_depth_b1hw=depth_gt,
        src_depth_bk1hw=src_data["depth_b1hw"],
        cur_invK_b44=cur_data["invK_s0_b44"],
        src_K_bk44=src_data["K_s0_b44"],
        cur_world_T_cam_b44=cur_data["world_T_cam_b44"],
        src_cam_T_world_bk44=src_data["cam_T_world_b44"],
    )
    loss = terms["ms_loss"] + 1.0 * grad_loss + 1.0 * normals_loss + 0.2 * mv_loss
    return {
        "loss": loss,
        "si_loss": terms["si_loss"],
        "grad_loss": grad_loss,
        "abs_loss": terms["abs_loss"],
        "normals_loss": normals_loss,
        "ms_loss": terms["ms_loss"],
        "inv_abs_loss": terms["inv_abs_loss"],
        "log_l1_loss": terms["log_l1_loss"],
        "mv_loss": mv_loss,
    }
