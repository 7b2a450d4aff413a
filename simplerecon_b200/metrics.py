"""Depth metrics, backed by the sm_90a kernel (csrc/srcv_metrics.cuh, DESIGN §4.12).

Mirrors ``compute_depth_metrics`` and ``compute_depth_metrics_batched`` of the reference's
``utils/metrics_utils.py`` (:7-120): same signatures, same dict keys in the same order.  The values
are views of one ``(B, 12)`` result computed in one pass (fp32 per-pixel terms as in the reference,
fp64 sums, exact counts), so they agree with the reference to the rounding of its fp32 sums, and the
a-metrics exactly.  ``depth_metrics`` is ``test.py:282-299`` in one call: it samples a prediction of
any resolution on the ground-truth grid (PyTorch's ``nearest`` or ``bilinear``), takes the validity
from a mask or ``gt > min_valid_depth``, and returns the metrics, the per-frame valid counts and
optionally the resampled prediction, without a host synchronisation.

CUDA tensors on an sm_90 device, or an exception: there is no CPU path.  fp16 / bf16 inputs are
computed from their fp32 upcasts; the continuous metrics then come back in the input dtype, as the
reference computes them, and the a-metrics in fp32 (the reference's ``.float()``).
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _native

KEYS = ("abs_diff", "abs_rel", "sq_rel", "rmse", "rmse_log", "a5", "a10", "a25", "a0", "a1", "a2", "a3")
_N_CONTINUOUS = 5
_DTYPES = (torch.float32, torch.float16, torch.bfloat16)
_MODES = {"nearest": _native.RESAMPLE_NEAREST, "bilinear": _native.RESAMPLE_BILINEAR}


def _require_cuda(t: torch.Tensor) -> None:
    """The device gate (tests/ patch exactly this to drive the host-emulated library)."""
    if t.device.type != "cuda":
        raise RuntimeError("simplerecon_b200 depth metrics run on CUDA (sm_90a) only; there is no CPU fallback")


def _lib():
    return _native.load()


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _check_inputs(named: dict) -> torch.device:
    tensors = {k: v for k, v in named.items() if v is not None}
    first = next(iter(tensors.values()))
    if any(t.device != first.device for t in tensors.values()):
        raise ValueError("depth-metric inputs live on different devices: " +
                         ", ".join(f"{k} {t.device}" for k, t in tensors.items()))
    for k in ("gt", "pred"):
        if named[k].dtype not in _DTYPES:
            raise ValueError(f"{k} must be float32, float16 or bfloat16, got {named[k].dtype}")
    _require_cuda(first)
    return first.device


def _run(gt, pred, valid, B, H, W, Hp, Wp, *, min_valid_depth=0.0, valid_source, resample, nan_mode, mult_a,
         want_upsampled=False):
    """gt (B*H*W), pred (B*Hp*Wp), valid (B*H*W) bool / uint8 or None -> (metrics (B,12) f32, counts (B,) i64, up)."""
    dev = gt.device
    g = gt.detach().to(torch.float32).contiguous()
    p = pred.detach().to(torch.float32).contiguous()
    v = valid.detach().contiguous().view(torch.uint8) if valid is not None else None
    args = _native.MetricsArgs(g.data_ptr(), p.data_ptr(), v.data_ptr() if v is not None else None,
                               float(min_valid_depth), B, H, W, Hp, Wp, resample, nan_mode, valid_source, int(bool(mult_a)))
    n = _lib().srcv_metrics_workspace_bytes(C.byref(args))
    if n == 0:
        raise ValueError(f"unsupported depth-metric shape B={B} H={H} W={W} Hp={Hp} Wp={Wp}")
    ws = torch.empty(n, device=dev, dtype=torch.uint8)
    metrics = torch.empty(B, len(KEYS), device=dev, dtype=torch.float32)
    counts = torch.empty(B, device=dev, dtype=torch.int64)
    up = torch.empty(B, H, W, device=dev, dtype=torch.float32) if want_upsampled else None
    with torch.cuda.device(dev):
        _native.check(_lib().srcv_depth_metrics_f32(
            C.byref(args), C.c_void_p(metrics.data_ptr()), C.c_void_p(counts.data_ptr()),
            C.c_void_p(up.data_ptr() if up is not None else 0), C.c_void_p(ws.data_ptr()), ws.numel(), _stream(dev)))
    return metrics, counts, up


def _as_dict(metrics: torch.Tensor, dtype: torch.dtype, row=None) -> dict:
    """{key: view of metrics[:, i]} (or of metrics[row, i]); continuous metrics in the inputs' dtype."""
    out = {}
    for i, k in enumerate(KEYS):
        m = metrics[:, i] if row is None else metrics[row, i]
        out[k] = m.to(dtype) if (i < _N_CONTINUOUS and dtype != torch.float32) else m
    return out


def compute_depth_metrics_batched(gt_bN, pred_bN, valid_masks_bN, mult_a=False):
    """reference utils/metrics_utils.py:51-120: per-frame metrics over the valid mask; each continuous
    metric is the nanmean of its terms, the a-metrics divide by the frame's valid count, and a frame
    without valid pixels gives NaN for all 12."""
    _check_inputs({"gt": gt_bN, "pred": pred_bN, "valid_masks": valid_masks_bN})
    if gt_bN.dim() != 2 or tuple(pred_bN.shape) != tuple(gt_bN.shape) or tuple(valid_masks_bN.shape) != tuple(gt_bN.shape):
        raise ValueError(f"expected (B, N) gt, pred and mask of one shape, got {tuple(gt_bN.shape)}, "
                         f"{tuple(pred_bN.shape)}, {tuple(valid_masks_bN.shape)}")
    if valid_masks_bN.dtype not in (torch.bool, torch.uint8):
        raise ValueError(f"valid_masks_bN must be bool, got {valid_masks_bN.dtype}")
    B, N = gt_bN.shape
    metrics, _, _ = _run(gt_bN, pred_bN, valid_masks_bN, B, 1, N, 1, N, valid_source=_native.METRICS_VALID_MASK,
                         resample=_native.RESAMPLE_IDENTITY, nan_mode=_native.METRICS_BATCHED, mult_a=mult_a)
    return _as_dict(metrics, torch.result_type(gt_bN, pred_bN))


def compute_depth_metrics(gt, pred, mult_a=False):
    """reference utils/metrics_utils.py:7-49: plain means over every element (already masked, any
    shape), so a NaN term makes its metric NaN; empty input gives NaN everywhere.  0-d values."""
    _check_inputs({"gt": gt, "pred": pred})
    if tuple(gt.shape) != tuple(pred.shape):
        raise ValueError(f"gt and pred shapes differ: {tuple(gt.shape)} vs {tuple(pred.shape)}")
    N = gt.numel()
    metrics, _, _ = _run(gt.reshape(-1), pred.reshape(-1), None, 1, 1, N, 1, N, valid_source=_native.METRICS_VALID_ALL,
                         resample=_native.RESAMPLE_IDENTITY, nan_mode=_native.METRICS_FLAT, mult_a=mult_a)
    return _as_dict(metrics, torch.result_type(gt, pred), row=0)


def depth_metrics(depth_gt_b1hw, depth_pred_b1hw, valid_mask_b1hw=None, min_valid_depth=None, mode="nearest",
                  mult_a=False, return_upsampled=False):
    """Batched metrics (compute_depth_metrics_batched's semantics) of a prediction of any resolution
    against the ground truth, in one launch pair and without a host synchronisation:

        metrics, valid_counts[, upsampled] = depth_metrics(gt, pred, min_valid_depth=0.5, mult_a=True,
                                                           return_upsampled=True)

    is test.py:282-299 — F.interpolate(pred, gt size, mode), valid = gt > 0.5,
    compute_depth_metrics_batched — with ``metrics`` (B, 12) fp32 in the order of ``KEYS``,
    ``valid_counts`` (B,) int64 (a frame with count 0 has NaN metrics: skip it with one read of the
    counts) and ``upsampled`` (B, 1, H, W) fp32, what F.interpolate returns.  Validity comes from
    ``valid_mask_b1hw`` (bool), or from ``gt > min_valid_depth`` in fp32, or, with neither, every pixel."""
    _check_inputs({"gt": depth_gt_b1hw, "pred": depth_pred_b1hw, "valid_mask": valid_mask_b1hw})
    if mode not in _MODES:
        raise ValueError(f"mode must be 'nearest' or 'bilinear', got {mode!r}")
    if depth_gt_b1hw.dim() != 4 or depth_pred_b1hw.dim() != 4 or depth_gt_b1hw.shape[1] != 1 or \
            depth_pred_b1hw.shape[1] != 1 or depth_pred_b1hw.shape[0] != depth_gt_b1hw.shape[0]:
        raise ValueError(f"expected (B,1,H,W) gt and (B,1,Hp,Wp) prediction, got {tuple(depth_gt_b1hw.shape)} and "
                         f"{tuple(depth_pred_b1hw.shape)}")
    if valid_mask_b1hw is not None and min_valid_depth is not None:
        raise ValueError("pass valid_mask_b1hw or min_valid_depth, not both")
    if valid_mask_b1hw is not None and (tuple(valid_mask_b1hw.shape) != tuple(depth_gt_b1hw.shape) or
                                        valid_mask_b1hw.dtype not in (torch.bool, torch.uint8)):
        raise ValueError(f"valid_mask_b1hw must be a bool tensor shaped like the ground truth "
                         f"{tuple(depth_gt_b1hw.shape)}, got {valid_mask_b1hw.dtype} {tuple(valid_mask_b1hw.shape)}")
    B, _, H, W = depth_gt_b1hw.shape
    Hp, Wp = depth_pred_b1hw.shape[-2:]
    source = (_native.METRICS_VALID_MASK if valid_mask_b1hw is not None else
              _native.METRICS_VALID_MIN_DEPTH if min_valid_depth is not None else _native.METRICS_VALID_ALL)
    metrics, counts, up = _run(depth_gt_b1hw, depth_pred_b1hw, valid_mask_b1hw, B, H, W, Hp, Wp,
                               min_valid_depth=min_valid_depth or 0.0, valid_source=source, resample=_MODES[mode],
                               nan_mode=_native.METRICS_BATCHED, mult_a=mult_a, want_upsampled=return_upsampled)
    if return_upsampled:
        return metrics, counts, up.view(B, 1, H, W)
    return metrics, counts


def metrics_to_dict(metrics_b12: torch.Tensor) -> dict:
    """(B, 12) -> {key: (B,) view}, the dict compute_depth_metrics_batched returns."""
    return {k: metrics_b12[:, i] for i, k in enumerate(KEYS)}
