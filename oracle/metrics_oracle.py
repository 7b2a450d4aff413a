"""CPU restatement of the reference's depth metrics — TEST INFRASTRUCTURE (only tests/, smoke() and
bench legs may import it).

Two modes:
  - fp32 (``compute_depth_metrics``, ``compute_depth_metrics_batched``): the reference's
    ``utils/metrics_utils.py`` (:7-49, :51-120) op for op, fp32 sums included; pinned bit for bit to
    the unmodified module in tests/test_metrics_oracle_vs_reference.py;
  - fp32 terms, fp64 sums (``metrics_fp64``): the same fp32 per-pixel terms, summed in fp64 with
    exact integer counts, each metric the fp32 rounding of the fp64 formula — what the kernel
    (csrc/srcv_metrics.cuh, DESIGN §4.12) computes.
And the two resamplings ``test.py:282-287`` and ``experiment_modules/depth_model.py:585-590`` run
before the metrics, with PyTorch's index rules (align_corners=False): ``resample_nearest``,
``resample_bilinear``.
"""
from __future__ import annotations

import numpy as np
import torch

KEYS = ("abs_diff", "abs_rel", "sq_rel", "rmse", "rmse_log", "a5", "a10", "a25", "a0", "a1", "a2", "a3")
# a-metric thresholds in key order (metrics_utils.py:14-21, :67-93): a0 repeats a10, a1 repeats a25
THRESHOLDS = (1.05, 1.10, 1.25, 1.10, 1.25, 1.25 ** 2, 1.25 ** 3)


def _thresh(gt, pred):
    """max(gt / pred, pred / gt), NaN-propagating (torch.max, :12 and :63-64)"""
    return torch.max(gt / pred, pred / gt)


def _continuous_terms(gt, pred):
    """the per-pixel terms of abs_diff, abs_rel, sq_rel, rmse, rmse_log in the reference's ops (:28-38, :99-109)"""
    return ((gt - pred).abs(), torch.abs(gt - pred) / gt, (gt - pred) ** 2 / gt, (gt - pred) ** 2,
            (torch.log(gt) - torch.log(pred)) ** 2)


def compute_depth_metrics(gt, pred, mult_a=False):
    """metrics_utils.py:7-49 — plain means over every element."""
    th = _thresh(gt, pred)
    a = [(th < t).float().mean() for t in THRESHOLDS]                        # :14-21
    if mult_a:
        a = [x * 100 for x in a]                                              # :24-26
    d, rel, sq_rel, sq, sq_log = _continuous_terms(gt, pred)
    cont = [torch.mean(d), torch.mean(rel), torch.mean(sq_rel), torch.sqrt(sq.mean()), torch.sqrt(sq_log.mean())]
    return dict(zip(KEYS, cont + a))


def compute_depth_metrics_batched(gt_bN, pred_bN, valid_masks_bN, mult_a=False):
    """metrics_utils.py:51-120 — invalid pixels become NaN and drop out of every nanmean."""
    gt_bN = gt_bN.clone()
    pred_bN = pred_bN.clone()
    gt_bN[~valid_masks_bN] = torch.nan                                        # :60-61
    pred_bN[~valid_masks_bN] = torch.nan
    th = torch.max(torch.stack([gt_bN / pred_bN, pred_bN / gt_bN], dim=2), dim=2)[0]   # :63-64
    a = []
    for t in THRESHOLDS:                                                      # :67-93
        v = (th < t).float()
        v[~valid_masks_bN] = torch.nan
        a.append(torch.nanmean(v, dim=1))
    if mult_a:
        a = [x * 100 for x in a]
    d, rel, sq_rel, sq, sq_log = _continuous_terms(gt_bN, pred_bN)            # :99-109
    cont = [torch.nanmean(d, dim=1), torch.nanmean(rel, dim=1), torch.nanmean(sq_rel, dim=1),
            torch.sqrt(torch.nanmean(sq, dim=1)), torch.sqrt(torch.nanmean(sq_log, dim=1))]
    return dict(zip(KEYS, cont + a))


def metrics_fp64(gt_bN, pred_bN, valid_bN=None, flat=False, mult_a=False):
    """fp32 inputs (B, N) -> (metrics (B, 12) fp32 in KEYS order, valid counts (B,) int64).

    Per-pixel terms in fp32 as above; sums in fp64, counts exact; a = count / valid count; each
    continuous metric is the mean of its non-NaN terms (batched) or, with ``flat``, NaN as soon as
    one term is NaN; rmse / rmse_log take the sqrt in fp64; every metric is rounded to fp32 last."""
    gt_bN, pred_bN = gt_bN.float(), pred_bN.float()
    valid = torch.ones_like(gt_bN, dtype=torch.bool) if valid_bN is None else valid_bN.bool()
    n = valid.sum(1)
    nd = n.double()
    th = torch.maximum(gt_bN / pred_bN, pred_bN / gt_bN)
    out = []
    for i, term in enumerate(_continuous_terms(gt_bN, pred_bN)):
        keep = valid & ~torch.isnan(term)
        s = torch.where(keep, term, torch.zeros_like(term)).double().sum(1)
        c = keep.sum(1).double()
        m = s / c
        if flat:
            m = torch.where(c == nd, m, torch.full_like(m, float("nan")))
        out.append(m.sqrt() if i >= 3 else m)
    out = [m.float() for m in out]
    for t in THRESHOLDS:
        a = ((th < t) & valid).sum(1).double() / nd
        a = a.float()
        out.append(a * 100 if mult_a else a)
    return torch.stack(out, 1), n


def _nearest_index(n_in: int, n_out: int) -> torch.Tensor:
    """min(floor(dst * fp32(in / out)), in - 1), every op in fp32"""
    scale = np.float32(n_in) / np.float32(n_out)
    dst = np.arange(n_out, dtype=np.float32)
    return torch.from_numpy(np.minimum(np.floor(dst * scale).astype(np.int64), n_in - 1))


def resample_nearest(x_b1hw: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """F.interpolate(x, (h, w), mode="nearest") (test.py:282-287)"""
    iy, ix = _nearest_index(x_b1hw.shape[-2], h), _nearest_index(x_b1hw.shape[-1], w)
    return x_b1hw[:, :, iy][:, :, :, ix]


def _fma32(a, b, c):
    """fp32 fused multiply-add: the fp64 product of two fp32 values is exact, one rounding to fp32
    (the fp64 sum may round first: off by one ulp at worst, in a vanishing share of cases)"""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def _linear_index(n_in: int, n_out: int):
    scale = np.float32(n_in) / np.float32(n_out)
    src = _fma32(scale, np.arange(n_out, dtype=np.float32) + np.float32(0.5), np.float32(-0.5))
    src = np.maximum(src, np.float32(0))
    i0 = src.astype(np.int64)
    i1 = i0 + (i0 < n_in - 1)                                                # PyTorch's clamp of the upper neighbour
    l1 = (src - i0.astype(np.float32)).astype(np.float32)
    return i0, i1, (np.float32(1) - l1).astype(np.float32), l1


def resample_bilinear(x_b1hw: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """F.interpolate(x, (h, w), mode="bilinear", align_corners=False) (depth_model.py:585-590), with the
    FMAs of PyTorch's CUDA kernel: h0 (w0 x00 + w1 x01) + h1 (w0 x10 + w1 x11) as
    fma(h0, fma(w0, x00, w1 x01), h1 fma(w0, x10, w1 x11)).  A same-size input is copied."""
    if tuple(x_b1hw.shape[-2:]) == (h, w):
        return x_b1hw.clone()
    x = x_b1hw.float().numpy()
    y0, y1, hl0, hl1 = (v[:, None] for v in _linear_index(x.shape[-2], h))
    x0, x1, wl0, wl1 = (v[None, :] for v in _linear_index(x.shape[-1], w))

    def pair(r):
        a, b = x[:, :, r, x0], x[:, :, r, x1]
        return _fma32(wl0, a, (wl1 * b).astype(np.float32))
    top, bot = pair(y0), pair(y1)
    return torch.from_numpy(_fma32(hl0, top, (hl1 * bot).astype(np.float32)))
