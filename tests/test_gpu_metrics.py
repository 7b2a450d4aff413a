"""GPU: the depth-metrics kernels through simplerecon_b200.metrics against the oracle's fp64-sum mode at the
sizes the reference runs them: test.py's evaluation (480x640 ground truth, 192x256 prediction, nearest,
gt > 0.5, mult_a), depth_model's high-res validation (bilinear to full resolution, then the flat metrics
of boolean-indexed 1-D tensors), the resampled map against torch's CUDA F.interpolate (nearest bit-equal,
bilinear within 1 ulp), determinism, a non-default stream, and a frame of more than 2^24 pixels."""
import pytest
import torch
import torch.nn.functional as F

import simplerecon_b200 as S
from oracle import metrics_oracle as M
from simplerecon_b200 import _native
from tests.test_emu_metrics import check_metrics, ulp_diff
from tests.test_metrics_oracle_vs_reference import make_batched_inputs, make_flat_inputs

pytestmark = pytest.mark.gpu


def _scan_batch(seed, B, H=480, W=640, Hp=192, Wp=256, dev="cuda"):
    g = torch.Generator(device="cpu").manual_seed(seed)
    gt = torch.rand(B, 1, H, W, generator=g) * 6
    gt[:, :, 100:180, 200:330] = 0.0                        # a hole in the ground truth
    pred = (torch.nn.functional.interpolate(gt[:, :, ::4, ::4], size=(Hp, Wp), mode="nearest") *
            torch.exp(torch.randn(B, 1, Hp, Wp, generator=g) * 0.15)).clamp_min(0.05)
    return gt.to(dev), pred.to(dev)


@pytest.mark.parametrize("B", [1, 8])
def test_test_py_evaluation(cuda_device, B):
    """test.py:282-299: nearest to 480x640, valid = gt > 0.5, batched metrics with mult_a"""
    gt, pred = _scan_batch(B, B)
    if B == 8:
        gt[5] = 0.2                                        # a frame without valid ground truth
    metrics, counts, up = S.depth_metrics(gt, pred, min_valid_depth=0.5, mult_a=True, return_upsampled=True)
    assert _native.last_variant() == "depth_metrics_f32"
    ref_up = F.interpolate(pred, size=(480, 640), mode="nearest")
    assert torch.equal(up, ref_up)
    valid = gt > 0.5
    check_metrics(metrics, valid.flatten(1).sum(1), gt.flatten(1), ref_up.flatten(1), valid.flatten(1), mult_a=True)
    ref32 = M.compute_depth_metrics_batched(gt.flatten(1).cpu(), ref_up.flatten(1).cpu(), valid.flatten(1).cpu(), mult_a=True)
    for i, k in enumerate(M.KEYS):
        r = ref32[k]
        if i >= 5:                                          # a-metrics: the reference's bits
            torch.testing.assert_close(metrics[:, i].cpu(), r, rtol=0, atol=0, equal_nan=True)
        else:                                               # the reference's fp32 sums are the inexact side
            torch.testing.assert_close(metrics[:, i].cpu(), r, rtol=1e-4, atol=0, equal_nan=True)
    if B == 8:
        assert counts[5].item() == 0 and metrics[5].isnan().all()


def test_high_res_validation_bilinear_then_flat(cuda_device):
    """depth_model.py:581-595: bilinear to the full-res ground truth, then compute_depth_metrics on the
    boolean-indexed 1-D tensors; and the same in one call through depth_metrics with the mask"""
    gt, pred = _scan_batch(3, 4)
    mask = gt > 0.1
    up_ref = F.interpolate(pred, size=gt.shape[-2:], mode="bilinear", align_corners=False)
    metrics, counts, up = S.depth_metrics(gt, pred, valid_mask_b1hw=mask, mode="bilinear", return_upsampled=True)
    assert ulp_diff(up, up_ref).max().item() <= 1
    check_metrics(metrics, mask.flatten(1).sum(1), gt.flatten(1), up.flatten(1), mask.flatten(1))
    d = S.compute_depth_metrics(gt[mask], up_ref[mask])
    assert list(d) == list(M.KEYS) and all(v.dim() == 0 and v.is_cuda for v in d.values())
    check_metrics(torch.stack(list(d.values()))[None], mask.sum()[None], gt[mask][None], up_ref[mask][None], flat=True)


@pytest.mark.parametrize("seed,mult_a", [(0, False), (1, True)])
def test_reference_functions_on_edge_cases(cuda_device, seed, mult_a):
    gt, pred, valid = (t.cuda() for t in make_batched_inputs(seed))
    d = S.compute_depth_metrics_batched(gt, pred, valid, mult_a=mult_a)
    check_metrics(torch.stack(list(d.values()), 1), valid.sum(1), gt, pred, valid, mult_a=mult_a)
    for case in ("finite", "nan", "empty", "edges"):
        g, p, ma = make_flat_inputs(case)
        f = S.compute_depth_metrics(g.cuda(), p.cuda(), mult_a=ma)
        check_metrics(torch.stack(list(f.values()))[None], torch.tensor([g.numel()]), g[None], p[None], flat=True,
                      mult_a=ma)


def test_deterministic_and_on_a_side_stream(cuda_device):
    gt, pred = _scan_batch(7, 6)
    runs = [S.depth_metrics(gt, pred, min_valid_depth=0.5, mode="bilinear")]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        runs.append(S.depth_metrics(gt, pred, min_valid_depth=0.5, mode="bilinear"))
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    for m, c in runs[1:]:
        assert torch.equal(m.view(torch.int32), runs[0][0].view(torch.int32)) and torch.equal(c, runs[0][1])


def test_frame_above_2_pow_24_pixels_counts_exactly(cuda_device):
    """4100 x 4100 = 16.8 M pixels: an fp32 mean of 0/1 values is no longer exact there; the counts are"""
    H = W = 4100
    g = torch.Generator(device="cuda").manual_seed(3)
    gt = torch.rand(1, 1, H, W, device="cuda", generator=g) * 4
    pred = torch.rand(1, 1, H // 2, W // 2, device="cuda", generator=g) * 4 + 0.01
    assert H * W > 2 ** 24
    metrics, counts, up = S.depth_metrics(gt, pred, min_valid_depth=0.5, return_upsampled=True)
    valid = gt > 0.5
    om, oc = M.metrics_fp64(gt.flatten(1), up.flatten(1), valid.flatten(1))
    assert counts.item() == oc.item() == valid.sum().item() > 2 ** 24 * 0.8
    torch.testing.assert_close(metrics[:, 5:], om[:, 5:], rtol=0, atol=0)
    assert ((metrics[:, :5].double() - om[:, :5].double()).abs() <= 1e-6 * om[:, :5].double().abs()).all()
