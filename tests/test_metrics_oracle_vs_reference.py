"""CPU: the depth-metrics oracle's fp32 mode (oracle/metrics_oracle.py) against the unmodified reference
``utils/metrics_utils.py`` — bit for bit, NaN and inf in the same places — on seeded inputs covering the
edge cases: threshold-boundary ratios, negative / zero / NaN / inf predictions, zero ground truth inside
the mask, empty frames and ``mult_a``.  The inputs and the reference's outputs are stored in
tests/golden/reference/metrics_oracle_vs_reference.npz (tests/golden/make_metrics_reference_golden.py);
the live comparison runs when ``$SIMPLERECON_REF`` names the reference tree."""
import importlib.util
import os

import pytest
import torch

from oracle import metrics_oracle as M
from oracle.ref_import import reference_available, reference_root
from tests import refgolden

MODULE = "metrics_oracle_vs_reference"
BATCHED_CASES = [(0, False), (1, True), (2, False)]
FLAT_CASES = ["finite", "finite_mult_a", "nan", "empty", "edges"]


def _fp32_boundaries():
    """fp32 ratios at and next to each threshold, and their inverses"""
    r = []
    for t in (1.05, 1.10, 1.25, 1.25 ** 2, 1.25 ** 3):
        tt = torch.tensor(t, dtype=torch.float32)
        for v in (tt, torch.nextafter(tt, torch.tensor(0.0)), torch.nextafter(tt, torch.tensor(2.0))):
            r += [v, 1 / v]
    return torch.stack(r)


def make_batched_inputs(seed: int, B: int = 4, N: int = 700):
    """(gt, pred, valid) with every edge case in frames 0-2 and an empty last frame"""
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(B, N, generator=g) * 6 + 0.1
    pred = gt * torch.exp(torch.randn(B, N, generator=g) * 0.25)
    valid = torch.rand(B, N, generator=g) > 0.3
    r = _fp32_boundaries()
    k = len(r)
    gt[:, :k] = torch.tensor([1.0, 2.0, 0.5, 4.0]).repeat(k)[:k]          # exact ratios on powers of two
    pred[:, :k] = gt[:, :k] * r
    pred[:, k:2 * k] = gt[:, k:2 * k] * r                                  # the same ratios on generic depths
    edge = slice(2 * k, 2 * k + 10)
    pred[:, edge] = torch.tensor([-1.0, -3.5, 0.0, -0.0, float("nan"), float("inf"), -float("inf"), 2.5, 0.0, 1.0])
    gt[:, 2 * k + 7:2 * k + 10] = torch.tensor([0.0, 0.0, float("nan")])    # zero gt with pred 2.5 and 0, NaN gt
    valid[:, :2 * k + 10] = True
    valid[B - 1] = False                                                  # a frame without valid pixels
    return gt, pred, valid


def make_flat_inputs(case: str):
    gt, pred, valid = make_batched_inputs(10 + FLAT_CASES.index(case))
    if case == "empty":
        return gt[0, :0], pred[0, :0], False
    m = valid[0]
    if case in ("finite", "finite_mult_a"):                                # drop the non-finite edge columns
        m = m & torch.isfinite(pred[0]) & (pred[0] > 0) & (gt[0] > 0)
    elif case == "nan":                                                    # one NaN prediction, otherwise finite
        m = m & torch.isfinite(pred[0]) & (pred[0] > 0) & (gt[0] > 0)
        pred = pred.clone()
        pred[0, m.nonzero()[5, 0]] = float("nan")
    return gt[0][m], pred[0][m], case == "finite_mult_a"


def _load_reference_metrics():
    """The reference's utils/metrics_utils.py, imported unmodified (it needs only torch, numpy, json)."""
    path = os.path.join(reference_root(), "utils", "metrics_utils.py")
    spec = importlib.util.spec_from_file_location("_simplerecon_ref_metrics_utils", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _pack(d: dict) -> dict:
    return {k: v.detach().reshape(-1).float() for k, v in d.items()}


def reference_outputs():
    """For tests/golden/make_metrics_reference_golden.py: the inputs and the reference's outputs."""
    ref = _load_reference_metrics()
    out = {}
    for seed, mult_a in BATCHED_CASES:
        gt, pred, valid = make_batched_inputs(seed)
        r = ref.compute_depth_metrics_batched(gt, pred, valid, mult_a=mult_a)
        assert list(r) == list(M.KEYS)
        out[f"batched_{seed}"] = {"gt": gt, "pred": pred, "valid": valid, **_pack(r)}
    for case in FLAT_CASES:
        gt, pred, mult_a = make_flat_inputs(case)
        r = ref.compute_depth_metrics(gt, pred, mult_a=mult_a)
        assert list(r) == list(M.KEYS)
        out[f"flat_{case}"] = {"gt": gt, "pred": pred, **_pack(r)}
    return out


def assert_bitwise(a: torch.Tensor, b: torch.Tensor, what=""):
    a, b = a.reshape(-1).float(), b.reshape(-1).float()
    assert a.shape == b.shape, what
    assert torch.equal(torch.isnan(a), torch.isnan(b)), what
    m = ~torch.isnan(a)
    assert torch.equal(a[m].view(torch.int32), b[m].view(torch.int32)), (what, a, b)


@pytest.mark.parametrize("seed,mult_a", BATCHED_CASES)
def test_batched_oracle_matches_stored_reference(seed, mult_a):
    G = refgolden.load(MODULE, f"batched_{seed}")
    gt, pred, valid = G["gt"], G["pred"], G["valid"]
    for stored, made in zip((gt, pred, valid), make_batched_inputs(seed)):   # the seeded inputs are reproducible
        assert_bitwise(stored, made)
    o = M.compute_depth_metrics_batched(gt, pred, valid, mult_a=mult_a)
    assert list(o) == list(M.KEYS)
    for k in M.KEYS:
        assert_bitwise(o[k], G[k], k)
    assert torch.isnan(G["abs_diff"][-1]) and torch.isnan(G["a5"][-1])      # the empty frame
    assert torch.isinf(G["abs_diff"][:-1]).all()                           # pred = inf
    assert torch.isinf(G["rmse_log"][:-1]).all()                           # pred = 0 -> log 0 = -inf
    assert (G["a5"][:-1] < (100 if mult_a else 1)).all()


@pytest.mark.parametrize("case", FLAT_CASES)
def test_flat_oracle_matches_stored_reference(case):
    G = refgolden.load(MODULE, f"flat_{case}")
    gt, pred, mult_a = make_flat_inputs(case)
    assert_bitwise(G["gt"], gt)
    assert_bitwise(G["pred"], pred)
    o = M.compute_depth_metrics(G["gt"], G["pred"], mult_a=mult_a)
    assert list(o) == list(M.KEYS)
    for k in M.KEYS:
        assert_bitwise(o[k], G[k], k)
    if case == "empty":
        assert all(torch.isnan(G[k]).all() for k in M.KEYS)
    if case == "nan":
        assert torch.isnan(G["rmse"]).all() and torch.isfinite(G["a5"]).all()


def test_fp32_threshold_constants():
    """pred = fp32(1.05) * gt on a power-of-two gt is not within a5: the comparison is in fp32"""
    gt = torch.tensor([1.0, 2.0])
    pred = gt * torch.tensor(1.05, dtype=torch.float32)
    assert M.compute_depth_metrics(gt, pred)["a5"].item() == 0.0
    assert M.compute_depth_metrics(gt, torch.nextafter(pred, torch.zeros(2)))["a5"].item() == 1.0


@pytest.mark.skipif(not reference_available(), reason="needs $SIMPLERECON_REF (the reference tree)")
def test_oracle_matches_live_reference():
    ref = _load_reference_metrics()
    for seed, mult_a in BATCHED_CASES:
        args = make_batched_inputs(seed)
        r, o = ref.compute_depth_metrics_batched(*args, mult_a=mult_a), M.compute_depth_metrics_batched(*args, mult_a=mult_a)
        assert list(r) == list(o)
        for k in M.KEYS:
            assert_bitwise(o[k], r[k], k)
    for case in FLAT_CASES:
        gt, pred, mult_a = make_flat_inputs(case)
        r, o = ref.compute_depth_metrics(gt, pred, mult_a=mult_a), M.compute_depth_metrics(gt, pred, mult_a=mult_a)
        assert list(r) == list(o)
        for k in M.KEYS:
            assert_bitwise(o[k], r[k], k)
